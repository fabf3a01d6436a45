// K-gnn: the parameter-free graph attention of the class decoder.
//
// Reference: Model.gnn_edge (code/pred_models.py:808-858) builds the dense [HW,HW] cosine matrix
// of F = l2_normalize([h ; mean_t scene_conv]); gnn_mask_edge (:885-909) adds -1e30 everywhere
// except the 3x3 neighbourhood (self included, borders clipped); gnn_node (:860-882) soft-maxes
// and multiplies by h; the caller adds the residual (:378, :651).  Only the <=9 unmasked entries
// of each row survive the softmax in fp32 (exp(-1e30) == 0), so this kernel evaluates exactly
// that 3x3 band:  h'_p = h_p + sum_q softmax_q(F^_p . F^_q) h_q.
//
// One warp walks one image row of one sample row with a 3x3 register window (8 h + 2 scene values
// per lane per cell) plus one column in flight: moving one cell to the right loads only the 3 new cells of a column,
// so every h row is fetched 3x (not 9x) through L1/L2, squared norms are computed once per loaded
// cell, and the centre-left dot product is the previous step's centre-right one.  Per cell: 7 dot
// products + 3 norms reduced by warp shuffles, a <=9-way softmax, 72 FMAs of weighted sum, and the
// result is written straight as the bf16 operand planes of the next cell step.
// HBM-bound by design: 4*HW*(256+64) bytes read, 4*HW*256 written per sample row (either operand format).
#include "mvb_common.cuh"
#include "mvb_kernels.h"

namespace mvb {

constexpr int GNN_WARPS = 4;

struct GnnCol {         // one window column: rows y-1, y, y+1
  float2 h[3][4];
  float2 s[3];
  float n[3];           // squared norm of [h ; s] (warp-reduced)
  float inv[3];         // tf.nn.l2_normalize's factor: rsqrt(max(n, 1e-12))
};

// Row pointers of the three window rows (this lane's 8 h channels / 2 scene channels), rows clamped into the image.
struct GnnRows {
  const float* h[3];
  const float* s[3];
};

// Raw loads of one window column, issued one step ahead of their use: with load-then-use the kernel was bound
// by the latency of these loads (ncu: 2.7 warps per issue stalled on the long scoreboard at 12 warps/SM).
// Out-of-image neighbours are not zero-filled: their coordinates are CLAMPED into the image (a valid, finite cell
// is loaded instead) and their softmax weight is exactly 0 (the `ok` mask below), so fma(0, finite, o) == o and the
// result is what a zero fill gives - without the branches, the zeroing moves and the predicates per load.
__device__ __forceinline__ void gnn_load_raw(GnnCol& c, const GnnRows& rows, int x, int W, bool has_scene) {
  const int xc = min(max(x, 0), W - 1);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const float4* p4 = reinterpret_cast<const float4*>(rows.h[r] + (long long)xc * kHidden);
    const float4 a = __ldg(p4), b = __ldg(p4 + 1);
    c.h[r][0] = make_float2(a.x, a.y); c.h[r][1] = make_float2(a.z, a.w);
    c.h[r][2] = make_float2(b.x, b.y); c.h[r][3] = make_float2(b.z, b.w);
    c.s[r] = has_scene ? __ldg(reinterpret_cast<const float2*>(rows.s[r] + (long long)xc * 64)) : make_float2(0.f, 0.f);
  }
}

__device__ __forceinline__ float gnn_dot(const GnnCol& a, int ra, const GnnCol& b, int rb) {
  float2 d = fmul2(a.h[ra][0], b.h[rb][0]);
#pragma unroll
  for (int k = 1; k < 4; ++k) d = ffma2(a.h[ra][k], b.h[rb][k], d);
  d = ffma2(a.s[ra], b.s[rb], d);
  return d.x + d.y;
}

// Squared norms of a loaded column (warp-reduced) and their normalisation factors.
__device__ __forceinline__ void gnn_norms(GnnCol& c) {
#pragma unroll
  for (int r = 0; r < 3; ++r) c.n[r] = gnn_dot(c, r, c, r);
#pragma unroll
  for (int r = 0; r < 3; ++r) c.n[r] = warp_sum(c.n[r]);
#pragma unroll
  for (int r = 0; r < 3; ++r) c.inv[r] = rsqrtf(fmaxf(c.n[r], 1e-12f));
}

// FMT = 1: the output is written in the f16f8 operand format (mvb_common.cuh), else as bf16x2 planes
template <int FMT>
__global__ void __launch_bounds__(GNN_WARPS * 32)
gnn_kernel(const float* __restrict__ h32, const int* __restrict__ row_map,
           const float* __restrict__ scene_mean, int beam, __nv_bfloat16* __restrict__ hp_out,
           long long plane_stride, int cpad_out, int ch_off, long long NS, Grid g) {
  const int lane = threadIdx.x & 31;
  const long long wid = (long long)blockIdx.x * GNN_WARPS + (threadIdx.x >> 5);
  if (wid >= NS * g.H) return;
  const long long s = wid / g.H;
  const int y = (int)(wid - s * g.H);
  const long long ss = row_map ? (long long)row_map[s] : s;
  const bool rok[3] = {y > 0, true, y < g.H - 1};
  const bool has_scene = scene_mean != nullptr;
  GnnRows rows;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int yy = min(max(y + r - 1, 0), g.H - 1);
    rows.h[r] = h32 + (ss * g.S + (long long)yy * g.Wp) * kHidden + lane * 8;
    rows.s[r] = has_scene ? scene_mean + ((s / beam) * (long long)g.H * g.W + (long long)yy * g.W) * 64 + lane * 2 : nullptr;
  }

  // Rotating 4-column register window (no register moves: the loop is unrolled by four and the roles
  // L / C / R / N(ext, in flight) rotate through the four structs): every column is requested one step before
  // its first use.  Measured at 2 560 rows of 36x18: 3 columns (load, then use) 1.86 ms; 4 columns 1.41 ms;
  // 5 columns (two steps ahead, 236 registers) 1.54 ms; an L1 prefetch instead of the fourth column 2.16 ms;
  // 4 columns + folded (transpose) reduction of the ten warp sums 1.54 ms (longer dependent shuffle chain);
  // forcing 3 CTAs/SM (168 registers, spills) 1.59 ms.
  GnnCol W0, W1, W2, W3;
  gnn_load_raw(W0, rows, -1, g.W, has_scene);     // masked out below (x == 0 has no left neighbours)
  gnn_load_raw(W1, rows, 0, g.W, has_scene);
  gnn_load_raw(W2, rows, 1, g.W, has_scene);
  gnn_norms(W0);
  gnn_norms(W1);
  float d_cl = 0.f;   // dot(centre, left-centre), carried from the previous cell
  auto step = [&](const GnnCol& L, const GnnCol& C, GnnCol& R, GnnCol& N, int x) {
    gnn_load_raw(N, rows, x + 2, g.W, has_scene);   // used by the next step
    gnn_norms(R);
    // dots of the centre cell (C,1) with its 8 neighbours; self = squared norm
    float d[9];
    d[0] = gnn_dot(C, 1, L, 0); d[1] = gnn_dot(C, 1, C, 0); d[2] = gnn_dot(C, 1, R, 0);
    d[5] = gnn_dot(C, 1, R, 1);
    d[6] = gnn_dot(C, 1, L, 2); d[7] = gnn_dot(C, 1, C, 2); d[8] = gnn_dot(C, 1, R, 2);
    d[0] = warp_sum(d[0]); d[1] = warp_sum(d[1]); d[2] = warp_sum(d[2]); d[5] = warp_sum(d[5]);
    d[6] = warp_sum(d[6]); d[7] = warp_sum(d[7]); d[8] = warp_sum(d[8]);
    d[3] = d_cl;
    d[4] = C.n[1];
    d_cl = d[5];
    const bool cokL = x > 0, cokR = x < g.W - 1;
    const bool ok[9] = {rok[0] && cokL, rok[0], rok[0] && cokR, cokL, true, cokR,
                        rok[2] && cokL, rok[2], rok[2] && cokR};
    const float iq[9] = {L.inv[0], C.inv[0], R.inv[0], L.inv[1], C.inv[1], R.inv[1], L.inv[2], C.inv[2], R.inv[2]};
    // tf.nn.l2_normalize: x * rsqrt(max(sum x^2, 1e-12))
    const float inv_p = C.inv[1];
    float e[9], m = -INFINITY;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      e[k] = d[k] * inv_p * iq[k];
      if (ok[k]) m = fmaxf(m, e[k]);
    }
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < 9; ++k) { e[k] = ok[k] ? __expf(e[k] - m) : 0.f; sum += e[k]; }
    const float inv_sum = 1.0f / sum;
    float2 o2[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) o2[c] = C.h[1][c];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float aL = e[r * 3 + 0] * inv_sum, aC = e[r * 3 + 1] * inv_sum, aR = e[r * 3 + 2] * inv_sum;
      const float2 aL2 = make_float2(aL, aL), aC2 = make_float2(aC, aC), aR2 = make_float2(aR, aR);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        o2[c] = ffma2(aL2, L.h[r][c], o2[c]);
        o2[c] = ffma2(aC2, C.h[r][c], o2[c]);
        o2[c] = ffma2(aR2, R.h[r][c], o2[c]);
      }
    }
    const float o[8] = {o2[0].x, o2[0].y, o2[1].x, o2[1].y, o2[2].x, o2[2].y, o2[3].x, o2[3].y};
    const long long orow = s * g.S + (long long)y * g.Wp + x;
    if constexpr (FMT) {
      store_f16f8_x8(hp_out, plane_stride, orow, ch_off + lane * 8, cpad_out, o);
    } else {
      uint32_t pk[kBf16Planes][4];
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        __nv_bfloat16 a[kBf16Planes], b[kBf16Planes];
        split_planes(o[2 * v], a);
        split_planes(o[2 * v + 1], b);
#pragma unroll
        for (int p = 0; p < kBf16Planes; ++p) pk[p][v] = pack_bf16x2(a[p], b[p]);
      }
#pragma unroll
      for (int p = 0; p < kBf16Planes; ++p) {
        uint4* po = reinterpret_cast<uint4*>(hp_out + p * plane_stride + orow * cpad_out + ch_off + lane * 8);
        *po = make_uint4(pk[p][0], pk[p][1], pk[p][2], pk[p][3]);
      }
    }
  };
  for (int x = 0; x < g.W; x += 4) {
    step(W0, W1, W2, W3, x);
    if (x + 1 < g.W) step(W1, W2, W3, W0, x + 1);
    if (x + 2 < g.W) step(W2, W3, W0, W1, x + 2);
    if (x + 3 < g.W) step(W3, W0, W1, W2, x + 3);
  }
}

// ----------------------------------------------------------------------------------------------------------------
// Second formulation (round 2): one CTA per sample row, image rows streamed through a shared-memory ring.
//
// The warp-per-image-row kernel above spends its issue slots on cross-lane work: ten 5-stage butterfly sums per cell
// (a dot product is spread over the 32 lanes) and a 9-way softmax that every lane repeats - ~510 instructions per
// cell, 6.2 ms for 10 240 rows of 36x18 (2.2 TB/s algorithmic; the HBM floor of the 11 GB it moves is 1.7 ms).
// Here the dot products are formed where the data is:
//   A(r)  when image row r arrives (one bulk async copy of W*1280 bytes into the ring), 16 lanes x 2 cells per task
//         form the five pair products of each of its cells with the row above and its right neighbour (every pair of
//         the 3x3 band is formed once - the band is symmetric) plus the squared norm: 3.5 vector loads per cell
//         instead of 5, reduced over 16 lanes;
//   B(y)  one thread per cell of row y collects its nine cosines from the rows y-1, y, y+1 and soft-maxes them
//         (done once, not by 32 lanes);
//   C(y)  one warp per 3 consecutive cells, 8 channels per lane: 15 neighbour vectors from shared memory for
//         3 outputs, written straight in the operand format of the next cell step.
// Shared-memory traffic (the bound of this formulation): ~9.5 KB per cell at 128 B/clk/SM.
// ----------------------------------------------------------------------------------------------------------------
constexpr int GT = 256;      // threads per CTA
constexpr int GNR = 4;       // ring slots (image rows y-1, y, y+1 and the one in flight)
constexpr int GD = 8;        // floats per cell in the pair-product table: U0 U1 U2 Rt Nn inv - -
constexpr int GW = 12;       // floats per cell in the weight table (9 used)

__host__ __device__ inline size_t gnn_rows_smem(int W) {
  return (size_t)W * (GNR * (kHidden + 64 + GD) + GW) * sizeof(float) + GNR * sizeof(uint64_t);
}

__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ float2 lo2(const float4& v) { return make_float2(v.x, v.y); }
__device__ __forceinline__ float2 hi2(const float4& v) { return make_float2(v.z, v.w); }
__device__ __forceinline__ void dot_acc(float2& acc, const float4& a, const float4& b) {
  acc = ffma2(lo2(a), lo2(b), acc);
  acc = ffma2(hi2(a), hi2(b), acc);
}

// 4 consecutive channels of one row into the operand buffer (FMT = 0: bf16x2 planes, 1: f16f8)
template <int FMT>
__device__ __forceinline__ void store_operand_x4(__nv_bfloat16* hp_out, long long plane_stride, long long row,
                                                 int ch, int cpad, const float (&v)[4]) {
  if constexpr (FMT) {
    uint32_t hw[2], b0 = 0u, b1 = 0u;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      uint32_t e0, e1;
      split_f16f8_x2(v[2 * i], v[2 * i + 1], hw[i], e0, e1);
      b0 |= e0 << (16 * i);
      b1 |= e1 << (16 * i);
    }
    *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(hp_out) + row * cpad + ch) = make_uint2(hw[0], hw[1]);
    uint8_t* b8 = reinterpret_cast<uint8_t*>(hp_out) + 2 * plane_stride + row * 2 * cpad;
    *reinterpret_cast<uint32_t*>(b8 + f8_off(ch, 0, cpad)) = b0;
    *reinterpret_cast<uint32_t*>(b8 + f8_off(ch, 1, cpad)) = b1;
  } else {
    uint32_t pk[kBf16Planes][2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      __nv_bfloat16 a[kBf16Planes], b[kBf16Planes];
      split_planes(v[2 * i], a);
      split_planes(v[2 * i + 1], b);
#pragma unroll
      for (int q = 0; q < kBf16Planes; ++q) pk[q][i] = pack_bf16x2(a[q], b[q]);
    }
#pragma unroll
    for (int q = 0; q < kBf16Planes; ++q)
      *reinterpret_cast<uint2*>(hp_out + q * plane_stride + row * cpad + ch) = make_uint2(pk[q][0], pk[q][1]);
  }
}

template <int FMT>
__global__ void __launch_bounds__(GT)
gnn_rows_kernel(const float* __restrict__ h32, const int* __restrict__ row_map,
                const float* __restrict__ scene_mean, int beam, __nv_bfloat16* __restrict__ hp_out,
                long long plane_stride, int cpad_out, int ch_off, Grid g) {
  extern __shared__ __align__(16) float gsm[];
  const int W = g.W, H = g.H;
  float* Hs = gsm;                               // [GNR][W][256]
  float* Ss = Hs + GNR * W * kHidden;            // [GNR][W][64]
  float* Dd = Ss + GNR * W * 64;                 // [GNR][W][GD]
  float* Wt = Dd + GNR * W * GD;                 // [W][GW]
  uint64_t* bar = reinterpret_cast<uint64_t*>(Wt + W * GW);
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);    // warp-uniform for the compiler: no per-shuffle re-convergence code
  const long long s = blockIdx.x;
  const long long ss = row_map ? (long long)row_map[s] : s;
  const float* hsrc = h32 + ss * g.S * kHidden;
  const float* ssrc = scene_mean ? scene_mean + (s / beam) * (long long)H * W * 64 : nullptr;
  auto slot = [](int r) { return (r + GNR) & (GNR - 1); };

  // zero: the whole ring (row -1 and, without scene features, every scene slot) and the tables
  for (int i = tid; i < W * (GNR * (kHidden + 64 + GD) + GW); i += GT) gsm[i] = 0.f;
  if (tid == 0) {
#pragma unroll
    for (int i = 0; i < GNR; ++i) mbar_init(&bar[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto issue = [&](int r) {                      // thread 0: image row r -> its ring slot
    const int sl = slot(r);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    mbar_expect_tx(&bar[sl], (uint32_t)(W * (kHidden + (ssrc ? 64 : 0)) * sizeof(float)));
    bulk_load(Hs + sl * W * kHidden, hsrc + (long long)r * g.Wp * kHidden, (uint32_t)(W * kHidden * sizeof(float)), &bar[sl]);
    if (ssrc) bulk_load(Ss + sl * W * 64, ssrc + (long long)r * W * 64, (uint32_t)(W * 64 * sizeof(float)), &bar[sl]);
  };
  auto wait_row = [&](int r) { mbar_wait(&bar[slot(r)], (uint32_t)((r / GNR) & 1)); };

  // A(r): pair products of row r with row r-1 and inside row r
  auto phase_a = [&](int r) {
    const float4* cur_h = reinterpret_cast<const float4*>(Hs + slot(r) * W * kHidden);
    const float4* up_h = reinterpret_cast<const float4*>(Hs + slot(r - 1) * W * kHidden);
    const float4* cur_s = reinterpret_cast<const float4*>(Ss + slot(r) * W * 64);
    const float4* up_s = reinterpret_cast<const float4*>(Ss + slot(r - 1) * W * 64);
    float* drow = Dd + slot(r) * W * GD;
    const int ntask = ((W + 1) >> 1) * 16;
    for (int base = warp * 32; base < ntask; base += GT) {
      const int idx = base + lane;
      const bool active = idx < ntask;
      const int q = min(idx, ntask - 1) >> 4, j = idx & 15;
      const int x0 = 2 * q, x1 = min(x0 + 1, W - 1), x2 = min(x0 + 2, W - 1), xm = max(x0 - 1, 0);
      float2 acc[10];
#pragma unroll
      for (int k = 0; k < 10; ++k) acc[k] = make_float2(0.f, 0.f);
      auto body = [&](const float4* cur, const float4* up, int f, int per) {
        const float4 p0 = cur[x0 * per + f], p1 = cur[x1 * per + f], p2 = cur[x2 * per + f];
        const float4 um = up[xm * per + f], u0 = up[x0 * per + f], u1 = up[x1 * per + f], u2 = up[x2 * per + f];
        dot_acc(acc[0], p0, um); dot_acc(acc[1], p0, u0); dot_acc(acc[2], p0, u1); dot_acc(acc[3], p0, p1);
        dot_acc(acc[4], p0, p0);
        dot_acc(acc[5], p1, u0); dot_acc(acc[6], p1, u1); dot_acc(acc[7], p1, u2); dot_acc(acc[8], p1, p2);
        dot_acc(acc[9], p1, p1);
      };
#pragma unroll
      for (int i = 0; i < 4; ++i) body(cur_h, up_h, j + 16 * i, kHidden / 4);
      body(cur_s, up_s, j, 16);
      float d[10];
#pragma unroll
      for (int k = 0; k < 10; ++k) d[k] = acc[k].x + acc[k].y;
      // (a transposed reduction - 11 shuffles instead of 40, every lane storing its own sum - was measured and is no
      // faster: the kernel is not bound by these instructions)
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) {
#pragma unroll
        for (int k = 0; k < 10; ++k) d[k] += __shfl_xor_sync(0xffffffffu, d[k], o);
      }
      if (active && j == 0) {
        float4* o0 = reinterpret_cast<float4*>(drow + x0 * GD);
        o0[0] = make_float4(d[0], d[1], d[2], d[3]);
        o0[1] = make_float4(d[4], rsqrtf(fmaxf(d[4], 1e-12f)), 0.f, 0.f);    // tf.nn.l2_normalize's factor
        if (x0 + 1 < W) {
          float4* o1 = reinterpret_cast<float4*>(drow + (x0 + 1) * GD);
          o1[0] = make_float4(d[5], d[6], d[7], d[8]);
          o1[1] = make_float4(d[9], rsqrtf(fmaxf(d[9], 1e-12f)), 0.f, 0.f);
        }
      }
    }
  };

  // B(y): the 9 softmax weights of every cell of row y.  Neighbours outside the image get weight 0 exactly; their
  // coordinates are clamped into the row, so whatever finite value is read there never reaches the result.
  auto phase_b = [&](int y) {
    const float* Dp = Dd + slot(y - 1) * W * GD;
    const float* Dy = Dd + slot(y) * W * GD;
    const float* Dn = Dd + slot(y + 1) * W * GD;
    for (int x = tid; x < W; x += GT) {
      const int xl = max(x - 1, 0), xr = min(x + 1, W - 1);
      const float d[9] = {Dy[x * GD + 0], Dy[x * GD + 1], Dy[x * GD + 2], Dy[xl * GD + 3], Dy[x * GD + 4],
                          Dy[x * GD + 3], Dn[xl * GD + 2], Dn[x * GD + 1], Dn[xr * GD + 0]};
      const float iq[9] = {Dp[xl * GD + 5], Dp[x * GD + 5], Dp[xr * GD + 5], Dy[xl * GD + 5], Dy[x * GD + 5],
                           Dy[xr * GD + 5], Dn[xl * GD + 5], Dn[x * GD + 5], Dn[xr * GD + 5]};
      const bool rt = y > 0, rb = y < H - 1, cl = x > 0, cr = x < W - 1;
      const bool ok[9] = {rt && cl, rt, rt && cr, cl, true, cr, rb && cl, rb, rb && cr};
      const float inv_p = iq[4];
      float e[9], m = -INFINITY;
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        e[k] = d[k] * inv_p * iq[k];
        if (ok[k]) m = fmaxf(m, e[k]);
      }
      float sum = 0.f;
#pragma unroll
      for (int k = 0; k < 9; ++k) { e[k] = ok[k] ? __expf(e[k] - m) : 0.f; sum += e[k]; }
      const float inv_sum = 1.0f / sum;
      float4* wo = reinterpret_cast<float4*>(Wt + x * GW);
      wo[0] = make_float4(e[0] * inv_sum, e[1] * inv_sum, e[2] * inv_sum, e[3] * inv_sum);
      wo[1] = make_float4(e[4] * inv_sum, e[5] * inv_sum, e[6] * inv_sum, e[7] * inv_sum);
      wo[2] = make_float4(e[8] * inv_sum, 0.f, 0.f, 0.f);
    }
  };

  // C(y): h'_p = h_p + sum_q a_pq h_q for 3 consecutive cells per warp; lane = channels [4 lane, +4) and [128 + 4 lane, +4)
  auto phase_c = [&](int y) {
    const float4* rows3[3] = {reinterpret_cast<const float4*>(Hs + slot(y - 1) * W * kHidden),
                              reinterpret_cast<const float4*>(Hs + slot(y) * W * kHidden),
                              reinterpret_cast<const float4*>(Hs + slot(y + 1) * W * kHidden)};
    const int nseg = (W + 2) / 3;
    for (int seg = warp; seg < nseg; seg += GT / 32) {
      const int xb = seg * 3;
      float a[3][9];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float4* wp = reinterpret_cast<const float4*>(Wt + min(xb + c, W - 1) * GW);
        const float4 w0 = wp[0], w1 = wp[1], w2 = wp[2];
        a[c][0] = w0.x; a[c][1] = w0.y; a[c][2] = w0.z; a[c][3] = w0.w;
        a[c][4] = w1.x; a[c][5] = w1.y; a[c][6] = w1.z; a[c][7] = w1.w; a[c][8] = w2.x;
      }
      float2 o[3][4];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int k = 0; k < 4; ++k) o[c][k] = make_float2(0.f, 0.f);
      }
#pragma unroll
      for (int col = 0; col < 5; ++col) {
        const int xc = min(max(xb + col - 1, 0), W - 1);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const float4 v0 = rows3[r][xc * (kHidden / 4) + lane], v1 = rows3[r][xc * (kHidden / 4) + 32 + lane];
          const float2 v[4] = {lo2(v0), hi2(v0), lo2(v1), hi2(v1)};
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const int dx = col - 1 - c;           // column of this vector relative to cell c
            if (dx < -1 || dx > 1) continue;
            const float wgt = a[c][r * 3 + dx + 1] + ((r == 1 && dx == 0) ? 1.0f : 0.0f);   // centre: + residual
            const float2 w2 = make_float2(wgt, wgt);
#pragma unroll
            for (int k = 0; k < 4; ++k) o[c][k] = ffma2(w2, v[k], o[c][k]);
          }
        }
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        if (xb + c >= W) continue;
        const long long orow = s * g.S + (long long)y * g.Wp + xb + c;
        const float lo[4] = {o[c][0].x, o[c][0].y, o[c][1].x, o[c][1].y};
        const float hi[4] = {o[c][2].x, o[c][2].y, o[c][3].x, o[c][3].y};
        store_operand_x4<FMT>(hp_out, plane_stride, orow, ch_off + 4 * lane, cpad_out, lo);
        store_operand_x4<FMT>(hp_out, plane_stride, orow, ch_off + 128 + 4 * lane, cpad_out, hi);
      }
    }
  };

  if (tid == 0) {
    issue(0);
    if (H > 1) issue(1);
  }
  wait_row(0);
  phase_a(0);
  for (int y = 0; y < H; ++y) {
    const int r = y + 1;
    if (r < H) {
      wait_row(r);
    } else {                                     // the row below the image: zeros
      float* hz = Hs + slot(r) * W * kHidden;
      float* sz = Ss + slot(r) * W * 64;
      for (int i = tid; i < W * kHidden; i += GT) hz[i] = 0.f;
      for (int i = tid; i < W * 64; i += GT) sz[i] = 0.f;
      __syncthreads();
    }
    if (tid == 0 && y + 2 < H) issue(y + 2);     // into the slot of row y-2, free since the barrier that ended C(y-1)
    phase_a(r);
    __syncthreads();
    phase_b(y);
    __syncthreads();
    phase_c(y);
    __syncthreads();
  }
}

int gnn_attend_fwd(const float* h32, const int* row_map, const float* scene_mean, int beam,
                   void* hp_out, long long hp_plane_stride, int cpad_out, int ch_off_out,
                   long long NS, int H, int W, int P, cudaStream_t stream) {
  MVB_REQUIRE(valid_planes(P), "gnn_attend_fwd: planes P=%d not 2 or %d", P, kPlanesF16F8);
  MVB_REQUIRE(h32 && hp_out && NS > 0 && beam >= 1, "gnn_attend_fwd: bad args");
  MVB_REQUIRE(cpad_out % 8 == 0 && ch_off_out % 8 == 0, "gnn_attend_fwd: pitch/offset must be multiples of 8");
  const Grid g = make_grid(H, W);
  __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(hp_out);
  const bool f16f8 = P == kPlanesF16F8;
  // shared-memory ring formulation when a ring of image rows fits (W <= 42), else the warp-per-image-row kernel
  const size_t smem = gnn_rows_smem(W);
  if (smem <= 220 * 1024 && ch_off_out % 4 == 0 && NS < (1ll << 31)) {
    auto kernel = f16f8 ? gnn_rows_kernel<1> : gnn_rows_kernel<0>;
    MVB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<(unsigned)NS, GT, smem, stream>>>(h32, row_map, scene_mean, beam, d, hp_plane_stride, cpad_out,
                                               ch_off_out, g);
    MVB_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return MVB_OK;
  }
  const long long warps = NS * H;
  const unsigned blocks = (unsigned)((warps + GNN_WARPS - 1) / GNN_WARPS);
  auto kernel = f16f8 ? gnn_kernel<1> : gnn_kernel<0>;
  kernel<<<blocks, GNN_WARPS * 32, 0, stream>>>(h32, row_map, scene_mean, beam, d, hp_plane_stride, cpad_out,
                                               ch_off_out, NS, g);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

}  // namespace mvb
