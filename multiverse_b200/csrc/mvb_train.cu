// Backward of the ConvLSTM cell (BPTT step), for Trainer (code/pred_models.py:1636-1742; the
// reference gets these from tf.gradients :1698 through tf.contrib.rnn.ConvLSTMCell).
//
//   lstm_gates_bwd   pointwise: (dh_t, dc_t, gates_t, c_{t-1}, c_t) -> dG_t (pre-activation gate
//                    gradients, bf16 planes, packed column order), dc_{t-1}, dbias
//   cell dgrad       dxh[r, c]  = sum_tap sum_g dG[r - shift(tap), g] * W[tap, c, g]
//                    = one wgmma implicit GEMM  [R, 9*1024] x [9*1024, cpad]   (same halo trick
//                    as the forward: a tap is a constant row shift of the dG matrix)
//   cell wgrad       dW[tap, c, g] = sum_r xh[r + shift(tap), c] * dG[r, g]
//                    = wgmma GEMM  dG^T [1024, R] x xh_tap [R, cpad] with K = the halo rows: both operands are
//                    read MN-major straight from the row-major planes (dG [2][R][1024], xh [2][R][cpad]) and the
//                    tap is a row shift of the TMA box, so no transposed copy exists.  Work items = 8 M tiles of 128
//                    gate columns x N tiles of (tap, channel) units x k-splits; every (tile, k-split) adds into its
//                    own fp32 slab of dW, which unpack_cell_wgrad sums (no atomics).
// Both GEMMs use the forward kernel's bf16x2 operand format (products a0*b0 + a0*b1 + a1*b0) and the same
// TMA / mbarrier pipeline with register accumulators.  dgrad tiles: two N tiles of cpad/2 (cpad 288, 320) or of 192
// / 256 columns (wider x blocks; the columns past cpad are zero-filled by TMA and not stored) when the x block is
// needed, one N = 256 tile (h block only) when it is not (regression encoder).
// Algorithmic FLOPs: dgrad = wgrad = forward (2*R*9*cpad*1024 each).
#include "mvb_common.cuh"
#include "mvb_kernels.h"
#include <stdlib.h>

namespace mvb {

constexpr int G_BLOCK_M = 128;                         // two MMA warpgroups of 64 rows
constexpr int G_BLOCK_K = 32;
constexpr int G_MMA_K = 16;
constexpr int G_MAX_BN = 256;
constexpr int G_THREADS = 384;
constexpr int G_A_PLANE = G_BLOCK_M * G_BLOCK_K * 2;   // 8 KB
constexpr int G_B_PLANE = G_MAX_BN * G_BLOCK_K * 2;    // 16 KB (smaller N tiles use part of it)
constexpr uint32_t G_SW64_LAYOUT = kSwizzle64B;
constexpr uint32_t G_SW64_SBO = 512;

enum { MODE_DGRAD = 0, MODE_WGRAD_MN = 1 };

struct GemmCfg {
  static constexpr int A_BYTES = kBf16Planes * G_A_PLANE;
  static constexpr int STAGE_BYTES = A_BYTES + kBf16Planes * G_B_PLANE;
  static constexpr int STAGES = (227 * 1024 - 2048) / STAGE_BYTES > 8 ? 8 : (227 * 1024 - 2048) / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
};

struct GemmParams {
  float* out;          // dgrad: [R, cpad] fp32;  wgrad: [ksplit][1024, 9*cpad] fp32 accumulator slabs (+=)
  long long R;         // halo rows
  int H, W;
  int cpad, bn;        // N tile
  int cxp;             // dgrad: width of the x block
  int need_x;          // dgrad: 1 -> two N tiles covering [0, cpad) (and up to 2 * bn); 0 -> one N tile [cxp, cxp+256) (h only)
  int num_kb;          // k-blocks per tile
  long long num_m_tiles;
  int num_n_tiles;
  // wgrad: operands are read MN-major straight from the row-major activations
  int ubn, nb;         // channels / 32-channel blocks of one (tap, chunk) unit
  int n_per_tap;       // units per tap (cpad / ubn)
  int upt;             // units per N tile (bn = upt * ubn): two 96-wide units are paired into N = 192
  int n_units;         // 9 * n_per_tap
  int ksplit;          // K (= halo rows) is split over this many work items, each with its own fp32 slab
  uint32_t lbo, sbo;   // descriptor strides of the MN-major SWIZZLE_64B tiles
};

// BN = N tile (columns of the accumulator).  Warpgroup 0 loads; warpgroups 1 and 2 multiply and store 64 rows each.
template <int MODE, int BN>
__global__ void __launch_bounds__(G_THREADS, 1)
pgemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
             const GemmParams prm) {
  using Cfg = GemmCfg;
  constexpr bool MN = MODE == MODE_WGRAD_MN;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const Grid g = make_grid(prm.H, prm.W);
  const long long num_tiles = prm.num_m_tiles * prm.num_n_tiles;
  const uint32_t stage_tx = (uint32_t)(Cfg::A_BYTES + kBf16Planes * BN * G_BLOCK_K * 2);

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA); prefetch_tmap(&tmB);
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    regs_dealloc<40>();
    if (warp == 0 && lane == 0) {
      // ===================== TMA producer =====================
      int stage = 0; uint32_t phase = 0;
      for (long long t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const long long mt = t / prm.num_n_tiles;
        const int ntile = (int)(t % prm.num_n_tiles);
        for (int kb = 0; kb < prm.num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
          uint8_t* sb = sa + Cfg::A_BYTES;
          mbar_expect_tx(&full_bar[stage], stage_tx);
          if (MODE == MODE_DGRAD) {
            // A = dG[rows - shift(tap), 32 gate columns];  B = Wd[N channels, tap*1024 + 32 gate columns]
            const int q = kb / 9, tap = kb - q * 9;
            const int shift = (tap / 3 - 1) * g.Wp + (tap % 3 - 1);
            tma_load_3d(sa, &tmA, &full_bar[stage], q * G_BLOCK_K, (int)(mt * G_BLOCK_M - shift), 0);
            tma_load_3d(sb, &tmB, &full_bar[stage], tap * kGates + q * G_BLOCK_K,
                        prm.need_x ? ntile * BN : prm.cxp, 0);
          } else {
            // MN-major: A = dG[32 halo rows (K), 4 blocks of 32 gate columns]; B = `upt` units, each
            // xh[32 halo rows + shift(tap), nb blocks of 32 channels]; ntile = (unit group, k-split)
            const int ks = ntile % prm.ksplit, grp = ntile / prm.ksplit;
            const int k0 = (ks * prm.num_kb + kb) * G_BLOCK_K;
            tma_load_4d(sa, &tmA, &full_bar[stage], 0, k0, (int)mt * 4, 0);
            for (int j = 0; j < prm.upt; ++j) {
              int u = grp * prm.upt + j;
              if (u >= prm.n_units) u = prm.n_units - 1;     // odd tail: duplicate, discarded by the epilogue
              const int tap = u / prm.n_per_tap, chunk = u - tap * prm.n_per_tap;
              const int shift = (tap / 3 - 1) * g.Wp + (tap % 3 - 1);
              for (int p = 0; p < kBf16Planes; ++p)
                tma_load_4d(sb + p * (BN * 64) + j * (prm.ubn * 64), &tmB, &full_bar[stage], 0, k0 + shift,
                            chunk * prm.nb, p);
            }
          }
          if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    regs_alloc<232>();
    // ===================== MMA + epilogue: rows [64 c, +64) of the tile =====================
    const int c = wg - 1;
    const bool leader = (threadIdx.x & 127) == 0;          // arrives on the barriers for the warpgroup
    constexpr uint32_t b_plane = (uint32_t)BN * G_BLOCK_K * 2;   // TMA packs planes back to back
    // this warpgroup's 64 rows: K-major: 64 rows of 64 B; MN-major: two 32-wide MN blocks of [32 K rows][64 B]
    const uint32_t a_wg = MN ? (uint32_t)c * 2 * 2048 : (uint32_t)c * 64 * 64;
    float acc[BN / 2];
    int stage = 0; uint32_t phase = 0;
    for (long long t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const long long mt = t / prm.num_n_tiles;
      const int ntile = (int)(t % prm.num_n_tiles);
      int prev = -1;
      for (int kb = 0; kb < prm.num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES);
        const uint32_t sb = sa + Cfg::A_BYTES;
        uint32_t accumulate = kb == 0 ? 0u : 1u;
        // the product of A plane pa and B plane pb over the k-block
        auto product = [&](int pa, int pb) {
#pragma unroll
          for (int k = 0; k < G_BLOCK_K / G_MMA_K; ++k) {
            uint64_t ad, bd;
            if (MN) {
              // one MMA consumes 16 K rows = two 8-row groups (sbo apart) of every 32-wide MN block
              ad = make_smem_desc(sa + pa * G_A_PLANE + a_wg + k * 2 * prm.sbo, prm.sbo, G_SW64_LAYOUT, prm.lbo);
              bd = make_smem_desc(sb + pb * b_plane + k * 2 * prm.sbo, prm.sbo, G_SW64_LAYOUT, prm.lbo);
            } else {
              ad = make_smem_desc(sa + pa * G_A_PLANE + a_wg + k * G_MMA_K * 2, G_SW64_SBO, G_SW64_LAYOUT);
              bd = make_smem_desc(sb + pb * b_plane + k * G_MMA_K * 2, G_SW64_SBO, G_SW64_LAYOUT);
            }
            wgmma_bf16<BN, MN ? 1 : 0, MN ? 1 : 0>(acc, ad, bd, accumulate);
            accumulate = 1u;
          }
        };
        wgmma_fence_regs(acc);
        wgmma_fence();
        product(0, 0);
        product(0, 1);
        product(1, 0);
        wgmma_commit();
        wgmma_fence_regs(acc);
        wgmma_wait<1>();                       // the previous k-block's MMAs have completed: refill its stage
        if (leader && prev >= 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (leader && prev >= 0) mbar_arrive(&empty_bar[prev]);
      // ===================== epilogue: registers -> fp32 global =====================
      // thread (warp w of the warpgroup, lane l) holds rows 16 w + l / 4 (+ 8) and columns 8 i + 2 (l % 4) (+ 1)
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const long long row = mt * G_BLOCK_M + 64 * c + 16 * (warp & 3) + (lane >> 2) + 8 * hr;
        bool valid;
        float* dst;
        int n_cols = BN;      // dgrad: columns of the tile inside [0, cpad)
        if (MODE == MODE_DGRAD) {
          valid = row < prm.R;
          if (valid) {
            const int rem = (int)(row % g.S);
            const int y = rem / g.Wp, x = rem - y * g.Wp;
            valid = (x < g.W) && (y < g.H);
          }
          dst = prm.out + row * prm.cpad + (prm.need_x ? ntile * BN : prm.cxp);
          n_cols = prm.need_x ? prm.cpad - ntile * BN : BN;
        } else {
          valid = row < kGates;
          dst = prm.out + (long long)(ntile % prm.ksplit) * kGates * 9LL * prm.cpad + row * (9LL * prm.cpad);
        }
        if (!valid) continue;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
          const int col = 8 * i + 2 * (lane & 3);
          if (MODE == MODE_DGRAD && col >= n_cols) continue;
          float2* d2 = reinterpret_cast<float2*>(dst + col);
          if (MN) {
            // column of the tile -> (unit, channel): dW[tap][chunk*ubn + c]; this (tile, k-split) owns its slab
            const int ju = col / prm.ubn;
            const int u = (ntile / prm.ksplit) * prm.upt + ju;
            if (u >= prm.n_units) continue;
            const int tap = u / prm.n_per_tap, chunk = u - tap * prm.n_per_tap;
            d2 = reinterpret_cast<float2*>(dst + tap * prm.cpad + chunk * prm.ubn + (col - ju * prm.ubn));
          }
          float2 o = make_float2(acc[4 * i + 2 * hr], acc[4 * i + 2 * hr + 1]);
          if (MN) { const float2 old = *d2; o.x += old.x; o.y += old.y; }
          *d2 = o;
        }
      }
    }
  }
}

// ----------------------------------------------------------------------------------
// pointwise LSTM backward
//   gates [R,1024] (activated i,j,f,o; packed column order tile*256 + gate*64 + j), c_prev, c [R,256]
//   dc_total = dc_in + dh*o*(1-tanh(c)^2);  dG = {di_pre, dj_pre, df_pre, do_pre};  dc_prev = dc_total*f
// block = 32 channel groups (8 channels each) x 8 rows
// ----------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
lstm_bwd_kernel(const float* __restrict__ gates, const float* __restrict__ c_prev,
                const float* __restrict__ c_new, const float* __restrict__ dh,
                const float* __restrict__ dc_in, __nv_bfloat16* __restrict__ dg_planes,
                long long plane_stride, float* __restrict__ dc_prev, float* __restrict__ dbias,
                long long NS, Grid g) {
  const int cg = threadIdx.x & 31;     // channel group: channels [8cg, 8cg+8)
  const int rl = threadIdx.x >> 5;     // row lane 0..7
  const int ch0 = cg * 8;
  const int colbase = (ch0 / 64) * 256 + (ch0 % 64);
  const int hw = g.H * g.W;
  float bsum[4][8];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int k = 0; k < 8; ++k) bsum[a][k] = 0.f;
  for (long long pix = (long long)blockIdx.x * 8 + rl; pix < NS * hw; pix += (long long)gridDim.x * 8) {
    const long long s = pix / hw;
    const int p = (int)(pix - s * hw);
    const long long row = s * g.S + (long long)(p / g.W) * g.Wp + (p % g.W);
    float gt[4][8], cp[8], cn[8], dhv[8], dcv[8];
    auto ld8 = [](const float* ptr, float (&o)[8]) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(ptr)), b = __ldg(reinterpret_cast<const float4*>(ptr) + 1);
      o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
    };
#pragma unroll
    for (int a = 0; a < 4; ++a) ld8(gates + row * kGates + colbase + a * 64, gt[a]);
    if (c_prev) ld8(c_prev + row * kHidden + ch0, cp);
    else {
#pragma unroll
      for (int k = 0; k < 8; ++k) cp[k] = 0.f;
    }
    ld8(c_new + row * kHidden + ch0, cn);
    ld8(dh + row * kHidden + ch0, dhv);
    if (dc_in) ld8(dc_in + row * kHidden + ch0, dcv);
    else {
#pragma unroll
      for (int k = 0; k < 8; ++k) dcv[k] = 0.f;
    }
    float dgv[4][8], dcp[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float ai = gt[0][k], aj = gt[1][k], af = gt[2][k], ao = gt[3][k];
      const float th = tanh_acc(cn[k]);
      const float dct = dcv[k] + dhv[k] * ao * (1.f - th * th);
      dgv[0][k] = dct * aj * ai * (1.f - ai);
      dgv[1][k] = dct * ai * (1.f - aj * aj);
      dgv[2][k] = dct * cp[k] * af * (1.f - af);
      dgv[3][k] = dhv[k] * th * ao * (1.f - ao);
      dcp[k] = dct * af;
#pragma unroll
      for (int a = 0; a < 4; ++a) bsum[a][k] += dgv[a][k];
    }
    float4* dc4 = reinterpret_cast<float4*>(dc_prev + row * kHidden + ch0);
    dc4[0] = make_float4(dcp[0], dcp[1], dcp[2], dcp[3]);
    dc4[1] = make_float4(dcp[4], dcp[5], dcp[6], dcp[7]);
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      uint32_t pk[kBf16Planes][4];
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        __nv_bfloat16 x0[kBf16Planes], x1[kBf16Planes];
        split_planes(dgv[a][2 * v], x0);
        split_planes(dgv[a][2 * v + 1], x1);
#pragma unroll
        for (int q = 0; q < kBf16Planes; ++q) pk[q][v] = pack_bf16x2(x0[q], x1[q]);
      }
#pragma unroll
      for (int q = 0; q < kBf16Planes; ++q)
        *reinterpret_cast<uint4*>(dg_planes + q * plane_stride + row * kGates + colbase + a * 64) =
            make_uint4(pk[q][0], pk[q][1], pk[q][2], pk[q][3]);
    }
  }
  // dbias: reduce the 8 row lanes through shared memory, one atomic per column per block
  __shared__ float red[8][32][33];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int k = 0; k < 8; ++k) red[rl][cg][a * 8 + k] = bsum[a][k];
  __syncthreads();
  if (rl == 0) {
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        float sacc = 0.f;
#pragma unroll
        for (int r = 0; r < 8; ++r) sacc += red[r][cg][a * 8 + k];
        atomicAdd(dbias + colbase + a * 64 + k, sacc);
      }
  }
}

// dgrad weights: Wd planes [2][cpad][9*1024], Wd[kc][tap*1024 + n_packed] = W_tf[tap][cin(kc)][col(n_packed)]
__global__ void pack_dgrad_kernel(const float* __restrict__ kernel, __nv_bfloat16* __restrict__ wd,
                                  int cx, int cxp, int cpad) {
  const long long ktot = 9LL * kGates;
  const long long total = (long long)cpad * ktot;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int kc = (int)(i / ktot);
    const int k = (int)(i - (long long)kc * ktot);
    const int tap = k / kGates, n = k - tap * kGates;
    const int tile = n / 256, gate = (n % 256) / 64, j = n % 64;
    const int col = gate * kHidden + tile * 64 + j;
    int cin = -1;
    if (kc < cx) cin = kc;
    else if (kc >= cxp) cin = cx + (kc - cxp);
    const float v = (cin >= 0) ? kernel[((long long)tap * (cx + kHidden) + cin) * kGates + col] : 0.f;
    __nv_bfloat16 pl[kBf16Planes];
    split_planes(v, pl);
    wd[i] = pl[0];
    wd[total + i] = pl[1];
  }
}

// dWp [1024][9*cpad] fp32 (packed) -> dkernel [3,3,cx+256,1024] (TF layout), dbias packed -> TF order
__global__ void unpack_wgrad_kernel(const float* __restrict__ dwp, const float* __restrict__ dbp,
                                    float* __restrict__ dkernel, float* __restrict__ dbiases, int cx,
                                    int cxp, int cpad, int comp, int accumulate, int slabs) {
  const int cin_tot = cx + kHidden;
  const long long total = 9LL * cin_tot * kGates;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % kGates);
    const int cin = (int)((i / kGates) % cin_tot);
    const int tap = (int)(i / ((long long)kGates * cin_tot));
    const int gate = col / kHidden, ch = col % kHidden;
    const int n = (ch / 64) * 256 + gate * 64 + (ch % 64);
    const int kc = cin < cx ? cin : cxp + (cin - cx);
    float v = 0.f;
    for (int sl = 0; sl < slabs; ++sl) {
      const float* d = dwp + (long long)sl * kGates * 9LL * cpad + (long long)n * (9LL * cpad) + tap * cpad;
      v += d[kc];
      if (comp && cin < cx) v += d[cx + cin];   // + residual block of the compensated x block
    }
    dkernel[i] = accumulate ? dkernel[i] + v : v;
    if (tap == 0 && cin == 0) dbiases[col] = accumulate ? dbiases[col] + dbp[n] : dbp[n];
  }
}

template <int MODE, int BN>
static int launch_pgemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& prm, int num_sms,
                        cudaStream_t stream) {
  using Cfg = GemmCfg;
  static SmemOptIn opt;
  MVB_CHECK_CUDA(smem_opt_in(opt, pgemm_kernel<MODE, BN>, Cfg::SMEM_BYTES));
  const long long tiles = prm.num_m_tiles * prm.num_n_tiles;
  const int grid = (int)(tiles < num_sms ? tiles : num_sms);
  pgemm_kernel<MODE, BN><<<grid, G_THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, prm);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

// x blocks of 32 to 256 channels
static bool valid_gemm_cpad(int cpad) { return cpad % 32 == 0 && cpad >= kHidden + 32 && cpad <= 2 * kHidden; }

static int num_sms_of_device(int* out) {
  int dev = 0;
  MVB_CHECK_CUDA(cudaGetDevice(&dev));
  MVB_CHECK_CUDA(cudaDeviceGetAttribute(out, cudaDevAttrMultiProcessorCount, dev));
  return MVB_OK;
}

int cell_dgrad(const void* dg_planes, const void* wd_planes, float* dxh, long long NS, int H, int W,
               int cpad, int P, int need_x, cudaStream_t stream) {
  MVB_REQUIRE(P == kBf16Planes, "cell_dgrad: planes P=%d must be 2 (the bf16x2 format)", P);
  MVB_REQUIRE(dg_planes && wd_planes && dxh && NS > 0, "cell_dgrad: bad args");
  MVB_REQUIRE(valid_gemm_cpad(cpad), "cell_dgrad: cpad=%d must be a multiple of 32 from 288 to 512", cpad);
  const int cxp = cpad - kHidden;
  const Grid g = make_grid(H, W);
  const long long R = NS * g.S;
  CUtensorMap tmA, tmB;
  int rc = encode_tmap_3d_bf16(&tmA, dg_planes, kGates, (uint64_t)R, kBf16Planes, kGates * 2ull,
                               (uint64_t)R * kGates * 2, G_BLOCK_K, G_BLOCK_M, kBf16Planes, 64);
  if (rc) return rc;
  const uint64_t ktot = 9ull * kGates;
  // with the x block: two N tiles of cpad/2 (144 / 160), or of 192 (cpad <= 384) or 256 columns; h only: one N tile
  // of 256
  const int bn = !need_x ? 256 : cpad <= 320 ? cpad / 2 : cpad <= 384 ? 192 : 256;
  rc = encode_tmap_3d_bf16(&tmB, wd_planes, ktot, (uint64_t)cpad, kBf16Planes, ktot * 2, ktot * cpad * 2, G_BLOCK_K,
                           bn, kBf16Planes, 64);
  if (rc) return rc;
  GemmParams prm = {};
  prm.out = dxh; prm.R = R; prm.H = H; prm.W = W; prm.cpad = cpad; prm.bn = bn; prm.cxp = cxp; prm.need_x = need_x;
  prm.num_kb = 9 * (kGates / G_BLOCK_K);
  prm.num_m_tiles = (R + G_BLOCK_M - 1) / G_BLOCK_M;
  prm.num_n_tiles = need_x ? 2 : 1;
  int sms = 0;
  if ((rc = num_sms_of_device(&sms))) return rc;
  switch (bn) {
    case 144: return launch_pgemm<MODE_DGRAD, 144>(tmA, tmB, prm, sms, stream);
    case 160: return launch_pgemm<MODE_DGRAD, 160>(tmA, tmB, prm, sms, stream);
    case 192: return launch_pgemm<MODE_DGRAD, 192>(tmA, tmB, prm, sms, stream);
    default: return launch_pgemm<MODE_DGRAD, 256>(tmA, tmB, prm, sms, stream);
  }
}

// K-split of the wgrad: every slab sums R / slabs halo rows, and the dW error grows with the rows a slab sums (1.5e-4
// of the 2e-4 bar at 45 k rows: micro-batch 128 of 36x18 on 2 slabs).  cpad 288: 5 slabs (its N tiles are fewer);
// cpad 320: 2; wider x blocks: 8.  At cpad 384 the whole-model gradient (summed over steps, scales and micro-batches)
// measured 3.6e-4 on 2 slabs, 2.2e-4 on 5 and 1.5e-4 on 8 (H100, micro-batch 128 of 36x18).
int cell_wgrad_mn_slabs(int cpad) { return cpad == 288 ? 5 : cpad == 320 ? 2 : 8; }

// wgrad N tiles: units of ubn channels of one tap, upt units per tile.  cpad 288: two 96-wide units (N = 192 keeps the
// MMA off the smem-bandwidth limit), cpad 320: one 160-wide unit; wider x blocks: the fewest units that fill a tile
// of 256, 192 or 160 columns with a unit width (a multiple of 32) that divides cpad.  cpad 352 and 416 (11 and 13 x
// 32) have no such unit wider than 32 channels: five 32-channel units per 160-column tile, i.e. five TMA boxes per
// plane and stage instead of one or two (correct, its cost not measured separately).
static void wgrad_units(int cpad, int* ubn, int* upt) {
  static const int kWidths[3] = {256, 192, 160};
  for (int u = 1; u <= 8; ++u)
    for (int bn : kWidths)
      if (bn % u == 0 && (bn / u) % 32 == 0 && cpad % (bn / u) == 0) { *ubn = bn / u; *upt = u; return; }
  *ubn = 32; *upt = 8;
}

int cell_wgrad_mn(const void* dg_planes, const void* xh_planes, float* dwp, long long NS, int H, int W,
                  int cpad, int P, cudaStream_t stream) {
  MVB_REQUIRE(P == kBf16Planes, "cell_wgrad_mn: planes P=%d must be 2 (the bf16x2 format)", P);
  MVB_REQUIRE(dg_planes && xh_planes && dwp && NS > 0, "cell_wgrad_mn: bad args");
  MVB_REQUIRE(valid_gemm_cpad(cpad), "cell_wgrad_mn: cpad=%d must be a multiple of 32 from 288 to 512", cpad);
  const Grid g = make_grid(H, W);
  const long long R = NS * g.S;
  GemmParams prm = {};
  wgrad_units(cpad, &prm.ubn, &prm.upt);
  prm.bn = prm.ubn * prm.upt;
  prm.nb = prm.ubn / 32; prm.n_per_tap = cpad / prm.ubn; prm.n_units = 9 * prm.n_per_tap;
  CUtensorMap tmA, tmB;
  {
    const uint64_t dims[4] = {32, (uint64_t)R, kGates / 32, (uint64_t)kBf16Planes};
    const uint64_t st[3] = {kGates * 2ull, 64, (uint64_t)R * kGates * 2};
    const uint32_t box[4] = {32, G_BLOCK_K, 4, (uint32_t)kBf16Planes};      // 128 gate columns per CTA tile
    int rc = encode_tmap_4d_bf16(&tmA, dg_planes, dims, st, box, 64);
    if (rc) return rc;
  }
  {
    const uint64_t dims[4] = {32, (uint64_t)R, (uint64_t)cpad / 32, (uint64_t)kBf16Planes};
    const uint64_t st[3] = {(uint64_t)cpad * 2, 64, (uint64_t)R * cpad * 2};
    const uint32_t box[4] = {32, G_BLOCK_K, (uint32_t)prm.nb, 1};
    int rc = encode_tmap_4d_bf16(&tmB, xh_planes, dims, st, box, 64);
    if (rc) return rc;
  }
  prm.out = dwp; prm.R = R; prm.H = H; prm.W = W; prm.cpad = cpad;
  const long long kb_total = (R + G_BLOCK_K - 1) / G_BLOCK_K;
  // work items = 8 M tiles (128 gate columns) x unit groups x k-splits: cpad 288: 8 x 14 x 5 = 560; cpad 320:
  // 8 x 18 x 2 = 288; wider x blocks 8 x (18 ... 27) x 8
  prm.ksplit = cell_wgrad_mn_slabs(cpad);
  prm.num_kb = (int)((kb_total + prm.ksplit - 1) / prm.ksplit);
  prm.num_m_tiles = kGates / G_BLOCK_M;
  prm.num_n_tiles = ((prm.n_units + prm.upt - 1) / prm.upt) * prm.ksplit;
  prm.lbo = 32 * 64;   // bytes between 32-wide MN blocks ([32 K rows][64 B] each)
  prm.sbo = 8 * 64;    // bytes between groups of 8 K rows
  int sms = 0;
  int rc = num_sms_of_device(&sms);
  if (rc) return rc;
  switch (prm.bn) {
    case 160: return launch_pgemm<MODE_WGRAD_MN, 160>(tmA, tmB, prm, sms, stream);
    case 192: return launch_pgemm<MODE_WGRAD_MN, 192>(tmA, tmB, prm, sms, stream);
    default: return launch_pgemm<MODE_WGRAD_MN, 256>(tmA, tmB, prm, sms, stream);
  }
}

int lstm_gates_bwd(const float* gates, const float* c_prev, const float* c_new, const float* dh,
                   const float* dc_in, void* dg_planes, long long plane_stride, float* dc_prev,
                   float* dbias_packed, long long NS, int H, int W, int P, cudaStream_t stream) {
  MVB_REQUIRE(P == kBf16Planes, "lstm_gates_bwd: planes P=%d must be 2 (the bf16x2 format)", P);
  MVB_REQUIRE(gates && c_new && dh && dg_planes && dc_prev && dbias_packed && NS > 0, "lstm_gates_bwd: bad args");
  const Grid g = make_grid(H, W);
  const long long pix = NS * H * W;
  const int blocks = (int)((pix + 7) / 8 < sm_count() * 8 ? (pix + 7) / 8 : sm_count() * 8);
  __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(dg_planes);
  lstm_bwd_kernel<<<blocks, 256, 0, stream>>>(gates, c_prev, c_new, dh, dc_in, d, plane_stride, dc_prev, dbias_packed,
                                              NS, g);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int pack_cell_weights_dgrad(const float* kernel, void* wd_planes, int cx, int P, cudaStream_t stream) {
  MVB_REQUIRE(P == kBf16Planes, "pack_cell_weights_dgrad: planes P=%d must be 2 (the bf16x2 format)", P);
  MVB_REQUIRE(kernel && wd_planes && cx >= 1, "pack_cell_weights_dgrad: bad args");
  const int cxp = (cx + 31) / 32 * 32, cpad = cxp + kHidden;
  __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(wd_planes);
  pack_dgrad_kernel<<<1184, 256, 0, stream>>>(kernel, d, cx, cxp, cpad);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int unpack_cell_wgrad(const float* dwp, const float* dbias_packed, float* dkernel, float* dbiases, int cx,
                      int comp, int accumulate, int slabs, cudaStream_t stream) {
  MVB_REQUIRE(dwp && dbias_packed && dkernel && dbiases && cx >= 1, "unpack_cell_wgrad: bad args");
  const int cxp = (cx + 31) / 32 * 32, cpad = cxp + kHidden;
  MVB_REQUIRE(slabs >= 1, "unpack_cell_wgrad: slabs=%d", slabs);
  unpack_wgrad_kernel<<<1184, 256, 0, stream>>>(dwp, dbias_packed, dkernel, dbiases, cx, cxp, cpad, comp, accumulate, slabs);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

}  // namespace mvb
