// K-head: grid heads of the decoders, fused with the feedback path of the rollout.
//
// Reference call sites: Model.hidden2grid (code/pred_models.py:925-959; conv3x3 [3,3,256,P], no bias)
// at :401,:422,:432 (in-loop), :467 (post-loop recompute - identical weights and inputs, so the
// in-loop result IS the fetched logit/offset map) and :550 (beam); argmax -> one_hot (:411-415);
// Model.grid_emb (:912-919; tanh(conv3x3 [3,3,P,E] + b)) at :442-446 and :662-666.
//
// One CTA per sample row.  Every h row (256 fp32) is read exactly once: a warp forms the 9*P
// per-tap partial dot products of its pixel, and the 3x3 gather happens in shared memory, so the
// kernel moves 4*HW*(256+P) bytes per sample row (HBM-bound).  The class head then does the
// argmax (first index on ties, as tf.argmax) and writes the embedded one-hot - tanh(b) everywhere
// except the <=9 cells around the arg-max - as the bf16 x-planes of the next cell step; the
// regression head embeds its own dense 2-channel output the same way.  The logits-fed variant of
// the class head (training without --train_w_onehot, :426-435) embeds its dense logits map instead.
#include "mvb_common.cuh"
#include "mvb_kernels.h"

namespace mvb {

constexpr int HEAD_THREADS = 256;

// x block (channels [0,E)) of xh_next for one sample row.
//   ONEHOT: input is one_hot(amax) (POUT == 1);  else the dense map `vals` [HW][POUT] in smem.
//   FMT = 1: written in the f16f8 operand format, else as bf16x2 planes.
template <int FMT, int POUT, bool ONEHOT = (POUT == 1)>
__device__ __forceinline__ void emb_write(const float* __restrict__ vals, int amax,
                                          const float* __restrict__ We, const float* __restrict__ be,
                                          int E, __nv_bfloat16* __restrict__ xh, long long plane_stride,
                                          int cpad, long long s, const Grid& g) {
  const int hw = g.H * g.W;
  const int groups = E / 8;
  const int ay = ONEHOT ? amax / g.W : 0, ax = ONEHOT ? amax % g.W : 0;
  for (int i = threadIdx.x; i < hw * groups; i += blockDim.x) {
    const int p = i / groups, e0 = (i % groups) * 8;
    const int y = p / g.W, x = p % g.W;
    float v[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = __ldg(be + e0 + c);
    if (ONEHOT) {
      // out[p] = sum_tap onehot[p + off(tap)] * We[tap]  ->  non-zero iff amax - p is a tap offset
      const int dy = ay - y, dx = ax - x;
      if (dy >= -1 && dy <= 1 && dx >= -1 && dx <= 1) {
        const int tap = (dy + 1) * 3 + (dx + 1);
#pragma unroll
        for (int c = 0; c < 8; ++c) v[c] += __ldg(We + tap * E + e0 + c);
      }
    } else {
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const int yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
        if (yy < 0 || yy >= g.H || xx < 0 || xx >= g.W) continue;
        float in[POUT];
#pragma unroll
        for (int ci = 0; ci < POUT; ++ci) in[ci] = vals[(yy * g.W + xx) * POUT + ci];
#pragma unroll
        for (int c = 0; c < 8; ++c)
#pragma unroll
          for (int ci = 0; ci < POUT; ++ci) v[c] = fmaf(in[ci], __ldg(We + (tap * POUT + ci) * E + e0 + c), v[c]);
      }
    }
    if (FMT) {      // f16f8 operand format (mvb_common.cuh)
#pragma unroll
      for (int c = 0; c < 8; ++c) v[c] = tanhf(v[c]);
      store_f16f8_x8(xh, plane_stride, s * g.S + (long long)y * g.Wp + x, e0, cpad, v);
      continue;
    }
    uint32_t pk[kBf16Planes][4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      __nv_bfloat16 a[kBf16Planes], b[kBf16Planes];
      split_planes(tanhf(v[2 * c]), a);
      split_planes(tanhf(v[2 * c + 1]), b);
#pragma unroll
      for (int q = 0; q < kBf16Planes; ++q) pk[q][c] = pack_bf16x2(a[q], b[q]);
    }
    const long long row = s * g.S + (long long)y * g.Wp + x;
#pragma unroll
    for (int q = 0; q < kBf16Planes; ++q)
      *reinterpret_cast<uint4*>(xh + q * plane_stride + row * cpad + e0) =
          make_uint4(pk[q][0], pk[q][1], pk[q][2], pk[q][3]);
  }
}

// DENSE_FB (POUT == 1 only): the feedback embeds the logits map itself, not one_hot(argmax)
template <int FMT, int POUT, bool DENSE_FB = false>
__global__ void __launch_bounds__(HEAD_THREADS)
head_kernel(const float* __restrict__ h32, const float* __restrict__ Wo, float* __restrict__ out,
            int* __restrict__ ids_out, const float* __restrict__ We, const float* __restrict__ be,
            int E, __nv_bfloat16* __restrict__ xh_next, long long plane_stride, int cpad, Grid g) {
  extern __shared__ float sm[];
  const int hw = g.H * g.W;
  float* w_s = sm;                                // [9][256][POUT]
  float* d_s = w_s + 9 * kHidden * POUT;          // [HW][9*POUT]
  float* o_s = d_s + (size_t)hw * 9 * POUT;       // [HW][POUT]
  __shared__ float red_v[HEAD_THREADS / 32];
  __shared__ int red_i[HEAD_THREADS / 32];
  __shared__ int amax_s;
  const long long s = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // weights transposed to [tap][po][256] so a lane's 8 channels are two 128-bit words
  for (int i = threadIdx.x; i < 9 * kHidden * POUT; i += blockDim.x) {
    const int po = i % POUT, ch = (i / POUT) % kHidden, t = i / (POUT * kHidden);
    w_s[(t * POUT + po) * kHidden + ch] = Wo[i];
  }
  __syncthreads();

  // phase 1: per-pixel, per-tap partial dot products.  The class head (POUT == 1) keeps its 72
  // weights in registers; the 2-output head reads them as 128-bit shared-memory words.
  // (packed fp32 pairs: one FFMA2 per two channels - the loop is bound by instruction issue, not by the FMA pipe)
  float2 wr[POUT == 1 ? 9 : 1][4];
  if (POUT == 1) {
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const float4 a = *reinterpret_cast<const float4*>(w_s + t * kHidden + lane * 8);
      const float4 b = *reinterpret_cast<const float4*>(w_s + t * kHidden + lane * 8 + 4);
      wr[t][0] = make_float2(a.x, a.y); wr[t][1] = make_float2(a.z, a.w);
      wr[t][2] = make_float2(b.x, b.y); wr[t][3] = make_float2(b.z, b.w);
    }
  }
  // the rows of the next TWO iterations are requested before the current one is consumed (load latency, not
  // bandwidth, bounds this loop)
  // (the pixel coordinates of the prefetched row advance incrementally: no division per iteration)
  constexpr int STEP = HEAD_THREADS / 32;
  const float* hbase = h32 + s * g.S * kHidden + lane * 8;
  int py = warp / g.W, px = warp % g.W;          // pixel of the row requested next
  auto fetch = [&](float4& lo, float4& hi) {
    const float4* p4 = reinterpret_cast<const float4*>(hbase + ((long long)py * g.Wp + px) * kHidden);
    lo = __ldg(p4); hi = __ldg(p4 + 1);
    px += STEP;
    while (px >= g.W) { px -= g.W; ++py; }
  };
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 na = z4, nb = z4, ma = z4, mb = z4;
  if (warp < hw) fetch(na, nb);
  if (warp + STEP < hw) fetch(ma, mb);
  for (int q = warp; q < hw; q += STEP) {
    const float4 a = na, b = nb;
    na = ma; nb = mb;
    if (q + 2 * STEP < hw) fetch(ma, mb);
    const float2 hv[4] = {make_float2(a.x, a.y), make_float2(a.z, a.w), make_float2(b.x, b.y), make_float2(b.z, b.w)};
    float part[9 * POUT];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
#pragma unroll
      for (int po = 0; po < POUT; ++po) {
        float2 acc;
        if (POUT == 1) {
          acc = fmul2(hv[0], wr[t][0]);
#pragma unroll
          for (int c = 1; c < 4; ++c) acc = ffma2(hv[c], wr[t][c], acc);
        } else {
          const float4 wa = *reinterpret_cast<const float4*>(w_s + (t * POUT + po) * kHidden + lane * 8);
          const float4 wb = *reinterpret_cast<const float4*>(w_s + (t * POUT + po) * kHidden + lane * 8 + 4);
          acc = fmul2(hv[0], make_float2(wa.x, wa.y));
          acc = ffma2(hv[1], make_float2(wa.z, wa.w), acc);
          acc = ffma2(hv[2], make_float2(wb.x, wb.y), acc);
          acc = ffma2(hv[3], make_float2(wb.z, wb.w), acc);
        }
        part[t * POUT + po] = acc.x + acc.y;
      }
    }
    // warp totals: groups of 8 values by the folding reduction (9 shuffles per 8 values), the rest by butterflies
    constexpr int NFOLD = (9 * POUT) / 8;
#pragma unroll
    for (int f = 0; f < NFOLD; ++f) {
      const float v8[8] = {part[f * 8 + 0], part[f * 8 + 1], part[f * 8 + 2], part[f * 8 + 3],
                           part[f * 8 + 4], part[f * 8 + 5], part[f * 8 + 6], part[f * 8 + 7]};
      const float tot = warp_fold8(v8, lane);
      if ((lane & 3) == 0) d_s[q * 9 * POUT + f * 8 + warp_fold8_index(lane)] = tot;
    }
#pragma unroll
    for (int t = NFOLD * 8; t < 9 * POUT; ++t) {
      const float tot = warp_sum(part[t]);
      if (lane == 0) d_s[q * 9 * POUT + t] = tot;
    }
  }
  __syncthreads();

  // phase 2: 3x3 gather -> logits / offsets
  float best = -INFINITY;
  int best_i = 0x7fffffff;
  for (int p = threadIdx.x; p < hw; p += blockDim.x) {
    const int y = p / g.W, x = p % g.W;
    float acc[POUT];
#pragma unroll
    for (int po = 0; po < POUT; ++po) acc[po] = 0.f;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
      if (yy < 0 || yy >= g.H || xx < 0 || xx >= g.W) continue;
#pragma unroll
      for (int po = 0; po < POUT; ++po) acc[po] += d_s[(yy * g.W + xx) * 9 * POUT + t * POUT + po];
    }
#pragma unroll
    for (int po = 0; po < POUT; ++po) {
      o_s[p * POUT + po] = acc[po];
      out[(s * hw + p) * POUT + po] = acc[po];
    }
    if (POUT == 1 && acc[0] > best) { best = acc[0]; best_i = p; }  // ascending p: first max wins
  }
  int amax = 0;
  if (POUT == 1) {
    // phase 3: block arg-max, ties -> lower index (tf.argmax)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
      if (ov > best || (ov == best && oi < best_i)) { best = ov; best_i = oi; }
    }
    if (lane == 0) { red_v[warp] = best; red_i[warp] = best_i; }
    __syncthreads();
    if (threadIdx.x == 0) {
      float bv = red_v[0]; int bi = red_i[0];
      for (int w = 1; w < HEAD_THREADS / 32; ++w)
        if (red_v[w] > bv || (red_v[w] == bv && red_i[w] < bi)) { bv = red_v[w]; bi = red_i[w]; }
      if (bi == 0x7fffffff) bi = 0;  // all-NaN row: tf.argmax returns 0
      amax_s = bi;
      if (ids_out) ids_out[s] = bi;
    }
    __syncthreads();
    amax = amax_s;
  } else {
    __syncthreads();
  }
  // phase 4: embedded feedback input of the next cell step
  if (xh_next) emb_write<FMT, POUT, POUT == 1 && !DENSE_FB>(o_s, amax, We, be, E, xh_next, plane_stride, cpad, s, g);
}

template <int FMT>
__global__ void __launch_bounds__(HEAD_THREADS)
emb_onehot_kernel(const int* __restrict__ ids, const float* __restrict__ We, const float* __restrict__ be,
                  int E, __nv_bfloat16* __restrict__ xh_next, long long plane_stride, int cpad, Grid g) {
  const long long s = blockIdx.x;
  emb_write<FMT, 1>(nullptr, ids[s], We, be, E, xh_next, plane_stride, cpad, s, g);
}

template <int FMT>
__global__ void __launch_bounds__(HEAD_THREADS)
emb_dense_kernel(const float* __restrict__ x, const float* __restrict__ We, const float* __restrict__ be,
                 int E, __nv_bfloat16* __restrict__ xh_next, long long plane_stride, int cpad, Grid g) {
  extern __shared__ float sm[];
  const long long s = blockIdx.x;
  const int hw = g.H * g.W;
  for (int i = threadIdx.x; i < hw * 2; i += blockDim.x) sm[i] = x[s * hw * 2 + i];
  __syncthreads();
  emb_write<FMT, 2>(sm, 0, We, be, E, xh_next, plane_stride, cpad, s, g);
}

template <int FMT, int POUT, bool DENSE_FB = false>
static int launch_head(const float* h32, const float* Wo, float* out, int* ids_out, const float* We,
                       const float* be, int E, void* xh_next, long long plane_stride, int cpad,
                       long long NS, const Grid& g, cudaStream_t stream) {
  const size_t smem = sizeof(float) * ((size_t)9 * kHidden * POUT + (size_t)g.H * g.W * (9 * POUT + POUT));
  static SmemOptIn opt;
  if (smem > 48 * 1024) {
    MVB_REQUIRE(smem <= 227 * 1024, "head_fwd: grid %dx%d needs %zu B shared memory", g.H, g.W, smem);
    MVB_CHECK_CUDA(smem_opt_in(opt, head_kernel<FMT, POUT, DENSE_FB>, smem));
  }
  head_kernel<FMT, POUT, DENSE_FB><<<(unsigned)NS, HEAD_THREADS, smem, stream>>>(
      h32, Wo, out, ids_out, We, be, E, reinterpret_cast<__nv_bfloat16*>(xh_next), plane_stride, cpad, g);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int head_fwd(const float* h32, const float* Wo, int Pout, float* out, int* ids_out, const float* We,
             const float* be, int E, void* xh_next, long long plane_stride, int cpad, long long NS,
             int H, int W, int P, cudaStream_t stream) {
  MVB_REQUIRE(valid_planes(P), "head_fwd: planes P=%d not 2 or %d", P, kPlanesF16F8);
  MVB_REQUIRE(Pout == 1 || Pout == 2, "head_fwd: Pout=%d", Pout);
  MVB_REQUIRE(h32 && Wo && out && NS > 0, "head_fwd: bad args");
  if (xh_next) MVB_REQUIRE(We && be && E > 0 && E % 8 == 0 && E <= cpad - kHidden && cpad % 8 == 0,
                           "head_fwd: emb needs We/be and E (=%d) a multiple of 8 within the x block", E);
  const Grid g = make_grid(H, W);
  if (P == kPlanesF16F8)
    return Pout == 1 ? launch_head<1, 1>(h32, Wo, out, ids_out, We, be, E, xh_next, plane_stride, cpad, NS, g, stream)
                     : launch_head<1, 2>(h32, Wo, out, ids_out, We, be, E, xh_next, plane_stride, cpad, NS, g, stream);
  return Pout == 1 ? launch_head<0, 1>(h32, Wo, out, ids_out, We, be, E, xh_next, plane_stride, cpad, NS, g, stream)
                   : launch_head<0, 2>(h32, Wo, out, ids_out, We, be, E, xh_next, plane_stride, cpad, NS, g, stream);
}

int head_class_fwd_dense(const float* h32, const float* Wo, float* out, int* ids_out, const float* We,
                         const float* be, int E, void* xh_next, long long plane_stride, int cpad, long long NS,
                         int H, int W, int P, cudaStream_t stream) {
  MVB_REQUIRE(P == kBf16Planes, "head_class_fwd_dense: planes P=%d must be 2 (a training format)", P);
  MVB_REQUIRE(h32 && Wo && out && NS > 0, "head_class_fwd_dense: bad args");
  if (xh_next) MVB_REQUIRE(We && be && E > 0 && E % 8 == 0 && E <= cpad - kHidden && cpad % 8 == 0,
                           "head_class_fwd_dense: emb needs We/be and E (=%d) a multiple of 8 within the x block", E);
  const Grid g = make_grid(H, W);
  return launch_head<0, 1, true>(h32, Wo, out, ids_out, We, be, E, xh_next, plane_stride, cpad, NS, g, stream);
}

int emb_onehot_fwd(const int* ids, const float* We, const float* be, int E, void* xh_next,
                   long long plane_stride, int cpad, long long NS, int H, int W, int P,
                   cudaStream_t stream) {
  MVB_REQUIRE(valid_planes(P), "emb_onehot_fwd: planes P=%d not 2 or %d", P, kPlanesF16F8);
  MVB_REQUIRE(ids && We && be && xh_next && NS > 0 && E > 0 && E % 8 == 0 && E <= cpad - kHidden,
              "emb_onehot_fwd: bad args (E=%d)", E);
  const Grid g = make_grid(H, W);
  __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(xh_next);
  if (P == kPlanesF16F8) emb_onehot_kernel<1><<<(unsigned)NS, HEAD_THREADS, 0, stream>>>(ids, We, be, E, d, plane_stride, cpad, g);
  else emb_onehot_kernel<0><<<(unsigned)NS, HEAD_THREADS, 0, stream>>>(ids, We, be, E, d, plane_stride, cpad, g);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int emb_dense_fwd(const float* x, const float* We, const float* be, int E, void* xh_next,
                  long long plane_stride, int cpad, long long NS, int H, int W, int P,
                  cudaStream_t stream) {
  MVB_REQUIRE(valid_planes(P), "emb_dense_fwd: planes P=%d not 2 or %d", P, kPlanesF16F8);
  MVB_REQUIRE(x && We && be && xh_next && NS > 0 && E > 0 && E % 8 == 0 && E <= cpad - kHidden,
              "emb_dense_fwd: bad args (E=%d)", E);
  const Grid g = make_grid(H, W);
  __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(xh_next);
  const size_t smem = sizeof(float) * (size_t)H * W * 2;
  MVB_REQUIRE(smem <= 48 * 1024, "emb_dense_fwd: grid too large");
  if (P == kPlanesF16F8) emb_dense_kernel<1><<<(unsigned)NS, HEAD_THREADS, smem, stream>>>(x, We, be, E, d, plane_stride, cpad, g);
  else emb_dense_kernel<0><<<(unsigned)NS, HEAD_THREADS, smem, stream>>>(x, We, be, E, d, plane_stride, cpad, g);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

}  // namespace mvb
