// Post-decode metrics of the multi-future evaluation on the device (SURVEY.md section 8 row f-3): what the
// reference computes per trajectory in host numpy loops AFTER pickling the decoded outputs,
//   minADE / minFDE over the K predicted trajectories   code/multifuture_eval_trajs.py:41-78 (get_min :16-21)
//   negative log-likelihood of the ground-truth cells     code/multifuture_eval_trajs_prob.py:113-131 (get_hw_prob,
//   under the beam mixture                                compute_nll, softmax :20-44), main loop :170-197
// here as two small kernels over the tensors the decoder already holds in HBM (mvb_decode_trajectories output,
// beam_outputs), so only [N,G]-sized results travel to the host instead of [N,K,Tp,HW] logits.
#include "mvb_common.cuh"
#include "mvb_kernels.h"
#include <float.h>

namespace mvb {

// dx^2 + dy^2 as numpy forms it: both squares rounded, then the add.  Written with explicit round-to-nearest
// intrinsics because nvcc would otherwise contract it to dx*dx then fma(dy, dy, .), which differs from numpy in the
// last bit whenever dy^2 is not exact in double (coordinates of unlike magnitude), and can flip a near-tie selection.
__device__ __forceinline__ double sq_dist(double dx, double dy) {
  return __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
}

// One warp per (trajectory n, ground-truth future g).
//   pred [N,K,Tp,2] fp32, gt [N,G,Tg,2] fp32, gt_len [N,G] (0 = no such future; <= min(Tp,Tg))
// The arithmetic is the reference's, in double like numpy on the float64 arrays it builds: per prediction k the
// per-step errors d[t] = sqrt((gx-px)^2 + (gy-py)^2), t < len; minADE picks the k with the smallest LEFT-TO-RIGHT sum
// of d (python `sum`), first index on ties (`list.index(min)`), and reports ITS per-step errors; minFDE picks the
// smallest d[len-1] the same way.
__global__ void min_ade_fde_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                   const int* __restrict__ gt_len, double* __restrict__ ade_err,
                                   int* __restrict__ ade_idx, double* __restrict__ fde, int* __restrict__ fde_idx,
                                   long long NG, int G, int K, int Tp, int Tg) {
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= NG) return;
  const long long n = wid / G;
  const int len = gt_len[wid];
  const float* g = gt + wid * Tg * 2;
  double best_sum = DBL_MAX, best_last = DBL_MAX;
  int best_k = 0x7fffffff, best_lk = 0x7fffffff;
  if (len > 0) {
    for (int k = lane; k < K; k += 32) {
      const float* p = pred + ((n * K + k) * Tp) * 2;
      double s = 0.0, last = 0.0;
      for (int t = 0; t < len; ++t) {
        const double dx = (double)g[2 * t] - (double)p[2 * t], dy = (double)g[2 * t + 1] - (double)p[2 * t + 1];
        last = sqrt(sq_dist(dx, dy));
        s += last;
      }
      if (s < best_sum) { best_sum = s; best_k = k; }          // lanes scan k in increasing order: first index wins
      if (last < best_last) { best_last = last; best_lk = k; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double os = __shfl_xor_sync(0xffffffffu, best_sum, o);
      const int ok = __shfl_xor_sync(0xffffffffu, best_k, o);
      if (os < best_sum || (os == best_sum && ok < best_k)) { best_sum = os; best_k = ok; }
      const double ol = __shfl_xor_sync(0xffffffffu, best_last, o);
      const int olk = __shfl_xor_sync(0xffffffffu, best_lk, o);
      if (ol < best_last || (ol == best_last && olk < best_lk)) { best_last = ol; best_lk = olk; }
    }
  }
  for (int t = lane; t < Tg; t += 32) {
    double d = 0.0;
    if (t < len) {
      const float* p = pred + ((n * K + best_k) * Tp) * 2;
      const double dx = (double)g[2 * t] - (double)p[2 * t], dy = (double)g[2 * t + 1] - (double)p[2 * t + 1];
      d = sqrt(sq_dist(dx, dy));
    }
    ade_err[wid * Tg + t] = d;
  }
  if (lane == 0) {
    ade_idx[wid] = len > 0 ? best_k : -1;
    fde[wid] = len > 0 ? best_last : 0.0;
    fde_idx[wid] = len > 0 ? best_lk : -1;
  }
}

// One block per (trajectory n, evaluated step j): the probability of each ground-truth cell under the beam mixture
//   p[v] = sum_b softmax_b(logprobs[n,:])[b] * softmax_v(logits[n,b,t_j,:])[v]
// and nll[n,j] = mean_g -log(p[gt_idx[n,j,g]] + DBL_EPSILON) over the present futures (gt_idx >= 0); count[n,j]
// = their number (0: the reference skips the step).  fp32 softmaxes like the reference's float32 numpy arrays, the
// logarithm in double (np.finfo(float).eps makes that sum float64).
constexpr int NLL_THREADS = 256;
__global__ void __launch_bounds__(NLL_THREADS)
beam_nll_kernel(const float* __restrict__ logits, const float* __restrict__ logprobs, const int* __restrict__ gt_idx,
                const int* __restrict__ steps, double* __restrict__ nll, int* __restrict__ count, int K, int Tp, int V,
                int J, int G) {
  extern __shared__ float sm[];            // [K] beam weights, [K] row max, [K] row sum(exp)
  float* wb = sm; float* mx = sm + K; float* se = sm + 2 * K;
  const long long n = blockIdx.x / J;
  const int j = blockIdx.x % J, t = steps[j];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = NLL_THREADS / 32;
  if (t < 0 || t >= Tp) {                  // step beyond this rollout
    if (threadIdx.x == 0) { nll[n * J + j] = 0.0; count[n * J + j] = 0; }
    return;
  }
  if (warp == 0) {                         // softmax over the K beam scores
    float m = -INFINITY;
    for (int b = lane; b < K; b += 32) m = fmaxf(m, logprobs[n * K + b]);
    m = warp_max(m);
    float s = 0.f;
    for (int b = lane; b < K; b += 32) s += expf(logprobs[n * K + b] - m);
    s = warp_sum(s);
    for (int b = lane; b < K; b += 32) wb[b] = expf(logprobs[n * K + b] - m) / s;
  }
  for (int b = warp; b < K; b += nwarps) {   // per beam: max and sum(exp) of its logit row at step t
    const float* row = logits + ((n * K + b) * (long long)Tp + t) * V;
    float m = -INFINITY;
    for (int v = lane; v < V; v += 32) m = fmaxf(m, row[v]);
    m = warp_max(m);
    float s = 0.f;
    for (int v = lane; v < V; v += 32) s += expf(row[v] - m);
    s = warp_sum(s);
    if (lane == 0) { mx[b] = m; se[b] = s; }
  }
  __syncthreads();
  double acc = 0.0; int cnt = 0;
  for (int gi = threadIdx.x; gi < G; gi += NLL_THREADS) {
    const int v = gt_idx[(n * J + j) * G + gi];
    if (v < 0 || v >= V) continue;
    float p = 0.f;
    for (int b = 0; b < K; ++b)
      p += expf(logits[((n * K + b) * (long long)Tp + t) * V + v] - mx[b]) / se[b] * wb[b];
    acc += -log((double)p + DBL_EPSILON);
    ++cnt;
  }
  // block reduction (G is small: a handful of futures per trajectory)
  __shared__ double racc[NLL_THREADS / 32];
  __shared__ int rcnt[NLL_THREADS / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { acc += __shfl_xor_sync(0xffffffffu, acc, o); cnt += __shfl_xor_sync(0xffffffffu, cnt, o); }
  if (lane == 0) { racc[warp] = acc; rcnt[warp] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0; int c = 0;
    for (int w = 0; w < nwarps; ++w) { a += racc[w]; c += rcnt[w]; }
    nll[n * J + j] = c ? a / c : 0.0;
    count[n * J + j] = c;
  }
}

int min_ade_fde(const float* pred, const float* gt, const int* gt_len, double* ade_err, int* ade_idx, double* fde,
                int* fde_idx, long long N, int G, int K, int Tp, int Tg, cudaStream_t stream) {
  MVB_REQUIRE(pred && gt && gt_len && ade_err && ade_idx && fde && fde_idx, "min_ade_fde: null pointer");
  MVB_REQUIRE(N > 0 && G > 0 && K > 0 && Tp > 0 && Tg > 0 && Tg <= Tp, "min_ade_fde: bad sizes N=%lld G=%d K=%d Tp=%d Tg=%d", N, G, K, Tp, Tg);
  const long long warps = N * G;
  const unsigned blocks = (unsigned)((warps * 32 + 255) / 256);
  min_ade_fde_kernel<<<blocks, 256, 0, stream>>>(pred, gt, gt_len, ade_err, ade_idx, fde, fde_idx, warps, G, K, Tp, Tg);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int beam_nll(const float* logits, const float* logprobs, const int* gt_idx, const int* steps, double* nll, int* count,
             long long N, int K, int Tp, int V, int J, int G, cudaStream_t stream) {
  MVB_REQUIRE(logits && logprobs && gt_idx && steps && nll && count, "beam_nll: null pointer");
  MVB_REQUIRE(N > 0 && K > 0 && Tp > 0 && V > 0 && J > 0 && G > 0 && N * J < 0x7fffffffLL, "beam_nll: bad sizes");
  beam_nll_kernel<<<(unsigned)(N * J), NLL_THREADS, 3 * K * sizeof(float), stream>>>(logits, logprobs, gt_idx, steps, nll,
                                                                                      count, K, Tp, V, J, G);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

}  // namespace mvb
