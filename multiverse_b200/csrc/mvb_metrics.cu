// Post-decode metrics of the multi-future evaluation on the device (SURVEY.md section 8 row f-3): what the
// reference computes per trajectory in host numpy loops AFTER pickling the decoded outputs,
//   minADE / minFDE over the K predicted trajectories   code/multifuture_eval_trajs.py:41-78 (get_min :16-21)
//   negative log-likelihood of the ground-truth cells     code/multifuture_eval_trajs_prob.py:113-131 (get_hw_prob,
//   under the beam mixture                                compute_nll, softmax :20-44), main loop :170-197
// here as two small kernels over the tensors the decoder already holds in HBM (mvb_decode_trajectories output,
// beam_outputs), so only [N,G]-sized results travel to the host instead of [N,K,Tp,HW] logits.
// The same minADE / minFDE code also scores the decode's selected cells directly (centre + offset in fp64, as
// multifuture_inference.py forms its points), the NLL takes per-row lengths of a ragged decode, and points_to_cells
// is the prob script's xys_to_indexes.
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

// Where the minADE / minFDE kernel reads its points: prediction k of trajectory n at step t, and future g (row ng =
// n * G + g) at step t, both as the double numpy computes with.
struct PredF32 {                 // fp32 points [N,K,Tp,2] (mvb_decode_trajectories output)
  const float* p; int K, Tp;
  __device__ __forceinline__ double2 at(long long n, int k, int t) const {
    const float* q = p + ((n * K + k) * Tp + t) * 2;
    return make_double2((double)q[0], (double)q[1]);
  }
};
struct PredCells {               // selected cells int32 [N,K,Tp] + their fp32 offsets [N,K,Tp,2], fp64 centres [V,2]
  const int* ids; const float* offs; const double* centers; int K, Tp, center_only;
  __device__ __forceinline__ double2 at(long long n, int k, int t) const {
    const long long i = (n * K + k) * Tp + t;
    const int v = ids[i];
    if (center_only) return make_double2(centers[2 * v], centers[2 * v + 1]);
    // one fp64 add of the widened offset: `centre + reg` of multifuture_inference.py:504-517 on float64 centres
    return make_double2(__dadd_rn(centers[2 * v], (double)offs[2 * i]), __dadd_rn(centers[2 * v + 1], (double)offs[2 * i + 1]));
  }
};
struct GtF32 {
  const float* g; int Tg;
  __device__ __forceinline__ double2 at(long long ng, int t) const {
    return make_double2((double)g[(ng * Tg + t) * 2], (double)g[(ng * Tg + t) * 2 + 1]);
  }
};
struct GtF64 {
  const double* g; int Tg;
  __device__ __forceinline__ double2 at(long long ng, int t) const {
    return make_double2(g[(ng * Tg + t) * 2], g[(ng * Tg + t) * 2 + 1]);
  }
};

template <class Pred, class Gt>
__device__ __forceinline__ double step_error(const Pred& pred, const Gt& gt, long long n, int k, long long ng, int t) {
  const double2 p = pred.at(n, k, t), g = gt.at(ng, t);
  return sqrt(sq_dist(g.x - p.x, g.y - p.y));
}

// One warp per (trajectory n, ground-truth future g).
//   gt_len [N,G] (0 = no such future; <= the prediction's length)
// The arithmetic is the reference's, in double like numpy on the float64 arrays it builds: per prediction k the
// per-step errors d[t] = sqrt((gx-px)^2 + (gy-py)^2), t < len; minADE picks the k with the smallest LEFT-TO-RIGHT sum
// of d (python `sum`), first index on ties (`list.index(min)`), and reports ITS per-step errors; minFDE picks the
// smallest d[len-1] the same way.  With row_len (the predictions' lengths [N], may be NULL) a future longer than its
// row's predictions, or a row longer than Tp, is not scored and sets err bit 1 (the script's `assert len(pred_out) >=
// pred_len`); with V > 0 a cell id outside [0, V) sets bit 2.
template <class Pred, class Gt>
__global__ void min_ade_fde_kernel(Pred pred, Gt gt, const int* __restrict__ gt_len, const int* __restrict__ row_len,
                                   const int* __restrict__ ids, int V, int* __restrict__ err,
                                   double* __restrict__ ade_err, int* __restrict__ ade_idx, double* __restrict__ fde,
                                   int* __restrict__ fde_idx, long long NG, int G, int K, int Tp, int Tg) {
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= NG) return;
  const long long n = wid / G;
  int len = gt_len[wid];
  if (row_len && len > 0 && (len > row_len[n] || row_len[n] > Tp)) {
    if (lane == 0) atomicOr(err, 1);
    len = 0;
  }
  if (V > 0 && len > 0) {        // the cells this future reads, checked before any centre is loaded
    bool bad = false;
    for (int i = lane; i < K * len; i += 32) {
      const int v = ids[(n * K + i / len) * Tp + i % len];
      bad |= v < 0 || v >= V;
    }
    if (__any_sync(0xffffffffu, bad)) {
      if (lane == 0) atomicOr(err, 2);
      len = 0;
    }
  }
  double best_sum = DBL_MAX, best_last = DBL_MAX;
  int best_k = 0x7fffffff, best_lk = 0x7fffffff;
  if (len > 0) {
    for (int k = lane; k < K; k += 32) {
      double s = 0.0, last = 0.0;
      for (int t = 0; t < len; ++t) {
        last = step_error(pred, gt, n, k, wid, t);
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
  for (int t = lane; t < Tg; t += 32) ade_err[wid * Tg + t] = t < len ? step_error(pred, gt, n, best_k, wid, t) : 0.0;
  if (lane == 0) {
    ade_idx[wid] = len > 0 ? best_k : -1;
    fde[wid] = len > 0 ? best_last : 0.0;
    fde_idx[wid] = len > 0 ? best_lk : -1;
  }
}

// One thread per point: xys_to_indexes of code/multifuture_eval_trajs_prob.py:45-63 on fp64 frame pixels.  Per axis
// i = ceil(c / gap) (IEEE division), 0 -> 1, minus 1, then numpy's indexing: -size <= i < 0 wraps, anything else
// outside [0, size) (NaN included) is an IndexError (err = 1, cell -1).
__device__ __forceinline__ bool axis_cell(double c, double gap, int size, int* out) {
  const double q = ceil(__ddiv_rn(c, gap));
  if (!(q >= -(double)size && q <= (double)size)) return false;
  long long i = (long long)q;
  i = (i == 0 ? 1 : i) - 1;
  if (i < -size) return false;
  *out = (int)(i < 0 ? i + size : i);
  return true;
}

__global__ void points_to_cells_kernel(const double* __restrict__ pts, int* __restrict__ cells, int* __restrict__ err,
                                       long long P, int H, int W, double h_gap, double w_gap) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= P) return;
  int x, y;
  const bool ok = axis_cell(pts[2 * i], w_gap, W, &x) & axis_cell(pts[2 * i + 1], h_gap, H, &y);
  cells[i] = ok ? y * W + x : -1;
  if (!ok) atomicOr(err, 1);
}

// One block per (trajectory n, evaluated step j): the probability of each ground-truth cell under the beam mixture
//   p[v] = sum_b softmax_b(logprobs[n,:])[b] * softmax_v(logits[n,b,t_j,:])[v]
// and nll[n,j] = mean_g -log(p[gt_idx[n,j,g]] + DBL_EPSILON) over the present futures (gt_idx >= 0); count[n,j]
// = their number (0: the reference skips the step, and a step at or past the row's length, lengths[n] or Tp without
// lengths, is not evaluated).  fp32 softmaxes like the reference's float32 numpy arrays, the
// logarithm in double (np.finfo(float).eps makes that sum float64).
constexpr int NLL_THREADS = 256;
__global__ void __launch_bounds__(NLL_THREADS)
beam_nll_kernel(const float* __restrict__ logits, const float* __restrict__ logprobs, const int* __restrict__ lengths,
                const int* __restrict__ gt_idx, const int* __restrict__ steps, double* __restrict__ nll,
                int* __restrict__ count, int K, int Tp, int V, int J, int G) {
  extern __shared__ float sm[];            // [K] beam weights, [K] row max, [K] row sum(exp)
  float* wb = sm; float* mx = sm + K; float* se = sm + 2 * K;
  const long long n = blockIdx.x / J;
  const int j = blockIdx.x % J, t = steps[j];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = NLL_THREADS / 32;
  if (t < 0 || t >= (lengths ? min(lengths[n], Tp) : Tp)) {    // step beyond this rollout
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
  min_ade_fde_kernel<<<blocks, 256, 0, stream>>>(PredF32{pred, K, Tp}, GtF32{gt, Tg}, gt_len, nullptr, nullptr, 0,
                                                 nullptr, ade_err, ade_idx, fde, fde_idx, warps, G, K, Tp, Tg);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int min_ade_fde_cells(const int* ids, const float* offs, const double* centers, int center_only, const int* lengths,
                      const double* gt, const int* gt_len, double* ade_err, int* ade_idx, double* fde, int* fde_idx,
                      int* err, long long N, int G, int K, int Tp, int V, int Tg, cudaStream_t stream) {
  MVB_REQUIRE(ids && (offs || center_only) && centers && lengths && gt && gt_len && ade_err && ade_idx && fde &&
              fde_idx && err, "min_ade_fde_cells: null pointer");
  MVB_REQUIRE(N > 0 && G > 0 && K > 0 && Tp > 0 && V > 0 && Tg > 0,
              "min_ade_fde_cells: bad sizes N=%lld G=%d K=%d Tp=%d V=%d Tg=%d", N, G, K, Tp, V, Tg);
  const long long warps = N * G;
  const unsigned blocks = (unsigned)((warps * 32 + 255) / 256);
  min_ade_fde_kernel<<<blocks, 256, 0, stream>>>(PredCells{ids, offs, centers, K, Tp, center_only}, GtF64{gt, Tg},
                                                 gt_len, lengths, ids, V, err, ade_err, ade_idx, fde, fde_idx, warps,
                                                 G, K, Tp, Tg);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int points_to_cells(const double* points, int* cells, int* err, long long P, int scene_h, int scene_w, int video_h,
                    int video_w, cudaStream_t stream) {
  MVB_REQUIRE(points && cells && err, "points_to_cells: null pointer");
  MVB_REQUIRE(P > 0 && scene_h > 0 && scene_w > 0 && video_h > 0 && video_w > 0, "points_to_cells: bad sizes");
  // the script's gaps, video_w * 1.0 / scene_w in Python floats
  const double w_gap = (double)video_w / (double)scene_w, h_gap = (double)video_h / (double)scene_h;
  points_to_cells_kernel<<<(unsigned)((P + 255) / 256), 256, 0, stream>>>(points, cells, err, P, scene_h, scene_w,
                                                                          h_gap, w_gap);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int beam_nll(const float* logits, const float* logprobs, const int* lengths, const int* gt_idx, const int* steps,
             double* nll, int* count, long long N, int K, int Tp, int V, int J, int G, cudaStream_t stream) {
  MVB_REQUIRE(logits && logprobs && gt_idx && steps && nll && count, "beam_nll: null pointer");
  MVB_REQUIRE(N > 0 && K > 0 && Tp > 0 && V > 0 && J > 0 && G > 0 && N * J < 0x7fffffffLL, "beam_nll: bad sizes");
  beam_nll_kernel<<<(unsigned)(N * J), NLL_THREADS, 3 * K * sizeof(float), stream>>>(logits, logprobs, lengths, gt_idx,
                                                                                      steps, nll, count, K, Tp, V, J, G);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

}  // namespace mvb
