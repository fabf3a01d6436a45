// K-beam: the per-step selection of the K-way multi-future rollout and its back-trace.
//
// Reference: decoder_loop_fn of Model.grid_decoder_beam_search (code/pred_models.py:547-606):
// log_softmax (:557) + running score (:560) + optional diverse penalty add_div_penalty
// (:1197-1223: rank of every entry inside its own beam row, obtained there with a full
// top_k(k=V) sort + invert_permutation; here by counting - rank = #greater + #equal-with-lower-
// index, which is what a stable descending sort yields), flatten to B*V (beam 0 only while
// time <= 1, :569-573), top_k(B, sorted) (:578; ties -> lower index), score reset while
// time <= fix_num_timestep (:581-584), ids = idx % V, parents = idx // V (:588-591).
// The (c,h) gather by parent (:611-623, gather_helper :1225-1251) is not a copy in this library:
// the kernel emits row_map = n*B + parent and the next K-gnn / K-cell launch reads its state
// through it.  Back-trace: tf.while_loop at :722-764.
//
// One CTA per sample; B*V fp32 candidates live in shared memory.  Latency-bound glue (<1 % of a
// rollout step), kept bit-faithful to fp32 TF arithmetic (no FMA contraction on the penalty).
#include <cstdlib>
#include "mvb_common.cuh"
#include "mvb_kernels.h"

namespace mvb {

constexpr int BEAM_THREADS = 256;

__device__ __forceinline__ void block_argmax(float& v, int& i, float* red_v, int* red_i) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
  }
  if (lane == 0) { red_v[warp] = v; red_i[warp] = i; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float bv = red_v[0]; int bi = red_i[0];
    for (int w = 1; w < BEAM_THREADS / 32; ++w)
      if (red_v[w] > bv || (red_v[w] == bv && red_i[w] < bi)) { bv = red_v[w]; bi = red_i[w]; }
    red_v[0] = bv; red_i[0] = bi;
  }
  __syncthreads();
  v = red_v[0]; i = red_i[0];
  __syncthreads();
}

__global__ void __launch_bounds__(BEAM_THREADS)
beam_step_kernel(const float* __restrict__ logits, const float* __restrict__ score_in,
                 float* __restrict__ score_out, int* __restrict__ ids_out,
                 int* __restrict__ parents_out, int* __restrict__ row_map_out, int B, int V,
                 int first_step, int zero_scores, int diverse, float log_gamma) {
  extern __shared__ float sm[];
  float* lp = sm;            // [B][V] log-probs (+score)
  float* cand = sm + (size_t)B * V;  // [B][V] candidates (penalised)
  __shared__ float red_v[BEAM_THREADS / 32];
  __shared__ int red_i[BEAM_THREADS / 32];
  __shared__ float row_stat[2];
  const long long n = blockIdx.x;
  const int rows = first_step ? 1 : B;   // all beams are identical at time 1 (:570-573)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // 1. log_softmax per beam row + running score
  for (int b = warp; b < rows; b += BEAM_THREADS / 32) {
    const float* lg = logits + (n * B + b) * V;
    float m = -INFINITY;
    for (int v = lane; v < V; v += 32) m = fmaxf(m, lg[v]);
    m = warp_max(m);
    float s = 0.f;
    for (int v = lane; v < V; v += 32) s += expf(lg[v] - m);
    s = warp_sum(s);
    const float lse = logf(s);
    const float sc = score_in ? score_in[n * B + b] : 0.f;
    for (int v = lane; v < V; v += 32) lp[b * V + v] = __fadd_rn(__fsub_rn(__fsub_rn(lg[v], m), lse), sc);
  }
  __syncthreads();
  // 2. diverse penalty: + log(gamma) * rank within the row
  for (int i = threadIdx.x; i < rows * V; i += blockDim.x) {
    float val = lp[i];
    if (diverse) {
      const int b = i / V, v = i - b * V;
      const float* r = lp + b * V;
      int rank = 0;
      for (int u = 0; u < V; ++u) {
        const float o = r[u];
        rank += (o > val) || (o == val && u < v);
      }
      val = __fadd_rn(val, __fmul_rn(log_gamma, (float)rank));
    }
    cand[i] = val;
  }
  __syncthreads();
  // 3. top-B, descending, ties -> lower flat index
  const int ncand = rows * V;
  for (int k = 0; k < B; ++k) {
    float bv = -INFINITY; int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < ncand; i += blockDim.x) {
      const float c = cand[i];
      if (c > bv) { bv = c; bi = i; }
    }
    block_argmax(bv, bi, red_v, red_i);
    if (bi == 0x7fffffff) bi = 0;
    if (threadIdx.x == 0) {
      cand[bi] = -INFINITY;
      // exhausted candidates (B > ncand) cannot happen: V >= B in every config
      const int parent = bi / V;
      score_out[n * B + k] = zero_scores ? 0.f : bv;
      ids_out[n * B + k] = bi - parent * V;
      parents_out[n * B + k] = parent;
      row_map_out[n * B + k] = (int)(n * B) + parent;
    }
    __syncthreads();
  }
  (void)row_stat;
}

// Same selection in O(B*V) per beam row instead of the O(V^2) rank count.  With log(gamma) <= 0 (every published
// setting: gamma = 0.01, or no penalty) the penalised value lp - |log gamma|*rank is non-increasing in the rank
// order of its row, and equal values keep index order, so an entry of rank >= B is preceded by B entries of its
// own row in the global order and can never be selected: the global top-B is the top-B of the rows' top-B lists.
// Each warp extracts the top-B of its rows by B arg-max sweeps over the row in shared memory (the k-th sweep's
// winner has rank k - the same rank the count gives, ties to the lower index); warp 0 then picks the B best of
// the <= B*B candidates, ties to the lower flat index.  Bit-identical outputs to beam_step_kernel.
__device__ __forceinline__ void warp_argmax(float& v, int& i, int& aux) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    const int oa = __shfl_xor_sync(0xffffffffu, aux, o);
    if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; aux = oa; }
  }
}

__global__ void __launch_bounds__(BEAM_THREADS)
beam_step_topk_kernel(const float* __restrict__ logits, const float* __restrict__ score_in,
                      float* __restrict__ score_out, int* __restrict__ ids_out,
                      int* __restrict__ parents_out, int* __restrict__ row_map_out, int B, int V,
                      int first_step, int zero_scores, int diverse, float log_gamma) {
  extern __shared__ float sm[];
  float* lp = sm;                                   // [rows][V] log-probs + score
  float* cv = sm + (size_t)B * V;                   // [rows][B] candidate values (penalised)
  int* ci = reinterpret_cast<int*>(cv + B * B);     // [rows][B] flat indices b*V + v
  const long long n = blockIdx.x;
  const int rows = first_step ? 1 : B;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int b = warp; b < rows; b += BEAM_THREADS / 32) {
    const float* lg = logits + (n * B + b) * V;
    float* r = lp + (size_t)b * V;
    float m = -INFINITY;
    for (int v = lane; v < V; v += 32) m = fmaxf(m, lg[v]);
    m = warp_max(m);
    float s = 0.f;
    for (int v = lane; v < V; v += 32) s += expf(lg[v] - m);
    s = warp_sum(s);
    const float lse = logf(s);
    const float sc = score_in ? score_in[n * B + b] : 0.f;
    for (int v = lane; v < V; v += 32) r[v] = __fadd_rn(__fsub_rn(__fsub_rn(lg[v], m), lse), sc);
    __syncwarp();
    for (int k = 0; k < B; ++k) {
      float bv = -INFINITY; int bi = 0x7fffffff, aux = 0;
      for (int v = lane; v < V; v += 32) {
        const float c = r[v];
        if (c > bv) { bv = c; bi = v; }
      }
      warp_argmax(bv, bi, aux);
      if (lane == 0) {
        if (bi == 0x7fffffff) bi = 0;
        cv[b * B + k] = diverse ? __fadd_rn(bv, __fmul_rn(log_gamma, (float)k)) : bv;
        ci[b * B + k] = b * V + bi;
        r[bi] = -INFINITY;
      }
      __syncwarp();
    }
  }
  __syncthreads();
  if (warp == 0) {
    const int ncand = rows * B;
    for (int k = 0; k < B; ++k) {
      float bv = -INFINITY; int bi = 0x7fffffff, pos = 0;
      for (int i = lane; i < ncand; i += 32) {
        const float c = cv[i];
        const int f = ci[i];
        if (c > bv || (c == bv && f < bi)) { bv = c; bi = f; pos = i; }
      }
      warp_argmax(bv, bi, pos);
      if (lane == 0) {
        if (bi == 0x7fffffff) bi = 0;
        cv[pos] = -INFINITY;
        ci[pos] = 0x7fffffff;
        const int parent = bi / V;
        score_out[n * B + k] = zero_scores ? 0.f : bv;
        ids_out[n * B + k] = bi - parent * V;
        parents_out[n * B + k] = parent;
        row_map_out[n * B + k] = (int)(n * B) + parent;
      }
      __syncwarp();
    }
  }
}

__global__ void __launch_bounds__(256)
beam_backtrace_kernel(const int* __restrict__ step_ids, const int* __restrict__ step_parents,
                      const float* __restrict__ step_logits, int* __restrict__ out_ids,
                      float* __restrict__ out_logits, long long N, int B, int Tp, int V) {
  extern __shared__ int src[];  // [Tp] source beam of each step for this (n, b)
  const long long nb = blockIdx.x;
  const long long n = nb / B;
  const int b = (int)(nb - n * B);
  if (threadIdx.x == 0) {
    int p = b;                                     // initial parents = range(B), :714-716
    for (int tau = Tp - 1; tau >= 0; --tau) {
      const long long o = ((long long)tau * N + n) * B + p;
      src[tau] = p;
      out_ids[(n * B + b) * Tp + tau] = step_ids[o];
      p = step_parents[o];
    }
  }
  __syncthreads();
  for (int tau = 0; tau < Tp; ++tau) {
    const float* s = step_logits + (((long long)tau * N + n) * B + src[tau]) * V;
    float* d = out_logits + ((n * B + b) * (long long)Tp + tau) * V;
    for (int v = threadIdx.x; v < V; v += blockDim.x) d[v] = s[v];
  }
}

// Post-decode (SURVEY.md §8 row f-3): trajectory point = centre[cell] + offset[cell] for the K selected cells,
// what the caller does on the host with the fetched [N,K,Tp,HW] logits and [N,Tp,HW,2] offsets
// (code/multifuture_inference.py:504-517, code/pred_utils.py:460-492).  ids [N,K,Tp]; offs [Tp,N,HW,2];
// centers [HW,2] -> out [N,K,Tp,2]: 1.9 KB per trajectory leave the device instead of 680 KB.
__global__ void decode_traj_kernel(const int* __restrict__ ids, const float* __restrict__ offs,
                                   const float* __restrict__ centers, float* __restrict__ out,
                                   long long N, int K, int Tp, int V) {
  const long long total = N * K * Tp;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i % Tp);
    const long long n = i / ((long long)Tp * K);
    const int id = ids[i];
    const float2 c = *reinterpret_cast<const float2*>(centers + 2 * id);
    const float2 o = *reinterpret_cast<const float2*>(offs + (((long long)t * N + n) * V + id) * 2);
    *reinterpret_cast<float2*>(out + 2 * i) = make_float2(c.x + o.x, c.y + o.y);
  }
}

int decode_trajectories(const int* ids, const float* offs, const float* centers, float* out, long long N,
                        int K, int Tp, int V, cudaStream_t stream) {
  MVB_REQUIRE(ids && offs && centers && out && N > 0 && K > 0 && Tp > 0 && V > 0, "decode_trajectories: bad args");
  const long long total = N * K * Tp;
  const int blocks = (int)((total + 255) / 256 < sm_count() * 8 ? (total + 255) / 256 : sm_count() * 8);
  decode_traj_kernel<<<blocks, 256, 0, stream>>>(ids, offs, centers, out, N, K, Tp, V);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int beam_step(const float* logits, const float* score_in, float* score_out, int* ids_out,
              int* parents_out, int* row_map_out, long long N, int B, int V, int first_step,
              int zero_scores, int diverse, float log_gamma, cudaStream_t stream) {
  MVB_REQUIRE(logits && score_out && ids_out && parents_out && row_map_out, "beam_step: null pointer");
  MVB_REQUIRE(N > 0 && B >= 1 && V >= B, "beam_step: bad sizes N=%lld B=%d V=%d", N, B, V);
  const char* full = getenv("MVB_BEAM_FULL_RANK");   // tests: force the O(V^2) rank-count kernel
  if ((!diverse || log_gamma <= 0.f) && !(full && full[0] == '1')) {
    const size_t smem_t = sizeof(float) * ((size_t)B * V + 2 * (size_t)B * B);
    MVB_REQUIRE(smem_t <= 227 * 1024, "beam_step: B*V=%d too large for shared memory", B * V);
    static SmemOptIn opt_t;
    if (smem_t > 48 * 1024) MVB_CHECK_CUDA(smem_opt_in(opt_t, beam_step_topk_kernel, smem_t));
    beam_step_topk_kernel<<<(unsigned)N, BEAM_THREADS, smem_t, stream>>>(logits, score_in, score_out, ids_out,
                                                                         parents_out, row_map_out, B, V, first_step,
                                                                         zero_scores, diverse, log_gamma);
    MVB_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return MVB_OK;
  }
  // log(gamma) > 0 rewards high ranks: no per-row bound on the winners, use the full rank count
  const size_t smem = sizeof(float) * 2 * (size_t)B * V;
  MVB_REQUIRE(smem <= 227 * 1024, "beam_step: B*V=%d too large for shared memory", B * V);
  static SmemOptIn opt;
  if (smem > 48 * 1024) MVB_CHECK_CUDA(smem_opt_in(opt, beam_step_kernel, smem));
  beam_step_kernel<<<(unsigned)N, BEAM_THREADS, smem, stream>>>(logits, score_in, score_out, ids_out,
                                                                parents_out, row_map_out, B, V, first_step,
                                                                zero_scores, diverse, log_gamma);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

// Parent-state gather of the beam decoder without graph attention (:611-623 then straight into the cell, :631-654
// with use_gnn off): h block of the children's f16f8 operand rows <- the fp32 h of their parents' rows.  The cell's
// A stage loads 2-D TMA boxes of consecutive halo rows, and one box spans several per-sample images, so the gather
// cannot happen there: this kernel writes it.  One warp per valid cell, 8 channels per lane (the layout the graph
// attention writes, packed cvt conversions); the x block, the channel padding and the halo rows are never written.
__global__ void __launch_bounds__(256)
beam_gather_h_kernel(const float* __restrict__ h32, const int* __restrict__ row_map, __nv_bfloat16* __restrict__ hp_out,
                     long long plane_stride, int cpad_out, long long cells, Grid g) {
  const int lane = threadIdx.x & 31;
  const long long cell = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (cell >= cells) return;
  const long long hw = (long long)g.H * g.W;
  const long long s = cell / hw;
  const int p = (int)(cell - s * hw);
  const int y = p / g.W, x = p - y * g.W;
  const long long off = (long long)y * g.Wp + x;
  const float4* src = reinterpret_cast<const float4*>(h32 + ((long long)row_map[s] * g.S + off) * kHidden + lane * 8);
  const float4 a = __ldg(src), b = __ldg(src + 1);
  const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  store_f16f8_x8(hp_out, plane_stride, s * g.S + off, cpad_out - kHidden + lane * 8, cpad_out, v);
}

int beam_gather_h(const float* h32, const int* row_map, void* hp_out, long long hp_plane_stride, int cpad_out,
                  long long NS, int H, int W, cudaStream_t stream) {
  MVB_REQUIRE(h32 && row_map && hp_out, "beam_gather_h: null pointer");
  MVB_REQUIRE(NS > 0 && H > 0 && W > 0, "beam_gather_h: bad sizes NS=%lld H=%d W=%d", NS, H, W);
  MVB_REQUIRE(cpad_out >= kHidden && cpad_out % 32 == 0,
              "beam_gather_h: cpad_out=%d is not an operand pitch (a multiple of 32, >= 256)", cpad_out);
  const Grid g = make_grid(H, W);
  MVB_REQUIRE(hp_plane_stride == NS * g.S * (long long)cpad_out,
              "beam_gather_h: plane stride %lld is not NS*(H+1)*(W+1)*cpad_out", hp_plane_stride);
  const long long cells = NS * H * W;
  MVB_REQUIRE((cells + 7) / 8 < (1ll << 31), "beam_gather_h: NS=%lld too large", NS);
  beam_gather_h_kernel<<<(unsigned)((cells + 7) / 8), 256, 0, stream>>>(
      h32, row_map, reinterpret_cast<__nv_bfloat16*>(hp_out), hp_plane_stride, cpad_out, cells, g);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

// ----------------------------------------------------------------------------------
// Image-row bands of the beam decoder.  A beam's state differs from that of its sample's base rollout (the same
// recurrence fed the no-selection input tanh(b) at every step) only near the cells its ancestry selected: the folded
// one-hot input changes the pre-activations of the 5x5 cells around the selected cell, and each later step spreads
// a difference by `radius` image rows (the 3x3 convolution, plus the 3x3 graph attention when it runs).  So
//   band[k] = clamp(widen(band[parent(k)], radius) U [y(id_k) - 2, y(id_k) + 2])
// and outside its band beam k's c and h are bit for bit the base's.  From the bands, the work list of the step's
// beam cell launch: 128-row M tiles (m0, m_end) covering GEMM rows [lo (W+1), (hi+1) (W+1)) of every beam.  Bands
// that meet across a sample boundary (one ends on the last image row, the next starts on the first: only the halo
// row between them) form one run of rows, tiled as one, so full bands give the launch's own tiling.
// One CTA: three block-wide scans over the beams (run start, run end, tile offset).
// ----------------------------------------------------------------------------------
constexpr int BAND_THREADS = 1024;

static long long beam_band_capacity(long long NS, int H, int W) {
  const Grid g = make_grid(H, W);
  return NS * ((g.S + 127) / 128 + 1);     // tiles of a beam's own rows: at most one more than its span needs
}

// exclusive scan of v over the block's threads in the order of `slot`, with an associative op and its identity
template <class Op>
__device__ long long block_scan_excl(long long v, long long identity, int slot, long long* sh, Op op) {
  long long x = v;
  sh[slot] = x;
  __syncthreads();
  for (int o = 1; o < BAND_THREADS; o <<= 1) {
    const long long u = slot >= o ? sh[slot - o] : identity;
    __syncthreads();
    x = op(u, x);
    sh[slot] = x;
    __syncthreads();
  }
  const long long r = slot ? sh[slot - 1] : identity;
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(BAND_THREADS)
beam_band_kernel(const int* __restrict__ ids, const int* __restrict__ parents, const int* __restrict__ band_in,
                 int* band_out, int* __restrict__ tiles, int* __restrict__ tile_count, int NS, int K, int radius,
                 Grid g) {
  __shared__ long long sh[BAND_THREADS];
  const int t = threadIdx.x;
  const int per = (NS + BAND_THREADS - 1) / BAND_THREADS;
  const int k0 = min(NS, t * per), k1 = min(NS, k0 + per);
  for (int k = k0; k < k1; ++k) {
    const int y = ids[k] / g.W;
    int lo = y - 2, hi = y + 2;
    if (band_in) {
      const int p = k - k % K + parents[k];
      lo = min(lo, band_in[2 * p] - radius);
      hi = max(hi, band_in[2 * p + 1] + radius);
    }
    band_out[2 * k] = max(lo, 0);
    band_out[2 * k + 1] = min(hi, g.H - 1);
  }
  __syncthreads();      // every band is visible to the block
  // beam k: GEMM rows [s_k, e_k) (through the trailing halo row when the band ends on the last image row); it
  // continues the run of beam k - 1 when that one ends there and this one starts on the first image row
  auto rows = [&](int k, long long& s, long long& e) {
    const int lo = band_out[2 * k], hi = band_out[2 * k + 1];
    s = (long long)k * g.S + (long long)lo * g.Wp;
    e = hi == g.H - 1 ? (long long)(k + 1) * g.S : (long long)k * g.S + (long long)(hi + 1) * g.Wp;
  };
  auto continues = [&](int k) { return k > 0 && k < NS && band_out[2 * k] == 0 && band_out[2 * k - 1] == g.H - 1; };
  auto lmax = [](long long a, long long b) { return a > b ? a : b; };
  auto lmin = [](long long a, long long b) { return a < b ? a : b; };
  auto lsum = [](long long a, long long b) { return a + b; };
  // first row of each beam's run: max-scan of the run starts
  long long agg = -1, s, e;
  for (int k = k0; k < k1; ++k) if (!continues(k)) { rows(k, s, e); agg = s; }
  const long long start_in = block_scan_excl(agg, -1LL, t, sh, lmax);
  // end row of each beam's run: reverse min-scan of the first run end in each thread's beams
  const long long kInf = 0x7fffffffffffffffLL;
  agg = kInf;
  for (int k = k0; k < k1; ++k) if (!continues(k + 1)) { rows(k, s, e); agg = e; break; }
  const long long end_in = block_scan_excl(agg, kInf, BAND_THREADS - 1 - t, sh, lmin);
  // a run's tiles start at its first row every 128 rows; beam k owns those whose m0 lies in [s_k, e_k)
  auto own = [](long long s, long long e, long long rs, long long& j0, long long& j1) {
    j0 = (s - rs + kCellTileRows - 1) / kCellTileRows; j1 = (e - rs + kCellTileRows - 1) / kCellTileRows;
  };
  long long rs = start_in, n = 0, j0, j1;
  for (int k = k0; k < k1; ++k) {
    rows(k, s, e);
    if (!continues(k)) rs = s;
    own(s, e, rs, j0, j1);
    n += j1 - j0;
  }
  long long o = block_scan_excl(n, 0LL, t, sh, lsum);
  if (t == BAND_THREADS - 1) *tile_count = (int)(o + n);
  long long re = 0;
  rs = start_in;
  for (int k = k0; k < k1; ++k) {
    rows(k, s, e);
    if (!continues(k)) rs = s;
    if (k == k0 || !continues(k)) {      // the last row of the run beam k belongs to
      int j = k;
      while (j + 1 < k1 && continues(j + 1)) ++j;
      long long sj, ej;
      rows(j, sj, ej);
      re = (j + 1 == k1 && continues(k1)) ? end_in : ej;
    }
    own(s, e, rs, j0, j1);
    for (long long j = j0; j < j1; ++j, ++o) {
      const long long m0 = rs + j * kCellTileRows;
      tiles[2 * o] = (int)m0;
      tiles[2 * o + 1] = (int)lmin(m0 + kCellTileRows, re);
    }
  }
}

int beam_band(const int* ids, const int* parents, const int* band_in, int* band_out, int* tiles, long long tiles_cap,
              int* tile_count, long long NS, int K, int radius, int H, int W, cudaStream_t stream) {
  MVB_REQUIRE(ids && band_out && tiles && tile_count && (!band_in || parents), "beam_band: null pointer");
  MVB_REQUIRE(band_in != band_out, "beam_band: the parents' bands and the new ones need separate buffers");
  MVB_REQUIRE(NS > 0 && K > 0 && NS % K == 0 && H > 0 && W > 0 && radius >= 0,
              "beam_band: bad sizes NS=%lld K=%d H=%d W=%d radius=%d", NS, K, H, W, radius);
  const Grid g = make_grid(H, W);
  MVB_REQUIRE(NS * g.S + kCellTileRows < 0x7fffffffLL, "beam_band: NS=%lld too large for int32 rows", NS);
  MVB_REQUIRE(tiles_cap >= beam_band_capacity(NS, H, W), "beam_band: %lld tile entries, %lld needed", tiles_cap,
              beam_band_capacity(NS, H, W));
  beam_band_kernel<<<1, BAND_THREADS, 0, stream>>>(ids, parents, band_in, band_out, tiles, tile_count, (int)NS, K,
                                                   radius, g);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

// c and h32 of the base rollout (sample k / K) into the valid rows of beam k outside its band: one CTA per (beam,
// image row), the row's W cells contiguous in both layouts.  The cell launch on the work list writes the other rows.
__global__ void __launch_bounds__(256)
beam_band_copy_kernel(const float4* __restrict__ base_c, const float4* __restrict__ base_h, const int* __restrict__ band,
                      float4* __restrict__ c, float4* __restrict__ h, int K, Grid g) {
  const long long k = blockIdx.x / g.H;
  const int y = (int)(blockIdx.x - k * g.H);
  if (y >= band[2 * k] && y <= band[2 * k + 1]) return;
  constexpr int V = kHidden / 4;      // float4 per row
  const long long src = ((k / K) * g.S + (long long)y * g.Wp) * V, dst = (k * g.S + (long long)y * g.Wp) * V;
  for (int i = threadIdx.x; i < g.W * V; i += blockDim.x) {
    c[dst + i] = __ldg(base_c + src + i);
    h[dst + i] = __ldg(base_h + src + i);
  }
}

int beam_band_copy(const float* base_c, const float* base_h32, const int* band, float* c, float* h32, long long NS,
                   int K, int H, int W, cudaStream_t stream) {
  MVB_REQUIRE(base_c && base_h32 && band && c && h32, "beam_band_copy: null pointer");
  MVB_REQUIRE(NS > 0 && K > 0 && NS % K == 0 && H > 0 && W > 0 && NS * H < (1ll << 31),
              "beam_band_copy: bad sizes NS=%lld K=%d H=%d W=%d", NS, K, H, W);
  beam_band_copy_kernel<<<(unsigned)(NS * H), 256, 0, stream>>>(
      reinterpret_cast<const float4*>(base_c), reinterpret_cast<const float4*>(base_h32), band,
      reinterpret_cast<float4*>(c), reinterpret_cast<float4*>(h32), K, make_grid(H, W));
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int beam_backtrace(const int* step_ids, const int* step_parents, const float* step_logits,
                   int* out_ids, float* out_logits, long long N, int B, int Tp, int V,
                   cudaStream_t stream) {
  MVB_REQUIRE(step_ids && step_parents && step_logits && out_ids && out_logits, "beam_backtrace: null pointer");
  MVB_REQUIRE(N > 0 && B >= 1 && Tp >= 1 && V >= 1, "beam_backtrace: bad sizes");
  beam_backtrace_kernel<<<(unsigned)(N * B), 256, sizeof(int) * Tp, stream>>>(
      step_ids, step_parents, step_logits, out_ids, out_logits, N, B, Tp, V);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

// The back-trace of a batch whose rows end at their own lengths: row n's trace starts at its last step
// lengths[n] - 1 (its selections stop there; the step buffers of a ragged rollout hold nothing for it beyond), and
// its outputs at the steps after it are zeros.
__global__ void __launch_bounds__(256)
beam_backtrace_ragged_kernel(const int* __restrict__ step_ids, const int* __restrict__ step_parents,
                             const float* __restrict__ step_logits, const int* __restrict__ lengths,
                             int* __restrict__ out_ids, float* __restrict__ out_logits, long long N, int B, int Tp,
                             int V) {
  extern __shared__ int src[];  // [Tp] source beam of each step for this (n, b)
  const long long nb = blockIdx.x;
  const long long n = nb / B;
  const int b = (int)(nb - n * B);
  const int len = lengths[n];
  if (threadIdx.x == 0) {
    int p = b;
    for (int tau = len - 1; tau >= 0; --tau) {
      const long long o = ((long long)tau * N + n) * B + p;
      src[tau] = p;
      out_ids[(n * B + b) * Tp + tau] = step_ids[o];
      p = step_parents[o];
    }
  }
  for (int tau = len + (int)threadIdx.x; tau < Tp; tau += blockDim.x) out_ids[(n * B + b) * Tp + tau] = 0;
  __syncthreads();
  for (int tau = 0; tau < Tp; ++tau) {
    float* d = out_logits + ((n * B + b) * (long long)Tp + tau) * V;
    if (tau < len) {
      const float* s = step_logits + (((long long)tau * N + n) * B + src[tau]) * V;
      for (int v = threadIdx.x; v < V; v += blockDim.x) d[v] = s[v];
    } else {
      for (int v = threadIdx.x; v < V; v += blockDim.x) d[v] = 0.f;
    }
  }
}

int beam_backtrace_ragged(const int* step_ids, const int* step_parents, const float* step_logits, const int* lengths,
                          int* out_ids, float* out_logits, long long N, int B, int Tp, int V, cudaStream_t stream) {
  MVB_REQUIRE(step_ids && step_parents && step_logits && lengths && out_ids && out_logits,
              "beam_backtrace_ragged: null pointer");
  MVB_REQUIRE(N > 0 && B >= 1 && Tp >= 1 && V >= 1, "beam_backtrace_ragged: bad sizes");
  beam_backtrace_ragged_kernel<<<(unsigned)(N * B), 256, sizeof(int) * Tp, stream>>>(
      step_ids, step_parents, step_logits, lengths, out_ids, out_logits, N, B, Tp, V);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

// The fp32 offsets of the selected cells: out[n,k,t] = offs[t, n, ids[n,k,t]] for t < lengths[n], zeros after
// (what a caller adds to the cell centres on the host, code/multifuture_inference.py:504-517, in its own precision).
__global__ void gather_offsets_kernel(const int* __restrict__ ids, const float* __restrict__ offs,
                                      const int* __restrict__ lengths, float* __restrict__ out, long long N, int K,
                                      int Tp, int V) {
  const long long total = N * K * Tp;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i % Tp);
    const long long n = i / ((long long)Tp * K);
    float2 o = make_float2(0.f, 0.f);
    if (t < lengths[n]) o = *reinterpret_cast<const float2*>(offs + (((long long)t * N + n) * V + ids[i]) * 2);
    *reinterpret_cast<float2*>(out + 2 * i) = o;
  }
}

int gather_offsets(const int* ids, const float* offs, const int* lengths, float* out, long long N, int K, int Tp,
                   int V, cudaStream_t stream) {
  MVB_REQUIRE(ids && offs && lengths && out && N > 0 && K > 0 && Tp > 0 && V > 0, "gather_offsets: bad args");
  const long long total = N * K * Tp;
  const int blocks = (int)((total + 255) / 256 < sm_count() * 8 ? (total + 255) / 256 : sm_count() * 8);
  gather_offsets_kernel<<<blocks, 256, 0, stream>>>(ids, offs, lengths, out, N, K, Tp, V);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

}  // namespace mvb
