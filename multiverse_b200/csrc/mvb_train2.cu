// Backward kernels of everything around the cell (all HBM- or latency-bound, fp32):
//   loss_fwd_bwd        Model.build_loss (code/pred_models.py:961-1040): sparse softmax CE (mean over
//                       N*Tp) and Huber(delta=1) (mean over N*Tp*HW*2), values + gradients
//   soft_ce_fwd_bwd     the --use_soft_grid_class CE (:986-989) against dense label maps
//   fg_count, masked_huber_fwd_bwd
//                       the --mask_grid_regression Huber (:999-1018): over the cells whose label is > 0 only
//   huber_traj_fwd_bwd, soft_ce_label_fwd_bwd, fg_count_label, masked_huber_traj_fwd_bwd
//                       the same losses with targets and label maps computed from the trajectories and label cells
//   head_bwd            hidden2grid (:925-959): dWo, dh
//   emb_onehot_bwd      grid_emb on a one-hot input (:442-446): dWe, dbe (no input gradient)
//   emb_dense_bwd       grid_emb on the 2-channel offset map: dWe, dbe, d(input)
//   gnn_bwd             graph attention (:808-909, residual :378): dh, d(scene_mean)
//   scene_conv_bwd      conv2d helper, stride 2, tanh (:157-160): dW, db, d(input)
//   enc_class_input_bwd scene_conv (.) one_hot (:210): scatter of the x-block gradient
//   scene_mean_bwd      reduce_mean over time (:828)
//   clip_adadelta       Trainer (:1698-1716): element-wise clip +-clip, Adadelta(rho, eps), weight decay
// The reference obtains all of these from tf.gradients (:1698).
#include "mvb_common.cuh"
#include "mvb_kernels.h"

namespace mvb {

__device__ __forceinline__ float block_sum_256(float v, float* red) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  if (threadIdx.x < (blockDim.x >> 5)) t = red[threadIdx.x];
  if (warp == 0) t = warp_sum(t);
  return t;   // valid in warp 0
}

// ------------------------------------------------------------------------------ loss
// one CTA per (n,t) row: CE over V logits; grad = (softmax - onehot) * scale
__global__ void __launch_bounds__(256)
ce_loss_kernel(const float* __restrict__ logits, const int* __restrict__ labels,
               float* __restrict__ dlogits, float* __restrict__ loss_sum, int V, float scale) {
  __shared__ float red[8];
  __shared__ float bc[2];
  const long long r = blockIdx.x;
  const float* lg = logits + r * V;
  float m = -INFINITY;
  for (int v = threadIdx.x; v < V; v += blockDim.x) m = fmaxf(m, lg[v]);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) { float t = red[0]; for (int i = 1; i < 8; ++i) t = fmaxf(t, red[i]); bc[0] = t; }
  __syncthreads();
  m = bc[0];
  float s = 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) s += expf(lg[v] - m);
  s = block_sum_256(s, red);
  if (threadIdx.x == 0) bc[1] = s;
  __syncthreads();
  s = bc[1];
  const float inv = 1.0f / s;
  const int lab = labels[r];
  const bool lab_ok = lab >= 0 && lab < V;      // TF's sparse_softmax_cross_entropy yields NaN loss / gradient rows for
  for (int v = threadIdx.x; v < V; v += blockDim.x) {      // an out-of-range label; never read lg[lab] out of bounds
    const float p = expf(lg[v] - m) * inv;
    dlogits[r * V + v] = lab_ok ? (p - (v == lab ? 1.f : 0.f)) * scale : NAN;
  }
  if (threadIdx.x == 0) atomicAdd(loss_sum, lab_ok ? (logf(s) + m - lg[lab]) * scale : NAN);
}

template <class Target>
__global__ void __launch_bounds__(256)
huber_loss_kernel(const float* __restrict__ pred, const Target target,
                  float* __restrict__ dpred, float* __restrict__ loss_sum, long long n, float scale) {
  __shared__ float red[8];
  float acc = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const float e = pred[i] - target(i);
    const float a = fabsf(e);
    acc += (a <= 1.f) ? 0.5f * e * e : a - 0.5f;
    dpred[i] = fminf(fmaxf(e, -1.f), 1.f) * scale;
  }
  acc = block_sum_256(acc, red);
  if (threadIdx.x == 0) atomicAdd(loss_sum, acc * scale);
}

// one CTA per (n,t) row: softmax_cross_entropy_with_logits against a dense label row y[V]:
//   loss = sum_v y_v (lse - l_v),  grad = (sum(y) softmax - y) * scale
// (the soft maps of :1085-1136 do not sum to one, and lose mass where the kernel is clipped at the border).
// y(r, v): a dense map (DenseMaps) or the rule of grid_label (LabelMaps)
struct DenseMaps {
  const float* y;
  int V;
  __device__ __forceinline__ float operator()(long long r, int v) const { return y[r * V + v]; }
};
struct LabelMaps {
  const int* labels;
  int mode, H, W;
  __device__ __forceinline__ float operator()(long long r, int v) const { return grid_label(labels[r], v, mode, H, W); }
};

template <class Maps>
__global__ void __launch_bounds__(256)
soft_ce_loss_kernel(const float* __restrict__ logits, const Maps y,
                    float* __restrict__ dlogits, float* __restrict__ loss_sum, int V, float scale) {
  __shared__ float red[8];
  __shared__ float bc[3];
  const long long r = blockIdx.x;
  const float* lg = logits + r * V;
  float m = -INFINITY;
  for (int v = threadIdx.x; v < V; v += blockDim.x) m = fmaxf(m, lg[v]);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) { float t = red[0]; for (int i = 1; i < 8; ++i) t = fmaxf(t, red[i]); bc[0] = t; }
  __syncthreads();
  m = bc[0];
  float s = 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) s += expf(lg[v] - m);
  s = block_sum_256(s, red);
  if (threadIdx.x == 0) bc[1] = s;
  __syncthreads();
  s = bc[1];
  const float lse = logf(s) + m;
  float sy = 0.f, l = 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    const float yv = y(r, v);
    sy += yv;
    l = fmaf(yv, lse - lg[v], l);
  }
  sy = block_sum_256(sy, red);
  if (threadIdx.x == 0) bc[2] = sy;
  l = block_sum_256(l, red);
  __syncthreads();
  sy = bc[2];
  const float inv = 1.0f / s;
  for (int v = threadIdx.x; v < V; v += blockDim.x)
    dlogits[r * V + v] = (sy * (expf(lg[v] - m) * inv) - y(r, v)) * scale;
  if (threadIdx.x == 0) atomicAdd(loss_sum, l * scale);
}

// foreground of the masked regression loss: cells with label > 0 (dense maps, or the maps of grid_label) or the
// label cell of each row (tf.one_hot of an in-range sparse label).  fg(i) over the cells [rows, V] of the maps
struct SoftFg {
  const float* soft;
  __device__ __forceinline__ bool operator()(long long i) const { return soft[i] > 0.f; }
};
struct SparseFg {
  const int* labels;
  int V;
  __device__ __forceinline__ bool operator()(long long i) const { return labels[i / V] == (int)(i % V); }
};
struct LabelFg {
  const int* labels;
  int mode, H, W;
  __device__ __forceinline__ bool operator()(long long i) const {
    const int hw = H * W;
    return grid_label(labels[i / hw], (int)(i % hw), mode, H, W) > 0.f;
  }
};
// ... or over the rows [rows] of sparse labels
struct RowFg {
  const int* labels;
  int V;
  __device__ __forceinline__ bool operator()(long long i) const { return labels[i] >= 0 && labels[i] < V; }
};

// count += the number of i in [0, n) with fg(i)
template <class Fg>
__global__ void __launch_bounds__(256)
fg_count_kernel(const Fg fg, long long n, double* __restrict__ count) {
  unsigned c = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    c += fg(i);
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, (double)c);       // integers: exact up to 2^53
}

// Huber(delta=1) over the foreground cells only (tf.where + tf.gather, Reduction.MEAN over the 2K gathered
// elements, div_no_nan: 0 when K = 0); dpred = 0 off the foreground.  K is read from the device: the count
// of the whole batch, which a micro-batch may be only a part of.
template <class Target, class Fg>
__global__ void __launch_bounds__(256)
masked_huber_kernel(const float2* __restrict__ pred, const Target target, float2* __restrict__ dpred, const Fg is_fg,
                    const double* __restrict__ fg_count, float* __restrict__ loss_sum, long long cells, float weight) {
  __shared__ float red[8];
  const double K = *fg_count;
  const float scale = K > 0.0 ? (float)(weight / (2.0 * K)) : 0.f;
  float acc = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < cells;
       i += (long long)gridDim.x * blockDim.x) {
    float2 d = make_float2(0.f, 0.f);
    if (is_fg(i)) {
      const float2 p = pred[i], t = target.cell(i);
      const float e0 = p.x - t.x, e1 = p.y - t.y, a0 = fabsf(e0), a1 = fabsf(e1);
      acc += ((a0 <= 1.f) ? 0.5f * e0 * e0 : a0 - 0.5f) + ((a1 <= 1.f) ? 0.5f * e1 * e1 : a1 - 0.5f);
      d = make_float2(fminf(fmaxf(e0, -1.f), 1.f) * scale, fminf(fmaxf(e1, -1.f), 1.f) * scale);
    }
    dpred[i] = d;
  }
  acc = block_sum_256(acc, red);
  if (threadIdx.x == 0) atomicAdd(loss_sum, acc * scale);
}

// ------------------------------------------------------------------------------ head backward
// one CTA per sample row; warp per pixel q:  for every tap with p = q - off(tap) valid:
//   dh[q] += dout[p] * Wo[tap];   dWo[tap] += dout[p] * h[q]
template <int POUT>
__global__ void __launch_bounds__(256)
head_bwd_kernel(const float* __restrict__ h32, const float* __restrict__ dout,
                const float* __restrict__ Wo, float* __restrict__ dWo, float* __restrict__ dh,
                int accumulate_dh, Grid g) {
  extern __shared__ float sm[];
  const int hw = g.H * g.W;
  float* w_s = sm;                          // [9][POUT][256]
  float* d_s = w_s + 9 * POUT * kHidden;    // [HW][POUT]
  float* acc_s = d_s + hw * POUT;           // [9][POUT][256] block accumulator of dWo
  const long long s = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 9 * kHidden * POUT; i += blockDim.x) {
    const int po = i % POUT, ch = (i / POUT) % kHidden, t = i / (POUT * kHidden);
    w_s[(t * POUT + po) * kHidden + ch] = Wo[i];
    acc_s[i] = 0.f;
  }
  for (int i = threadIdx.x; i < hw * POUT; i += blockDim.x) d_s[i] = dout[s * hw * POUT + i];
  __syncthreads();
  float dw[9 * POUT][8];
#pragma unroll
  for (int a = 0; a < 9 * POUT; ++a)
#pragma unroll
    for (int c = 0; c < 8; ++c) dw[a][c] = 0.f;
  for (int q = warp; q < hw; q += 8) {
    const int y = q / g.W, x = q % g.W;
    const long long row = s * g.S + (long long)y * g.Wp + x;
    const float4* p4 = reinterpret_cast<const float4*>(h32 + row * kHidden + lane * 8);
    const float4 a = __ldg(p4), b = __ldg(p4 + 1);
    const float hv[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    float dhv[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) dhv[c] = 0.f;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int py = y - (t / 3 - 1), px = x - (t % 3 - 1);
      if (py < 0 || py >= g.H || px < 0 || px >= g.W) continue;
#pragma unroll
      for (int po = 0; po < POUT; ++po) {
        const float gd = d_s[(py * g.W + px) * POUT + po];
        const float4 wa = *reinterpret_cast<const float4*>(w_s + (t * POUT + po) * kHidden + lane * 8);
        const float4 wb = *reinterpret_cast<const float4*>(w_s + (t * POUT + po) * kHidden + lane * 8 + 4);
        dhv[0] = fmaf(gd, wa.x, dhv[0]); dhv[1] = fmaf(gd, wa.y, dhv[1]); dhv[2] = fmaf(gd, wa.z, dhv[2]); dhv[3] = fmaf(gd, wa.w, dhv[3]);
        dhv[4] = fmaf(gd, wb.x, dhv[4]); dhv[5] = fmaf(gd, wb.y, dhv[5]); dhv[6] = fmaf(gd, wb.z, dhv[6]); dhv[7] = fmaf(gd, wb.w, dhv[7]);
#pragma unroll
        for (int c = 0; c < 8; ++c) dw[t * POUT + po][c] = fmaf(gd, hv[c], dw[t * POUT + po][c]);
      }
    }
    float4* o4 = reinterpret_cast<float4*>(dh + row * kHidden + lane * 8);
    if (accumulate_dh) {
      const float4 oa = o4[0], ob = o4[1];
      o4[0] = make_float4(oa.x + dhv[0], oa.y + dhv[1], oa.z + dhv[2], oa.w + dhv[3]);
      o4[1] = make_float4(ob.x + dhv[4], ob.y + dhv[5], ob.z + dhv[6], ob.w + dhv[7]);
    } else {
      o4[0] = make_float4(dhv[0], dhv[1], dhv[2], dhv[3]);
      o4[1] = make_float4(dhv[4], dhv[5], dhv[6], dhv[7]);
    }
  }
  // block-reduce dWo through shared memory, then one global atomic per element
#pragma unroll
  for (int a = 0; a < 9 * POUT; ++a)
#pragma unroll
    for (int c = 0; c < 8; ++c) atomicAdd(&acc_s[a * kHidden + lane * 8 + c], dw[a][c]);
  __syncthreads();
  for (int i = threadIdx.x; i < 9 * kHidden * POUT; i += blockDim.x) {
    // acc_s is [t][po][ch]; dWo is TF layout [t][ch][po]
    const int ch = i % kHidden, po = (i / kHidden) % POUT, t = i / (kHidden * POUT);
    atomicAdd(dWo + (t * kHidden + ch) * POUT + po, acc_s[i]);
  }
}

// ------------------------------------------------------------------------------ emb backward
// x = tanh(pre), pre = be + conv3x3(in, We);  dpre = dx * (1 - x^2)
// one CTA per sample row.  ONEHOT (POUT == 1): in = one_hot(id);  else in = dense [HW][POUT] map (POUT = 1: the
// class decoder's logits feedback, 2: the offset map).  The channels run in groups of EG whose dpre [HW][EG] fits in
// shared memory; dbe and dWe of a channel are summed in the same order whatever the grouping, d_in adds the groups'
// partial sums in channel order.
template <int POUT, bool ONEHOT = (POUT == 1)>
__global__ void __launch_bounds__(256)
emb_bwd_kernel(const float* __restrict__ dxh, int cpad, const int* __restrict__ ids,
               const float* __restrict__ in_map, const float* __restrict__ We,
               const float* __restrict__ be, int E, int EG, float* __restrict__ dWe, float* __restrict__ dbe,
               float* __restrict__ d_in, int accumulate_din, Grid g) {
  extern __shared__ float sm[];
  const int hw = g.H * g.W;
  float* in_s = sm;                      // [HW][POUT] (dense input)
  float* dpre_s = in_s + hw * 2;         // [HW][eg]: the current channel group [e0, e0 + eg)
  const long long s = blockIdx.x;
  const int amax = ONEHOT ? ids[s] : 0;
  const int ay = amax / g.W, ax = amax % g.W;
  if (!ONEHOT)
    for (int i = threadIdx.x; i < hw * POUT; i += blockDim.x) in_s[i] = in_map[s * hw * POUT + i];
  for (int e0 = 0; e0 < E; e0 += EG) {
    const int eg = E - e0 < EG ? E - e0 : EG;
    __syncthreads();                     // in_s is loaded / the previous group's dpre has been read
    // pass 1: dpre for every (pixel, e)
    for (int i = threadIdx.x; i < hw * eg; i += blockDim.x) {
      const int p = i / eg, e = e0 + i % eg;
      const int y = p / g.W, x = p % g.W;
      float pre = be[e];
      if (ONEHOT) {
        const int dy = ay - y, dx = ax - x;
        if (dy >= -1 && dy <= 1 && dx >= -1 && dx <= 1) pre += We[((dy + 1) * 3 + (dx + 1)) * E + e];
      } else {
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
          if (yy < 0 || yy >= g.H || xx < 0 || xx >= g.W) continue;
#pragma unroll
          for (int ci = 0; ci < POUT; ++ci) pre = fmaf(in_s[(yy * g.W + xx) * POUT + ci], We[(t * POUT + ci) * E + e], pre);
        }
      }
      const float xv = tanhf(pre);
      const long long row = s * g.S + (long long)y * g.Wp + x;
      dpre_s[i] = dxh[row * cpad + e] * (1.f - xv * xv);
    }
    __syncthreads();
    // pass 2: dbe, dWe (thread per (tap, po, e)), d_in (thread per (pixel, po))
    for (int i = threadIdx.x; i < eg; i += blockDim.x) {
      float a = 0.f;
      for (int p = 0; p < hw; ++p) a += dpre_s[p * eg + i];
      atomicAdd(dbe + e0 + i, a);
    }
    for (int i = threadIdx.x; i < 9 * POUT * eg; i += blockDim.x) {
      const int el = i % eg, po = (i / eg) % POUT, t = i / (eg * POUT);
      float a = 0.f;
      if (ONEHOT) {
        // out[p] += onehot[p + off(t)] * We[t]  ->  only p = amax - off(t)
        const int y = ay - (t / 3 - 1), x = ax - (t % 3 - 1);
        if (y >= 0 && y < g.H && x >= 0 && x < g.W) a = dpre_s[(y * g.W + x) * eg + el];
      } else {
        for (int p = 0; p < hw; ++p) {
          const int yy = p / g.W + t / 3 - 1, xx = p % g.W + t % 3 - 1;
          if (yy < 0 || yy >= g.H || xx < 0 || xx >= g.W) continue;
          a = fmaf(in_s[(yy * g.W + xx) * POUT + po], dpre_s[p * eg + el], a);
        }
      }
      atomicAdd(dWe + (t * POUT + po) * E + e0 + el, a);
    }
    if (!ONEHOT && d_in) {
      for (int i = threadIdx.x; i < hw * POUT; i += blockDim.x) {
        const int q = i / POUT, po = i % POUT;
        const int y = q / g.W, x = q % g.W;
        float a = 0.f;
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          const int py = y - (t / 3 - 1), px = x - (t % 3 - 1);   // out[p] uses in[p + off] -> p = q - off
          if (py < 0 || py >= g.H || px < 0 || px >= g.W) continue;
          const float* dp = dpre_s + (py * g.W + px) * eg;
          const float* wv = We + (t * POUT + po) * E + e0;
          for (int e = 0; e < eg; ++e) a = fmaf(dp[e], wv[e], a);
        }
        const long long o = s * hw * POUT + i;
        d_in[o] = (accumulate_din || e0 > 0) ? d_in[o] + a : a;
      }
    }
  }
}

// ------------------------------------------------------------------------------ GNN backward
// forward: F = [h ; s], Fh = F / n (n = sqrt(max(|F|^2, eps))), e_pq = Fh_p . Fh_q, a = softmax_q,
//          out_p = h_p + sum_q a_pq h_q.
// pass 1 (warp per cell p): recompute a_pq, da_pq = g_p . h_q, de_pq = a_pq (da_pq - sum_r a_pr da_pr);
//          store a[p][9], de[p][9], inv_n[p].
// pass 2 (warp per cell p): dh_p = g_p + sum_q a_qp g_q + dF_p[:256],  ds_p = dF_p[256:],
//          dFh_p = sum_q (de_pq + de_qp) Fh_q,  dF_p = (dFh_p - (dFh_p . Fh_p) Fh_p) / n_p.
__global__ void __launch_bounds__(256)
gnn_bwd_pass1_kernel(const float* __restrict__ h32, const float* __restrict__ scene,
                     const float* __restrict__ gout, float* __restrict__ a_out,
                     float* __restrict__ de_out, float* __restrict__ invn_out, long long NS, Grid g) {
  const int lane = threadIdx.x & 31;
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int hw = g.H * g.W;
  if (wid >= NS * hw) return;
  const long long s = wid / hw;
  const int pix = (int)(wid - s * hw);
  const int y = pix / g.W, x = pix - y * g.W;
  auto ld8 = [&](const float* base, long long row, float (&o)[8]) {
    const float4* p4 = reinterpret_cast<const float4*>(base + row * kHidden + lane * 8);
    const float4 a = __ldg(p4), b = __ldg(p4 + 1);
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
  };
  const long long rowp = s * g.S + (long long)y * g.Wp + x;
  float hp[8], gp[8], sp[2] = {0.f, 0.f};
  ld8(h32, rowp, hp);
  ld8(gout, rowp, gp);
  if (scene) {
    const float2 c = __ldg(reinterpret_cast<const float2*>(scene + ((s * g.H + y) * g.W + x) * 64 + lane * 2));
    sp[0] = c.x; sp[1] = c.y;
  }
  float dot[9], nrm[9], da[9];
  bool ok[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
    ok[k] = (yy >= 0) && (yy < g.H) && (xx >= 0) && (xx < g.W);
    float d = 0.f, q = 0.f, a = 0.f;
    if (ok[k]) {
      float hq[8];
      ld8(h32, s * g.S + (long long)yy * g.Wp + xx, hq);
#pragma unroll
      for (int c = 0; c < 8; ++c) { d = fmaf(hp[c], hq[c], d); q = fmaf(hq[c], hq[c], q); a = fmaf(gp[c], hq[c], a); }
      if (scene) {
        const float2 sq = __ldg(reinterpret_cast<const float2*>(scene + ((s * g.H + yy) * g.W + xx) * 64 + lane * 2));
        d = fmaf(sp[0], sq.x, d); d = fmaf(sp[1], sq.y, d);
        q = fmaf(sq.x, sq.x, q); q = fmaf(sq.y, sq.y, q);
      }
    }
    dot[k] = warp_sum(d); nrm[k] = warp_sum(q); da[k] = warp_sum(a);
  }
  const float inv_p = rsqrtf(fmaxf(nrm[4], 1e-12f));
  float e[9], m = -INFINITY;
#pragma unroll
  for (int k = 0; k < 9; ++k) { e[k] = dot[k] * inv_p * rsqrtf(fmaxf(nrm[k], 1e-12f)); if (ok[k]) m = fmaxf(m, e[k]); }
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) { e[k] = ok[k] ? __expf(e[k] - m) : 0.f; sum += e[k]; }
  const float inv_sum = 1.f / sum;
  float bar = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) { e[k] *= inv_sum; bar = fmaf(e[k], da[k], bar); }
  if (lane < 9) {
    float av = 0.f, dv = 0.f;
#pragma unroll
    for (int k = 0; k < 9; ++k) if (lane == k) { av = e[k]; dv = e[k] * (da[k] - bar); }
    a_out[(s * hw + pix) * 9 + lane] = av;
    de_out[(s * hw + pix) * 9 + lane] = dv;
  }
  if (lane == 0) invn_out[s * hw + pix] = inv_p;
}

__global__ void __launch_bounds__(256)
gnn_bwd_pass2_kernel(const float* __restrict__ h32, const float* __restrict__ scene,
                     const float* __restrict__ gout, const float* __restrict__ a_in,
                     const float* __restrict__ de_in, const float* __restrict__ invn,
                     float* __restrict__ dh, int accumulate_dh, float* __restrict__ dscene,
                     long long NS, Grid g) {
  const int lane = threadIdx.x & 31;
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int hw = g.H * g.W;
  if (wid >= NS * hw) return;
  const long long s = wid / hw;
  const int pix = (int)(wid - s * hw);
  const int y = pix / g.W, x = pix - y * g.W;
  auto ld8 = [&](const float* base, long long row, float (&o)[8]) {
    const float4* p4 = reinterpret_cast<const float4*>(base + row * kHidden + lane * 8);
    const float4 a = __ldg(p4), b = __ldg(p4 + 1);
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
  };
  const long long rowp = s * g.S + (long long)y * g.Wp + x;
  float hp[8], acc[8], dfh[8], dfs[2] = {0.f, 0.f}, sp[2] = {0.f, 0.f};
  ld8(h32, rowp, hp);
  ld8(gout, rowp, acc);                       // residual: dh_p = g_p + ...
#pragma unroll
  for (int c = 0; c < 8; ++c) dfh[c] = 0.f;
  if (scene) {
    const float2 c = __ldg(reinterpret_cast<const float2*>(scene + ((s * g.H + y) * g.W + x) * 64 + lane * 2));
    sp[0] = c.x; sp[1] = c.y;
  }
  const float inv_p = invn[s * hw + pix];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
    if (yy < 0 || yy >= g.H || xx < 0 || xx >= g.W) continue;
    const long long q = s * hw + yy * g.W + xx;
    const float a_qp = a_in[q * 9 + (8 - k)];          // p is neighbour (8-k) of q
    const float w = de_in[(s * hw + pix) * 9 + k] + de_in[q * 9 + (8 - k)];
    const float inv_q = invn[q];
    float hq[8], gq[8];
    const long long rowq = s * g.S + (long long)yy * g.Wp + xx;
    ld8(h32, rowq, hq);
    ld8(gout, rowq, gq);
    const float wq = w * inv_q;
#pragma unroll
    for (int c = 0; c < 8; ++c) { acc[c] = fmaf(a_qp, gq[c], acc[c]); dfh[c] = fmaf(wq, hq[c], dfh[c]); }
    if (scene) {
      const float2 sq = __ldg(reinterpret_cast<const float2*>(scene + ((s * g.H + yy) * g.W + xx) * 64 + lane * 2));
      dfs[0] = fmaf(wq, sq.x, dfs[0]); dfs[1] = fmaf(wq, sq.y, dfs[1]);
    }
  }
  // projection through the normalisation: dF = (dFh - (dFh . Fh) Fh) / n   (zero if |F|^2 < eps)
  float proj = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) proj = fmaf(dfh[c], hp[c], proj);
  proj = fmaf(dfs[0], sp[0], proj); proj = fmaf(dfs[1], sp[1], proj);
  proj = warp_sum(proj) * inv_p * inv_p;     // (dFh . F) / n^2
  const bool clamped = inv_p >= 1e6f;        // |F|^2 <= 1e-12: l2_normalize is x * const there
  float4* o4 = reinterpret_cast<float4*>(dh + rowp * kHidden + lane * 8);
  float r[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) r[c] = acc[c] + (clamped ? dfh[c] : dfh[c] - proj * hp[c]) * inv_p;
  if (accumulate_dh) {
    const float4 oa = o4[0], ob = o4[1];
    o4[0] = make_float4(oa.x + r[0], oa.y + r[1], oa.z + r[2], oa.w + r[3]);
    o4[1] = make_float4(ob.x + r[4], ob.y + r[5], ob.z + r[6], ob.w + r[7]);
  } else {
    o4[0] = make_float4(r[0], r[1], r[2], r[3]);
    o4[1] = make_float4(r[4], r[5], r[6], r[7]);
  }
  if (scene && dscene) {
    float2* ds = reinterpret_cast<float2*>(dscene + ((s * g.H + y) * g.W + x) * 64 + lane * 2);
    const float d0 = (clamped ? dfs[0] : dfs[0] - proj * sp[0]) * inv_p;
    const float d1 = (clamped ? dfs[1] : dfs[1] - proj * sp[1]) * inv_p;
    const float2 old = *ds;
    *ds = make_float2(old.x + d0, old.y + d1);
  }
}

// ------------------------------------------------------------------------------ scene CNN backward
// dpre = dout * (1 - out^2);  db += sum dpre;  dW[k][oc] += patch[k] * dpre[oc];  din += W . dpre
// block = 4 k-groups x Cout(=64) threads; each thread keeps KPG partial sums of dW in registers over
// the block's strip of output pixels and flushes them with one atomic per element at the end.
template <int KPG>
__global__ void __launch_bounds__(256)
scene_conv_bwd_kernel(const float* __restrict__ in, const float* __restrict__ Wt,
                      const float* __restrict__ out, const float* __restrict__ dout,
                      float* __restrict__ dW, float* __restrict__ db, float* __restrict__ din,
                      long long F, int IH, int IW, int OH, int OW, int pad_t, int pad_l, int Cin,
                      int Cout) {
  extern __shared__ float sm[];
  float* patch = sm;                    // [4*KPG] (zero padded beyond 9*Cin)
  float* dpre_s = sm + 4 * KPG;         // [Cout]
  const int oc = threadIdx.x % Cout, kg = threadIdx.x / Cout;
  const int K = 9 * Cin;
  const long long total_pix = F * OH * OW;
  float acc[KPG];
#pragma unroll
  for (int k = 0; k < KPG; ++k) acc[k] = 0.f;
  float dbacc = 0.f;
  for (long long pix = blockIdx.x; pix < total_pix; pix += gridDim.x) {
    const int ox = (int)(pix % OW);
    const int oy = (int)((pix / OW) % OH);
    const long long f = pix / ((long long)OW * OH);
    __syncthreads();
    for (int i = threadIdx.x; i < 4 * KPG; i += blockDim.x) {
      float v = 0.f;
      if (i < K) {
        const int ci = i % Cin, tap = i / Cin;
        const int iy = oy * 2 - pad_t + tap / 3, ix = ox * 2 - pad_l + tap % 3;
        if (iy >= 0 && iy < IH && ix >= 0 && ix < IW) v = in[((f * IH + iy) * IW + ix) * Cin + ci];
      }
      patch[i] = v;
    }
    const float o = out[pix * Cout + oc];
    const float dp = dout[pix * Cout + oc] * (1.f - o * o);
    if (kg == 0) { dpre_s[oc] = dp; dbacc += dp; }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < KPG; ++k) acc[k] = fmaf(patch[kg * KPG + k], dp, acc[k]);
    if (din) {
      for (int i = threadIdx.x; i < K; i += blockDim.x) {
        const int ci = i % Cin, tap = i / Cin;
        const int iy = oy * 2 - pad_t + tap / 3, ix = ox * 2 - pad_l + tap % 3;
        if (iy < 0 || iy >= IH || ix < 0 || ix >= IW) continue;
        float a = 0.f;
        for (int c = 0; c < Cout; ++c) a = fmaf(Wt[(long long)i * Cout + c], dpre_s[c], a);
        atomicAdd(din + ((f * IH + iy) * IW + ix) * Cin + ci, a);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < KPG; ++k)
    if (kg * KPG + k < K) atomicAdd(dW + (long long)(kg * KPG + k) * Cout + oc, acc[k]);
  if (kg == 0) atomicAdd(db + oc, dbacc);
}

__global__ void enc_class_input_bwd_kernel(const float* __restrict__ dxh, int cpad,
                                           const int* __restrict__ frame_idx,
                                           const int* __restrict__ label, float* __restrict__ dscene,
                                           Grid g) {
  const long long s = blockIdx.x;
  const int c = threadIdx.x;
  const int lb = label[s], hw = g.H * g.W;
  if (lb < 0 || lb >= hw) return;
  const long long row = s * g.S + (long long)(lb / g.W) * g.Wp + (lb % g.W);
  atomicAdd(dscene + ((long long)frame_idx[s] * hw + lb) * 64 + c, dxh[row * cpad + c]);
}

// backward of enc_class_input_mix: the x-block gradient of the two weighted pixels goes to the scene features
__global__ void enc_class_input_mix_bwd_kernel(const float* __restrict__ dxh, int cpad, const int* __restrict__ frame_idx,
                                               const int* __restrict__ label, const int* __restrict__ label2, float beta,
                                               float* __restrict__ dscene, Grid g) {
  const long long s = blockIdx.x;
  const int c = threadIdx.x;
  const int hw = g.H * g.W;
  const int l1 = label[s], l2 = label2[s];
  const float w1 = beta, w2 = 1.0f - beta;
  auto add = [&](int lb, float wgt) {
    if (lb < 0 || lb >= hw) return;
    const long long row = s * g.S + (long long)(lb / g.W) * g.Wp + (lb % g.W);
    atomicAdd(dscene + ((long long)frame_idx[s] * hw + lb) * 64 + c, dxh[row * cpad + c] * wgt);
  };
  if (l1 == l2) {
    add(l1, w1 + w2);
  } else {
    add(l1, w1);
    add(l2, w2);
  }
}

__global__ void scene_mean_bwd_kernel(const float* __restrict__ dmean, const int* __restrict__ fidx,
                                      float* __restrict__ dscene, long long N, int T, long long HWC) {
  const long long total = N * HWC;
  const float inv = 1.0f / (float)T;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / HWC, e = i - n * HWC;
    const float v = dmean[i] * inv;
    for (int t = 0; t < T; ++t) atomicAdd(dscene + (long long)fidx[n * T + t] * HWC + e, v);
  }
}

// ------------------------------------------------------------------------------ optimizer
// g = clip(g + wd * w [if decayed], +-clip);  Adadelta (tf.train.AdadeltaOptimizer, rho, eps):
//   acc = rho*acc + (1-rho) g^2;  upd = sqrt(acc_upd+eps) * rsqrt(acc+eps) * g;
//   acc_upd = rho*acc_upd + (1-rho) upd^2;  w -= lr * upd
__global__ void clip_adadelta_kernel(float* __restrict__ w, const float* __restrict__ grad,
                                     float* __restrict__ acc, float* __restrict__ acc_upd,
                                     long long n, float lr, float rho, float eps, float clip,
                                     float wd, float gscale) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float gv = fmaf(wd, w[i], grad[i] * gscale);
    if (clip > 0.f) gv = fminf(fmaxf(gv, -clip), clip);
    const float a = rho * acc[i] + (1.f - rho) * gv * gv;
    const float u = sqrtf(acc_upd[i] + eps) * rsqrtf(a + eps) * gv;
    acc[i] = a;
    acc_upd[i] = rho * acc_upd[i] + (1.f - rho) * u * u;
    w[i] -= lr * u;
  }
}

// The other three optimizers Trainer offers (code/pred_models.py:1667-1681), same gradient preparation (wd * w added,
// 1/G scaling, element-wise clip):
//   kind 1  tf.train.MomentumOptimizer(lr, 0.9):   a = m a + g;  w -= lr a                        (s1 = a)
//   kind 2  tf.train.AdamOptimizer(lr):            m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;
//                                                  w -= lr sqrt(1-b2^t)/(1-b1^t) m / (sqrt(v) + eps)   (s1 = m, s2 = v)
//   kind 3  tf.train.RMSPropOptimizer(lr):         ms = d ms + (1-d) g^2;  mom = mu mom + lr g rsqrt(ms + eps);
//                                                  w -= mom      (s1 = ms, initialised to ONE by TF; s2 = mom)
__global__ void clip_update_kernel(float* __restrict__ w, const float* __restrict__ grad, float* __restrict__ s1,
                                   float* __restrict__ s2, long long n, int kind, float lr, float p1, float p2,
                                   float eps, float clip, float wd, float gscale) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float gv = fmaf(wd, w[i], grad[i] * gscale);
    if (clip > 0.f) gv = fminf(fmaxf(gv, -clip), clip);
    if (kind == 1) {
      const float a = p1 * s1[i] + gv;
      s1[i] = a;
      w[i] -= lr * a;
    } else if (kind == 2) {
      const float m = p1 * s1[i] + (1.f - p1) * gv;
      const float v = p2 * s2[i] + (1.f - p2) * gv * gv;
      s1[i] = m; s2[i] = v;
      w[i] -= lr * m / (sqrtf(v) + eps);          // lr already carries sqrt(1-b2^t)/(1-b1^t)
    } else {
      const float ms = p1 * s1[i] + (1.f - p1) * gv * gv;
      const float mom = p2 * s2[i] + lr * gv * rsqrtf(ms + eps);
      s1[i] = ms; s2[i] = mom;
      w[i] -= mom;
    }
  }
}

// ------------------------------------------------------------------------------ launchers
static inline int grid_for(long long n, int threads) {
  const long long b = (n + threads - 1) / threads;
  return (int)(b < sm_count() * 16 ? (b > 0 ? b : 1) : sm_count() * 16);
}

int loss_fwd_bwd(const float* logits, const int* labels, float* dlogits, long long rows, int V,
                 float cls_scale, const float* reg, const float* target, float* dreg, long long nreg,
                 float reg_scale, float* loss_out, cudaStream_t stream) {
  MVB_REQUIRE(loss_out, "loss_fwd_bwd: null loss_out");
  if (logits) {
    MVB_REQUIRE(labels && dlogits && rows > 0 && V > 0, "loss_fwd_bwd: bad CE args");
    ce_loss_kernel<<<(unsigned)rows, 256, 0, stream>>>(logits, labels, dlogits, loss_out, V, cls_scale / (float)rows);
    MVB_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
  }
  if (reg) {
    MVB_REQUIRE(target && dreg && nreg > 0, "loss_fwd_bwd: bad Huber args");
    huber_loss_kernel<<<grid_for(nreg, 256), 256, 0, stream>>>(reg, DenseOffsets{target}, dreg, loss_out + 1, nreg,
                                                               reg_scale / (float)nreg);
    MVB_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
  }
  return MVB_OK;
}

int soft_ce_fwd_bwd(const float* logits, const float* labels, float* dlogits, long long rows, int V, float cls_scale,
                    float* loss_out, cudaStream_t stream) {
  MVB_REQUIRE(logits && labels && dlogits && loss_out && rows > 0 && V > 0, "soft_ce_fwd_bwd: bad args");
  soft_ce_loss_kernel<<<(unsigned)rows, 256, 0, stream>>>(logits, DenseMaps{labels, V}, dlogits, loss_out, V,
                                                           cls_scale / (float)rows);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int fg_count(const float* soft, const int* labels, long long rows, int V, double* count, cudaStream_t stream) {
  MVB_REQUIRE((soft || labels) && count && rows > 0 && V > 0, "fg_count: bad args");
  if (soft) fg_count_kernel<<<grid_for(rows * V, 256), 256, 0, stream>>>(SoftFg{soft}, rows * V, count);
  else fg_count_kernel<<<grid_for(rows, 256), 256, 0, stream>>>(RowFg{labels, V}, rows, count);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

// ---- the same losses with their targets and label maps computed from the trajectories and the label cells
// (SURVEY.md §8 row f-1): reg fp32 [Tp,N,H*W,2]; pred_traj fp64 [N,Tp,2]; centers fp64 [H*W,2]; labels int32 [Tp,N];
// mode: --soft_grid 1-7, or 0 for the sparse labels
static inline TrajOffsets pred_offsets(const double* traj, const double* centers, long long N, int Tp, int hw) {
  return TrajOffsets{traj, centers, N, 2LL * Tp, 2, hw};
}

int huber_traj_fwd_bwd(const float* reg, const double* pred_traj, const double* centers, float* dreg, long long N,
                       int Tp, int V, float reg_scale, float* loss_out, cudaStream_t stream) {
  MVB_REQUIRE(reg && pred_traj && centers && dreg && loss_out && N > 0 && Tp > 0 && V > 0,
              "huber_traj_fwd_bwd: bad args");
  const long long nreg = N * Tp * V * 2;
  huber_loss_kernel<<<grid_for(nreg, 256), 256, 0, stream>>>(reg, pred_offsets(pred_traj, centers, N, Tp, V), dreg,
                                                             loss_out + 1, nreg, reg_scale / (float)nreg);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int soft_ce_label_fwd_bwd(const float* logits, const int* labels, int mode, float* dlogits, long long rows, int H,
                          int W, float cls_scale, float* loss_out, cudaStream_t stream) {
  MVB_REQUIRE(logits && labels && dlogits && loss_out && rows > 0 && H > 0 && W > 0 && mode >= 1 && mode <= 7,
              "soft_ce_label_fwd_bwd: bad args (mode %d)", mode);
  soft_ce_loss_kernel<<<(unsigned)rows, 256, 0, stream>>>(logits, LabelMaps{labels, mode, H, W}, dlogits, loss_out,
                                                           H * W, cls_scale / (float)rows);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int fg_count_label(const int* labels, int mode, long long rows, int H, int W, double* count, cudaStream_t stream) {
  MVB_REQUIRE(labels && count && rows > 0 && H > 0 && W > 0 && mode >= 0 && mode <= 7,
              "fg_count_label: bad args (mode %d)", mode);
  const long long cells = rows * H * W;
  fg_count_kernel<<<grid_for(cells, 256), 256, 0, stream>>>(LabelFg{labels, mode, H, W}, cells, count);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int masked_huber_traj_fwd_bwd(const float* reg, const double* pred_traj, const double* centers, float* dreg,
                              const int* labels, int mode, long long N, int Tp, int H, int W, const double* count,
                              float reg_scale, float* loss_out, cudaStream_t stream) {
  MVB_REQUIRE(reg && pred_traj && centers && dreg && labels && count && loss_out && N > 0 && Tp > 0 && H > 0 &&
              W > 0 && mode >= 0 && mode <= 7, "masked_huber_traj_fwd_bwd: bad args (mode %d)", mode);
  const long long cells = N * Tp * H * W;
  masked_huber_kernel<<<grid_for(cells, 256), 256, 0, stream>>>(
      reinterpret_cast<const float2*>(reg), pred_offsets(pred_traj, centers, N, Tp, H * W),
      reinterpret_cast<float2*>(dreg), LabelFg{labels, mode, H, W}, count, loss_out + 1, cells, reg_scale);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int masked_huber_fwd_bwd(const float* reg, const float* target, float* dreg, const float* soft, const int* labels,
                         long long rows, int V, const double* count, float reg_scale, float* loss_out,
                         cudaStream_t stream) {
  MVB_REQUIRE(reg && target && dreg && (soft || labels) && count && loss_out && rows > 0 && V > 0,
              "masked_huber_fwd_bwd: bad args");
  const long long cells = rows * V;
  const DenseOffsets tg{target};
  float2* d = reinterpret_cast<float2*>(dreg);
  if (soft)
    masked_huber_kernel<<<grid_for(cells, 256), 256, 0, stream>>>(reinterpret_cast<const float2*>(reg), tg, d,
                                                                  SoftFg{soft}, count, loss_out + 1, cells, reg_scale);
  else
    masked_huber_kernel<<<grid_for(cells, 256), 256, 0, stream>>>(reinterpret_cast<const float2*>(reg), tg, d,
                                                                  SparseFg{labels, V}, count, loss_out + 1, cells,
                                                                  reg_scale);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int head_bwd(const float* h32, const float* dout, const float* Wo, int Pout, float* dWo, float* dh,
             int accumulate_dh, long long NS, int H, int W, cudaStream_t stream) {
  MVB_REQUIRE(h32 && dout && Wo && dWo && dh && NS > 0 && (Pout == 1 || Pout == 2), "head_bwd: bad args");
  const Grid g = make_grid(H, W);
  const size_t smem = sizeof(float) * ((size_t)2 * 9 * kHidden * Pout + (size_t)H * W * Pout);
  if (Pout == 1) {
    head_bwd_kernel<1><<<(unsigned)NS, 256, smem, stream>>>(h32, dout, Wo, dWo, dh, accumulate_dh, g);
  } else {
    static SmemOptIn opt;
    MVB_CHECK_CUDA(smem_opt_in(opt, head_bwd_kernel<2>, 100 * 1024));
    MVB_REQUIRE(smem <= 100 * 1024, "head_bwd: grid too large");
    head_bwd_kernel<2><<<(unsigned)NS, 256, smem, stream>>>(h32, dout, Wo, dWo, dh, accumulate_dh, g);
  }
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int emb_bwd(const float* dxh, int cpad, const int* ids, const float* in_map, const float* We,
            const float* be, int E, int Pout, float* dWe, float* dbe, float* d_in, int accumulate_din,
            long long NS, int H, int W, cudaStream_t stream) {
  MVB_REQUIRE(dxh && We && be && dWe && dbe && NS > 0 && E > 0, "emb_bwd: bad args");
  MVB_REQUIRE((Pout == 1 && (ids || in_map)) || (Pout == 2 && in_map),
              "emb_bwd: need ids or in_map (Pout=1) or in_map (Pout=2)");
  const Grid g = make_grid(H, W);
  // channel group: all E channels where [HW][2 + E] floats fit, else the widest multiple of 8 that does
  constexpr size_t kSmemMax = 160 * 1024;
  const size_t hw = (size_t)H * W;
  const long long fit = (long long)(kSmemMax / sizeof(float) / hw) - 2;
  const int EG = fit >= E ? E : (int)(fit / 8 * 8);
  MVB_REQUIRE(EG >= 8, "emb_bwd: grid %dx%d too large", H, W);
  const size_t smem = sizeof(float) * hw * (2 + EG);
  static SmemOptIn opt1, opt1d, opt2;
  MVB_CHECK_CUDA(smem_opt_in(opt1, emb_bwd_kernel<1>, kSmemMax));
  MVB_CHECK_CUDA(smem_opt_in(opt1d, emb_bwd_kernel<1, false>, kSmemMax));
  MVB_CHECK_CUDA(smem_opt_in(opt2, emb_bwd_kernel<2>, kSmemMax));
  if (Pout == 1 && ids) emb_bwd_kernel<1><<<(unsigned)NS, 256, smem, stream>>>(dxh, cpad, ids, in_map, We, be, E, EG, dWe, dbe, d_in, accumulate_din, g);
  else if (Pout == 1) emb_bwd_kernel<1, false><<<(unsigned)NS, 256, smem, stream>>>(dxh, cpad, ids, in_map, We, be, E, EG, dWe, dbe, d_in, accumulate_din, g);
  else emb_bwd_kernel<2><<<(unsigned)NS, 256, smem, stream>>>(dxh, cpad, ids, in_map, We, be, E, EG, dWe, dbe, d_in, accumulate_din, g);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int gnn_bwd(const float* h32, const float* scene_mean, const float* gout, float* work, float* dh,
            int accumulate_dh, float* dscene_mean, long long NS, int H, int W, cudaStream_t stream) {
  MVB_REQUIRE(h32 && gout && work && dh && NS > 0, "gnn_bwd: bad args");
  const Grid g = make_grid(H, W);
  const long long cells = NS * H * W;
  float* a_buf = work;
  float* de_buf = work + cells * 9;
  float* invn = work + cells * 18;
  const unsigned blocks = (unsigned)((cells + 7) / 8);
  gnn_bwd_pass1_kernel<<<blocks, 256, 0, stream>>>(h32, scene_mean, gout, a_buf, de_buf, invn, NS, g);
  MVB_CHECK_CUDA(cudaGetLastError());
  gnn_bwd_pass2_kernel<<<blocks, 256, 0, stream>>>(h32, scene_mean, gout, a_buf, de_buf, invn, dh, accumulate_dh, dscene_mean, NS, g);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(2);
  return MVB_OK;
}

int scene_conv_bwd(const float* in, const float* W, const float* out, const float* dout, float* dW,
                   float* db, float* din, long long F, int IH, int IW, int Cin, int Cout,
                   cudaStream_t stream) {
  MVB_REQUIRE(in && W && out && dout && dW && db && F > 0 && Cout == 64, "scene_conv_bwd: bad args (Cout must be 64)");
  MVB_REQUIRE(9 * Cin <= 4 * 144, "scene_conv_bwd: Cin=%d too large", Cin);
  const int OH = (IH + 1) / 2, OW = (IW + 1) / 2;
  const int tot_h = (OH - 1) * 2 + 3 - IH > 0 ? (OH - 1) * 2 + 3 - IH : 0;
  const int tot_w = (OW - 1) * 2 + 3 - IW > 0 ? (OW - 1) * 2 + 3 - IW : 0;
  const long long total_pix = F * OH * OW;
  const unsigned blocks = (unsigned)(total_pix < sm_count() * 8 ? total_pix : sm_count() * 8);
  if (9 * Cin <= 4 * 25) {
    scene_conv_bwd_kernel<25><<<blocks, 256, sizeof(float) * (100 + 64), stream>>>(
        in, W, out, dout, dW, db, din, F, IH, IW, OH, OW, tot_h / 2, tot_w / 2, Cin, Cout);
  } else {
    scene_conv_bwd_kernel<144><<<blocks, 256, sizeof(float) * (576 + 64), stream>>>(
        in, W, out, dout, dW, db, din, F, IH, IW, OH, OW, tot_h / 2, tot_w / 2, Cin, Cout);
  }
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

// ------------------------------------------------------------------------------ SimAug input attack step
// One step of SimAug's white-box attack on the scene input (SimAug/code/pred_models.py:96-124): the targeted
// FGSM / PGD update  adv <- clip(adv - step * sign(grad), lower, upper)  with the bounds of :142-143,
// lower = clip(x - eps, -1, 1), upper = clip(x + eps, -1, 1), x = the clean input.
__global__ void adv_step_kernel(const float* __restrict__ x, const float* __restrict__ adv, const float* __restrict__ g,
                                float* __restrict__ out, float eps, float step, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float lo = fminf(fmaxf(x[i] - eps, -1.f), 1.f), hi = fminf(fmaxf(x[i] + eps, -1.f), 1.f);
    const float gi = g[i];
    const float sg = gi > 0.f ? 1.f : (gi < 0.f ? -1.f : 0.f);          // tf.sign
    out[i] = fminf(fmaxf(adv[i] - step * sg, lo), hi);                  // tf.clip_by_value: min(max(v, lo), hi)
  }
}
// mixup of :149-166:  out = a * w + b * (1 - w)
__global__ void mix_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, float w,
                           long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = a[i] * w + b[i] * (1.f - w);
}

// per-row sparse softmax cross entropy, no gradient: SimAug's multi-view selection ranks the M views of a sample by
// the mean of these over the predicted steps (SimAug/code/pred_models.py:386-392, :413-416)
__global__ void __launch_bounds__(256)
ce_rows_kernel(const float* __restrict__ logits, const int* __restrict__ labels, float* __restrict__ loss, int V) {
  __shared__ float red[8];
  __shared__ float bc;
  const long long r = blockIdx.x;
  const float* lg = logits + r * V;
  float m = -INFINITY;
  for (int v = threadIdx.x; v < V; v += blockDim.x) m = fmaxf(m, lg[v]);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) { float t = red[0]; for (int i = 1; i < 8; ++i) t = fmaxf(t, red[i]); bc = t; }
  __syncthreads();
  m = bc;
  float s = 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) s += expf(lg[v] - m);
  s = block_sum_256(s, red);
  if (threadIdx.x == 0) {
    const int lab = labels[r];
    loss[r] = (lab >= 0 && lab < V) ? logf(s) + m - lg[lab] : NAN;      // TF: NaN for an out-of-range label
  }
}
int ce_rows(const float* logits, const int* labels, float* loss, long long rows, int V, cudaStream_t stream) {
  MVB_REQUIRE(logits && labels && loss && rows > 0 && V > 0, "ce_rows: bad args");
  ce_rows_kernel<<<(unsigned)rows, 256, 0, stream>>>(logits, labels, loss, V);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int adv_step(const float* x, const float* adv, const float* grad, float* out, float eps, float step, long long n,
             cudaStream_t stream) {
  MVB_REQUIRE(x && adv && grad && out && n > 0 && eps >= 0.f, "adv_step: bad args");
  const long long b = (n + 255) / 256;
  adv_step_kernel<<<(unsigned)(b < sm_count() * 16 ? b : sm_count() * 16), 256, 0, stream>>>(x, adv, grad, out, eps, step, n);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}
int mix(const float* a, const float* b, float* out, float w, long long n, cudaStream_t stream) {
  MVB_REQUIRE(a && b && out && n > 0, "mix: bad args");
  const long long bl = (n + 255) / 256;
  mix_kernel<<<(unsigned)(bl < sm_count() * 16 ? bl : sm_count() * 16), 256, 0, stream>>>(a, b, out, w, n);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int enc_class_input_bwd(const float* dxh, int cpad, const int* frame_idx, const int* label,
                        float* dscene, long long NS, int H, int W, cudaStream_t stream) {
  MVB_REQUIRE(dxh && frame_idx && label && dscene && NS > 0, "enc_class_input_bwd: bad args");
  enc_class_input_bwd_kernel<<<(unsigned)NS, 64, 0, stream>>>(dxh, cpad, frame_idx, label, dscene, make_grid(H, W));
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int enc_class_input_mix_bwd(const float* dxh, int cpad, const int* frame_idx, const int* label, const int* label2,
                            float beta, float* dscene, long long NS, int H, int W, cudaStream_t stream) {
  MVB_REQUIRE(dxh && frame_idx && label && label2 && dscene && NS > 0, "enc_class_input_mix_bwd: bad args");
  enc_class_input_mix_bwd_kernel<<<(unsigned)NS, 64, 0, stream>>>(dxh, cpad, frame_idx, label, label2, beta, dscene, make_grid(H, W));
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int scene_mean_bwd(const float* dmean, const int* frame_idx, float* dscene, long long N, int T,
                   long long HWC, cudaStream_t stream) {
  MVB_REQUIRE(dmean && frame_idx && dscene && N > 0 && T > 0, "scene_mean_bwd: bad args");
  scene_mean_bwd_kernel<<<grid_for(N * HWC, 256), 256, 0, stream>>>(dmean, frame_idx, dscene, N, T, HWC);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int clip_adadelta(float* w, const float* grad, float* acc, float* acc_upd, long long n, float lr,
                  float rho, float eps, float clip, float wd, float gscale, cudaStream_t stream) {
  MVB_REQUIRE(w && grad && acc && acc_upd && n > 0, "clip_adadelta: bad args");
  clip_adadelta_kernel<<<grid_for(n, 256), 256, 0, stream>>>(w, grad, acc, acc_upd, n, lr, rho, eps, clip, wd, gscale);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int clip_update(float* w, const float* grad, float* s1, float* s2, long long n, int kind, float lr, float p1, float p2,
                float eps, float clip, float wd, float gscale, cudaStream_t stream) {
  MVB_REQUIRE(w && grad && s1 && n > 0 && kind >= 1 && kind <= 3 && (kind == 1 || s2), "clip_update: bad args (kind %d)", kind);
  clip_update_kernel<<<grid_for(n, 256), 256, 0, stream>>>(w, grad, s1, s2, n, kind, lr, p1, p2, eps, clip, wd, gscale);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

}  // namespace mvb
