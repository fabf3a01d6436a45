// Layout kernels at the API boundary: NHWC fp32 (the reference's placeholder layout,
// code/pred_models.py:62-115) <-> the library's halo layout / bf16 operand planes, and the
// class-encoder input of code/pred_models.py:210.  All HBM-bound, one pass.
#include "mvb_common.cuh"
#include "mvb_kernels.h"

namespace mvb {

// One thread per (pixel, channel); channel fastest so reads and writes coalesce.  FMT = 1: f16f8 operand format.
template <int FMT, class Src>
__global__ void nhwc_to_planes_kernel(const Src src, __nv_bfloat16* __restrict__ dst,
                                      long long plane_stride, int cpad, int ch_off, long long NS,
                                      Grid g, int C, int comp) {
  const long long total = NS * g.H * g.W * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long pix = i / C;
    const int x = (int)(pix % g.W);
    const long long t = pix / g.W;
    const int y = (int)(t % g.H);
    const long long s = t / g.H;
    const long long row = s * g.S + (long long)y * g.Wp + x;
    const float v = src(i);
    if (FMT) {      // f16f8 operand format (mvb_common.cuh)
      store_f16f8(dst, plane_stride, row, ch_off + c, cpad, v);
      continue;
    }
    __nv_bfloat16 pl[kBf16Planes];
    split_planes(v, pl);
    __nv_bfloat16* d = dst + row * cpad + ch_off + c;
    d[0] = pl[0];
    d[plane_stride] = pl[1];
    if (comp) {
      // Compensated x block for large-magnitude inputs (the regression encoder is fed raw pixel
      // offsets up to ~1.9e3, code/pred_models.py:232): the padded channels carry the terms the
      // 3-product plane scheme drops, so the MMA itself restores fp32-grade accuracy:
      //   A: [x | r=x-x0-x1 | x | x1]   B: [W | W | W-w0-w1 | w1]   (pack_weights_kernel)
      const float r = (v - __bfloat162float(pl[0])) - __bfloat162float(pl[1]);
      __nv_bfloat16 rp[kBf16Planes];
      split_planes(r, rp);
      d[C] = rp[0];
      d[plane_stride + C] = rp[1];
      d[2 * C] = pl[0];
      d[plane_stride + 2 * C] = pl[1];
      d[3 * C] = pl[1];
      d[plane_stride + 3 * C] = __float2bfloat16_rn(0.f);
    }
  }
}

__global__ void nhwc_halo_copy_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                      long long NS, Grid g, int C, int to_nhwc) {
  const int c4 = C / 4;
  const long long total = NS * g.H * g.W * c4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % c4);
    const long long pix = i / c4;
    const int x = (int)(pix % g.W);
    const long long t = pix / g.W;
    const int y = (int)(t % g.H);
    const long long s = t / g.H;
    const long long row = s * g.S + (long long)y * g.Wp + x;
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    if (to_nhwc) d4[pix * c4 + c] = s4[row * c4 + c];
    else d4[row * c4 + c] = s4[pix * c4 + c];
  }
}

// One block of 64 threads per sample row: thread c handles scene channel c.
template <int FMT>
__global__ void enc_class_input_kernel(const float* __restrict__ scene_conv,
                                       const int* __restrict__ frame_idx,
                                       const int* __restrict__ label,
                                       const int* __restrict__ prev_label,
                                       __nv_bfloat16* __restrict__ xh, long long plane_stride,
                                       int cpad, Grid g) {
  const long long s = blockIdx.x;
  const int c = threadIdx.x;  // 0..63
  const int hw = g.H * g.W;
  if (prev_label) {
    const int pl = prev_label[s];
    if (pl >= 0 && pl < hw) {
      const long long row = s * g.S + (long long)(pl / g.W) * g.Wp + (pl % g.W);
      if (FMT) {
        store_f16f8(xh, plane_stride, row, c, cpad, 0.f);
      } else {
        xh[row * cpad + c] = __float2bfloat16_rn(0.f);
        xh[plane_stride + row * cpad + c] = __float2bfloat16_rn(0.f);
      }
    }
  }
  __syncthreads();  // same-pixel clear/set ordering inside the block
  const int lb = label[s];
  if (lb >= 0 && lb < hw) {
    const long long row = s * g.S + (long long)(lb / g.W) * g.Wp + (lb % g.W);
    const float v = scene_conv[((long long)frame_idx[s] * hw + lb) * 64 + c];
    if (FMT) { store_f16f8(xh, plane_stride, row, c, cpad, v); return; }
    __nv_bfloat16 pl[kBf16Planes];
    split_planes(v, pl);
    xh[row * cpad + c] = pl[0];
    xh[plane_stride + row * cpad + c] = pl[1];
  }
}

// SimAug multiview_exp 3 (SimAug/code/pred_models.py:616-638): the observed grid class is a mix of two one-hot maps,
// beta * one_hot(label) + one_hot(label2) * (1 - beta), so two pixels of the x block carry scene features (one, with the
// fp32 sum of the two weights, when both labels name the same cell).  The x block must be zero on entry.
template <int FMT>
__global__ void enc_class_input_mix_kernel(const float* __restrict__ scene_conv, const int* __restrict__ frame_idx,
                                           const int* __restrict__ label, const int* __restrict__ label2, float beta,
                                           __nv_bfloat16* __restrict__ xh, long long plane_stride, int cpad, Grid g) {
  const long long s = blockIdx.x;
  const int c = threadIdx.x;  // 0..63
  const int hw = g.H * g.W;
  const int l1 = label[s], l2 = label2[s];
  const float w1 = beta, w2 = 1.0f - beta;
  auto put = [&](int lb, float wgt) {
    if (lb < 0 || lb >= hw) return;
    const long long row = s * g.S + (long long)(lb / g.W) * g.Wp + (lb % g.W);
    const float v = scene_conv[((long long)frame_idx[s] * hw + lb) * 64 + c] * wgt;
    if (FMT) { store_f16f8(xh, plane_stride, row, c, cpad, v); return; }
    __nv_bfloat16 pl[kBf16Planes];
    split_planes(v, pl);
    xh[row * cpad + c] = pl[0];
    xh[plane_stride + row * cpad + c] = pl[1];
  };
  if (l1 == l2) {
    put(l1, w1 + w2);
  } else {
    put(l1, w1);
    put(l2, w2);
  }
}

int enc_class_input_mix(const float* scene_conv, const int* frame_idx, const int* label, const int* label2, float beta,
                        void* xh_planes, long long plane_stride, int cpad, long long NS, int H, int W, int P,
                        cudaStream_t stream) {
  MVB_REQUIRE(valid_planes(P), "enc_class_input_mix: planes P=%d not 2 or %d", P, kPlanesF16F8);
  MVB_REQUIRE(scene_conv && frame_idx && label && label2 && xh_planes && NS > 0, "enc_class_input_mix: bad args");
  const Grid g = make_grid(H, W);
  __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(xh_planes);
  if (P == kPlanesF16F8) enc_class_input_mix_kernel<1><<<(unsigned)NS, 64, 0, stream>>>(scene_conv, frame_idx, label, label2, beta, d, plane_stride, cpad, g);
  else enc_class_input_mix_kernel<0><<<(unsigned)NS, 64, 0, stream>>>(scene_conv, frame_idx, label, label2, beta, d, plane_stride, cpad, g);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int nhwc_to_planes(const float* src, void* dst_planes, long long plane_stride, int cpad, int ch_off,
                   long long NS, int H, int W, int C, int P, int comp, cudaStream_t stream) {
  MVB_REQUIRE(valid_planes(P), "nhwc_to_planes: planes P=%d not 2 or %d", P, kPlanesF16F8);
  MVB_REQUIRE(src && dst_planes && NS > 0 && C > 0 && ch_off + C <= cpad, "nhwc_to_planes: bad args");
  MVB_REQUIRE(!comp || (P == kBf16Planes && ch_off + 4 * C <= cpad - kHidden), "nhwc_to_planes: compensated block needs planes=2 and 4*C inside the x block");
  const Grid g = make_grid(H, W);
  const long long total = NS * H * W * C;
  const int threads = 256;
  const int blocks = (int)((total + threads - 1) / threads < sm_count() * 16 ? (total + threads - 1) / threads : sm_count() * 16);
  __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(dst_planes);
  const DenseOffsets s{src};
  if (P == kPlanesF16F8) nhwc_to_planes_kernel<1><<<blocks, threads, 0, stream>>>(s, d, plane_stride, cpad, ch_off, NS, g, C, 0);
  else nhwc_to_planes_kernel<0><<<blocks, threads, 0, stream>>>(s, d, plane_stride, cpad, ch_off, NS, g, C, comp);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

// nhwc_to_planes of the offsets float32(traj[s] - centre) [NS,H,W,2] into channels [0, 2) of the bf16x2 planes (and
// the compensation channels [2, 8) under comp), computed in the kernel instead of read from a dense tensor: the
// regression encoder's input straight from the observed trajectories (point s at traj + s * traj_stride doubles).
int traj_to_planes(const double* traj, long long traj_stride, const double* centers, void* dst_planes,
                   long long plane_stride, int cpad, long long NS, int H, int W, int comp, cudaStream_t stream) {
  MVB_REQUIRE(traj && centers && dst_planes && NS > 0 && H > 0 && W > 0 && traj_stride >= 2 &&
              (comp ? 8 : 2) <= cpad - kHidden, "traj_to_planes: bad args");
  const Grid g = make_grid(H, W);
  const long long total = NS * H * W * 2;
  const int threads = 256;
  const int blocks = (int)((total + threads - 1) / threads < sm_count() * 16 ? (total + threads - 1) / threads : sm_count() * 16);
  const TrajOffsets s{traj, centers, NS, traj_stride, 0, H * W};
  nhwc_to_planes_kernel<0><<<blocks, threads, 0, stream>>>(s, reinterpret_cast<__nv_bfloat16*>(dst_planes),
                                                           plane_stride, cpad, 0, NS, g, 2, comp);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

// Feed generation on the device (SURVEY.md §8 row f-1): what get_grid_input does per trajectory on the host
// (code/multifuture_inference.py:115-156 == code/preprocess.py:436-475): cell index = ceil(x / gap) (0 -> 1) - 1 per
// axis, offsets = point - centre of every cell.  Double arithmetic on the caller's float64 points and centres, so
// labels are bit-identical to numpy's and the fp32 offsets equal numpy's float64 result cast to float32.
__global__ void traj_to_grid_kernel(const double* __restrict__ traj, const double* __restrict__ centers,
                                    double h_gap, double w_gap, int* __restrict__ labels,
                                    float* __restrict__ regress, long long NT, int H, int W) {
  const int hw = H * W;
  const long long total = NT * hw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long p = i / hw;
    const int cell = (int)(i - p * hw);
    const double x = traj[2 * p], y = traj[2 * p + 1];
    if (cell == 0) {
      long long xi = (long long)ceil(x / w_gap), yi = (long long)ceil(y / h_gap);
      if (xi == 0) xi = 1;
      if (yi == 0) yi = 1;
      labels[p] = (int)((yi - 1) * W + (xi - 1));
    }
    reinterpret_cast<float2*>(regress)[i] =
        make_float2((float)(x - centers[2 * cell]), (float)(y - centers[2 * cell + 1]));
  }
}

int traj_to_grid(const double* traj, const double* centers, double h_gap, double w_gap, int* labels,
                 float* regress, long long NT, int H, int W, cudaStream_t stream) {
  MVB_REQUIRE(traj && centers && labels && regress && NT > 0 && H > 0 && W > 0 && h_gap > 0 && w_gap > 0,
              "traj_to_grid: bad args");
  const long long total = NT * H * W;
  const int blocks = (int)((total + 255) / 256 < sm_count() * 16 ? (total + 255) / 256 : sm_count() * 16);
  traj_to_grid_kernel<<<blocks, 256, 0, stream>>>(traj, centers, h_gap, w_gap, labels, regress, NT, H, W);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int nhwc_halo_copy(const float* src, float* dst, long long NS, int H, int W, int C, int to_nhwc,
                   cudaStream_t stream) {
  MVB_REQUIRE(src && dst && NS > 0 && C > 0 && C % 4 == 0, "nhwc_halo_copy: bad args (C=%d must be a multiple of 4)", C);
  const Grid g = make_grid(H, W);
  const long long total = NS * H * W * (C / 4);
  const int threads = 256;
  const int blocks = (int)((total + threads - 1) / threads < sm_count() * 16 ? (total + threads - 1) / threads : sm_count() * 16);
  nhwc_halo_copy_kernel<<<blocks, threads, 0, stream>>>(src, dst, NS, g, C, to_nhwc);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int enc_class_input(const float* scene_conv, const int* frame_idx, const int* label,
                    const int* prev_label, void* xh_planes, long long plane_stride, int cpad,
                    long long NS, int H, int W, int P, cudaStream_t stream) {
  MVB_REQUIRE(valid_planes(P), "enc_class_input: planes P=%d not 2 or %d", P, kPlanesF16F8);
  MVB_REQUIRE(scene_conv && frame_idx && label && xh_planes && NS > 0, "enc_class_input: bad args");
  const Grid g = make_grid(H, W);
  __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(xh_planes);
  if (P == kPlanesF16F8) enc_class_input_kernel<1><<<(unsigned)NS, 64, 0, stream>>>(scene_conv, frame_idx, label, prev_label, d, plane_stride, cpad, g);
  else enc_class_input_kernel<0><<<(unsigned)NS, 64, 0, stream>>>(scene_conv, frame_idx, label, prev_label, d, plane_stride, cpad, g);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

}  // namespace mvb
