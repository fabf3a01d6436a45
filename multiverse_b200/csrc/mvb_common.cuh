// Common device/host helpers for libmultiverse_b200 (H100, sm_90a only).
//
// Internal "halo" layout used by every kernel of the hot path:
//   a location grid of H x W cells is stored with ONE shared zero column and ONE
//   shared zero row: pixel (n, y, x) lives at row  r = n*S + y*(W+1) + x  with
//   S = (H+1)*(W+1);  x == W and y == H are zero cells that are never written.
//   A 3x3 "SAME" tap (dy,dx) is then the constant row shift  (dy-1)*(W+1)+(dx-1)
//   for every pixel of every image, so the im2col A-operand of the ConvLSTM GEMM is
//   a plain 2-D TMA box of the activation matrix [rows, channels] at a shifted row
//   coordinate (rows < 0 / >= R are zero-filled by TMA).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "mvb_wgmma.cuh"

namespace mvb {

constexpr int kHidden = 256;          // enc/dec hidden size of every published config
constexpr int kGates = 4 * kHidden;   // i, j, f, o

// ----------------------------------------------------------------------------------
// error plumbing (C-ABI: int return codes + thread-local message)
// ----------------------------------------------------------------------------------
enum : int {
  MVB_OK = 0,
  MVB_ERR_INVALID = 1,
  MVB_ERR_CUDA = 2,
  MVB_ERR_DRIVER = 3,
};

void set_error(const char* fmt, ...);
const char* get_error();

#define MVB_CHECK_CUDA(expr)                                                      \
  do {                                                                            \
    cudaError_t _e = (expr);                                                      \
    if (_e != cudaSuccess) {                                                      \
      mvb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),      \
                     __FILE__, __LINE__);                                         \
      return mvb::MVB_ERR_CUDA;                                                   \
    }                                                                             \
  } while (0)

#define MVB_REQUIRE(cond, ...)                                                    \
  do {                                                                            \
    if (!(cond)) {                                                                \
      mvb::set_error(__VA_ARGS__);                                                \
      return mvb::MVB_ERR_INVALID;                                                \
    }                                                                             \
  } while (0)

// ----------------------------------------------------------------------------------
// halo-layout index helpers
// ----------------------------------------------------------------------------------
struct Grid {
  int H, W;      // valid cells
  int Wp;        // W + 1
  int S;         // (H+1)*(W+1) rows per sample
};
__host__ __device__ inline Grid make_grid(int H, int W) {
  Grid g; g.H = H; g.W = W; g.Wp = W + 1; g.S = (H + 1) * (W + 1); return g;
}

// ----------------------------------------------------------------------------------
// Inputs of the training step (SURVEY.md §8 row f-1), read either from dense fp32 tensors or computed where they are
// consumed from the trajectories: kernels that take one of these as a template parameter run the same arithmetic on
// the same values either way.
// ----------------------------------------------------------------------------------
// dense fp32 offsets: element i of [rows, V, 2], or cell i of [rows, V] as a pair
struct DenseOffsets {
  const float* p;
  __device__ __forceinline__ float operator()(long long i) const { return p[i]; }
  __device__ __forceinline__ float2 cell(long long i) const { return reinterpret_cast<const float2*>(p)[i]; }
};
// float32(point - centre) computed in double, as traj_to_grid and the host's float64 preprocessing cast to float32.
// Row r of [rows, H*W, 2] is the point traj + (r % n) * row_stride + (r / n) * step_stride (in doubles); centers
// fp64 [H*W, 2].
struct TrajOffsets {
  const double* traj;
  const double* centers;
  long long n, row_stride, step_stride;
  int hw;
  __device__ __forceinline__ float2 cell(long long i) const {
    const long long r = i / hw;
    const int v = (int)(i - r * hw);
    const double* p = traj + (r % n) * row_stride + (r / n) * step_stride;
    return make_float2((float)(p[0] - centers[2 * v]), (float)(p[1] - centers[2 * v + 1]));
  }
  __device__ __forceinline__ float operator()(long long i) const {
    const float2 o = cell(i >> 1);
    return (i & 1) ? o.y : o.x;
  }
};

// Grid-class label of cell v for the label cell `lab` under --soft_grid `mode` (code/pred_models.py:1085-1136, as
// pred_models._soft_labels builds the maps): the 3x3 (modes 1-6) or 5x5 (mode 7) kernel value at the cell's offset
// from the label cell, 0 outside the kernel; a negative label indexes from the end, as numpy's m[cls] does.
// mode 0: the one-hot map of a label in [0, H*W).  Values are float32 of the float64 table entries.
__device__ __forceinline__ float grid_label(int lab, int v, int mode, int H, int W) {
  const int hw = H * W;
  if (mode == 0) return lab == v ? 1.f : 0.f;
  if (lab < -hw || lab >= hw) return 0.f;
  const int cell = lab < 0 ? lab + hw : lab;
  const int r = mode == 7 ? 2 : 1;
  const int dy = v / W - cell / W + r, dx = v % W - cell % W + r;
  if (dy < 0 || dy > 2 * r || dx < 0 || dx > 2 * r) return 0.f;
  if (mode == 7) {
    if (dy == 2 && dx == 2) return (float)0.8;
    return (dy >= 1 && dy <= 3 && dx >= 1 && dx <= 3) ? (float)0.0125 : (float)0.0625;
  }
  const bool centre = dy == 1 && dx == 1;
  switch (mode) {
    case 1: return centre ? (float)1.0 : (float)0.1;
    case 2: return centre ? (float)1.0 : (float)0.01;
    case 3: return centre ? (float)1.0 : (float)0.05;
    case 4: return centre ? (float)0.9 : (float)0.0125;
    case 5: return centre ? (float)0.6 : (float)0.05;
    default: return centre ? (float)0.2 : (float)0.1;
  }
}

// ----------------------------------------------------------------------------------
// "bf16x2" operand format (planes code kBf16Planes): v = p0 + p1 + O(2^-18 |v|), both planes bf16; the product
// of two such operands is accumulated as a0*b0 + a0*b1 + a1*b0 (a1*b1, 2^-18 of the result, is dropped).
// A plane tensor is [2][rows][cpad] bf16.
// ----------------------------------------------------------------------------------
constexpr int kBf16Planes = 2;
__device__ __forceinline__ void split_planes(float v, __nv_bfloat16 (&out)[kBf16Planes]) {
  out[0] = __float2bfloat16_rn(v);
  out[1] = __float2bfloat16_rn(v - __bfloat162float(out[0]));
}

// ----------------------------------------------------------------------------------
// "f16f8" operand format (planes code kPlanesF16F8): v = a0 + a1 with a0 = fp16(v); the tensor cores see
//   a0 (fp16 plane), e0 = e4m3(a0) and e1 = e4m3(a1 * 2^12) (two fp8 planes), and the product of two such
// operands is accumulated as   a0*b0 (fp16 wgmma)  +  e0(a)*e0'(b)  +  e1(a)*e1'(b)  (e4m3 wgmma, twice the rate)
// where for the WEIGHT operand e0' = e4m3(b1) and e1' = e4m3(b0 * 2^-12): the two fp8 products are the cross
// terms a0*b1 and a1*b0 to 4 significant bits, i.e. to 2^-17 of the main product; a1*b1 (2^-24) is dropped.
// All three products have the same scale, so they share ONE fp32 accumulator.  2 bf16-pass equivalents
// instead of 3 at the accuracy class of the bf16 x 2-plane scheme.
// Buffer layout for R rows of cpad channels: [fp16 R*cpad][fp8: R rows of 2*cpad bytes] = the bytes of two bf16
// planes, so the same allocations serve both formats.  Inside an fp8 row the two planes are interleaved per K chunk
// of the cell kernel, so that ONE 128-byte TMA row carries both (f8_off): per 64-channel chunk of the x block
// [e0 (64) | e1 (64)], a trailing 32-channel chunk as [e0 (32) | e1 (32)], then per 64-channel chunk of the h block
// [e0 (64) | e1 (64)],  cxp = cpad - 256 (a multiple of 32).  For cxp <= 64 the x block is [e0 (cxp) | e1 (cxp)].
// ----------------------------------------------------------------------------------
constexpr int kPlanesF16F8 = 16;
constexpr float kF8ResidualScale = 4096.f;   // 2^12: residual of an fp16 rounding, brought into e4m3's range

// the `planes` codes of the two operand formats; kernels that serve both take FMT = 0 (bf16x2) or 1 (f16f8)
inline bool valid_planes(int P) { return P == kBf16Planes || P == kPlanesF16F8; }

// byte offset inside an fp8 row of channel c, plane p
__host__ __device__ __forceinline__ int f8_off(int c, int p, int cpad) {
  const int hoff = cpad - kHidden;
  if (c >= hoff) { const int cc = c - hoff; return 2 * hoff + (cc >> 6) * 128 + p * 64 + (cc & 63); }
  const int c0 = c & ~63, width = hoff - c0 < 64 ? hoff - c0 : 64;     // c's x chunk: 64 channels, or a trailing 32
  return 2 * c0 + p * width + (c & 63);
}

__device__ __forceinline__ uint8_t to_e4m3(float v) {
  return (uint8_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3);
}
// two values -> their fp16 pair, the e4m3 pair of the fp16 values and the e4m3 pair of the scaled residuals
// (packed conversions: 1 + 1 + 1 cvt for two values; low half / low byte = the first value)
__device__ __forceinline__ void split_f16f8_x2(float v0, float v1, uint32_t& h2, uint32_t& e0, uint32_t& e1) {
  const __half2 h = __floats2half2_rn(v0, v1);
  h2 = *reinterpret_cast<const uint32_t*>(&h);
  e0 = (uint32_t)__nv_cvt_halfraw2_to_fp8x2(static_cast<__half2_raw>(h), __NV_SATFINITE, __NV_E4M3);
  const float2 f = __half22float2(h);
  e1 = (uint32_t)__nv_cvt_float2_to_fp8x2(make_float2((v0 - f.x) * kF8ResidualScale, (v1 - f.y) * kF8ResidualScale),
                                          __NV_SATFINITE, __NV_E4M3);
}
// 8 consecutive channels -> 16 B of fp16 and 8 B of each fp8 plane
__device__ __forceinline__ void split_f16f8_x8(const float (&v)[8], uint4& f16, uint2& p0, uint2& p1) {
  uint32_t hw[4], b0[2] = {0u, 0u}, b1[2] = {0u, 0u};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t e0, e1;
    split_f16f8_x2(v[2 * i], v[2 * i + 1], hw[i], e0, e1);
    b0[i >> 1] |= e0 << (16 * (i & 1));
    b1[i >> 1] |= e1 << (16 * (i & 1));
  }
  f16 = make_uint4(hw[0], hw[1], hw[2], hw[3]);
  p0 = make_uint2(b0[0], b0[1]);
  p1 = make_uint2(b1[0], b1[1]);
}
// store 8 consecutive channels [ch, ch+8) (ch % 8 == 0) of one row into an f16f8 operand buffer (base = start of
// the fp16 region, plane_stride = rows * cpad = elements of it)
__device__ __forceinline__ void store_f16f8_x8(void* base, long long plane_stride, long long row, int ch, int cpad,
                                               const float (&v)[8]) {
  uint4 f16; uint2 p0, p1;
  split_f16f8_x8(v, f16, p0, p1);
  *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(base) + row * cpad + ch) = f16;
  uint8_t* b8 = reinterpret_cast<uint8_t*>(base) + 2 * plane_stride + row * 2 * cpad;
  *reinterpret_cast<uint2*>(b8 + f8_off(ch, 0, cpad)) = p0;
  *reinterpret_cast<uint2*>(b8 + f8_off(ch, 1, cpad)) = p1;
}

// one element
__device__ __forceinline__ void store_f16f8(void* base, long long plane_stride, long long row, int ch, int cpad,
                                            float v) {
  const __half a0 = __float2half_rn(v);
  const float f0 = __half2float(a0);
  reinterpret_cast<__half*>(base)[row * cpad + ch] = a0;
  uint8_t* b8 = reinterpret_cast<uint8_t*>(base) + 2 * plane_stride + row * 2 * cpad;
  b8[f8_off(ch, 0, cpad)] = to_e4m3(f0);
  b8[f8_off(ch, 1, cpad)] = to_e4m3((v - f0) * kF8ResidualScale);
}

__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 lo, __nv_bfloat16 hi) {
  return (uint32_t)__bfloat16_as_ushort(lo) | ((uint32_t)__bfloat16_as_ushort(hi) << 16);
}

// ----------------------------------------------------------------------------------
// activations: fp32, ~1e-6 accurate (MUFU.EX2 is 2^-22; tanh.approx at 2^-11 is NOT
// acceptable for the 1e-4 parity bar, so it is never used)
// ----------------------------------------------------------------------------------
// MUFU.RCP (1 ulp) instead of the correctly rounded __frcp_rn (MUFU + Newton fix-up, ~5 instructions): the gate
// epilogue of the cell evaluates five of these per state element and is co-critical with the f16f8 mainloop
__device__ __forceinline__ float rcp_fast(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float sigmoid_acc(float x) {
  return rcp_fast(1.0f + __expf(-x));
}
__device__ __forceinline__ float tanh_acc(float x) {
  // 1 - 2/(exp(2x)+1): exact limits at +-inf, abs error ~1e-7
  return 1.0f - 2.0f * rcp_fast(__expf(2.0f * x) + 1.0f);
}

// ----------------------------------------------------------------------------------
// warp reductions
// ----------------------------------------------------------------------------------
// Opt-in to more than 48 KB of dynamic shared memory: once per (kernel, device) and again whenever a launch needs
// more than was granted.  The attribute lives in the device's context, so a process that drives several GPUs
// through this library needs it set on each of them; a racing second thread at worst repeats the idempotent call.
struct SmemOptIn { size_t granted[64] = {}; };
template <class Kernel>
inline cudaError_t smem_opt_in(SmemOptIn& st, Kernel kernel, size_t bytes) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (bytes <= st.granted[dev]) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) st.granted[dev] = bytes;
  return e;
}

// Number of SMs of the current device (cached per device; 132 on the H100 SXM): grid-stride launchers size their grids in
// multiples of it instead of a hard-coded constant.
inline int sm_count() {
  static int cached[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (!cached[dev]) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

// Sums each of v[0..7] over the warp with 9 shuffles instead of 8 butterflies (40): at every halving step a lane
// keeps one half of its values and hands the other half to its partner.  Lane l returns the warp total of value
// ((l >> 4) & 1) * 4 + ((l >> 3) & 1) * 2 + ((l >> 2) & 1); the four lanes that share l >> 2 hold the same total.
__device__ __forceinline__ float warp_fold8(const float (&v)[8], int lane) {
  const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4;
  float a[4], b[2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    a[i] = (h16 ? v[i + 4] : v[i]) + __shfl_xor_sync(0xffffffffu, h16 ? v[i] : v[i + 4], 16);
#pragma unroll
  for (int i = 0; i < 2; ++i)
    b[i] = (h8 ? a[i + 2] : a[i]) + __shfl_xor_sync(0xffffffffu, h8 ? a[i] : a[i + 2], 8);
  float c = (h4 ? b[1] : b[0]) + __shfl_xor_sync(0xffffffffu, h4 ? b[0] : b[1], 4);
  c += __shfl_xor_sync(0xffffffffu, c, 2);
  c += __shfl_xor_sync(0xffffffffu, c, 1);
  return c;
}
__device__ __forceinline__ int warp_fold8_index(int lane) { return ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1); }

// fp32 pairs: the graph-attention and head kernels write their dot products and weighted sums on float2; each lane
// is one correctly rounded fma / mul (H100 has no packed fp32 FMA instruction).
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ----------------------------------------------------------------------------------
// PTX wrappers: mbarrier, TMA, clusters, wgmma descriptors
// ----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}

// 3-D tiled TMA load, completes on an mbarrier with complete_tx::bytes.
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// 4-D tiled TMA load.
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ---- clusters: CTAs of one cluster exchange operand tiles and barrier arrivals ----
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// TMA load multicast to the CTAs of `mask`: the box lands at the same smem offset in each of them and each of
// their barriers (same offset) receives the transaction bytes.
__device__ __forceinline__ void tma_load_3d_mc(void* dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                               int c1, int c2, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4, %5}], [%2], %6;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "h"(mask)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d_mc(void* dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                               int c1, int c2, int c3, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "h"(mask)
      : "memory");
}
// arrive on the barrier at the same offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n"
      ".reg .b32 ra;\n"
      "mapa.shared::cluster.u32 ra, %0, %1;\n"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(cta)
      : "memory");
}

// Register budget of a warpgroup (setmaxnreg): the TMA producer warpgroup hands its registers to the MMA
// warpgroups, whose fp32 accumulators live in registers.
template <int R>
__device__ __forceinline__ void regs_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void regs_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// K-major or MN-major shared-memory matrix descriptor of wgmma (sm_90): start address, leading / stride byte offsets
// and the swizzle of the TMA-written tile (layout_type 1 = 128B, 2 = 64B, 3 = 32B).  The hardware applies the swizzle
// to the absolute shared-memory address bits, like the TMA unit that wrote the tile, so a descriptor may start at
// any 16-byte step inside a swizzled row (K) and at any row.  sbo = byte stride between 8-row groups.
constexpr uint32_t kSwizzle128B = 1, kSwizzle64B = 2;
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t sbo_bytes,
                                                   uint32_t layout_type, uint32_t lbo_bytes = 0) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)(lbo_bytes >> 4) << 16;
  d |= (uint64_t)(sbo_bytes >> 4) << 32;
  d |= (uint64_t)layout_type << 62;
  return d;
}
// the same as {lo, hi} halves: only `lo` (address >> 4) moves along K / rows
constexpr uint32_t smem_desc_hi(uint32_t sbo_bytes, uint32_t layout_type) {
  return (sbo_bytes >> 4) | (layout_type << 30);
}
__device__ __forceinline__ uint64_t desc_of(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }

// ----------------------------------------------------------------------------------
// host: TMA descriptor encode through the runtime's driver entry point (no -lcuda)
// ----------------------------------------------------------------------------------
int encode_tmap_3d_bf16(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1,
                        uint64_t d2, uint64_t stride1_bytes, uint64_t stride2_bytes,
                        uint32_t b0, uint32_t b1, uint32_t b2, int swizzle_bytes);
int encode_tmap_3d_u8(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                      uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t b0, uint32_t b1, uint32_t b2,
                      int swizzle_bytes);
int encode_tmap_4d_bf16(CUtensorMap* out, const void* base, const uint64_t (&dims)[4],
                        const uint64_t (&strides_bytes)[3], const uint32_t (&box)[4],
                        int swizzle_bytes);
int encode_tmap_4d_u8(CUtensorMap* out, const void* base, const uint64_t (&dims)[4],
                      const uint64_t (&strides_bytes)[3], const uint32_t (&box)[4], int swizzle_bytes);

}  // namespace mvb
