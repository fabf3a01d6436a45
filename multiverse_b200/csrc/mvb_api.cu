// extern "C" surface of libmultiverse_b200 (declared in include/multiverse_b200.h) plus the
// host-side plumbing shared by the kernels: error string, launch counter, TMA descriptor encode.
#include "mvb_common.cuh"
#include "mvb_kernels.h"
#include "../../include/multiverse_b200.h"

#include <string.h>

namespace mvb {

static thread_local char g_err[512] = "";
static thread_local long long g_launches = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }
void count_launch(int n) { g_launches += n; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
    set_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s",
              cudaGetErrorString(e));
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

static int encode_tmap_3d_any(CUtensorMapDataType dt, CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                        uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t b0, uint32_t b1,
                        uint32_t b2, int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return MVB_ERR_DRIVER;
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
  cuuint32_t box[3] = {b0, b1, b2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUtensorMapSwizzle sw = swizzle_bytes == 128  ? CU_TENSOR_MAP_SWIZZLE_128B
                          : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                          : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = fn(out, dt, 3, const_cast<void*>(base), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (dims %llu,%llu,%llu box %u,%u,%u)",
              (int)r, (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, b0,
              b1, b2);
    return MVB_ERR_DRIVER;
  }
  return MVB_OK;
}

int encode_tmap_3d_bf16(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                        uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t b0, uint32_t b1,
                        uint32_t b2, int swizzle_bytes) {
  return encode_tmap_3d_any(CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, out, base, d0, d1, d2, stride1_bytes, stride2_bytes,
                            b0, b1, b2, swizzle_bytes);
}
int encode_tmap_3d_u8(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                      uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t b0, uint32_t b1, uint32_t b2,
                      int swizzle_bytes) {
  return encode_tmap_3d_any(CU_TENSOR_MAP_DATA_TYPE_UINT8, out, base, d0, d1, d2, stride1_bytes, stride2_bytes,
                            b0, b1, b2, swizzle_bytes);
}

static int encode_tmap_4d_any(CUtensorMapDataType dt, CUtensorMap* out, const void* base, const uint64_t (&dims)[4],
                              const uint64_t (&strides_bytes)[3], const uint32_t (&box)[4], int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return MVB_ERR_DRIVER;
  cuuint64_t d[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t st[3] = {strides_bytes[0], strides_bytes[1], strides_bytes[2]};
  cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUtensorMapSwizzle sw = swizzle_bytes == 128  ? CU_TENSOR_MAP_SWIZZLE_128B
                          : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                          : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = fn(out, dt, 4, const_cast<void*>(base), d, st, bx, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(4d) failed with CUresult %d (dims %llu,%llu,%llu,%llu)", (int)r,
              (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
              (unsigned long long)dims[3]);
    return MVB_ERR_DRIVER;
  }
  return MVB_OK;
}

int encode_tmap_4d_bf16(CUtensorMap* out, const void* base, const uint64_t (&dims)[4],
                        const uint64_t (&strides_bytes)[3], const uint32_t (&box)[4],
                        int swizzle_bytes) {
  return encode_tmap_4d_any(CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, out, base, dims, strides_bytes, box, swizzle_bytes);
}
int encode_tmap_4d_u8(CUtensorMap* out, const void* base, const uint64_t (&dims)[4],
                      const uint64_t (&strides_bytes)[3], const uint32_t (&box)[4], int swizzle_bytes) {
  return encode_tmap_4d_any(CU_TENSOR_MAP_DATA_TYPE_UINT8, out, base, dims, strides_bytes, box, swizzle_bytes);
}

}  // namespace mvb

using namespace mvb;

static inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }

extern "C" {

const char* mvb_last_error(void) { return get_error(); }
int mvb_abi_version(void) { return 17; }
int mvb_cell_last_variant(void) { return cell_last_variant(); }
long long mvb_cell_variants_seen(int reset) { return (long long)cell_variants_seen(reset); }
long long mvb_launch_count(void) { return g_launches; }
void mvb_reset_launch_count(void) { g_launches = 0; }

int mvb_cell_cpad(int cx) { return (cx + 31) / 32 * 32 + kHidden; }

int mvb_pack_cell_weights(const float* kernel, const float* biases, void* w_planes,
                          float* bias_packed, int cx, int planes, int comp, void* stream) {
  return pack_cell_weights(kernel, biases, w_planes, bias_packed, cx, planes, comp, S(stream));
}

int mvb_convlstm_cell_fwd(const void* xh_planes, const void* w_planes, const float* bias_packed,
                          const float* c_in, const int32_t* row_map, float* c_out, float* h32_out,
                          void* hp_out, int64_t hp_plane_stride, int cpad_out, int ch_off_out,
                          int64_t NS, int H, int W, int cpad, int planes, float forget_bias,
                          void* stream) {
  CellStep s{};
  s.xh = xh_planes; s.w = w_planes; s.bias = bias_packed; s.c_in = c_in; s.row_map = row_map; s.c_out = c_out;
  s.h32_out = h32_out; s.hp_out = hp_out; s.hp_plane_stride = hp_plane_stride; s.cpad_out = cpad_out;
  s.ch_off_out = ch_off_out; s.NS = NS; s.H = H; s.W = W; s.cpad = cpad; s.planes = planes; s.forget_bias = forget_bias;
  return cell_fwd(s, S(stream));
}
int mvb_cell_xfold_tables(const float* kernel, const float* biases, const float* We, const float* be,
                          int E, float* table_B, float* table_T2, void* stream) {
  return cell_xfold_tables(kernel, biases, We, be, E, table_B, table_T2, S(stream));
}
int mvb_convlstm_cell_fwd_onehot(const void* xh_planes, const void* w_planes, const float* table_B,
                                 const float* table_T2, const int32_t* ids, const float* c_in,
                                 const int32_t* row_map, const int32_t* tiles, const int32_t* tile_count,
                                 float* c_out, float* h32_out, void* hp_out,
                                 int64_t hp_plane_stride, int cpad_out, int ch_off_out, int64_t NS, int H,
                                 int W, int cpad, int planes, float forget_bias, void* stream) {
  CellStep s{};
  s.xh = xh_planes; s.w = w_planes; s.xf_B = table_B; s.xf_T2 = table_T2; s.xf_ids = ids; s.c_in = c_in;
  s.row_map = row_map; s.c_out = c_out; s.h32_out = h32_out; s.hp_out = hp_out; s.hp_plane_stride = hp_plane_stride;
  s.cpad_out = cpad_out; s.ch_off_out = ch_off_out; s.NS = NS; s.H = H; s.W = W; s.cpad = cpad; s.planes = planes;
  s.forget_bias = forget_bias; s.tiles = tiles; s.tile_count = tile_count;
  return cell_fwd(s, S(stream));
}
int mvb_convlstm_cell_fwd_xdense(const void* xh_planes, const void* w_planes, const float* bias_packed,
                                 const float* x_in, const float* x_weights, const float* c_in, float* c_out,
                                 float* h32_out, void* hp_out, int64_t hp_plane_stride, int cpad_out, int ch_off_out,
                                 int64_t NS, int H, int W, int cpad, int planes, float forget_bias, void* stream) {
  MVB_REQUIRE(x_in && x_weights, "mvb_convlstm_cell_fwd_xdense: null x input / weights");
  CellStep s{};
  s.xh = xh_planes; s.w = w_planes; s.bias = bias_packed; s.xr_in = x_in; s.xr_W = x_weights; s.c_in = c_in;
  s.c_out = c_out; s.h32_out = h32_out; s.hp_out = hp_out; s.hp_plane_stride = hp_plane_stride; s.cpad_out = cpad_out;
  s.ch_off_out = ch_off_out; s.NS = NS; s.H = H; s.W = W; s.cpad = cpad; s.planes = planes; s.forget_bias = forget_bias;
  return cell_fwd(s, S(stream));
}
int mvb_cell_xdense_weights(const float* kernel_tf, float* x_weights, void* stream) {
  return cell_xdense_weights(kernel_tf, x_weights, S(stream));
}
int mvb_convlstm_cell_fwd_xsparse(const void* xh_planes, const void* w_planes, const float* bias_packed,
                                  const float* x_table, const int32_t* label, const float* c_in, float* c_out,
                                  float* h32_out, void* hp_out, int64_t hp_plane_stride, int cpad_out, int ch_off_out,
                                  int64_t NS, int H, int W, int cpad, int planes, float forget_bias, void* stream) {
  MVB_REQUIRE(x_table && label, "mvb_convlstm_cell_fwd_xsparse: null table / labels");
  CellStep s{};
  s.xh = xh_planes; s.w = w_planes; s.bias = bias_packed; s.xs_tab = x_table; s.xs_label = label; s.c_in = c_in;
  s.c_out = c_out; s.h32_out = h32_out; s.hp_out = hp_out; s.hp_plane_stride = hp_plane_stride; s.cpad_out = cpad_out;
  s.ch_off_out = ch_off_out; s.NS = NS; s.H = H; s.W = W; s.cpad = cpad; s.planes = planes; s.forget_bias = forget_bias;
  return cell_fwd(s, S(stream));
}
int mvb_cell_xsparse_weights(const float* kernel_tf, int cx, float* x_weights, void* stream) {
  return cell_xsparse_weights(kernel_tf, cx, x_weights, S(stream));
}
int mvb_cell_xsparse_table(const float* scene_conv, const int32_t* frame_idx, const int32_t* label,
                           const float* x_weights, float* x_table, int64_t NS, int H, int W, void* stream) {
  return cell_xsparse_table(scene_conv, frame_idx, label, x_weights, x_table, NS, H, W, S(stream));
}
int mvb_convlstm_cell_fwd_onehot_fanout(const void* xh_planes, const void* w_planes, const float* table_B,
                                        const float* table_T2, const int32_t* ids, const float* c_in,
                                        float* c_out, float* h32_out, float* workspace, int64_t NS, int fanout, int H,
                                        int W, int cpad, int planes, float forget_bias, void* stream) {
  CellStep s{};
  s.xh = xh_planes; s.w = w_planes; s.xf_B = table_B; s.xf_T2 = table_T2; s.xf_ids = ids; s.c_in = c_in;
  s.c_out = c_out; s.h32_out = h32_out; s.fanout_ws = workspace; s.NS = NS; s.fanout = fanout; s.H = H; s.W = W;
  s.cpad = cpad; s.planes = planes; s.forget_bias = forget_bias;
  return cell_fwd(s, S(stream));
}

int mvb_convlstm_cell_fwd_train(const void* xh_planes, const void* w_planes,
                                const float* bias_packed, const float* c_in, float* c_out,
                                float* h32_out, void* hp_out, int64_t hp_plane_stride, int cpad_out,
                                int ch_off_out, float* gates_out, int64_t NS, int H, int W, int cpad,
                                int planes, float forget_bias, void* stream) {
  CellStep s{};
  s.xh = xh_planes; s.w = w_planes; s.bias = bias_packed; s.c_in = c_in; s.c_out = c_out; s.h32_out = h32_out;
  s.hp_out = hp_out; s.hp_plane_stride = hp_plane_stride; s.cpad_out = cpad_out; s.ch_off_out = ch_off_out;
  s.gates_out = gates_out; s.NS = NS; s.H = H; s.W = W; s.cpad = cpad; s.planes = planes; s.forget_bias = forget_bias;
  return cell_fwd(s, S(stream));
}
int mvb_lstm_gates_bwd(const float* gates, const float* c_prev, const float* c_new, const float* dh,
                       const float* dc_in, void* dg_planes, int64_t plane_stride, float* dc_prev,
                       float* dbias_packed, int64_t NS, int H, int W, int planes, void* stream) {
  return lstm_gates_bwd(gates, c_prev, c_new, dh, dc_in, dg_planes, plane_stride, dc_prev,
                        dbias_packed, NS, H, W, planes, S(stream));
}
int mvb_pack_cell_weights_dgrad(const float* kernel, void* wd_planes, int cx, int planes,
                                void* stream) {
  return pack_cell_weights_dgrad(kernel, wd_planes, cx, planes, S(stream));
}
int mvb_cell_dgrad(const void* dg_planes, const void* wd_planes, float* dxh, int64_t NS, int H,
                   int W, int cpad, int planes, int need_dx, void* stream) {
  return cell_dgrad(dg_planes, wd_planes, dxh, NS, H, W, cpad, planes, need_dx, S(stream));
}
int mvb_cell_wgrad_direct(const void* dg_planes, const void* xh_planes, float* dw_packed, int64_t NS,
                          int H, int W, int cpad, int planes, void* stream) {
  return cell_wgrad_mn(dg_planes, xh_planes, dw_packed, NS, H, W, cpad, planes, S(stream));
}
int mvb_unpack_cell_wgrad(const float* dw_packed, const float* dbias_packed, float* dkernel,
                          float* dbiases, int cx, int comp, int accumulate, int slabs, void* stream) {
  return unpack_cell_wgrad(dw_packed, dbias_packed, dkernel, dbiases, cx, comp, accumulate, slabs,
                           S(stream));
}
int mvb_cell_wgrad_slabs(int cpad) { return cell_wgrad_mn_slabs(cpad); }

int mvb_loss_fwd_bwd(const float* logits, const int32_t* labels, float* dlogits, int64_t rows, int V,
                     float cls_weight, const float* reg, const float* target, float* dreg,
                     int64_t nreg, float reg_weight, float* loss_out, void* stream) {
  return loss_fwd_bwd(logits, labels, dlogits, rows, V, cls_weight, reg, target, dreg, nreg,
                      reg_weight, loss_out, S(stream));
}
int mvb_soft_ce_fwd_bwd(const float* logits, const float* labels, float* dlogits, int64_t rows, int V,
                        float cls_weight, float* loss_out, void* stream) {
  return soft_ce_fwd_bwd(logits, labels, dlogits, rows, V, cls_weight, loss_out, S(stream));
}
int mvb_fg_count(const float* soft_labels, const int32_t* labels, int64_t rows, int V, double* count, void* stream) {
  return fg_count(soft_labels, labels, rows, V, count, S(stream));
}
int mvb_masked_huber_fwd_bwd(const float* reg, const float* target, float* dreg, const float* soft_labels,
                             const int32_t* labels, int64_t rows, int V, const double* fg_count, float reg_weight,
                             float* loss_out, void* stream) {
  return masked_huber_fwd_bwd(reg, target, dreg, soft_labels, labels, rows, V, fg_count, reg_weight, loss_out,
                              S(stream));
}
int mvb_huber_traj_fwd_bwd(const float* reg, const double* pred_traj, const double* centers, float* dreg, int64_t N,
                           int Tp, int V, float reg_weight, float* loss_out, void* stream) {
  return huber_traj_fwd_bwd(reg, pred_traj, centers, dreg, N, Tp, V, reg_weight, loss_out, S(stream));
}
int mvb_soft_ce_label_fwd_bwd(const float* logits, const int32_t* labels, int soft_grid, float* dlogits, int64_t rows,
                              int H, int W, float cls_weight, float* loss_out, void* stream) {
  return soft_ce_label_fwd_bwd(logits, labels, soft_grid, dlogits, rows, H, W, cls_weight, loss_out, S(stream));
}
int mvb_fg_count_label(const int32_t* labels, int soft_grid, int64_t rows, int H, int W, double* fg_count,
                       void* stream) {
  return fg_count_label(labels, soft_grid, rows, H, W, fg_count, S(stream));
}
int mvb_masked_huber_traj_fwd_bwd(const float* reg, const double* pred_traj, const double* centers, float* dreg,
                                  const int32_t* labels, int soft_grid, int64_t N, int Tp, int H, int W,
                                  const double* fg_count, float reg_weight, float* loss_out, void* stream) {
  return masked_huber_traj_fwd_bwd(reg, pred_traj, centers, dreg, labels, soft_grid, N, Tp, H, W, fg_count,
                                   reg_weight, loss_out, S(stream));
}
int mvb_head_bwd(const float* h32, const float* dout, const float* Wo, int Pout, float* dWo,
                 float* dh, int accumulate_dh, int64_t NS, int H, int W, void* stream) {
  return head_bwd(h32, dout, Wo, Pout, dWo, dh, accumulate_dh, NS, H, W, S(stream));
}
int mvb_emb_bwd(const float* dxh, int cpad, const int32_t* ids, const float* in_map, const float* We,
                const float* be, int E, int Pout, float* dWe, float* dbe, float* d_in,
                int accumulate_din, int64_t NS, int H, int W, void* stream) {
  return emb_bwd(dxh, cpad, ids, in_map, We, be, E, Pout, dWe, dbe, d_in, accumulate_din, NS, H, W,
                 S(stream));
}
int mvb_gnn_attend_bwd(const float* h32, const float* scene_mean, const float* gout, float* work,
                       float* dh, int accumulate_dh, float* dscene_mean, int64_t NS, int H, int W,
                       void* stream) {
  return gnn_bwd(h32, scene_mean, gout, work, dh, accumulate_dh, dscene_mean, NS, H, W, S(stream));
}
int mvb_scene_conv_bwd(const float* in, const float* W, const float* out, const float* dout,
                       float* dW, float* db, float* din, int64_t F, int IH, int IW, int Cin, int Cout,
                       void* stream) {
  return scene_conv_bwd(in, W, out, dout, dW, db, din, F, IH, IW, Cin, Cout, S(stream));
}
int mvb_enc_class_input_bwd(const float* dxh, int cpad, const int32_t* frame_idx,
                            const int32_t* label, float* dscene, int64_t NS, int H, int W,
                            void* stream) {
  return enc_class_input_bwd(dxh, cpad, frame_idx, label, dscene, NS, H, W, S(stream));
}
int mvb_scene_time_mean_bwd(const float* dmean, const int32_t* frame_idx, float* dscene, int64_t N,
                            int T, int64_t HWC, void* stream) {
  return scene_mean_bwd(dmean, frame_idx, dscene, N, T, HWC, S(stream));
}
int mvb_clip_adadelta(float* w, const float* grad, float* acc, float* acc_upd, int64_t n, float lr,
                      float rho, float eps, float clip, float wd, float grad_scale, void* stream) {
  return clip_adadelta(w, grad, acc, acc_upd, n, lr, rho, eps, clip, wd, grad_scale, S(stream));
}

int mvb_nhwc_to_planes(const float* src, void* dst_planes, int64_t plane_stride, int cpad,
                       int ch_off, int64_t NS, int H, int W, int C, int planes, int comp,
                       void* stream) {
  return nhwc_to_planes(src, dst_planes, plane_stride, cpad, ch_off, NS, H, W, C, planes, comp,
                        S(stream));
}
int mvb_traj_to_grid(const double* traj, const double* centers, double h_gap, double w_gap, int32_t* labels,
                     float* regress, int64_t NT, int H, int W, void* stream) {
  return traj_to_grid(traj, centers, h_gap, w_gap, labels, regress, NT, H, W, S(stream));
}
int mvb_traj_to_planes(const double* traj, int64_t traj_stride, const double* centers, void* dst_planes,
                       int64_t plane_stride, int cpad, int64_t NS, int H, int W, int comp, void* stream) {
  return traj_to_planes(traj, traj_stride, centers, dst_planes, plane_stride, cpad, NS, H, W, comp, S(stream));
}
int mvb_nhwc_to_halo(const float* src, float* dst, int64_t NS, int H, int W, int C, void* stream) {
  return nhwc_halo_copy(src, dst, NS, H, W, C, 0, S(stream));
}
int mvb_halo_to_nhwc(const float* src, float* dst, int64_t NS, int H, int W, int C, void* stream) {
  return nhwc_halo_copy(src, dst, NS, H, W, C, 1, S(stream));
}

int mvb_enc_class_input(const float* scene_conv, const int32_t* frame_idx, const int32_t* label,
                        const int32_t* prev_label, void* xh_planes, int64_t plane_stride, int cpad,
                        int64_t NS, int H, int W, int planes, void* stream) {
  return enc_class_input(scene_conv, frame_idx, label, prev_label, xh_planes, plane_stride, cpad,
                         NS, H, W, planes, S(stream));
}

int mvb_scene_conv_fwd(const float* in, const float* W, const float* b, float* out, int64_t F,
                       int IH, int IW, int Cin, int Cout, void* stream) {
  return scene_conv_fwd(in, W, b, out, F, IH, IW, Cin, Cout, S(stream));
}
int mvb_scene_time_mean(const float* scene_conv, const int32_t* frame_idx, float* out, int64_t N,
                        int T, int64_t HWC, void* stream) {
  return scene_time_mean(scene_conv, frame_idx, out, N, T, HWC, S(stream));
}

int mvb_gnn_attend_fwd(const float* h32, const int32_t* row_map, const float* scene_mean,
                       int beam, void* hp_out, int64_t hp_plane_stride, int cpad_out,
                       int ch_off_out, int64_t NS, int H, int W, int planes, void* stream) {
  return gnn_attend_fwd(h32, row_map, scene_mean, beam, hp_out, hp_plane_stride, cpad_out,
                        ch_off_out, NS, H, W, planes, S(stream));
}

int mvb_head_class_fwd(const float* h32, const float* Wo, float* logits_out, int32_t* ids_out,
                       const float* We, const float* be, int E, void* xh_next,
                       int64_t plane_stride, int cpad, int64_t NS, int H, int W, int planes,
                       void* stream) {
  return head_fwd(h32, Wo, 1, logits_out, ids_out, We, be, E, xh_next, plane_stride, cpad, NS, H,
                  W, planes, S(stream));
}
int mvb_head_class_fwd_dense(const float* h32, const float* Wo, float* logits_out, int32_t* ids_out,
                             const float* We, const float* be, int E, void* xh_next, int64_t plane_stride, int cpad,
                             int64_t NS, int H, int W, int planes, void* stream) {
  return head_class_fwd_dense(h32, Wo, logits_out, ids_out, We, be, E, xh_next, plane_stride, cpad, NS, H, W,
                              planes, S(stream));
}
int mvb_head_reg_fwd(const float* h32, const float* Wo, float* off_out, const float* We,
                     const float* be, int E, void* xh_next, int64_t plane_stride, int cpad,
                     int64_t NS, int H, int W, int planes, void* stream) {
  return head_fwd(h32, Wo, 2, off_out, nullptr, We, be, E, xh_next, plane_stride, cpad, NS, H, W,
                  planes, S(stream));
}
int mvb_emb_onehot_fwd(const int32_t* ids, const float* We, const float* be, int E, void* xh_next,
                       int64_t plane_stride, int cpad, int64_t NS, int H, int W, int planes,
                       void* stream) {
  return emb_onehot_fwd(ids, We, be, E, xh_next, plane_stride, cpad, NS, H, W, planes, S(stream));
}
int mvb_emb_dense_fwd(const float* x, const float* We, const float* be, int E, void* xh_next,
                      int64_t plane_stride, int cpad, int64_t NS, int H, int W, int planes,
                      void* stream) {
  return emb_dense_fwd(x, We, be, E, xh_next, plane_stride, cpad, NS, H, W, planes, S(stream));
}

int mvb_beam_step(const float* logits, const float* score_in, float* score_out, int32_t* ids_out,
                  int32_t* parents_out, int32_t* row_map_out, int64_t N, int B, int V,
                  int first_step, int zero_scores, int diverse, float log_gamma, void* stream) {
  return beam_step(logits, score_in, score_out, ids_out, parents_out, row_map_out, N, B, V,
                   first_step, zero_scores, diverse, log_gamma, S(stream));
}
int mvb_decode_trajectories(const int32_t* ids, const float* offsets, const float* centers, float* out,
                            int64_t N, int K, int Tp, int V, void* stream) {
  return decode_trajectories(ids, offsets, centers, out, N, K, Tp, V, S(stream));
}
int mvb_clip_update(float* w, const float* grad, float* slot1, float* slot2, int64_t n, int kind, float lr, float p1,
                    float p2, float eps, float clip, float wd, float grad_scale, void* stream) {
  return clip_update(w, grad, slot1, slot2, n, kind, lr, p1, p2, eps, clip, wd, grad_scale, S(stream));
}
int mvb_adv_step(const float* x, const float* adv, const float* grad, float* out, float eps, float step, int64_t n,
                 void* stream) {
  return adv_step(x, adv, grad, out, eps, step, n, S(stream));
}
int mvb_mix(const float* a, const float* b, float* out, float w, int64_t n, void* stream) {
  return mix(a, b, out, w, n, S(stream));
}
int mvb_ce_rows(const float* logits, const int32_t* labels, float* loss, int64_t rows, int V, void* stream) {
  return ce_rows(logits, labels, loss, rows, V, S(stream));
}
int mvb_enc_class_input_mix(const float* scene_conv, const int32_t* frame_idx, const int32_t* label,
                            const int32_t* label2, float beta, void* xh_planes, int64_t plane_stride, int cpad,
                            int64_t NS, int H, int W, int planes, void* stream) {
  return enc_class_input_mix(scene_conv, frame_idx, label, label2, beta, xh_planes, plane_stride, cpad, NS, H, W,
                             planes, S(stream));
}
int mvb_enc_class_input_mix_bwd(const float* dxh, int cpad, const int32_t* frame_idx, const int32_t* label,
                                const int32_t* label2, float beta, float* dscene, int64_t NS, int H, int W,
                                void* stream) {
  return enc_class_input_mix_bwd(dxh, cpad, frame_idx, label, label2, beta, dscene, NS, H, W, S(stream));
}
int mvb_min_ade_fde(const float* pred, const float* gt, const int32_t* gt_len, double* ade_err, int32_t* ade_idx,
                    double* fde, int32_t* fde_idx, int64_t N, int G, int K, int Tp, int Tg, void* stream) {
  return min_ade_fde(pred, gt, gt_len, ade_err, ade_idx, fde, fde_idx, N, G, K, Tp, Tg, S(stream));
}
int mvb_beam_nll(const float* logits, const float* logprobs, const int32_t* gt_idx, const int32_t* steps, double* nll,
                 int32_t* count, int64_t N, int K, int Tp, int V, int J, int G, void* stream) {
  return beam_nll(logits, logprobs, nullptr, gt_idx, steps, nll, count, N, K, Tp, V, J, G, S(stream));
}
int mvb_beam_nll_ragged(const float* logits, const float* logprobs, const int32_t* lengths, const int32_t* gt_idx,
                        const int32_t* steps, double* nll, int32_t* count, int64_t N, int K, int Tp, int V, int J,
                        int G, void* stream) {
  MVB_REQUIRE(lengths, "beam_nll_ragged: null lengths");
  return beam_nll(logits, logprobs, lengths, gt_idx, steps, nll, count, N, K, Tp, V, J, G, S(stream));
}
int mvb_min_ade_fde_cells(const int32_t* ids, const float* offsets, const double* centers, int center_only,
                          const int32_t* lengths, const double* gt, const int32_t* gt_len, double* ade_err,
                          int32_t* ade_idx, double* fde, int32_t* fde_idx, int32_t* err, int64_t N, int G, int K,
                          int Tp, int V, int Tg, void* stream) {
  return min_ade_fde_cells(ids, offsets, centers, center_only, lengths, gt, gt_len, ade_err, ade_idx, fde, fde_idx,
                           err, N, G, K, Tp, V, Tg, S(stream));
}
int mvb_points_to_cells(const double* points, int32_t* cells, int32_t* err, int64_t P, int scene_h, int scene_w,
                        int video_h, int video_w, void* stream) {
  return points_to_cells(points, cells, err, P, scene_h, scene_w, video_h, video_w, S(stream));
}
int mvb_beam_backtrace(const int32_t* step_ids, const int32_t* step_parents,
                       const float* step_logits, int32_t* out_ids, float* out_logits, int64_t N,
                       int B, int Tp, int V, void* stream) {
  return beam_backtrace(step_ids, step_parents, step_logits, out_ids, out_logits, N, B, Tp, V,
                        S(stream));
}
int mvb_beam_backtrace_ragged(const int32_t* step_ids, const int32_t* step_parents, const float* step_logits,
                              const int32_t* lengths, int32_t* out_ids, float* out_logits, int64_t N, int B, int Tp,
                              int V, void* stream) {
  return beam_backtrace_ragged(step_ids, step_parents, step_logits, lengths, out_ids, out_logits, N, B, Tp, V,
                               S(stream));
}
int mvb_gather_offsets(const int32_t* ids, const float* offsets, const int32_t* lengths, float* out, int64_t N, int K,
                       int Tp, int V, void* stream) {
  return gather_offsets(ids, offsets, lengths, out, N, K, Tp, V, S(stream));
}
int mvb_beam_gather_h_f16f8(const float* h32, const int32_t* row_map, void* hp_out, int64_t hp_plane_stride,
                            int cpad_out, int64_t NS, int H, int W, void* stream) {
  return beam_gather_h(h32, row_map, hp_out, hp_plane_stride, cpad_out, NS, H, W, S(stream));
}
int mvb_beam_band(const int32_t* ids, const int32_t* parents, const int32_t* band_in, int32_t* band_out,
                  int32_t* tiles, int64_t tiles_cap, int32_t* tile_count, int64_t NS, int K, int radius, int H, int W,
                  void* stream) {
  return beam_band(ids, parents, band_in, band_out, tiles, tiles_cap, tile_count, NS, K, radius, H, W, S(stream));
}
int mvb_beam_band_copy(const float* base_c, const float* base_h32, const int32_t* band, float* c, float* h32,
                       int64_t NS, int K, int H, int W, void* stream) {
  return beam_band_copy(base_c, base_h32, band, c, h32, NS, K, H, W, S(stream));
}

}  // extern "C"
