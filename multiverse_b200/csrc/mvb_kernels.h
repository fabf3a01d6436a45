// Internal C++ launchers (one per kernel group); the extern "C" wrappers live in mvb_api.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace mvb {

void count_launch(int n);

// mvb_cell.cu
constexpr int kCellTileRows = 128;    // M rows of a cell kernel tile (and of a beam_band work-list entry at most)
// One ConvLSTM cell step.  Callers value-initialise it (`CellStep s{};`) and set the fields they use; a null pointer is
// an input not read or an output not written.  At most one x source (x-fold, sparse, dense) replaces the x block.
struct CellStep {
  const void *xh, *w;             // operand planes [R, cpad] and packed weights (mvb_pack_cell_weights)
  const float *bias, *c_in;       // [1024] packed (may be null with x-fold, whose tables fold it in); [R_src, 256]
  const int* row_map;             // [NS] source sample row of c_in for each sample row (null: identity)
  float *c_out, *h32_out;         // [R, 256]
  void* hp_out;                   // operand planes whose h block receives h': plane stride, row pitch, channel offset
  long long hp_plane_stride; int cpad_out, ch_off_out;
  long long NS; int H, W, cpad;
  int planes; float forget_bias;  // planes: format of xh and w | (format of hp_out << 8) when that differs
  float* gates_out;               // [R, 1024] activated gates for the backward pass (bf16x2 only)
  const float *xf_B, *xf_T2; const int* xf_ids;   // x-fold: tables [9][1024], [9][25][1024]; arg-max cells [NS]
  const float* xs_tab; const int* xs_label;       // sparse x: table rows [NS, 9, 1024]; label cells [NS]
  const float *xr_in, *xr_W;                      // dense x: raw input [NS, H, W, 2] fp32; weights [18][1024]
  int fanout;                     // > 1: each x-fold row is the parent of `fanout` child rows of c_out / h32_out,
  float* fanout_ws;               // through the parents' raw accumulators [R, 1024] fp32 (xh null: already there,
                                  // from an earlier step on the same parents: the GEMM is skipped)
  const int *tiles, *tile_count;  // work list of M tiles (m0, m_end) [*tile_count][2] (mvb_beam_band), or null
};
int cell_fwd(const CellStep& s, cudaStream_t stream);
int cell_xdense_weights(const float* kernel, float* out, cudaStream_t stream);
int cell_xsparse_weights(const float* kernel, int cx, float* out, cudaStream_t stream);
int cell_xsparse_table(const float* scene_conv, const int* frame_idx, const int* label, const float* Wx, float* tab,
                       long long NS, int H, int W, cudaStream_t stream);
int cell_last_variant();
unsigned long long cell_variants_seen(int reset);
int cell_xfold_tables(const float* kernel, const float* biases, const float* We, const float* be, int E,
                      float* Bt, float* T2, cudaStream_t stream);
int pack_cell_weights(const float* kernel, const float* biases, void* w_planes, float* bias_packed,
                      int cx, int P, int comp, cudaStream_t stream);

// mvb_layout.cu
int nhwc_to_planes(const float* src, void* dst_planes, long long plane_stride, int cpad, int ch_off,
                   long long NS, int H, int W, int C, int P, int comp, cudaStream_t stream);
int traj_to_grid(const double* traj, const double* centers, double h_gap, double w_gap, int* labels,
                 float* regress, long long NT, int H, int W, cudaStream_t stream);
int traj_to_planes(const double* traj, long long traj_stride, const double* centers, void* dst_planes,
                   long long plane_stride, int cpad, long long NS, int H, int W, int comp, cudaStream_t stream);
int nhwc_halo_copy(const float* src, float* dst, long long NS, int H, int W, int C, int to_nhwc,
                   cudaStream_t stream);
int enc_class_input(const float* scene_conv, const int* frame_idx, const int* label,
                    const int* prev_label, void* xh_planes, long long plane_stride, int cpad,
                    long long NS, int H, int W, int P, cudaStream_t stream);

// mvb_scene.cu
int scene_conv_fwd(const float* in, const float* W, const float* b, float* out, long long F, int IH,
                   int IW, int Cin, int Cout, cudaStream_t stream);
int scene_time_mean(const float* scene_conv, const int* frame_idx, float* out, long long N, int T,
                    long long HWC, cudaStream_t stream);

// mvb_gnn.cu
int gnn_attend_fwd(const float* h32, const int* row_map, const float* scene_mean, int beam,
                   void* hp_out, long long hp_plane_stride, int cpad_out, int ch_off_out,
                   long long NS, int H, int W, int P, cudaStream_t stream);

// mvb_head.cu
int head_fwd(const float* h32, const float* Wo, int Pout, float* out, int* ids_out, const float* We,
             const float* be, int E, void* xh_next, long long plane_stride, int cpad, long long NS,
             int H, int W, int P, cudaStream_t stream);
int head_class_fwd_dense(const float* h32, const float* Wo, float* out, int* ids_out, const float* We,
                         const float* be, int E, void* xh_next, long long plane_stride, int cpad, long long NS,
                         int H, int W, int P, cudaStream_t stream);
int emb_onehot_fwd(const int* ids, const float* We, const float* be, int E, void* xh_next,
                   long long plane_stride, int cpad, long long NS, int H, int W, int P,
                   cudaStream_t stream);
int emb_dense_fwd(const float* x, const float* We, const float* be, int E, void* xh_next,
                  long long plane_stride, int cpad, long long NS, int H, int W, int P,
                  cudaStream_t stream);

// mvb_beam.cu
int decode_trajectories(const int* ids, const float* offs, const float* centers, float* out, long long N,
                        int K, int Tp, int V, cudaStream_t stream);
int beam_step(const float* logits, const float* score_in, float* score_out, int* ids_out,
              int* parents_out, int* row_map_out, long long N, int B, int V, int first_step,
              int zero_scores, int diverse, float log_gamma, cudaStream_t stream);
int beam_backtrace(const int* step_ids, const int* step_parents, const float* step_logits,
                   int* out_ids, float* out_logits, long long N, int B, int Tp, int V,
                   cudaStream_t stream);
int beam_backtrace_ragged(const int* step_ids, const int* step_parents, const float* step_logits, const int* lengths,
                          int* out_ids, float* out_logits, long long N, int B, int Tp, int V, cudaStream_t stream);
int gather_offsets(const int* ids, const float* offs, const int* lengths, float* out, long long N, int K, int Tp,
                   int V, cudaStream_t stream);
int beam_gather_h(const float* h32, const int* row_map, void* hp_out, long long hp_plane_stride, int cpad_out,
                  long long NS, int H, int W, cudaStream_t stream);
int beam_band(const int* ids, const int* parents, const int* band_in, int* band_out, int* tiles, long long tiles_cap,
              int* tile_count, long long NS, int K, int radius, int H, int W, cudaStream_t stream);
int beam_band_copy(const float* base_c, const float* base_h32, const int* band, float* c, float* h32, long long NS,
                   int K, int H, int W, cudaStream_t stream);

// mvb_metrics.cu
int min_ade_fde(const float* pred, const float* gt, const int* gt_len, double* ade_err, int* ade_idx, double* fde,
                int* fde_idx, long long N, int G, int K, int Tp, int Tg, cudaStream_t stream);
int min_ade_fde_cells(const int* ids, const float* offs, const double* centers, int center_only, const int* lengths,
                      const double* gt, const int* gt_len, double* ade_err, int* ade_idx, double* fde, int* fde_idx,
                      int* err, long long N, int G, int K, int Tp, int V, int Tg, cudaStream_t stream);
int points_to_cells(const double* points, int* cells, int* err, long long P, int scene_h, int scene_w, int video_h,
                    int video_w, cudaStream_t stream);
// lengths [N] may be NULL (every row Tp steps)
int beam_nll(const float* logits, const float* logprobs, const int* lengths, const int* gt_idx, const int* steps,
             double* nll, int* count, long long N, int K, int Tp, int V, int J, int G, cudaStream_t stream);

// mvb_train.cu
int cell_dgrad(const void* dg_planes, const void* wd_planes, float* dxh, long long NS, int H, int W,
               int cpad, int P, int need_x, cudaStream_t stream);
int cell_wgrad_mn(const void* dg_planes, const void* xh_planes, float* dwp, long long NS, int H, int W,
                  int cpad, int P, cudaStream_t stream);
int lstm_gates_bwd(const float* gates, const float* c_prev, const float* c_new, const float* dh,
                   const float* dc_in, void* dg_planes, long long plane_stride, float* dc_prev,
                   float* dbias_packed, long long NS, int H, int W, int P, cudaStream_t stream);
int pack_cell_weights_dgrad(const float* kernel, void* wd_planes, int cx, int P, cudaStream_t stream);
int unpack_cell_wgrad(const float* dwp, const float* dbias_packed, float* dkernel, float* dbiases,
                      int cx, int comp, int accumulate, int slabs, cudaStream_t stream);
int cell_wgrad_mn_slabs(int cpad);

// mvb_train2.cu
int loss_fwd_bwd(const float* logits, const int* labels, float* dlogits, long long rows, int V,
                 float cls_scale, const float* reg, const float* target, float* dreg, long long nreg,
                 float reg_scale, float* loss_out, cudaStream_t stream);
int soft_ce_fwd_bwd(const float* logits, const float* labels, float* dlogits, long long rows, int V, float cls_scale,
                    float* loss_out, cudaStream_t stream);
int fg_count(const float* soft, const int* labels, long long rows, int V, double* count, cudaStream_t stream);
int masked_huber_fwd_bwd(const float* reg, const float* target, float* dreg, const float* soft, const int* labels,
                         long long rows, int V, const double* count, float reg_scale, float* loss_out,
                         cudaStream_t stream);
int huber_traj_fwd_bwd(const float* reg, const double* pred_traj, const double* centers, float* dreg, long long N,
                       int Tp, int V, float reg_scale, float* loss_out, cudaStream_t stream);
int soft_ce_label_fwd_bwd(const float* logits, const int* labels, int mode, float* dlogits, long long rows, int H,
                          int W, float cls_scale, float* loss_out, cudaStream_t stream);
int fg_count_label(const int* labels, int mode, long long rows, int H, int W, double* count, cudaStream_t stream);
int masked_huber_traj_fwd_bwd(const float* reg, const double* pred_traj, const double* centers, float* dreg,
                              const int* labels, int mode, long long N, int Tp, int H, int W, const double* count,
                              float reg_scale, float* loss_out, cudaStream_t stream);
int head_bwd(const float* h32, const float* dout, const float* Wo, int Pout, float* dWo, float* dh,
             int accumulate_dh, long long NS, int H, int W, cudaStream_t stream);
int emb_bwd(const float* dxh, int cpad, const int* ids, const float* in_map, const float* We,
            const float* be, int E, int Pout, float* dWe, float* dbe, float* d_in, int accumulate_din,
            long long NS, int H, int W, cudaStream_t stream);
int gnn_bwd(const float* h32, const float* scene_mean, const float* gout, float* work, float* dh,
            int accumulate_dh, float* dscene_mean, long long NS, int H, int W, cudaStream_t stream);
int scene_conv_bwd(const float* in, const float* W, const float* out, const float* dout, float* dW,
                   float* db, float* din, long long F, int IH, int IW, int Cin, int Cout,
                   cudaStream_t stream);
int enc_class_input_bwd(const float* dxh, int cpad, const int* frame_idx, const int* label,
                        float* dscene, long long NS, int H, int W, cudaStream_t stream);
int scene_mean_bwd(const float* dmean, const int* frame_idx, float* dscene, long long N, int T,
                   long long HWC, cudaStream_t stream);
int clip_update(float* w, const float* grad, float* s1, float* s2, long long n, int kind, float lr, float p1, float p2,
                float eps, float clip, float wd, float gscale, cudaStream_t stream);
int adv_step(const float* x, const float* adv, const float* grad, float* out, float eps, float step, long long n,
             cudaStream_t stream);
int mix(const float* a, const float* b, float* out, float w, long long n, cudaStream_t stream);
int ce_rows(const float* logits, const int* labels, float* loss, long long rows, int V, cudaStream_t stream);
int enc_class_input_mix(const float* scene_conv, const int* frame_idx, const int* label, const int* label2, float beta,
                        void* xh_planes, long long plane_stride, int cpad, long long NS, int H, int W, int P,
                        cudaStream_t stream);
int enc_class_input_mix_bwd(const float* dxh, int cpad, const int* frame_idx, const int* label, const int* label2,
                            float beta, float* dscene, long long NS, int H, int W, cudaStream_t stream);
int clip_adadelta(float* w, const float* grad, float* acc, float* acc_upd, long long n, float lr,
                  float rho, float eps, float clip, float wd, float gscale, cudaStream_t stream);

}  // namespace mvb
