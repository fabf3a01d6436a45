/* libmultiverse_b200 - C ABI of the H100-native Multiverse ConvRNN hot path.
 *
 * The reference (JunweiLiang/Multiverse, code/pred_models.py) has no FFI: its device work is
 * TensorFlow-1.15 op dispatch behind `sess.run` (pred_models.py:1732 train, :1779 test,
 * multifuture_inference.py:471 K-way decode).  Each entry point below replaces the TF ops of one
 * group of call sites; the citation on every function is the reference code it stands in for.
 * INTEGRATION.md shows the ctypes binding (the reference is pure Python) a maintainer would add.
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer on the current device
 *     unless noted; the caller (PyTorch in this repo) owns all memory, nothing is allocated
 *     or retained by the library; work is enqueued asynchronously on `stream`
 *     (a cudaStream_t passed as void*; NULL = legacy default stream).
 *   - return 0 on success, non-zero on error; mvb_last_error() returns a thread-local message.
 *   - activations use the library's "halo" layout: a grid of H x W cells is stored as
 *     S = (H+1)*(W+1) rows per sample, row = y*(W+1)+x, the extra column/row are zeros that
 *     the library never writes.  Operands are stored in one of two formats, selected by a `planes`
 *     argument: planes == 2 ("bf16x2") stores an fp32 value as two bf16 summands (v = p0 + p1) in a
 *     plane tensor [2][rows][cpad] bf16; planes == MVB_PLANES_F16F8 selects the inference format
 *     described at mvb_pack_cell_weights.  Any other value is refused.
 *   - NS is the number of sample rows (batch, or batch*beam); fp32 state tensors are
 *     [NS*S, 256]; the hidden size is fixed at 256 (enc/dec_hidden_size of every published config).
 */
#ifndef MULTIVERSE_B200_H_
#define MULTIVERSE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- library ------------------------------------------------------------------------- */
const char* mvb_last_error(void);
/* ABI version of this header (bumped on any signature change). */
int mvb_abi_version(void);
/* Number of kernels this library has launched on the calling thread since the last reset
 * (bench.py reports it as gpu_launches). */
long long mvb_launch_count(void);
void mvb_reset_launch_count(void);

/* ---- a1: ConvLSTM cell (tf.contrib.rnn.ConvLSTMCell built at pred_models.py:189-202,
 *      :236-249; called through dynamic_rnn :212,:232 and raw_rnn :455,:678) -------------- */

/* Channels per tap of the packed K dimension for an input of cx channels: roundup(cx,32)+256. */
int mvb_cell_cpad(int cx);

/* Pack a TF ConvLSTM `kernel` [3,3,cx+256,1024] (HWIO; gate order i,j,f,o) and `biases` [1024]
 * (host layout of the TF variables, but resident on the device) into
 *   w_planes   bf16 [2][1024][9*cpad]   (row = tile*256 + gate*64 + ch%64, K-major)
 *   bias_packed fp32 [1024]             (same row order).
 * comp != 0 (needs planes == 2 and 4*cx <= roundup(cx,32)): "compensated x block" for inputs of
 * large magnitude (the regression encoder's raw pixel offsets, pred_models.py:232): the zero
 * padding of the x block instead carries [W | W | W-w0-w1 | w1] against the activation side's
 * [x | x-x0-x1 | x | x1] (mvb_nhwc_to_planes with comp), so the terms the 3-product bf16 scheme
 * drops are added back by the same MMAs and the x contribution is exact to fp32.
 *
 * planes == MVB_PLANES_F16F8 (16) selects the "f16f8" operand format everywhere a `planes` argument appears
 * (inference only): an operand value v = a0 + a1, a0 = fp16(v), is stored as one fp16 plane and two e4m3 planes
 * e0 = e4m3(a0), e1 = e4m3(a1 * 2^12) - for R rows of cpad channels [fp16 R*cpad][fp8 R rows of 2*cpad bytes], the
 * same bytes as two bf16 planes; inside an fp8 row the planes are interleaved per K chunk: [x block: e0 | e1]
 * then per 64 channels of the h block [e0 (64) | e1 (64)] - and the cell accumulates a0*b0 (fp16 tensor-core pass)
 * + the two cross terms as e4m3 passes at twice the rate into the same fp32 accumulator: 2 bf16-pass equivalents
 * instead of 3 at the accuracy class of planes == 2.  w_planes then holds [fp16 1024*9*cpad][fp8 1024*9 rows of
 * 2*cpad bytes][fp32 1024 column scales] (4*1024*9*cpad + 4096 bytes; weights are stored times a per-column power
 * of two).  comp must be 0. */
#define MVB_PLANES_F16F8 16
int mvb_pack_cell_weights(const float* kernel, const float* biases, void* w_planes,
                          float* bias_packed, int cx, int planes, int comp, void* stream);
/* Which cell kernel the calling process launched last: planes * 2 + (1 if the CTA-pair / weight-multicast
 * variant ran), -1 before the first launch.  Lets tests assert that the variant they mean to check ran. */
int mvb_cell_last_variant(void);
/* Bit mask of the cell kernel variants launched since the last call with reset != 0: bit (f * 2 + pair), f = 0 for
 * planes == 2 and 1 for MVB_PLANES_F16F8; pair = the CTA-pair (cluster of two) variant. */
long long mvb_cell_variants_seen(int reset);

/* One cell step over NS sample rows:  (c_in, xh) -> (c_out, h).
 *   xh_planes  bf16 [2][NS*S][cpad]: concat([x (cx, zero-padded to roundup(cx,32)), h (256)])
 *   c_in       fp32 [*,256] or NULL (zero state); row_map int32 [NS] (source sample row of c_in
 *              for each sample row - the beam search's parent gather, pred_models.py:611-623) or NULL
 *   c_out      fp32 [NS*S,256];  h32_out fp32 [NS*S,256] or NULL
 *   hp_out     bf16 planes of h written at channel offset ch_off_out of rows with pitch cpad_out
 *              (the h block of the NEXT step's xh), plane stride hp_plane_stride elements; or NULL
 *   planes     format of xh_planes and w_planes | (format of hp_out << 8) when the two differ
 * Semantics: g = conv3x3_SAME(concat[x,h]) + biases; i,j,f,o = split(g);
 *   c' = sigmoid(f+forget_bias)*c + sigmoid(i)*tanh(j);  h' = tanh(c')*sigmoid(o). */
int mvb_convlstm_cell_fwd(const void* xh_planes, const void* w_planes, const float* bias_packed,
                          const float* c_in, const int32_t* row_map, float* c_out, float* h32_out,
                          void* hp_out, int64_t hp_plane_stride, int cpad_out, int ch_off_out,
                          int64_t NS, int H, int W, int cpad, int planes, float forget_bias,
                          void* stream);

/* Class-decoder cell step whose input is grid_emb(one_hot(ids)) (pred_models.py:411-446, :602-666).
 * That input is tanh(b) everywhere except the 3x3 cells around ids[s], so its contribution to the
 * gate pre-activations is exactly two table rows per cell (mvb_cell_xfold_tables): the x chunks of
 * the K loop are skipped (1/9 of the MMAs) and the x block of xh_planes is never read.
 *   table_B  fp32 [9][1024]      (border class of the cell; biases folded in)
 *   table_T2 fp32 [9][25][1024]  (border class of ids[s]; 5x5 offset of the cell to ids[s])
 * tiles / tile_count (or NULL: every row): a work list from mvb_beam_band, int32 [*tile_count][2] (m0, m_end) of
 * GEMM rows; only the rows [m0, m_end) of its entries are computed and written. */
int mvb_cell_xfold_tables(const float* kernel, const float* biases, const float* We, const float* be,
                          int E, float* table_B, float* table_T2, void* stream);
int mvb_convlstm_cell_fwd_onehot(const void* xh_planes, const void* w_planes, const float* table_B,
                                 const float* table_T2, const int32_t* ids, const float* c_in,
                                 const int32_t* row_map, const int32_t* tiles, const int32_t* tile_count,
                                 float* c_out, float* h32_out, void* hp_out,
                                 int64_t hp_plane_stride, int cpad_out, int ch_off_out, int64_t NS, int H,
                                 int W, int cpad, int planes, float forget_bias, void* stream);
/* The cell of the regression encoder (code/pred_models.py:196-202, :232-234), whose 2-channel input holds raw pixel
 * offsets of up to +-1.9e3: the h block goes through the tensor cores (any operand format, normally f16f8), the x block
 * is added in fp32 in the gate epilogue, sum over the 9 taps and the 2 channels of x_in[p + off(tap)][ch] *
 * x_weights[tap * 2 + ch][column] (zero outside the image) - every bit of the input counts, at 2 instead of 3 tensor
 * passes.  x_in fp32 [NS,H,W,2] NHWC without halo; x_weights fp32 [18][1024] from mvb_cell_xdense_weights (rows
 * (tap, channel) of the TF kernel [3,3,2+256,1024] in the packed column order); the x block of xh_planes is not read.
 * Other arguments as mvb_convlstm_cell_fwd. */
int mvb_convlstm_cell_fwd_xdense(const void* xh_planes, const void* w_planes, const float* bias_packed,
                                 const float* x_in, const float* x_weights, const float* c_in, float* c_out,
                                 float* h32_out, void* hp_out, int64_t hp_plane_stride, int cpad_out, int ch_off_out,
                                 int64_t NS, int H, int W, int cpad, int planes, float forget_bias, void* stream);
int mvb_cell_xdense_weights(const float* kernel_tf, float* x_weights, void* stream);
/* The cell of the class encoder (code/pred_models.py:189-195, :210-215), whose 64-channel input scene_conv (.) one_hot
 * is non-zero at ONE cell per sample row: instead of spending a K chunk of the GEMM on it, mvb_cell_xsparse_table
 * forms per sample row the nine products  x_table[s][tap][:] = scene_conv[frame_idx[s]][label[s]][:] . W[tap][:64][:]
 * (fp32; x_weights fp32 [9*64][1024] from mvb_cell_xsparse_weights(kernel_tf, 64, ...), packed column order) and the
 * gate epilogue adds row `tap = label - p` of it to the <= 9 cells p around the label (labels outside [0,HW) add
 * nothing, like mvb_enc_class_input).  The x block of xh_planes is not read.  Other arguments as
 * mvb_convlstm_cell_fwd. */
int mvb_convlstm_cell_fwd_xsparse(const void* xh_planes, const void* w_planes, const float* bias_packed,
                                  const float* x_table, const int32_t* label, const float* c_in, float* c_out,
                                  float* h32_out, void* hp_out, int64_t hp_plane_stride, int cpad_out, int ch_off_out,
                                  int64_t NS, int H, int W, int cpad, int planes, float forget_bias, void* stream);
int mvb_cell_xsparse_weights(const float* kernel_tf, int cx, float* x_weights, void* stream);
int mvb_cell_xsparse_table(const float* scene_conv, const int32_t* frame_idx, const int32_t* label,
                           const float* x_weights, float* x_table, int64_t NS, int H, int W, void* stream);

/* First K-row step of the beam decoder (pred_models.py:611-666 right after the first selection): the K = fanout
 * children of a sample share their parent - the same graph-attended h and the same c - and differ only in the
 * selected cell ids[s*K + k], i.e. in the folded table rows.  The GEMM runs once per PARENT row (xh_planes, c_in:
 * NS sample rows; its raw accumulators go to `workspace`, fp32 [NS*S, 1024], caller-allocated) and a second,
 * HBM-bound kernel emits the K children (c_out, h32_out: NS*K sample rows, child-major within a sample): 1/K of the
 * MMAs, identical values. */
/* xh_planes NULL: `workspace` already holds the accumulators of these parent rows (an earlier call on the same
 * operands and weights): the GEMM is skipped and only the children are emitted (fanout >= 1). */
int mvb_convlstm_cell_fwd_onehot_fanout(const void* xh_planes, const void* w_planes, const float* table_B,
                                        const float* table_T2, const int32_t* ids, const float* c_in,
                                        float* c_out, float* h32_out, float* workspace, int64_t NS, int fanout,
                                        int H, int W, int cpad, int planes, float forget_bias, void* stream);

/* ---- a13: BPTT step of the cell (Trainer, pred_models.py:1636-1742; tf.gradients :1698 through
 *      ConvLSTMCell) ------------------------------------------------------------------------ */

/* Forward step that also stores the activated gates i,j,f,o as fp32 [NS*S,1024] in the packed
 * column order (tile*256 + gate*64 + ch%64) for the backward pass. */
int mvb_convlstm_cell_fwd_train(const void* xh_planes, const void* w_planes,
                                const float* bias_packed, const float* c_in, float* c_out,
                                float* h32_out, void* hp_out, int64_t hp_plane_stride, int cpad_out,
                                int ch_off_out, float* gates_out, int64_t NS, int H, int W, int cpad,
                                int planes, float forget_bias, void* stream);
/* Pointwise LSTM backward: (dh_t, dc_t (or NULL = 0), gates_t, c_{t-1} (or NULL = 0), c_t) ->
 * dg_planes bf16 [2][NS*S][1024] (pre-activation gate gradients; halo rows are never written and
 * must be zero), dc_prev fp32, dbias_packed[1024] += column sums.  The backward entry points take
 * planes == 2 only. */
int mvb_lstm_gates_bwd(const float* gates, const float* c_prev, const float* c_new, const float* dh,
                       const float* dc_in, void* dg_planes, int64_t plane_stride, float* dc_prev,
                       float* dbias_packed, int64_t NS, int H, int W, int planes, void* stream);
/* TF kernel [3,3,cx+256,1024] -> dgrad operand planes bf16 [2][cpad][9*1024]. */
int mvb_pack_cell_weights_dgrad(const float* kernel, void* wd_planes, int cx, int planes,
                                void* stream);
/* dxh fp32 [NS*S, cpad] = conv3x3^T(dG, W): gradient w.r.t. concat([x, h]) of the step; the h block
 * (columns [cpad-256, cpad)) always, the x block only if need_dx (the regression encoder's input is data). */
int mvb_cell_dgrad(const void* dg_planes, const void* wd_planes, float* dxh, int64_t NS, int H,
                   int W, int cpad, int planes, int need_dx, void* stream);
/* dw_packed += dG^T x im2col(xh): weight gradient of the step.  Both operands are read MN-major
 * straight from the row-major planes (dG [2][NS*S][1024], xh [2][NS*S][cpad]); the tap is a row
 * shift of the TMA box.  dw_packed: fp32 [mvb_cell_wgrad_slabs(cpad)][1024][9*cpad], accumulated (+=). */
int mvb_cell_wgrad_direct(const void* dg_planes, const void* xh_planes, float* dw_packed, int64_t NS,
                          int H, int W, int cpad, int planes, void* stream);
/* packed accumulators -> gradients of the TF variables kernel [3,3,cx+256,1024], biases [1024]
 * (accumulate != 0: +=). */
int mvb_unpack_cell_wgrad(const float* dw_packed, const float* dbias_packed, float* dkernel,
                          float* dbiases, int cx, int comp, int accumulate, int slabs, void* stream);
/* Number of fp32 slabs [1024][9*cpad] mvb_cell_wgrad_direct accumulates into (its K split: every
 * (tile, k-split) work item owns one slab region, so no atomics); dw_packed must hold that many,
 * zero-initialised, and mvb_unpack_cell_wgrad sums them. */
int mvb_cell_wgrad_slabs(int cpad);

/* ---- a12: loss (Model.build_loss, pred_models.py:961-1040) --------------------------------
 * loss_out[0] += cls_weight * mean_rows CE(logits[rows,V], labels);  dlogits = its gradient.
 * loss_out[1] += reg_weight * mean Huber_delta1(reg - target) over nreg elements; dreg = gradient.
 * Either half may be skipped by passing NULL for logits / reg. */
int mvb_loss_fwd_bwd(const float* logits, const int32_t* labels, float* dlogits, int64_t rows, int V,
                     float cls_weight, const float* reg, const float* target, float* dreg,
                     int64_t nreg, float reg_weight, float* loss_out, void* stream);
/* --use_soft_grid_class (:986-989): loss_out[0] += cls_weight * mean_rows softmax_cross_entropy_with_logits(
 * labels[rows,V], logits[rows,V]) = sum_v y_v (logsumexp(l) - l_v);  dlogits = (sum(y) softmax(l) - y) * cls_weight
 * / rows (the label maps need not sum to one). */
int mvb_soft_ce_fwd_bwd(const float* logits, const float* labels, float* dlogits, int64_t rows, int V,
                        float cls_weight, float* loss_out, void* stream);
/* --mask_grid_regression (:999-1018): the foreground is the cells whose label is > 0 - of the dense maps
 * soft_labels fp32 [rows,V], or (soft_labels NULL) the cell labels[r] of each row of int32 [rows] that lies in [0,V).
 * mvb_fg_count: *fg_count += its size K (an fp64 scalar on the device, exact to 2^53; the caller zeroes it).
 * mvb_masked_huber_fwd_bwd: loss_out[1] += reg_weight * sum_fg Huber_delta1(reg - target) / (2 K), both channels
 * of every foreground cell of reg / target fp32 [rows,V,2]; dreg = its gradient, zero off the foreground.  K is read
 * from *fg_count, so a micro-batch can be divided by the count of its whole batch (or, data parallel, by the
 * all-reduced count over the number of ranks); K = 0 gives a zero loss and
 * gradient (TF's div_no_nan).  No host synchronisation. */
int mvb_fg_count(const float* soft_labels, const int32_t* labels, int64_t rows, int V, double* fg_count,
                 void* stream);
int mvb_masked_huber_fwd_bwd(const float* reg, const float* target, float* dreg, const float* soft_labels,
                             const int32_t* labels, int64_t rows, int V, const double* fg_count, float reg_weight,
                             float* loss_out, void* stream);
/* The same losses with their targets and label maps computed where they are read (f-1, training), so that no
 * dense target or label map exists:  reg / dreg fp32 [Tp,N,H*W,2]; pred_traj fp64 [N,Tp,2] frame pixels; centers
 * fp64 [H*W,2]; labels int32 [Tp,N] label cells.  The target of cell v of row (t, n) is
 * float32(pred_traj[n,t] - centers[v]) computed in fp64 (as mvb_traj_to_grid); the label map of a row is that of
 * --use_soft_grid_class with --soft_grid `soft_grid` (1-7: the 3x3 / 5x5 tables of pred_models.py:1085-1136 around the
 * label cell, a negative label counted from the end), or the one-hot map of an in-range label for soft_grid 0.
 * Each equals the dense entry point above fed the tensors the host builds from the same data, bit for bit in
 * every element (the loss sums are accumulated across blocks in no fixed order, as there):
 *   mvb_huber_traj_fwd_bwd        = the Huber half of mvb_loss_fwd_bwd (nreg = N*Tp*H*W*2 = Tp*N*V*2)
 *   mvb_soft_ce_label_fwd_bwd     = mvb_soft_ce_fwd_bwd (rows = Tp*N, V = H*W; soft_grid 1-7)
 *   mvb_fg_count_label            = mvb_fg_count (soft_grid 0-7; rows = Tp*N label cells)
 *   mvb_masked_huber_traj_fwd_bwd = mvb_masked_huber_fwd_bwd (soft_grid 0-7) */
int mvb_huber_traj_fwd_bwd(const float* reg, const double* pred_traj, const double* centers, float* dreg, int64_t N,
                           int Tp, int V, float reg_weight, float* loss_out, void* stream);
int mvb_soft_ce_label_fwd_bwd(const float* logits, const int32_t* labels, int soft_grid, float* dlogits, int64_t rows,
                              int H, int W, float cls_weight, float* loss_out, void* stream);
int mvb_fg_count_label(const int32_t* labels, int soft_grid, int64_t rows, int H, int W, double* fg_count,
                       void* stream);
int mvb_masked_huber_traj_fwd_bwd(const float* reg, const double* pred_traj, const double* centers, float* dreg,
                                  const int32_t* labels, int soft_grid, int64_t N, int Tp, int H, int W,
                                  const double* fg_count, float reg_weight, float* loss_out, void* stream);
/* ---- a13: backward of the heads / embedding / attention / scene CNN (tf.gradients :1698) ----
 * hidden2grid: dWo[3,3,256,Pout] += ..., dh[NS*S,256] (=|+=) conv3x3^T(dout[NS,HW,Pout], Wo). */
int mvb_head_bwd(const float* h32, const float* dout, const float* Wo, int Pout, float* dWo,
                 float* dh, int accumulate_dh, int64_t NS, int H, int W, void* stream);
/* grid_emb: dxh = gradient w.r.t. concat([x,h]) rows (x block = columns [0,E)); input is
 * one_hot(ids) (Pout=1), the dense map in_map[NS,HW,1] (Pout=1, ids NULL: the logits fed back by the class decoder
 * when training without --train_w_onehot) or in_map[NS,HW,2] (Pout=2); a dense input also yields d_in
 * (accumulate_din: +=). */
int mvb_emb_bwd(const float* dxh, int cpad, const int32_t* ids, const float* in_map, const float* We,
                const float* be, int E, int Pout, float* dWe, float* dbe, float* d_in,
                int accumulate_din, int64_t NS, int H, int W, void* stream);
/* graph attention: gout = gradient w.r.t. its output; work = fp32 scratch of 19*NS*H*W floats. */
int mvb_gnn_attend_bwd(const float* h32, const float* scene_mean, const float* gout, float* work,
                       float* dh, int accumulate_dh, float* dscene_mean, int64_t NS, int H, int W,
                       void* stream);
int mvb_scene_conv_bwd(const float* in, const float* W, const float* out, const float* dout,
                       float* dW, float* db, float* din, int64_t F, int IH, int IW, int Cin, int Cout,
                       void* stream);
int mvb_enc_class_input_bwd(const float* dxh, int cpad, const int32_t* frame_idx,
                            const int32_t* label, float* dscene, int64_t NS, int H, int W,
                            void* stream);
int mvb_scene_time_mean_bwd(const float* dmean, const int32_t* frame_idx, float* dscene, int64_t N,
                            int T, int64_t HWC, void* stream);
/* Trainer (:1698-1716): g = clip(grad*grad_scale + wd*w, +-clip) (clip <= 0: off), then
 * tf.train.AdadeltaOptimizer(lr, rho, eps) on (w, acc, acc_upd), all fp32 [n]. */
int mvb_clip_adadelta(float* w, const float* grad, float* acc, float* acc_upd, int64_t n, float lr,
                      float rho, float eps, float clip, float wd, float grad_scale, void* stream);

/* ---- layout conversion at the API boundary (placeholders are NHWC, pred_models.py:62-115) */

/* fp32 NHWC [NS,H,W,C] -> bf16 planes written at channel offset ch_off of halo rows (pitch cpad);
 * comp != 0 also writes the compensation channels [ch_off+C, ch_off+4C) (see above). */
int mvb_nhwc_to_planes(const float* src, void* dst_planes, int64_t plane_stride, int cpad,
                       int ch_off, int64_t NS, int H, int W, int C, int planes, int comp,
                       void* stream);
/* fp32 NHWC [NS,H,W,C] <-> fp32 halo [NS*S, C] (halo cells are left untouched / skipped). */
int mvb_nhwc_to_halo(const float* src, float* dst, int64_t NS, int H, int W, int C, void* stream);
int mvb_halo_to_nhwc(const float* src, float* dst, int64_t NS, int H, int W, int C, void* stream);

/* ---- a3/k11: class-encoder input, scene_conv (.) one_hot(obs cell) (pred_models.py:210) ---
 * Writes the single non-zero pixel of step t into the x block (channels [0,64)) of xh and
 * clears the pixel written two steps earlier into the same buffer.
 *   scene_conv fp32 [F,H,W,64] (per unique frame), frame_idx int32 [NS] (obs_scene[:,t]),
 *   label int32 [NS] (grid_obs_labels[:,t]), prev_label int32 [NS] or NULL. */
int mvb_enc_class_input(const float* scene_conv, const int32_t* frame_idx, const int32_t* label,
                        const int32_t* prev_label, void* xh_planes, int64_t plane_stride, int cpad,
                        int64_t NS, int H, int W, int planes, void* stream);

/* ---- a4: scene CNN (pred_models.py:146-165; conv2d helper :1333-1373) ------------------
 * out = tanh(conv3x3 stride 2 SAME(in, W) + b), fp32 NHWC; TF SAME padding. */
int mvb_scene_conv_fwd(const float* in, const float* W, const float* b, float* out, int64_t F,
                       int IH, int IW, int Cin, int Cout, void* stream);
/* scene_mean[n] = mean_t scene_conv[frame_idx[n,t]]  (gnn_edge, pred_models.py:826-828). */
int mvb_scene_time_mean(const float* scene_conv, const int32_t* frame_idx, float* out, int64_t N,
                        int T, int64_t HWC, void* stream);

/* ---- a7-a9: graph attention (gnn_edge :808-858, gnn_mask_edge :885-909, gnn_node :860-882,
 *      residual :378/:651):  h' = h + softmax_{q in N3x3(p)}(cos(F_p,F_q)) . h_q,
 *      F = [h ; scene_mean].  Reads fp32 h (halo; sample row row_map[s] if given - the beam
 *      parent gather), writes the bf16 planes of h' into the h block of the next xh. */
int mvb_gnn_attend_fwd(const float* h32, const int32_t* row_map, const float* scene_mean,
                       int beam, void* hp_out, int64_t hp_plane_stride, int cpad_out,
                       int ch_off_out, int64_t NS, int H, int W, int planes, void* stream);

/* ---- a10/a11 + argmax: heads (hidden2grid :925-959, grid_emb :912-919, argmax/one_hot
 *      :411-415) ---------------------------------------------------------------------------
 * Class head: logits[s, HW] = conv3x3(h, Wo[3,3,256,1]); ids[s] = argmax (first index on ties);
 * if xh_next: x block <- planes of tanh(conv3x3(one_hot(ids), We[3,3,1,E]) + be).
 *   logits_out fp32 [NS,HW] (standard row-major cells); ids_out int32 [NS] or NULL. */
int mvb_head_class_fwd(const float* h32, const float* Wo, float* logits_out, int32_t* ids_out,
                       const float* We, const float* be, int E, void* xh_next,
                       int64_t plane_stride, int cpad, int64_t NS, int H, int W, int planes,
                       void* stream);
/* Class head of the training-mode decoder without --train_w_onehot (:426-435): as mvb_head_class_fwd, but
 * the x block receives tanh(conv3x3(logits, We[3,3,1,E]) + be) - the embedded logits map itself, not the one-hot
 * of its arg-max.  planes == 2 only (a training format). */
int mvb_head_class_fwd_dense(const float* h32, const float* Wo, float* logits_out, int32_t* ids_out,
                             const float* We, const float* be, int E, void* xh_next, int64_t plane_stride, int cpad,
                             int64_t NS, int H, int W, int planes, void* stream);
/* Regression head: off[s,HW,2] = conv3x3(h, Wo[3,3,256,2]);
 * if xh_next: x block <- planes of tanh(conv3x3(off, We[3,3,2,E]) + be). */
int mvb_head_reg_fwd(const float* h32, const float* Wo, float* off_out, const float* We,
                     const float* be, int E, void* xh_next, int64_t plane_stride, int cpad,
                     int64_t NS, int H, int W, int planes, void* stream);
/* x block <- planes of tanh(conv3x3(one_hot(ids), We) + be) for given ids (decoder step 0 and
 * the beam search's chosen cells, pred_models.py:602-606, :662-666). */
int mvb_emb_onehot_fwd(const int32_t* ids, const float* We, const float* be, int E, void* xh_next,
                       int64_t plane_stride, int cpad, int64_t NS, int H, int W, int planes,
                       void* stream);
/* x block <- planes of tanh(conv3x3(x, We[3,3,2,E]) + be) for a dense NHWC fp32 input [NS,H,W,2]
 * (regression decoder step 0, pred_models.py:386-387, :442-446). */
int mvb_emb_dense_fwd(const float* x, const float* We, const float* be, int E, void* xh_next,
                      int64_t plane_stride, int cpad, int64_t NS, int H, int W, int planes,
                      void* stream);

/* ---- a6: beam step (pred_models.py:547-606; add_div_penalty :1197-1223) ------------------
 * Per sample n over its B beams: lp = log_softmax(logits) + score; optional
 * lp += log(gamma) * rank_within_row(lp); candidates = all B*V (first_step: beam 0 only);
 * top-B (descending, ties -> lower flat index); score' (zeroed if zero_scores);
 * ids = idx % V; parents = idx / V; row_map_out[n*B+b] = n*B + parents (for the state gather). */
int mvb_beam_step(const float* logits, const float* score_in, float* score_out, int32_t* ids_out,
                  int32_t* parents_out, int32_t* row_map_out, int64_t N, int B, int V,
                  int first_step, int zero_scores, int diverse, float log_gamma, void* stream);
/* The other optimizers of Trainer (pred_models.py:1667-1681), fused with the same gradient preparation as
 * mvb_clip_adadelta (g = grad * grad_scale + wd * w, then clip to +-clip if clip > 0):
 *   kind 1 MomentumOptimizer(lr, p1 = 0.9): slot1 = p1 slot1 + g; w -= lr slot1
 *   kind 2 AdamOptimizer: slot1 (m), slot2 (v), p1 = beta1, p2 = beta2; `lr` must carry sqrt(1-beta2^t)/(1-beta1^t)
 *   kind 3 RMSPropOptimizer: slot1 = ms (initialise to ONE like TF), slot2 = mom, p1 = decay 0.9, p2 = momentum 0.0,
 *          eps 1e-10 */
int mvb_clip_update(float* w, const float* grad, float* slot1, float* slot2, int64_t n, int kind, float lr, float p1,
                    float p2, float eps, float clip, float wd, float grad_scale, void* stream);

/* ---- f-4: SimAug's white-box attack on the scene input (SimAug/code/pred_models.py:60-170) ----------------------
 * The gradient of the (targeted) classification loss with respect to the scene features comes out of the ordinary
 * backward pass: mvb_scene_conv_bwd with a non-NULL `din` for the FIRST scene convolution accumulates d loss / d input
 * (fp32 [F,SH,SW,SC]).  One attack step (:96-124, bounds :142-143), element-wise over n values:
 *   out = clip(adv - step * sign(grad), clip(x - eps, -1, 1), clip(x + eps, -1, 1))      (FGSM: step = eps; PGD: step size)
 * and the mixup of :149-166: out = a * w + b * (1 - w). */
int mvb_adv_step(const float* x, const float* adv, const float* grad, float* out, float eps, float step, int64_t n,
                 void* stream);
int mvb_mix(const float* a, const float* b, float* out, float w, int64_t n, void* stream);
/* Per-row sparse softmax cross entropy without gradient, loss[r] = logsumexp(logits[r,:]) - logits[r, labels[r]] (NaN
 * for a label outside [0,V), as TensorFlow): what SimAug's multi-view augmentation ranks the M views of a sample by
 * (mean over the predicted steps, SimAug/code/pred_models.py:386-392, :413-416, :465-470).  logits fp32 [rows,V]. */
int mvb_ce_rows(const float* logits, const int32_t* labels, float* loss, int64_t rows, int V, void* stream);
/* multiview_exp 3 (SimAug/code/pred_models.py:616-638): the class encoder's input with the observed grid class mixed
 * from two views, scene_conv (.) (beta * one_hot(label) + one_hot(label2) * (1 - beta)): two weighted feature pixels
 * per sample row (one, weighted beta + (1 - beta) in fp32, when the labels coincide) into an x block that is zero on
 * entry; and its backward (x-block gradient -> d scene_conv, atomically added).  Shapes as mvb_enc_class_input. */
int mvb_enc_class_input_mix(const float* scene_conv, const int32_t* frame_idx, const int32_t* label,
                            const int32_t* label2, float beta, void* xh_planes, int64_t plane_stride, int cpad,
                            int64_t NS, int H, int W, int planes, void* stream);
int mvb_enc_class_input_mix_bwd(const float* dxh, int cpad, const int32_t* frame_idx, const int32_t* label,
                                const int32_t* label2, float beta, float* dscene, int64_t NS, int H, int W,
                                void* stream);

/* ---- f-3: multi-future evaluation metrics on the device ------------------------------------------------------
 * minADE / minFDE of code/multifuture_eval_trajs.py:41-78 (get_min :16-21): for every trajectory n and ground-truth
 * future g (gt_len[n,g] steps, 0 = absent) the prediction k in [0,K) with the smallest left-to-right SUM of per-step
 * L2 errors (first index on ties) -> its per-step errors ade_err [N,G,Tg] fp64 (0 beyond the length) and index
 * ade_idx [N,G]; and the smallest final-step error fde [N,G] fp64 with its index.  Double arithmetic on the fp32
 * inputs, i.e. the reference's numpy float64 results bit for bit.
 *   pred fp32 [N,K,Tp,2] (mvb_decode_trajectories output), gt fp32 [N,G,Tg,2], Tg <= Tp. */
int mvb_min_ade_fde(const float* pred, const float* gt, const int32_t* gt_len, double* ade_err, int32_t* ade_idx,
                    double* fde, int32_t* fde_idx, int64_t N, int G, int K, int Tp, int Tg, void* stream);
/* NLL of code/multifuture_eval_trajs_prob.py:113-131,170-197: for trajectory n and evaluated step steps[j] the grid
 * distribution p = sum_b softmax(logprobs[n,:])[b] * softmax(logits[n,b,steps[j],:]) (get_hw_prob) and
 * nll[n,j] = mean over the present ground-truth cells gt_idx[n,j,g] >= 0 of -log(p[cell] + DBL_EPSILON)
 * (compute_nll); count[n,j] = number of present cells (0: the reference skips that step).
 *   logits fp32 [N,K,Tp,V] and logprobs fp32 [N,K] = beam_outputs[0], [2]; gt_idx int32 [N,J,G]; steps int32 [J]. */
int mvb_beam_nll(const float* logits, const float* logprobs, const int32_t* gt_idx, const int32_t* steps, double* nll,
                 int32_t* count, int64_t N, int K, int Tp, int V, int J, int G, void* stream);
/* mvb_beam_nll of a batch whose rows end at their own lengths (lengths int32 [N], the decode's out["_lengths"]):
 * logits [N,K,Tp,V] as the ragged decode leaves them (zeros after each row's length), and a step steps[j] >=
 * lengths[n] is not evaluated for row n (count 0).  With every length Tp it equals mvb_beam_nll bit for bit. */
int mvb_beam_nll_ragged(const float* logits, const float* logprobs, const int32_t* lengths, const int32_t* gt_idx,
                        const int32_t* steps, double* nll, int32_t* count, int64_t N, int K, int Tp, int V, int J,
                        int G, void* stream);
/* mvb_min_ade_fde on the decode's selections instead of fp32 points: prediction k's point at step t is
 *   centers[ids[n,k,t]] + (double)offsets[n,k,t]    (center_only: centers[ids[n,k,t]])
 * one fp64 add, as multifuture_inference.py:504-517 forms it on float64 centres, against fp64 ground truth
 * gt [N,G,Tg,2] (gt_len [N,G], 0 = absent).  Same selections and errors as mvb_min_ade_fde (shared code); greedy
 * decodes are K = 1.  ids int32 [N,K,Tp] (beam_outputs[1] or the arg-max), offsets fp32 [N,K,Tp,2]
 * (mvb_gather_offsets; unread with center_only, may be NULL), centers fp64 [V,2], lengths int32 [N] (the rows'
 * prediction lengths).  *err |= 1 for a future longer than its row's predictions (or a row longer than Tp), |= 2 for
 * an id outside [0, V); such futures are not scored (index -1).  err is not cleared. */
int mvb_min_ade_fde_cells(const int32_t* ids, const float* offsets, const double* centers, int center_only,
                          const int32_t* lengths, const double* gt, const int32_t* gt_len, double* ade_err,
                          int32_t* ade_idx, double* fde, int32_t* fde_idx, int32_t* err, int64_t N, int G, int K,
                          int Tp, int V, int Tg, void* stream);
/* xys_to_indexes of code/multifuture_eval_trajs_prob.py:45-63: points fp64 [P,2] frame pixels -> cells int32 [P] =
 * y * scene_w + x of the grid cell, per axis ceil(c / gap) with gap = video / scene in fp64, 0 counted as 1, minus
 * one, negative indices wrapped as numpy indexes.  An index outside [-size, size) sets *err = 1 (numpy's IndexError)
 * and that cell to -1.  err is not cleared. */
int mvb_points_to_cells(const double* points, int32_t* cells, int32_t* err, int64_t P, int scene_h, int scene_w,
                        int video_h, int video_w, void* stream);

/* Back-trace (pred_models.py:689-764): step_ids/step_parents int32 [Tp,N,B], step_logits fp32
 * [Tp,N,B,V] -> out_ids int32 [N,B,Tp], out_logits fp32 [N,B,Tp,V]. */
int mvb_beam_backtrace(const int32_t* step_ids, const int32_t* step_parents,
                       const float* step_logits, int32_t* out_ids, float* out_logits, int64_t N,
                       int B, int Tp, int V, void* stream);
/* Back-trace of a batch whose rows end at their own lengths (1 <= lengths[n] <= Tp, int32 [N]): row n's trace starts
 * at its own last step lengths[n] - 1, and out_ids / out_logits of row n at the steps t >= lengths[n] are zeros.
 * Shapes as mvb_beam_backtrace; steps >= lengths[n] of the step buffers are not read for row n. */
int mvb_beam_backtrace_ragged(const int32_t* step_ids, const int32_t* step_parents, const float* step_logits,
                              const int32_t* lengths, int32_t* out_ids, float* out_logits, int64_t N, int B, int Tp,
                              int V, void* stream);

/* Parent-state gather of the beam decoder without graph attention (use_gnn off: pred_models.py:611-623, then the
 * gathered h goes straight into the cell): for every sample row s < NS and valid cell, the h block (channels
 * [cpad_out - 256, cpad_out)) of row s of hp_out <- the f16f8 operand values of h32 row row_map[s] (fp32 halo).
 * hp_out is an f16f8 operand buffer of NS*(H+1)*(W+1) rows (hp_plane_stride = that times cpad_out); its x block,
 * channel padding and halo rows are not written. */
int mvb_beam_gather_h_f16f8(const float* h32, const int32_t* row_map, void* hp_out, int64_t hp_plane_stride,
                            int cpad_out, int64_t NS, int H, int W, void* stream);

/* Image-row bands of the beam decoder (DESIGN.md 3.2).  Beam k's c and h equal those of its sample's base rollout
 * (the same recurrence fed the no-selection input; ids outside the grid, e.g. (H+3)*W) outside the rows
 *   band[k] = clamp(widen(band_in[parent(k)], radius) U [y(ids[k]) - 2, y(ids[k]) + 2])
 * (radius 2 with the graph attention, 1 without; band_in NULL at the fan-out: no parent band).  ids, parents int32
 * [NS] (NS = N*K; parents within the sample, as mvb_beam_step writes them), bands int32 [NS][2] (first, last row).
 * Also writes the work list of the step's cell launch (mvb_convlstm_cell_fwd_onehot): int32 (m0, m_end) pairs of
 * 128-row M tiles over the bands' GEMM rows, tiles_cap >= NS * (ceil((H+1)(W+1) / 128) + 1) of them, and their
 * count.  Everything stays on the device. */
int mvb_beam_band(const int32_t* ids, const int32_t* parents, const int32_t* band_in, int32_t* band_out,
                  int32_t* tiles, int64_t tiles_cap, int32_t* tile_count, int64_t NS, int K, int radius, int H, int W,
                  void* stream);
/* c, h32 fp32 [NS*(H+1)*(W+1), 256] halo: the valid rows of beam k outside band[k] <- rows of sample k / K of the
 * base rollout's base_c, base_h32 ([N*(H+1)*(W+1), 256]).  The rows inside the bands are not touched. */
int mvb_beam_band_copy(const float* base_c, const float* base_h32, const int32_t* band, float* c, float* h32,
                       int64_t NS, int K, int H, int W, void* stream);

/* ---- f-1 (next row): feed generation on the device (multifuture_inference.py:115-156, preprocess.py:436-475):
 *      traj fp64 [NT,2] frame pixels, centers fp64 [H*W,2] (the caller's scene_grid_centers) ->
 *      labels int32 [NT] (cell of every point), regress fp32 [NT,H,W,2] (point - centre of every cell). */
int mvb_traj_to_grid(const double* traj, const double* centers, double h_gap, double w_gap, int32_t* labels,
                     float* regress, int64_t NT, int H, int W, void* stream);
/* The regression encoder's input from the trajectories (training): = mvb_nhwc_to_planes(src, ..., ch_off 0, C 2,
 * bf16x2 planes, comp) of src[s,y,x] = float32(traj[s * traj_stride + (0,1)] - centers[y*W+x]) (fp64 difference),
 * without src: traj fp64 points of NS rows, traj_stride >= 2 doubles apart (one time step of [N,T,2]). */
int mvb_traj_to_planes(const double* traj, int64_t traj_stride, const double* centers, void* dst_planes,
                       int64_t plane_stride, int cpad, int64_t NS, int H, int W, int comp, void* stream);

/* ---- f-3 (next row): post-decode on the device (multifuture_inference.py:504-517,
 *      pred_utils.py:460-492): out[n,k,t] = centers[ids[n,k,t]] + offsets[t,n,ids[n,k,t]].
 *      ids int32 [N,K,Tp]; offsets fp32 [Tp,N,V,2] (mvb_head_reg_fwd layout); centers fp32 [V,2]. */
int mvb_decode_trajectories(const int32_t* ids, const float* offsets, const float* centers, float* out,
                            int64_t N, int K, int Tp, int V, void* stream);
/* The fp32 offsets of the selected cells alone, for a caller that adds them to the centres in its own precision
 * (multifuture_inference.py:495-517 in float64): out[n,k,t] = offsets[t,n,ids[n,k,t]] for t < lengths[n], zeros
 * after.  ids int32 [N,K,Tp]; offsets fp32 [Tp,N,V,2]; lengths int32 [N] (1..Tp); out fp32 [N,K,Tp,2]. */
int mvb_gather_offsets(const int32_t* ids, const float* offsets, const int32_t* lengths, float* out, int64_t N, int K,
                       int Tp, int V, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MULTIVERSE_B200_H_ */
