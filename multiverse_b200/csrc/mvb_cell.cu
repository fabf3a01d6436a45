// K-cell: the fused ConvLSTM cell of the Multiverse encoder/decoder.
//
// Replaces, per call, what the reference runs as tf.contrib.rnn.ConvLSTMCell.call
// (built at code/pred_models.py:189-202 and :236-249, driven by dynamic_rnn :212/:232
// and raw_rnn :455/:678):  concat([x,h]) -> conv3x3 SAME -> +biases -> split i,j,f,o ->
// c' = sigmoid(f+forget_bias)*c + sigmoid(i)*tanh(j);  h' = tanh(c')*sigmoid(o).
//
// Formulation: one persistent warp-specialised wgmma GEMM
//     G[R, 1024] = A[R, 9*Cpad] * Bt[1024, 9*Cpad]^T
// over the halo layout (mvb_common.cuh): the A k-block for tap t / channel chunk q is
// the rows [m0+shift(t), +128) x channels [64q, +64) of the activation matrix, read in place from one TMA-loaded
// stage per chunk, so the 3x3 im2col never exists in memory.  fp32 parity on 16-bit tensor cores comes from one of
// two operand formats (mvb_common.cuh): bf16x2, x = x0 + x1 with both planes bf16 (mvb::split_planes), whose products
// a0*b0 + a0*b1 + a1*b0 (3 MMAs, error ~2^-17) go into the same fp32 accumulator; or f16f8, an fp16 pass and an e4m3
// cross-term pass at twice the rate (2 bf16-pass equivalents) at the same accuracy.
// Output columns are gate-interleaved (tile of 256 = 4 gates x 64 channels) so every
// thread holds i,j,f,o of its channels in its accumulator registers and emits (c', h') directly - the gate
// pre-activations never reach HBM.
//
// Warp roles (384 threads, 1 CTA/SM, persistent over tiles):
//   warpgroup 0      TMA producer (one thread), registers handed to the others (setmaxnreg)
//   warpgroups 1, 2  MMA + epilogue: each owns 64 rows of the 128-row tile, all 256 columns (128 fp32
//                    accumulators per thread)
// f16f8 launches of many M tiles per SM run cell_fwd_epi_kernel instead: tiles of 128 x 128 (4 gates x 32
// channels) and a fourth warpgroup that runs the epilogue of one tile from shared memory while the MMA warpgroups compute the next.
#include "mvb_common.cuh"
#include "mvb_kernels.h"
#include <stdlib.h>

namespace mvb {

constexpr int BLOCK_M = kCellTileRows;
constexpr int BLOCK_N = 256;
constexpr int XPAD = 32;      // the x block is zero-padded to a multiple of 32 channels (cpad = roundup(cx,32) + 256)
constexpr int kMaxXBlock = 256;   // widest x block of the GEMM: four 64-channel chunks (emb_size up to 256)
constexpr int CHUNK = 64;     // channels per K chunk: 64 16-bit elements = 128 B = one SWIZZLE_128B row
constexpr int ROW_BYTES = 128;
constexpr int MMA_K = 16;       // K of one 16-bit wgmma
constexpr int TILE_CH = 64;   // hidden channels per N tile
constexpr int N_TILES = kGates / BLOCK_N;  // 4
constexpr int NUM_THREADS = 384;
constexpr int B_SLOT_BYTES = BLOCK_N * ROW_BYTES;  // 32 KB: 256 weight rows x 128 B
constexpr uint32_t SW128_LAYOUT = kSwizzle128B;
constexpr uint32_t SW128_SBO = 8 * ROW_BYTES;      // 1024 B between 8-row groups

// Shared-memory rings.  The TMA unit writes about one box row per clock into shared memory whatever the row's width,
// so the stages are made of full 128-byte rows and no activation row is loaded once per tap:
//   B ring: slots of 256 rows x 128 B = 64 channels of ONE plane of the weight tile (SWIZZLE_128B): per (chunk,
//           tap) 2 slots (bf16x2: one per weight plane), or one per pass (f16f8: the fp16 plane, then both e4m3 planes
//           interleaved in one row).
//   A ring: one stage per 64-channel chunk: rows [m0 - (Wp+1), m0 + 128 + (Wp+1)) of every activation plane,
//           rounded up to a multiple of 8 rows (RA8).  The nine taps of the chunk read THE SAME stage through wgmma
//           descriptors that start (dy Wp + dx) rows into it (see make_smem_desc).
// Layout: [B slots][A stages][barriers: full, empty (kMaxBSlots each), afull, aempty (kMaxAStages each)].
constexpr int kSmemLimit = 227 * 1024;
constexpr int kSmemExtra = 1024 /*alignment*/ + 512 /*barriers*/;
constexpr int kMaxBSlots = 8;
constexpr int kMaxAStages = 4;
static_assert((2 * kMaxBSlots + 2 * kMaxAStages) * 8 <= 512, "the barrier area holds every ring's barriers");

struct CellRing {
  int b_slots, a_stages, a_stage_bytes;
  constexpr int smem_bytes() const { return b_slots * B_SLOT_BYTES + a_stages * a_stage_bytes + kSmemExtra; }
};

template <int FMT>
struct CellCfg {
  static constexpr int MAX_RA8 = 256;           // TMA box limit: 128 + 2 (W + 2) <= 256  ->  W <= 62
  static constexpr CellRing ring(int ra8) {
    if (FMT == 0) {
      // bf16x2: both planes of a chunk in one stage, two stages; 4 weight slots when they fit beside them, else 3
      const int a = kBf16Planes * ra8 * ROW_BYTES;
      return CellRing{(4 * B_SLOT_BYTES + 2 * a + 2048 <= kSmemLimit) ? 4 : 3, 2, a};
    }
    // f16f8: a pass loads one 128-byte row per A row (the fp16 plane, or both e4m3 planes interleaved), so a stage
    // holds one plane.  As many weight slots as fit beside two stages (5 at every width up to 62), then a third
    // stage where it still fits (W <= 21: 36x18, 18x9).
    const int a = ra8 * ROW_BYTES;
    int b = (kSmemLimit - kSmemExtra - 2 * a) / B_SLOT_BYTES;
    if (b > kMaxBSlots) b = kMaxBSlots;
    return CellRing{b, CellRing{b, 3, a}.smem_bytes() <= kSmemLimit ? 3 : 2, a};
  }
};
static_assert(CellCfg<1>::ring(168).b_slots == 5 && CellCfg<1>::ring(168).a_stages == 3, "36x18: 5 slots, 3 stages");
static_assert(CellCfg<1>::ring(152).b_slots == 5 && CellCfg<1>::ring(152).a_stages == 3, "18x9: 5 slots, 3 stages");
static_assert(CellCfg<1>::ring(200).b_slots == 5 && CellCfg<1>::ring(200).a_stages == 2, "18x32: 5 slots, 2 stages");
static_assert(CellCfg<1>::ring(256).b_slots == 5 && CellCfg<1>::ring(256).a_stages == 2 &&
              CellCfg<1>::ring(256).smem_bytes() <= kSmemLimit, "4x62: 5 slots, 2 stages");
static_assert(CellCfg<0>::ring(168).b_slots == 4 && CellCfg<0>::ring(200).b_slots == 3, "bf16x2 rings unchanged");

// Phase profile (built with -DMVB_CELL_PROBE only, tools/probe_cell_phases.py): clock64() cycles of every warpgroup's
// first thread, summed over all CTAs of the launches since the last read.  The product build has none of it.
enum CellProbePhase {
  kProbeFullWait, kProbeAFullWait, kProbeMmaWait, kProbeEpilogue, kProbeConsumer,    // MMA warpgroups
  kProbeEmptyWait, kProbeAEmptyWait, kProbeProducer,                                 // TMA producer thread
  // cell_fwd_epi_kernel: the MMA warpgroups' wait for a free staging buffer (their kProbeEpilogue is the staging
  // write), the epilogue warpgroup's wait for a staged tile and the rest of its time
  kProbeFreeWait, kProbeStagedWait, kProbeEpiBusy,
  kProbeTiles, kProbePhases
};
#ifdef MVB_CELL_PROBE
__device__ unsigned long long g_cell_probe[kProbePhases];
#define CELL_PROBE(...) __VA_ARGS__
#define CELL_PROBED(ph, ...) do { const long long t0_ = clock64(); __VA_ARGS__; probe[ph] += clock64() - t0_; } while (0)
#else
#define CELL_PROBE(...)
#define CELL_PROBED(ph, ...) __VA_ARGS__
#endif

struct CellParams {
  const float* bias;        // [1024] packed (tile, gate, channel) order
  const float* col_scale;   // f16f8 only: [1024] 2^-S of every packed column (the weights are stored times 2^S)
  const float* c_in;        // [R_src, 256] or nullptr (zero state)
  const int* row_map;       // [NS] source sample-row of c_in, or nullptr (identity)
  float* c_out;             // [R, 256]
  float* h32_out;           // [R, 256] or nullptr
  float* gates_out;         // [R, 1024] activated gates (packed column order) for training, or nullptr
  // "x-fold" (class decoder only): the input is grid_emb(one_hot(id)), i.e. tanh(b) everywhere except
  // the 3x3 cells around id, so its whole contribution to the pre-activations is a table look-up:
  // xf_B[border class of the cell][1024] (bias folded in) + xf_T2[border class of id][5x5 offset][1024]
  // for the <=25 cells around id.  The x chunk is then skipped in the K loop (skip_x).
  const float* xf_B;        // [9][1024] packed column order, or nullptr
  const float* xf_T2;       // [9][25][1024]
  const int* xf_ids;        // [NS] arg-max cell of every sample row
  int skip_x;               // x-fold: the x chunk of the K loop is skipped
  // dense raw x block of two channels, added in fp32 in the epilogue instead of going through the tensor cores
  // (regression encoder: the +-1.9e3 pixel offsets need all 24 bits, which neither operand format carries in 2 passes):
  // sparse x block (class encoder: scene features at ONE cell per sample row): per-sample table rows
  // xs_tab[sample][tap][1024] = features(label cell) . W[tap], added to the <= 9 cells around the label
  const float* xs_tab;      // [NS, 9, 1024] fp32 packed column order, or nullptr
  const int* xs_label;      // [NS]
  const float* xr_in;       // [NS, H, W, 2] fp32 NHWC (no halo), or nullptr
  const float* xr_W;        // [9 taps * 2 channels][1024] fp32, packed column order
  int order;                // work order, see work_index()
  CellRing ring;            // shared-memory rings of this launch (CellCfg<FMT>::ring)
  float* preact_out;        // [R, 1024] raw accumulators (packed column order) instead of the state update: first stage of
                            // the fan-out step (fanout_children_kernel turns every parent row into its K children)
  int hp_mixed;             // hp_out is written in the f16f8 format (else bf16x2 planes)
  __nv_bfloat16* hp_out;    // [2][R][cpad_out] plane base or nullptr
  long long hp_plane_stride;  // elements between planes of hp_out
  int cpad_out;             // row pitch of hp_out (elements)
  int ch_off_out;           // channel offset of the h block inside hp_out rows
  long long R;              // total halo rows
  // work list (beam decoder, mvb_beam_band): M tiles (m0, m_end) pairs [*tile_count][2], or nullptr (the launch's
  // 128-row blocks in order); a tile's stores are clipped to [m0, m_end)
  const int* tiles;
  const int* tile_count;
  int H, W;
  int cpad;                 // K channels per tap (multiple of 32)
  float forget_bias;
};

// The state update of one element from its four gate pre-activations, with the roundings spelled out so that the
// cell epilogue and the fan-out kernel produce the same bits:  c' = sigmoid(f + forget_bias) c + sigmoid(i) tanh(j);
// h' = tanh(c') sigmoid(o).
struct GateOut { float ai, aj, af, ao, c, h; };
__device__ __forceinline__ GateOut lstm_update(float xi, float xj, float xf, float xo, float cprev, float forget_bias) {
  GateOut r;
  r.ai = sigmoid_acc(xi); r.aj = tanh_acc(xj); r.af = sigmoid_acc(__fadd_rn(xf, forget_bias)); r.ao = sigmoid_acc(xo);
  r.c = __fmaf_rn(r.af, cprev, __fmul_rn(r.ai, r.aj));
  r.h = __fmul_rn(tanh_acc(r.c), r.ao);
  return r;
}
// pre-activation from the accumulator: acc * (column scale, f16f8 only) + (bias + x-fold table row)
template <int FMT>
__device__ __forceinline__ float preact(float acc, float scale, float q) {
  return FMT ? __fmaf_rn(acc, scale, q) : __fadd_rn(acc, q);
}

// Per-row context of the epilogue: where the row's state comes from and which input tables apply to it.
struct EpiRow {
  long long row, src_row, psmp;
  int py, px;
  bool valid;
  const float* xfb;     // x-fold: table row of this cell's border class (bias included), else nullptr
  const float* xft;     // x-fold / sparse-x table row of this cell for its sample row, else nullptr
};

__device__ __forceinline__ EpiRow epi_row(const CellParams& prm, const Grid& g, long long row, long long m_end) {
  EpiRow r;
  r.row = row; r.src_row = row; r.psmp = 0; r.py = 0; r.px = 0; r.xfb = nullptr; r.xft = nullptr;
  r.valid = row < m_end;
  if (!r.valid) return r;
  const long long smp = row / g.S;
  const int rem = (int)(row - smp * g.S);
  const int y = rem / g.Wp, x = rem - y * g.Wp;
  r.valid = (x < g.W) && (y < g.H);
  if (!r.valid) return r;
  if (prm.row_map) r.src_row = (long long)prm.row_map[smp] * g.S + rem;
  r.py = y; r.px = x; r.psmp = smp;
  if (prm.xf_B) {
    const int cy = y == 0 ? 0 : (y == g.H - 1 ? 2 : 1), cx = x == 0 ? 0 : (x == g.W - 1 ? 2 : 1);
    r.xfb = prm.xf_B + (cy * 3 + cx) * kGates;
    // x-fold table row of this cell for the sample row whose arg-max cell is `a` (nullptr outside its 5x5)
    const int a = prm.xf_ids[smp];
    const int ay = a / g.W, ax = a - ay * g.W;
    const int ry = y - ay, rx = x - ax;
    if (ry >= -2 && ry <= 2 && rx >= -2 && rx <= 2) {
      const int acy = ay == 0 ? 0 : (ay == g.H - 1 ? 2 : 1), acx = ax == 0 ? 0 : (ax == g.W - 1 ? 2 : 1);
      r.xft = prm.xf_T2 + ((long long)(acy * 3 + acx) * 25 + (ry + 2) * 5 + (rx + 2)) * kGates;
    }
  }
  if (prm.xs_tab) {          // out[p] += in[p + off(tap)] . W[tap] with the input at the label cell only
    const int l = prm.xs_label[smp];
    if (l >= 0 && l < g.H * g.W) {
      const int ly = l / g.W, dy = ly - y, dx = (l - ly * g.W) - x;
      if (dy >= -1 && dy <= 1 && dx >= -1 && dx <= 1)
        r.xft = prm.xs_tab + ((long long)smp * 9 + (dy + 1) * 3 + (dx + 1)) * kGates;
    }
  }
  return r;
}

// M tiles of a launch, and the rows [m0, m_end) that tile i computes and stores: the launch's 128-row blocks in order,
// or entry i of the work list.  An index past the list (rank 1 of a pair on an odd count) stores nothing.
__device__ __forceinline__ long long m_tile_count(const CellParams& prm) {
  return prm.tiles ? (long long)__ldg(prm.tile_count) : (prm.R + BLOCK_M - 1) / BLOCK_M;
}
__device__ __forceinline__ void m_tile_rows(const CellParams& prm, long long count, long long i, long long& m0,
                                            long long& m_end) {
  if (!prm.tiles) { m0 = i * BLOCK_M; m_end = prm.R; }
  else if (i < count) { m0 = __ldg(prm.tiles + 2 * i); m_end = __ldg(prm.tiles + 2 * i + 1); }
  else { m0 = 0; m_end = 0; }
}

// c of the row's channels ch, ch + 1 from the previous step (zero state without c_in).  The epilogue fetches all of
// its rows' c before the tile's last MMAs complete (the rows are scattered by row_map, so each is an HBM round trip).
__device__ __forceinline__ float2 epi_cprev(const CellParams& prm, const EpiRow& r, int ch) {
  return (prm.c_in && !prm.preact_out && r.valid)
             ? __ldg(reinterpret_cast<const float2*>(prm.c_in + r.src_row * kHidden + ch)) : make_float2(0.f, 0.f);
}

// What the pre-activations of one row and two adjacent packed columns j, j + 1 of every gate add to the
// accumulators: q = bias (or bias-folded table) + x-fold / sparse-x table row + dense x path, and the f16f8 column
// scales.  Loaded for both rows of a column pair before either is stored (epi_pair), so that the loads of one row do
// not wait for the stores of the other.
struct EpiIn { float q[4][2], sc[4][2]; };
template <int FMT>
__device__ __forceinline__ EpiIn epi_inputs(const CellParams& prm, const Grid& g, const EpiRow& r, int nt, int j) {
  EpiIn in = {};
  if (prm.preact_out || !r.valid) return in;
  const int col = nt * BLOCK_N + j;             // packed column of gate 0
  const float* bptr = (r.xfb ? r.xfb : prm.bias) + col;
  float (&q)[4][2] = in.q;
#pragma unroll
  for (int gt = 0; gt < 4; ++gt) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(bptr + gt * TILE_CH));
    q[gt][0] = b.x; q[gt][1] = b.y;
  }
  if (r.xft) {
#pragma unroll
    for (int gt = 0; gt < 4; ++gt) {
      const float2 t = __ldg(reinterpret_cast<const float2*>(r.xft + col + gt * TILE_CH));
      q[gt][0] = __fadd_rn(q[gt][0], t.x); q[gt][1] = __fadd_rn(q[gt][1], t.y);
    }
  }
  if (prm.xr_W) {           // + sum over taps and the two channels of x * W, fp32
#pragma unroll 1
    for (int k = 0; k < 18; ++k) {
      const int tp = k >> 1, yy = r.py + tp / 3 - 1, xx = r.px + tp % 3 - 1;
      const float xk = (yy >= 0 && yy < g.H && xx >= 0 && xx < g.W)
                           ? __ldg(prm.xr_in + ((r.psmp * g.H + yy) * g.W + xx) * 2 + (k & 1)) : 0.f;
#pragma unroll
      for (int gt = 0; gt < 4; ++gt) {
        const float2 w = __ldg(reinterpret_cast<const float2*>(prm.xr_W + k * kGates + col + gt * TILE_CH));
        q[gt][0] = __fmaf_rn(xk, w.x, q[gt][0]); q[gt][1] = __fmaf_rn(xk, w.y, q[gt][1]);
      }
    }
  }
  if (FMT == 1) {
#pragma unroll
    for (int gt = 0; gt < 4; ++gt) {
      const float2 s2 = __ldg(reinterpret_cast<const float2*>(prm.col_scale + col + gt * TILE_CH));
      in.sc[gt][0] = s2.x; in.sc[gt][1] = s2.y;
    }
  }
  return in;
}

// The epilogue of one row and two adjacent packed columns j, j + 1 of every gate (a[gate][e] = accumulators of
// column gate * 64 + j + e of N tile nt, cprev = epi_cprev of its channels, in = epi_inputs): state update and every
// requested output.
template <int FMT>
__device__ __forceinline__ void epi_pair(const CellParams& prm, const EpiRow& r, int nt, int j, const float (&a)[4][2],
                                         float2 cprev, const EpiIn& in) {
  const int col = nt * BLOCK_N + j;             // packed column of gate 0
  const int ch = nt * TILE_CH + j;              // hidden channel
  if (prm.preact_out) {
    float* gp = prm.preact_out + r.row * kGates + col;
#pragma unroll
    for (int gt = 0; gt < 4; ++gt) *reinterpret_cast<float2*>(gp + gt * TILE_CH) = make_float2(a[gt][0], a[gt][1]);
    return;
  }
  const float (&q)[4][2] = in.q;
  const float (&sc)[4][2] = in.sc;
  GateOut o[2];
#pragma unroll
  for (int e = 0; e < 2; ++e)
    o[e] = lstm_update(preact<FMT>(a[0][e], sc[0][e], q[0][e]), preact<FMT>(a[1][e], sc[1][e], q[1][e]),
                       preact<FMT>(a[2][e], sc[2][e], q[2][e]), preact<FMT>(a[3][e], sc[3][e], q[3][e]),
                       e ? cprev.y : cprev.x, prm.forget_bias);
  if (prm.gates_out) {
    float* gp = prm.gates_out + r.row * kGates + col;
    *reinterpret_cast<float2*>(gp + 0 * TILE_CH) = make_float2(o[0].ai, o[1].ai);
    *reinterpret_cast<float2*>(gp + 1 * TILE_CH) = make_float2(o[0].aj, o[1].aj);
    *reinterpret_cast<float2*>(gp + 2 * TILE_CH) = make_float2(o[0].af, o[1].af);
    *reinterpret_cast<float2*>(gp + 3 * TILE_CH) = make_float2(o[0].ao, o[1].ao);
  }
  *reinterpret_cast<float2*>(prm.c_out + r.row * kHidden + ch) = make_float2(o[0].c, o[1].c);
  if (prm.h32_out) *reinterpret_cast<float2*>(prm.h32_out + r.row * kHidden + ch) = make_float2(o[0].h, o[1].h);
  if (prm.hp_out && prm.hp_mixed) {
    uint32_t h2, e0, e1;
    split_f16f8_x2(o[0].h, o[1].h, h2, e0, e1);
    const int c = prm.ch_off_out + ch;
    *reinterpret_cast<uint32_t*>(reinterpret_cast<__half*>(prm.hp_out) + r.row * prm.cpad_out + c) = h2;
    uint8_t* b8 = reinterpret_cast<uint8_t*>(prm.hp_out) + 2 * prm.hp_plane_stride + r.row * 2 * prm.cpad_out;
    *reinterpret_cast<uint16_t*>(b8 + f8_off(c, 0, prm.cpad_out)) = (uint16_t)e0;
    *reinterpret_cast<uint16_t*>(b8 + f8_off(c, 1, prm.cpad_out)) = (uint16_t)e1;
  } else if (prm.hp_out) {
    __nv_bfloat16 p0[kBf16Planes], p1[kBf16Planes];
    split_planes(o[0].h, p0);
    split_planes(o[1].h, p1);
#pragma unroll
    for (int p = 0; p < kBf16Planes; ++p)
      *reinterpret_cast<uint32_t*>(prm.hp_out + p * prm.hp_plane_stride + r.row * prm.cpad_out + prm.ch_off_out + ch) =
          pack_bf16x2(p0[p], p1[p]);
  }
}

// MMA steps of x chunk q (channels [64 q, +64) of the x block, cut at its end cxp): K16 steps of a 16-bit plane,
// K32 steps of one e4m3 plane, and the distance in 16-byte units from e0 to e1 in an fp8 row (f8_off).
__device__ __forceinline__ void x_chunk_steps(int q, int cxp, int cpad, int& ks16, int& ks8, uint32_t& poff) {
  const int c16 = q * CHUNK, width = cxp - c16 < CHUNK ? cxp - c16 : CHUNK;
  ks16 = width / MMA_K;
  ks8 = width / 32;
  poff = (uint32_t)(f8_off(c16, 1, cpad) - f8_off(c16, 0, cpad)) >> 4;
}

// MC = true: clusters of two CTAs work on two M tiles of the same N tile in lock step; each loads half of every B
// (weight) tile and TMA-multicasts it to both, so the L2 -> shared-memory traffic per CTA and stage drops from
// 48 KB to 32 KB (bf16x2).  A slot may be refilled once the MMA warpgroups of BOTH CTAs have consumed it (empty
// barrier count 4: two warpgroups per CTA arrive on their own and on the peer's barrier).
// FMT = 1: f16f8 operands (FMT = 0: bf16x2).  tmA / tmB then describe the fp16 regions (one
// "plane") and tmA8 / tmB8 the two fp8 planes; per 64-channel chunk and tap each warpgroup sends four e4m3 MMAs
// (K = 32 each) and four fp16 MMAs (K = 16 each) into the same accumulator: 2 bf16-pass equivalents instead of 3.
template <bool MC, int FMT>
__global__ void __launch_bounds__(NUM_THREADS, 1)
cell_fwd_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmA8, const __grid_constant__ CUtensorMap tmB8,
                const CellParams prm) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  const int ra8 = (BLOCK_M + 2 * (prm.W + 2) + 7) & ~7;     // rows of an A stage
  const int a_stage_bytes = prm.ring.a_stage_bytes;
  const int a_load_bytes = FMT ? ra8 * ROW_BYTES : a_stage_bytes;     // f16f8: one plane per pass
  const int b_slots = prm.ring.b_slots, a_stages = prm.ring.a_stages;
  uint8_t* smem_a = smem + b_slots * B_SLOT_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_a + a_stages * a_stage_bytes);
  uint64_t* empty_bar = full_bar + kMaxBSlots;
  uint64_t* afull_bar = empty_bar + kMaxBSlots;
  uint64_t* aempty_bar = afull_bar + kMaxAStages;
  CELL_PROBE(long long probe[kProbePhases] = {};)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;                    // 0: TMA producer; 1, 2: MMA + epilogue of rows [64 (wg - 1), +64)
  const Grid g = make_grid(prm.H, prm.W);
  // K chunks of 64 channels: the nqx x chunks [64 q, +64) - of which only the cxp channels of the x block are
  // multiplied, so the last one may be half a chunk - then the four chunks of the h block [cxp + 64 j, +64).  fp8 rows
  // (f16f8): both e4m3 planes of a chunk side by side (mvb_common.cuh f8_off), 2 * cpad bytes per row.
  const int cxp = prm.cpad - kHidden;
  const int nqx = (cxp + CHUNK - 1) / CHUNK;
  const int q_begin = prm.skip_x ? nqx : 0;
  const int NQ = nqx + kHidden / CHUNK;
  // f16f8: two passes over K, the e4m3 cross terms first and then the fp16 main products.  The e4m3 MMAs accumulate
  // with a short internal sum (about 14 significant bits of the accumulator), so they run while the accumulator holds
  // only their own small sum (~2^-11 of the result); the fp16 MMAs, exact in fp32, then add the main products.
  constexpr int NPASS = FMT ? 2 : 1;
  constexpr int NS = FMT ? 1 : kBf16Planes;    // B slots per (pass, chunk, tap)
  const long long num_m_tiles = m_tile_count(prm);
  // work index w -> (m tile, n tile).  MC: the pair shares w; rank r takes m tile 2*(w / N_TILES) + r.
  const uint32_t rank = MC ? cluster_ctarank() : 0u;
  const long long num_tiles = (MC ? (num_m_tiles + 1) / 2 : num_m_tiles) * N_TILES;
  const long long w_begin = MC ? (long long)(blockIdx.x >> 1) : (long long)blockIdx.x;
  const long long w_step = MC ? (long long)(gridDim.x >> 1) : (long long)gridDim.x;
  // iteration it of this CTA (pair) -> work index.  order 1 (default): the N tiles of an M tile run back to back on
  // the same CTA (pair), so its operand rows are re-read from L2 by the SM that fetched them; order 0: strided
  // (the N tiles of an M tile run concurrently on neighbouring CTAs).
  auto work_index = [&](long long it) -> long long {
    return prm.order ? (w_begin + (it / N_TILES) * w_step) * N_TILES + it % N_TILES : w_begin + it * w_step;
  };
  auto tile_rows = [&](long long w, long long& m0, long long& m_end) {
    m_tile_rows(prm, num_m_tiles, (w / N_TILES) * (MC ? 2 : 1) + rank, m0, m_end);
  };

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    if (FMT == 1) { prefetch_tmap(&tmA8); prefetch_tmap(&tmB8); }
#pragma unroll 1
    for (int s = 0; s < b_slots; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], MC ? 4 : 2); }
#pragma unroll 1
    for (int s = 0; s < a_stages; ++s) { mbar_init(&afull_bar[s], 1); mbar_init(&aempty_bar[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  if (MC) cluster_sync_all();     // the peer's barriers exist before anything is sent to them

  if (wg == 0) {
    regs_dealloc<40>();
    if (warp == 0 && lane == 0) {
      // ===================== TMA producer =====================
      int slot = 0, astage = 0; uint32_t phase = 0, aphase = 0;
      CELL_PROBE(const long long probe_t0 = clock64();)
      for (long long it = 0, t; (t = work_index(it)) < num_tiles; ++it) {
        long long m0, m_end;
        tile_rows(t, m0, m_end);
        const int n0 = (int)(t % N_TILES) * BLOCK_N;
        // chunk-major K order: the x block - whose terms can be orders of magnitude larger than the h terms (raw
        // pixel offsets in the regression encoder) - is accumulated first, so the small h products are never added
        // onto a large transient partial sum.
        for (int pass = 0; pass < NPASS; ++pass)
        for (int q = q_begin; q < NQ; ++q) {
          const int c16 = q < nqx ? q * CHUNK : cxp + (q - nqx) * CHUNK;     // 16-bit channel coordinate
          const int c8 = f8_off(c16, 0, prm.cpad);                          // fp8 byte coordinate
          const bool f8 = FMT == 1 && pass == 0;
          CELL_PROBED(kProbeAEmptyWait, mbar_wait(&aempty_bar[astage], aphase ^ 1));
          uint8_t* sa = smem_a + astage * a_stage_bytes;
          mbar_expect_tx(&afull_bar[astage], a_load_bytes);
          if (f8) tma_load_3d(sa, &tmA8, &afull_bar[astage], c8, (int)(m0 - g.Wp - 1), 0);
          else tma_load_3d(sa, &tmA, &afull_bar[astage], c16, (int)(m0 - g.Wp - 1), 0);
          if (++astage == a_stages) { astage = 0; aphase ^= 1; }
          for (int tap = 0; tap < 9; ++tap) {
#pragma unroll
            for (int sl = 0; sl < NS; ++sl) {
              CELL_PROBED(kProbeEmptyWait, mbar_wait(&empty_bar[slot], phase ^ 1));
              uint8_t* sb = smem + slot * B_SLOT_BYTES;
              mbar_expect_tx(&full_bar[slot], B_SLOT_BYTES);
              const CUtensorMap* tm = f8 ? &tmB8 : &tmB;
              const int kcol = f8 ? tap * 2 * prm.cpad + c8 : tap * prm.cpad + c16;
              // MC: this CTA's half (128 rows) of the slot, delivered to both CTAs of the pair
              if (MC) tma_load_3d_mc(sb + rank * (B_SLOT_BYTES / 2), tm, &full_bar[slot], kcol,
                                     n0 + (int)rank * (BLOCK_N / 2), sl, (uint16_t)3);
              else tma_load_3d(sb, tm, &full_bar[slot], kcol, n0, sl);
              if (++slot == b_slots) { slot = 0; phase ^= 1; }
            }
          }
        }
      }
#ifdef MVB_CELL_PROBE
      atomicAdd(&g_cell_probe[kProbeEmptyWait], (unsigned long long)probe[kProbeEmptyWait]);
      atomicAdd(&g_cell_probe[kProbeAEmptyWait], (unsigned long long)probe[kProbeAEmptyWait]);
      atomicAdd(&g_cell_probe[kProbeProducer], (unsigned long long)(clock64() - probe_t0));
#endif
    }
  } else {
    regs_alloc<232>();
    // ===================== MMA + epilogue (one warpgroup per 64 rows of the tile) =====================
    const int c = wg - 1;
    const bool leader = (threadIdx.x & 127) == 0;          // arrives on the barriers for the warpgroup
    constexpr uint32_t kHi = smem_desc_hi(SW128_SBO, SW128_LAYOUT);
    const uint32_t a_plane_lo = (uint32_t)(ra8 * ROW_BYTES) >> 4;
    const uint32_t a_wg_lo = (uint32_t)(64 * c) * (ROW_BYTES >> 4);      // this warpgroup's 64 rows of the A tile
    int slot = 0, astage = 0; uint32_t phase = 0, aphase = 0;
    float acc[128];
    // release of the previous batch of MMAs' operands, once they have completed
    int rel_slot = -1, rel_astage = -1;
    auto release = [&]() {
      if (leader && rel_slot >= 0) {
        if (MC) { mbar_arrive_remote(&empty_bar[rel_slot], 0); mbar_arrive_remote(&empty_bar[rel_slot], 1); }
        else mbar_arrive(&empty_bar[rel_slot]);
        if (rel_astage >= 0) mbar_arrive(&aempty_bar[rel_astage]);
      }
      rel_slot = -1; rel_astage = -1;
    };
    CELL_PROBE(const long long probe_t0 = clock64();)
    for (long long it = 0, t; (t = work_index(it)) < num_tiles; ++it) {
      CELL_PROBE(++probe[kProbeTiles];)
      long long m0, m_end;
      tile_rows(t, m0, m_end);
      const int nt = (int)(t % N_TILES);
      uint32_t fresh = 1;                      // the tile's first MMA overwrites the accumulator
      auto mma16 = [&](uint32_t a_lo, uint32_t b_lo) {
        if (FMT == 1) wgmma_f16<256, 0, 0>(acc, desc_of(a_lo, kHi), desc_of(b_lo, kHi), fresh ^ 1u);
        else wgmma_bf16<256, 0, 0>(acc, desc_of(a_lo, kHi), desc_of(b_lo, kHi), fresh ^ 1u);
        fresh = 0;
      };
      auto mma8 = [&](uint32_t a_lo, uint32_t b_lo) {
        wgmma_e4m3_n256(acc, desc_of(a_lo, kHi), desc_of(b_lo, kHi), fresh ^ 1u);
        fresh = 0;
      };
      for (int pass = 0; pass < NPASS; ++pass)
      for (int q = q_begin; q < NQ; ++q) {
        const bool f8 = FMT == 1 && pass == 0;
        CELL_PROBED(kProbeAFullWait, mbar_wait(&afull_bar[astage], aphase));
        const uint32_t sa_lo = (smem_u32(smem_a + astage * a_stage_bytes) >> 4) + a_wg_lo;
        for (int tap = 0; tap < 9; ++tap) {
          // the tap's A tile: the stage's rows starting (dy-1) Wp + (dx-1) + (Wp+1) = dy Wp + dx rows in
          const uint32_t a_lo = sa_lo + (uint32_t)((tap / 3) * g.Wp + (tap % 3)) * (ROW_BYTES >> 4);
#pragma unroll
          for (int sl = 0; sl < NS; ++sl) {
            CELL_PROBED(kProbeFullWait, mbar_wait(&full_bar[slot], phase));
            const uint32_t b_lo = smem_u32(smem + slot * B_SLOT_BYTES) >> 4;
            wgmma_fence_regs(acc);
            wgmma_fence();
            if (q >= nqx) {
              // ---- h chunk: 64 channels = 4 K16 steps per 16-bit plane pair, 4 K32 steps over the two e4m3 planes ----
              if (f8) {
                for (int k = 0; k < 4; ++k) mma8(a_lo + 2 * k, b_lo + 2 * k);    // [e0 (64 B) | e1 (64 B)]
              } else {
                // bf16x2: B plane 0 against A planes 0 and 1, B plane 1 against A plane 0 (a0b0 + a1b0 + a0b1);
                // f16f8: the fp16 planes
#pragma unroll
                for (int pa = 0; pa < (FMT ? 1 : kBf16Planes - sl); ++pa)
#pragma unroll
                  for (int k = 0; k < 4; ++k) mma16(a_lo + pa * a_plane_lo + 2 * k, b_lo + 2 * k);
              }
            } else {
              // ---- x chunk (only cells whose input is not folded): 64 channels, or 32 for a trailing half chunk ----
              int ks16, ks8; uint32_t poff;
              x_chunk_steps(q, cxp, prm.cpad, ks16, ks8, poff);
              if (f8) {
                for (int pk = 0; pk < 2 * ks8; ++pk) {
                  const uint32_t o = (pk / ks8) * poff + (pk % ks8) * 2;
                  mma8(a_lo + o, b_lo + o);
                }
              } else {
                for (int pa = 0; pa < (FMT ? 1 : kBf16Planes - sl); ++pa)
                  for (int k = 0; k < ks16; ++k) mma16(a_lo + pa * a_plane_lo + 2 * k, b_lo + 2 * k);
              }
            }
            wgmma_commit();
            wgmma_fence_regs(acc);
            // the previous batch has completed: its slot (and A stage) can be refilled
            CELL_PROBED(kProbeMmaWait, wgmma_wait<1>());
            release();
            rel_slot = slot;
            if (tap == 8 && sl == NS - 1) rel_astage = astage;     // this CTA's nine taps have consumed the A stage
            if (++slot == b_slots) { slot = 0; phase ^= 1; }
          }
        }
        if (++astage == a_stages) { astage = 0; aphase ^= 1; }
      }
      // ===================== epilogue =====================
      // thread (warp w of the warpgroup, lane l) holds rows 16 w + l / 4 (+ 8) and columns 8 i + 2 (l % 4) (+ 1);
      // column gate * 64 + j of the N tile is gate `gate` of channel j: each thread owns all four gates of its channels.
      // The rows' context and c are loaded while the last MMAs run, all at once rather than one pair after another's
      // stores.
      CELL_PROBE(const long long probe_e0 = clock64();)
      const long long rbase = m0 + 64 * c + 16 * (warp & 3) + (lane >> 2);
      EpiRow rows[2];
      float2 cprev[2][8];
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        rows[hr] = epi_row(prm, g, rbase + 8 * hr, m_end);
#pragma unroll
        for (int ip = 0; ip < 8; ++ip) cprev[hr][ip] = epi_cprev(prm, rows[hr], nt * TILE_CH + 8 * ip + 2 * (lane & 3));
      }
      CELL_PROBE(const long long probe_w0 = clock64();)
      wgmma_wait<0>();
      CELL_PROBE(const long long probe_w = clock64() - probe_w0; probe[kProbeMmaWait] += probe_w;)
      wgmma_fence_regs(acc);
      release();
#pragma unroll
      for (int ip = 0; ip < 8; ++ip) {
        const int j = 8 * ip + 2 * (lane & 3);
        EpiIn in[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) in[hr] = epi_inputs<FMT>(prm, g, rows[hr], nt, j);
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          if (!rows[hr].valid) continue;
          float a[4][2];
#pragma unroll
          for (int gt = 0; gt < 4; ++gt) {
            a[gt][0] = acc[4 * (8 * gt + ip) + 2 * hr];
            a[gt][1] = acc[4 * (8 * gt + ip) + 2 * hr + 1];
          }
          epi_pair<FMT>(prm, rows[hr], nt, j, a, cprev[hr][ip], in[hr]);
        }
      }
      CELL_PROBE(probe[kProbeEpilogue] += clock64() - probe_e0 - probe_w;)
    }
#ifdef MVB_CELL_PROBE
    if (leader) {
      for (int p = kProbeFullWait; p <= kProbeEpilogue; ++p) atomicAdd(&g_cell_probe[p], (unsigned long long)probe[p]);
      atomicAdd(&g_cell_probe[kProbeConsumer], (unsigned long long)(clock64() - probe_t0));
      atomicAdd(&g_cell_probe[kProbeTiles], (unsigned long long)probe[kProbeTiles]);
    }
#endif
  }

  __syncthreads();
  if (MC) cluster_sync_all();     // the peer may still send into this CTA's smem / barriers
}

// ----------------------------------------------------------------------------------
// f16f8 cell with an epilogue warpgroup (the f16f8 kernel of large launches, kEpiWgMinTilesPerSm; MVB_CELL_EPI_WG=0
// runs cell_fwd_kernel instead, MVB_CELL_EPI_WG=1 this one at every size).
// Tiles of 128 rows x 128 columns, 512 threads, 1 CTA/SM, persistent over tiles:
//   warpgroup 0      TMA producer (one thread)
//   warpgroups 1, 2  MMA only: each owns 64 rows of the tile (m64n128: 64 fp32 accumulators per thread).  When a
//                    tile's MMAs have completed they copy the accumulators into a 64 KB fp32 staging buffer in shared
//                    memory and start the next tile at once
//   warpgroup 3      the epilogue of the staged tile (epi_row, epi_cprev, epi_inputs, epi_pair: the same functions of
//                    the same accumulators as cell_fwd_kernel) while the MMA warpgroups run the next tile's mainloop
// The mainloop is cell_fwd_kernel's f16f8 one (both passes, e4m3 first; halo'd A stages read by all nine taps; pair
// multicast of the weight slots).  A weight slot still serves 128 rows, so the weight bytes per FLOP are unchanged;
// an A stage now serves eight N tiles instead of four.
// Columns: N tile nt of 128 holds all four gates of 32 channels: packed columns T * 256 + gate * 64 + 32 h + [0, 32)
// with T = nt / 2, h = nt % 2.  Its weight rows are four 32-row groups of the packed weights, loaded as one 4-D TMA
// box (rows = [32 rows][2 halves][16 (tile, gate)]), so the packed column order of the weights and of every table
// is the one cell_fwd_kernel reads.
// ----------------------------------------------------------------------------------
constexpr int EW_BLOCK_N = 128;
constexpr int EW_TILE_CH = EW_BLOCK_N / 4;                  // 32 channels per N tile
constexpr int EW_N_TILES = kGates / EW_BLOCK_N;             // 8
constexpr int EW_THREADS = 512;
constexpr int EW_SLOT_BYTES = EW_BLOCK_N * ROW_BYTES;       // 16 KB: 128 weight rows x 128 B
constexpr int EW_STAGING_BYTES = BLOCK_M * EW_BLOCK_N * 4;  // 64 KB: the fp32 accumulators of one tile
// setmaxnreg budgets: producer, each MMA warpgroup, the epilogue warpgroup
constexpr int kEwRegsProducer = 40, kEwRegsMma = 152, kEwRegsEpi = 168;
static_assert(128 * (kEwRegsProducer + 2 * kEwRegsMma + kEwRegsEpi) <= 65536, "the four warpgroups fit the register file");

// Layout: [staging][B slots][A stages][barriers: full, empty (kMaxBSlots each), afull, aempty (kMaxAStages each),
// staged, staging free].  Three A stages where 6 weight slots of 16 KB still fit beside them and the staging buffer
// (36x18, 18x9), else two stages and as many slots as fit (6 at 18x32 and 4x62): measured on the beam launch, the third
// stage is worth a slot, a sixth slot is worth more than the third stage.
struct CellEpiCfg {
  static constexpr int slots(int a, int stages) {
    const int b = (kSmemLimit - kSmemExtra - EW_STAGING_BYTES - stages * a) / EW_SLOT_BYTES;
    return b > kMaxBSlots ? kMaxBSlots : b;
  }
  static constexpr CellRing ring(int ra8) {
    const int a = ra8 * ROW_BYTES;
    return slots(a, 3) >= 6 ? CellRing{slots(a, 3), 3, a} : CellRing{slots(a, 2), 2, a};
  }
  static constexpr int smem_bytes(const CellRing& r) {
    return EW_STAGING_BYTES + r.b_slots * EW_SLOT_BYTES + r.a_stages * r.a_stage_bytes + kSmemExtra;
  }
};
static_assert((2 * kMaxBSlots + 2 * kMaxAStages + 2) * 8 <= 512, "the barrier area holds the staging barriers too");
static_assert(CellEpiCfg::ring(168).b_slots == 6 && CellEpiCfg::ring(168).a_stages == 3 &&
              CellEpiCfg::smem_bytes(CellEpiCfg::ring(168)) <= kSmemLimit, "36x18: 6 slots, 3 stages");
static_assert(CellEpiCfg::ring(152).b_slots == 6 && CellEpiCfg::ring(152).a_stages == 3 &&
              CellEpiCfg::smem_bytes(CellEpiCfg::ring(152)) <= kSmemLimit, "18x9: 6 slots, 3 stages");
static_assert(CellEpiCfg::ring(200).b_slots == 6 && CellEpiCfg::ring(200).a_stages == 2 && CellEpiCfg::smem_bytes(CellEpiCfg::ring(200)) <= kSmemLimit,
              "18x32: 6 slots, 2 stages");
static_assert(CellEpiCfg::ring(256).b_slots == 6 && CellEpiCfg::ring(256).a_stages == 2 && CellEpiCfg::smem_bytes(CellEpiCfg::ring(256)) <= kSmemLimit,
              "4x62: 6 slots, 2 stages");

// fp32 offset of (row r, column col) of the staging buffer: rows of 128 floats whose 16-byte chunks are XOR-swizzled
// by the row, so that the float2 accesses of the accumulator fragment layout (8 rows x 4 threads per 8-column group)
// - the MMA warpgroups' writes and the epilogue warpgroup's reads alike - touch 32 different banks per 16 threads.
__device__ __forceinline__ int staging_off(int r, int col) {
  return r * EW_BLOCK_N + ((((col >> 2) ^ ((r & 3) << 1))) << 2) + (col & 3);
}

template <bool MC>
__global__ void __launch_bounds__(EW_THREADS, 1)
cell_fwd_epi_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmA8, const __grid_constant__ CUtensorMap tmB8,
                    const CellParams prm) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  const int ra8 = (BLOCK_M + 2 * (prm.W + 2) + 7) & ~7;     // rows of an A stage
  const int a_stage_bytes = prm.ring.a_stage_bytes;           // one plane: ra8 rows of 128 B
  const int b_slots = prm.ring.b_slots, a_stages = prm.ring.a_stages;
  float* staging = reinterpret_cast<float*>(smem);
  uint8_t* smem_b = smem + EW_STAGING_BYTES;
  uint8_t* smem_a = smem_b + b_slots * EW_SLOT_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_a + a_stages * a_stage_bytes);
  uint64_t* empty_bar = full_bar + kMaxBSlots;
  uint64_t* afull_bar = empty_bar + kMaxBSlots;
  uint64_t* aempty_bar = afull_bar + kMaxAStages;
  uint64_t* staged_bar = aempty_bar + kMaxAStages;   // every MMA thread has written its accumulators to the staging
  uint64_t* free_bar = staged_bar + 1;               // every epilogue thread has read the staged tile
  CELL_PROBE(long long probe[kProbePhases] = {};)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;                    // 0: TMA producer; 1, 2: MMA of rows [64 (wg - 1), +64); 3: epilogue
  const Grid g = make_grid(prm.H, prm.W);
  const int cxp = prm.cpad - kHidden;
  const int nqx = (cxp + CHUNK - 1) / CHUNK;   // x chunks, then the four h chunks (as in cell_fwd_kernel)
  const int q_begin = prm.skip_x ? nqx : 0;
  const int NQ = nqx + kHidden / CHUNK;
  const long long num_m_tiles = m_tile_count(prm);
  const uint32_t rank = MC ? cluster_ctarank() : 0u;
  const long long num_tiles = (MC ? (num_m_tiles + 1) / 2 : num_m_tiles) * EW_N_TILES;
  const long long w_begin = MC ? (long long)(blockIdx.x >> 1) : (long long)blockIdx.x;
  const long long w_step = MC ? (long long)(gridDim.x >> 1) : (long long)gridDim.x;
  auto work_index = [&](long long it) -> long long {      // as in cell_fwd_kernel, with eight N tiles per M tile
    return prm.order ? (w_begin + (it / EW_N_TILES) * w_step) * EW_N_TILES + it % EW_N_TILES : w_begin + it * w_step;
  };
  auto tile_rows = [&](long long w, long long& m0, long long& m_end) {
    m_tile_rows(prm, num_m_tiles, (w / EW_N_TILES) * (MC ? 2 : 1) + rank, m0, m_end);
  };

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA); prefetch_tmap(&tmB); prefetch_tmap(&tmA8); prefetch_tmap(&tmB8);
#pragma unroll 1
    for (int s = 0; s < b_slots; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], MC ? 4 : 2); }
#pragma unroll 1
    for (int s = 0; s < a_stages; ++s) { mbar_init(&afull_bar[s], 1); mbar_init(&aempty_bar[s], 2); }
    mbar_init(staged_bar, 256);
    mbar_init(free_bar, 128);
    fence_barrier_init();
  }
  __syncthreads();
  if (MC) cluster_sync_all();     // the peer's barriers exist before anything is sent to them

  if (wg == 0) {
    regs_dealloc<kEwRegsProducer>();
    if (warp == 0 && lane == 0) {
      // ===================== TMA producer =====================
      int slot = 0, astage = 0; uint32_t phase = 0, aphase = 0;
      CELL_PROBE(const long long probe_t0 = clock64();)
      for (long long it = 0, t; (t = work_index(it)) < num_tiles; ++it) {
        long long m0, m_end;
        tile_rows(t, m0, m_end);
        const int nt = (int)(t % EW_N_TILES);
        const int half = nt & 1, tg0 = (nt >> 1) * 4;      // 32-row half and (tile, gate) index of gate 0
        for (int pass = 0; pass < 2; ++pass)
        for (int q = q_begin; q < NQ; ++q) {
          const int c16 = q < nqx ? q * CHUNK : cxp + (q - nqx) * CHUNK;
          const int c8 = f8_off(c16, 0, prm.cpad);
          const bool f8 = pass == 0;
          CELL_PROBED(kProbeAEmptyWait, mbar_wait(&aempty_bar[astage], aphase ^ 1));
          uint8_t* sa = smem_a + astage * a_stage_bytes;
          mbar_expect_tx(&afull_bar[astage], a_stage_bytes);
          if (f8) tma_load_3d(sa, &tmA8, &afull_bar[astage], c8, (int)(m0 - g.Wp - 1), 0);
          else tma_load_3d(sa, &tmA, &afull_bar[astage], c16, (int)(m0 - g.Wp - 1), 0);
          if (++astage == a_stages) { astage = 0; aphase ^= 1; }
          for (int tap = 0; tap < 9; ++tap) {
            CELL_PROBED(kProbeEmptyWait, mbar_wait(&empty_bar[slot], phase ^ 1));
            uint8_t* sb = smem_b + slot * EW_SLOT_BYTES;
            mbar_expect_tx(&full_bar[slot], EW_SLOT_BYTES);
            const CUtensorMap* tm = f8 ? &tmB8 : &tmB;
            const int kcol = f8 ? tap * 2 * prm.cpad + c8 : tap * prm.cpad + c16;
            // MC: this CTA's two gates (64 rows) of the slot, delivered to both CTAs of the pair
            if (MC) tma_load_4d_mc(sb + rank * (EW_SLOT_BYTES / 2), tm, &full_bar[slot], kcol, 0, half,
                                   tg0 + 2 * (int)rank, (uint16_t)3);
            else tma_load_4d(sb, tm, &full_bar[slot], kcol, 0, half, tg0);
            if (++slot == b_slots) { slot = 0; phase ^= 1; }
          }
        }
      }
#ifdef MVB_CELL_PROBE
      atomicAdd(&g_cell_probe[kProbeEmptyWait], (unsigned long long)probe[kProbeEmptyWait]);
      atomicAdd(&g_cell_probe[kProbeAEmptyWait], (unsigned long long)probe[kProbeAEmptyWait]);
      atomicAdd(&g_cell_probe[kProbeProducer], (unsigned long long)(clock64() - probe_t0));
#endif
    }
  } else if (wg < 3) {
    regs_alloc<kEwRegsMma>();
    // ===================== MMA (one warpgroup per 64 rows of the tile) =====================
    const int c = wg - 1;
    const bool leader = (threadIdx.x & 127) == 0;          // arrives on the ring barriers for the warpgroup
    constexpr uint32_t kHi = smem_desc_hi(SW128_SBO, SW128_LAYOUT);
    const uint32_t a_wg_lo = (uint32_t)(64 * c) * (ROW_BYTES >> 4);      // this warpgroup's 64 rows of the A tile
    int slot = 0, astage = 0; uint32_t phase = 0, aphase = 0, free_phase = 0;
    float acc[64];
    // Two MMA batches (weight slots) in flight per warpgroup: a slot of 128 columns is 512 tensor clocks, half of
    // cell_fwd_kernel's, and with one batch in flight the barrier / fence / wait of every slot left the tensor pipe
    // idle.  A batch's slot (and, after its ninth tap, A stage) is released once the batch after next is issued and
    // wgmma.wait_group 2 has returned.
    constexpr int D = 2;
    int rq_slot[D], rq_astage[D];
#pragma unroll
    for (int i = 0; i < D; ++i) { rq_slot[i] = -1; rq_astage[i] = -1; }
    auto release_one = [&](int rs, int ra) {
      if (leader && rs >= 0) {
        if (MC) { mbar_arrive_remote(&empty_bar[rs], 0); mbar_arrive_remote(&empty_bar[rs], 1); }
        else mbar_arrive(&empty_bar[rs]);
        if (ra >= 0) mbar_arrive(&aempty_bar[ra]);
      }
    };
    CELL_PROBE(const long long probe_t0 = clock64();)
    for (long long it = 0, t; (t = work_index(it)) < num_tiles; ++it) {
      CELL_PROBE(++probe[kProbeTiles];)
      uint32_t fresh = 1;                      // the tile's first MMA overwrites the accumulator
      for (int pass = 0; pass < 2; ++pass)
      for (int q = q_begin; q < NQ; ++q) {
        const bool f8 = pass == 0;
        CELL_PROBED(kProbeAFullWait, mbar_wait(&afull_bar[astage], aphase));
        const uint32_t sa_lo = (smem_u32(smem_a + astage * a_stage_bytes) >> 4) + a_wg_lo;
        for (int tap = 0; tap < 9; ++tap) {
          const uint32_t a_lo = sa_lo + (uint32_t)((tap / 3) * g.Wp + (tap % 3)) * (ROW_BYTES >> 4);
          CELL_PROBED(kProbeFullWait, mbar_wait(&full_bar[slot], phase));
          const uint32_t b_lo = smem_u32(smem_b + slot * EW_SLOT_BYTES) >> 4;
          wgmma_fence_regs(acc);
          wgmma_fence();
          if (q >= nqx) {
            if (f8) {
              for (int k = 0; k < 4; ++k) {           // [e0 (64 B) | e1 (64 B)]
                wgmma_e4m3_n128(acc, desc_of(a_lo + 2 * k, kHi), desc_of(b_lo + 2 * k, kHi), fresh ^ 1u);
                fresh = 0;
              }
            } else {
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                wgmma_f16<128, 0, 0>(acc, desc_of(a_lo + 2 * k, kHi), desc_of(b_lo + 2 * k, kHi), fresh ^ 1u);
                fresh = 0;
              }
            }
          } else {
            // ---- x chunk (only cells whose input is not folded): 64 channels, or 32 for a trailing half chunk ----
            int ks16, ks8; uint32_t poff;
            x_chunk_steps(q, cxp, prm.cpad, ks16, ks8, poff);
            if (f8) {
              for (int pk = 0; pk < 2 * ks8; ++pk) {
                const uint32_t o = (pk / ks8) * poff + (pk % ks8) * 2;
                wgmma_e4m3_n128(acc, desc_of(a_lo + o, kHi), desc_of(b_lo + o, kHi), fresh ^ 1u);
                fresh = 0;
              }
            } else {
              for (int k = 0; k < ks16; ++k) {
                wgmma_f16<128, 0, 0>(acc, desc_of(a_lo + 2 * k, kHi), desc_of(b_lo + 2 * k, kHi), fresh ^ 1u);
                fresh = 0;
              }
            }
          }
          wgmma_commit();
          wgmma_fence_regs(acc);
          CELL_PROBED(kProbeMmaWait, wgmma_wait<D>());
          release_one(rq_slot[0], rq_astage[0]);
#pragma unroll
          for (int i = 0; i + 1 < D; ++i) { rq_slot[i] = rq_slot[i + 1]; rq_astage[i] = rq_astage[i + 1]; }
          rq_slot[D - 1] = slot;
          rq_astage[D - 1] = tap == 8 ? astage : -1;
          if (++slot == b_slots) { slot = 0; phase ^= 1; }
        }
        if (++astage == a_stages) { astage = 0; aphase ^= 1; }
      }
      CELL_PROBED(kProbeMmaWait, wgmma_wait<0>());
      wgmma_fence_regs(acc);
#pragma unroll
      for (int i = 0; i < D; ++i) { release_one(rq_slot[i], rq_astage[i]); rq_slot[i] = -1; rq_astage[i] = -1; }
      // ===================== accumulators -> staging =====================
      // thread (warp w, lane l) holds rows 16 w + l / 4 (+ 8) and columns 8 i + 2 (l % 4) (+ 1) of its 64 rows
      CELL_PROBED(kProbeFreeWait, mbar_wait(free_bar, free_phase ^ 1));
      free_phase ^= 1;
      CELL_PROBE(const long long probe_e0 = clock64();)
      const int r0 = 64 * c + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
      for (int i = 0; i < EW_BLOCK_N / 8; ++i)
#pragma unroll
        for (int hr = 0; hr < 2; ++hr)
          *reinterpret_cast<float2*>(staging + staging_off(r0 + 8 * hr, 8 * i + 2 * (lane & 3))) =
              make_float2(acc[4 * i + 2 * hr], acc[4 * i + 2 * hr + 1]);
      mbar_arrive(staged_bar);
      CELL_PROBE(probe[kProbeEpilogue] += clock64() - probe_e0;)
    }
#ifdef MVB_CELL_PROBE
    if (leader) {
      for (int p = kProbeFullWait; p <= kProbeEpilogue; ++p) atomicAdd(&g_cell_probe[p], (unsigned long long)probe[p]);
      atomicAdd(&g_cell_probe[kProbeFreeWait], (unsigned long long)probe[kProbeFreeWait]);
      atomicAdd(&g_cell_probe[kProbeConsumer], (unsigned long long)(clock64() - probe_t0));
      atomicAdd(&g_cell_probe[kProbeTiles], (unsigned long long)probe[kProbeTiles]);
    }
#endif
  } else {
    regs_alloc<kEwRegsEpi>();
    // ===================== epilogue of the staged tile =====================
    // thread (warp w, lane l) takes rows 32 w + 8 k + l / 4 (k < 4) and channel pairs 8 ip + 2 (l % 4) (ip < 4) of the
    // N tile's 32 channels: the accumulator fragment layout, so that its staging reads are free of bank conflicts.
    // Two rows at a time (ptxas allocates every warpgroup's registers under the 128 of the launch bound): their
    // context and c are loaded first - for the first two while the tile is still being computed.
    const int ew = warp & 3, lc = 2 * (lane & 3);
    uint32_t staged_phase = 0;
    CELL_PROBE(const long long probe_t0 = clock64();)
    for (long long it = 0, t; (t = work_index(it)) < num_tiles; ++it) {
      long long m0, m_end;
      tile_rows(t, m0, m_end);
      const int nt = (int)(t % EW_N_TILES);
      const int tn = nt >> 1, jh = (nt & 1) * EW_TILE_CH;   // 256-column tile and this N tile's first channel in it
      const int rb = 32 * ew + (lane >> 2);
#pragma unroll 1
      for (int k2 = 0; k2 < 4; k2 += 2) {
        EpiRow rows[2];
        float2 cprev[2][4];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          rows[hr] = epi_row(prm, g, m0 + rb + 8 * (k2 + hr), m_end);
#pragma unroll
          for (int ip = 0; ip < 4; ++ip) cprev[hr][ip] = epi_cprev(prm, rows[hr], tn * TILE_CH + jh + 8 * ip + lc);
        }
        if (k2 == 0) {
          CELL_PROBED(kProbeStagedWait, mbar_wait(staged_bar, staged_phase));
          staged_phase ^= 1;
        }
#pragma unroll
        for (int ip = 0; ip < 4; ++ip) {
          const int j = jh + 8 * ip + lc;            // packed column of gate 0 in the 256-column tile tn
          EpiIn in[2];
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) in[hr] = epi_inputs<1>(prm, g, rows[hr], tn, j);
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            if (!rows[hr].valid) continue;
            float a[4][2];
#pragma unroll
            for (int gt = 0; gt < 4; ++gt) {
              const float2 v = *reinterpret_cast<const float2*>(
                  staging + staging_off(rb + 8 * (k2 + hr), gt * EW_TILE_CH + 8 * ip + lc));
              a[gt][0] = v.x; a[gt][1] = v.y;
            }
            epi_pair<1>(prm, rows[hr], tn, j, a, cprev[hr][ip], in[hr]);
          }
        }
      }
      mbar_arrive(free_bar);
    }
#ifdef MVB_CELL_PROBE
    if ((threadIdx.x & 127) == 0) {
      atomicAdd(&g_cell_probe[kProbeStagedWait], (unsigned long long)probe[kProbeStagedWait]);
      atomicAdd(&g_cell_probe[kProbeEpiBusy],
                (unsigned long long)(clock64() - probe_t0 - probe[kProbeStagedWait]));
    }
#endif
  }

  __syncthreads();
  if (MC) cluster_sync_all();     // the peer may still send into this CTA's smem / barriers
}

// ----------------------------------------------------------------------------------
// Fan-out step of the beam decoder (the first K-row step: every child's parent is its sample's single t0 row, so the
// K children share the graph-attended h, the GEMM and c, and differ only in the folded table rows of their selected
// cell).  Stage 1 = the cell kernel with preact_out (one GEMM per PARENT row, raw accumulators to HBM: 4 KB per cell);
// stage 2 = this kernel: one warp per parent cell keeps the 1024 accumulators, the bias-folded table row and c in
// registers and emits the K children (c', h') - HBM-bound on its 2 KB of stores per child cell, where the round-1
// in-epilogue fan-out ran the K passes on 8 warps per SM (25 ms against a 2.5 ms HBM bound).
// Bit-identical to the K-times tiled launch: same preact() / lstm_update() roundings.
// ----------------------------------------------------------------------------------
template <int FMT>
__global__ void __launch_bounds__(256)
fanout_children_kernel(const float* __restrict__ acc, const float* __restrict__ col_scale,
                       const float* __restrict__ xf_B, const float* __restrict__ xf_T2, const int* __restrict__ ids,
                       const float* __restrict__ c_in, float* __restrict__ c_out, float* __restrict__ h32_out,
                       long long NS, int K, Grid g, float forget_bias) {
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int hw = g.H * g.W;
  if (wid >= NS * hw) return;
  const long long smp = wid / hw;
  const int cell = (int)(wid - smp * hw);
  const int y = cell / g.W, x = cell - y * g.W;
  const int rem = y * g.Wp + x;
  const long long prow = smp * g.S + rem;
  const int ch0 = lane * 8;                                  // this lane's 8 hidden channels
  const int col0 = (ch0 / TILE_CH) * BLOCK_N + ch0 % TILE_CH;   // packed column of gate 0 (gate g: + g * 64)
  const int cy = y == 0 ? 0 : (y == g.H - 1 ? 2 : 1), cx = x == 0 ? 0 : (x == g.W - 1 ? 2 : 1);
  float a[4][8], q0[4][8], sc[4][8], cp[8];
#pragma unroll
  for (int gt = 0; gt < 4; ++gt) {
    const float4* ap = reinterpret_cast<const float4*>(acc + prow * kGates + col0 + gt * TILE_CH);
    const float4* bp = reinterpret_cast<const float4*>(xf_B + (cy * 3 + cx) * kGates + col0 + gt * TILE_CH);
    const float4* sp = reinterpret_cast<const float4*>((FMT ? col_scale : xf_B) + col0 + gt * TILE_CH);
#pragma unroll
    for (int v = 0; v < 2; ++v) {
      const float4 av = __ldg(ap + v), bv = __ldg(bp + v), sv = __ldg(sp + v);
      a[gt][4 * v] = av.x; a[gt][4 * v + 1] = av.y; a[gt][4 * v + 2] = av.z; a[gt][4 * v + 3] = av.w;
      q0[gt][4 * v] = bv.x; q0[gt][4 * v + 1] = bv.y; q0[gt][4 * v + 2] = bv.z; q0[gt][4 * v + 3] = bv.w;
      sc[gt][4 * v] = sv.x; sc[gt][4 * v + 1] = sv.y; sc[gt][4 * v + 2] = sv.z; sc[gt][4 * v + 3] = sv.w;
    }
  }
  {
    const float4* cq = reinterpret_cast<const float4*>(c_in + prow * kHidden + ch0);
    const float4 c0 = __ldg(cq), c1 = __ldg(cq + 1);
    cp[0] = c0.x; cp[1] = c0.y; cp[2] = c0.z; cp[3] = c0.w; cp[4] = c1.x; cp[5] = c1.y; cp[6] = c1.z; cp[7] = c1.w;
  }
  for (int k = 0; k < K; ++k) {
    const long long osmp = smp * K + k;
    const int id = ids[osmp];
    const int ay = id / g.W, ax = id - ay * g.W;
    const int ry = y - ay, rx = x - ax;
    const float* tp = nullptr;      // x-fold table row of this cell for the child's selected cell (inside its 5x5)
    if (ry >= -2 && ry <= 2 && rx >= -2 && rx <= 2) {
      const int acy = ay == 0 ? 0 : (ay == g.H - 1 ? 2 : 1), acx = ax == 0 ? 0 : (ax == g.W - 1 ? 2 : 1);
      tp = xf_T2 + ((long long)(acy * 3 + acx) * 25 + (ry + 2) * 5 + (rx + 2)) * kGates + col0;
    }
    float cn[8], hn[8];
#pragma unroll
    for (int v = 0; v < 8; ++v) {
      float q[4];
#pragma unroll
      for (int gt = 0; gt < 4; ++gt) q[gt] = tp ? __fadd_rn(q0[gt][v], __ldg(tp + gt * TILE_CH + v)) : q0[gt][v];
      const GateOut r = lstm_update(preact<FMT>(a[0][v], sc[0][v], q[0]), preact<FMT>(a[1][v], sc[1][v], q[1]),
                                    preact<FMT>(a[2][v], sc[2][v], q[2]), preact<FMT>(a[3][v], sc[3][v], q[3]),
                                    cp[v], forget_bias);
      cn[v] = r.c; hn[v] = r.h;
    }
    const long long orow = osmp * g.S + rem;
    float4* co = reinterpret_cast<float4*>(c_out + orow * kHidden + ch0);
    co[0] = make_float4(cn[0], cn[1], cn[2], cn[3]); co[1] = make_float4(cn[4], cn[5], cn[6], cn[7]);
    float4* ho = reinterpret_cast<float4*>(h32_out + orow * kHidden + ch0);
    ho[0] = make_float4(hn[0], hn[1], hn[2], hn[3]); ho[1] = make_float4(hn[4], hn[5], hn[6], hn[7]);
  }
}

// ----------------------------------------------------------------------------------
// weight packing:  TF kernel [3,3,Cx+256,1024] (HWIO, gate order i,j,f,o) + biases
//   -> planes bf16 [2][1024][9*cpad]  (row = tile*256 + gate*64 + j,  k = tap*cpad + kc)
//   -> bias fp32 [1024] in the same row order
// kc < cx: input channel kc;  cx <= kc < cxp: zero;  kc >= cxp: hidden channel kc-cxp.
// ----------------------------------------------------------------------------------
__global__ void pack_weights_kernel(const float* __restrict__ kernel, const float* __restrict__ biases,
                                    __nv_bfloat16* __restrict__ wp, float* __restrict__ bias_packed,
                                    int cx, int cxp, int cpad, int comp) {
  const long long ktot = 9LL * cpad;
  const long long total = (long long)kGates * ktot;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i / ktot);
    const int k = (int)(i - (long long)n * ktot);
    const int tap = k / cpad, kcn = k - tap * cpad;
    const int tile = n / BLOCK_N, gate = (n % BLOCK_N) / TILE_CH, j = n % TILE_CH;
    const int col = gate * kHidden + tile * TILE_CH + j;
    int cin = -1, blk = 0;
    if (kcn >= cxp) cin = cx + (kcn - cxp);
    else if (!comp) { if (kcn < cx) cin = kcn; }
    else if (kcn < 4 * cx) { blk = kcn / cx; cin = kcn - blk * cx; }
    const float v = (cin >= 0) ? kernel[((long long)tap * (cx + kHidden) + cin) * kGates + col] : 0.f;
    __nv_bfloat16 pl[kBf16Planes];
    split_planes(v, pl);
    if (comp && kcn < cxp) {
      // compensated x block (see nhwc_to_planes_kernel): [W | W | W-w0-w1 | w1]
      if (blk == 2) {
        split_planes((v - __bfloat162float(pl[0])) - __bfloat162float(pl[1]), pl);
      } else if (blk == 3) {
        pl[0] = pl[1];
        pl[1] = __float2bfloat16_rn(0.f);
      }
    }
    wp[i] = pl[0];
    wp[total + i] = pl[1];
    if (k == 0) bias_packed[n] = biases[col];
  }
}

// x-fold tables of a class-decoder cell (packed column order n = tile*256 + gate*64 + j):
//   X0[e] = tanh(be[e]);  delta[k][e] = tanh(be[e] + We[8-k][e]) - X0[e]   (k = 3x3 position around the arg-max;
//   the one-hot at a reaches cell q = a + k through tap a - q, i.e. tap index 8 - k)
//   B[cls][n]        = bias[n] + sum_{tap valid at a cell of border class cls} X0 . W[tap][:E][n]
//   T2[acls][r][n]   = sum_{tap: q = p + off(tap) in 3x3(a), q inside the grid} delta[k(q)] . W[tap][:E][n],  r = p - a
__global__ void xfold_tables_kernel(const float* __restrict__ kernel, const float* __restrict__ biases,
                                    const float* __restrict__ We, const float* __restrict__ be, int E,
                                    float* __restrict__ Bt, float* __restrict__ T2) {
  const int total = (9 + 9 * 25) * kGates;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int n = i % kGates, item = i / kGates;
    const int tile = n / BLOCK_N, gate = (n % BLOCK_N) / TILE_CH, j = n % TILE_CH;
    const int col = gate * kHidden + tile * TILE_CH + j;
    const int cin_tot = E + kHidden;
    float acc = 0.f;
    if (item < 9) {
      const int cy = item / 3, cx = item % 3;
      acc = biases[col];
      for (int t = 0; t < 9; ++t) {
        const int oy = t / 3 - 1, ox = t % 3 - 1;
        if ((cy == 0 && oy < 0) || (cy == 2 && oy > 0) || (cx == 0 && ox < 0) || (cx == 2 && ox > 0)) continue;
        for (int e = 0; e < E; ++e) acc = fmaf(tanhf(be[e]), kernel[((long long)t * cin_tot + e) * kGates + col], acc);
      }
      Bt[item * kGates + n] = acc;
    } else {
      const int it2 = item - 9, acls = it2 / 25, rr = it2 % 25;
      const int acy = acls / 3, acx = acls % 3;
      const int ry = rr / 5 - 2, rx = rr % 5 - 2;
      for (int t = 0; t < 9; ++t) {
        const int ky = ry + t / 3 - 1, kx = rx + t % 3 - 1;      // q - a
        if (ky < -1 || ky > 1 || kx < -1 || kx > 1) continue;
        if ((acy == 0 && ky < 0) || (acy == 2 && ky > 0) || (acx == 0 && kx < 0) || (acx == 2 && kx > 0)) continue;
        const int k = (ky + 1) * 3 + (kx + 1);
        for (int e = 0; e < E; ++e) {
          const float d = tanhf(be[e] + We[(8 - k) * E + e]) - tanhf(be[e]);
          acc = fmaf(d, kernel[((long long)t * cin_tot + e) * kGates + col], acc);
        }
      }
      T2[(long long)it2 * kGates + n] = acc;
    }
  }
}

// weights of the dense x path: rows (tap, channel) of the TF kernel [3,3,2+256,1024] in the packed column order
__global__ void xdense_weights_kernel(const float* __restrict__ kernel, float* __restrict__ out) {
  const int total = 18 * kGates;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int n = i % kGates, k = i / kGates, tap = k >> 1, ch = k & 1;
    const int tile = n / BLOCK_N, gate = (n % BLOCK_N) / TILE_CH, j = n % TILE_CH;
    const int col = gate * kHidden + tile * TILE_CH + j;
    out[i] = kernel[((long long)tap * (2 + kHidden) + ch) * kGates + col];
  }
}
int cell_xdense_weights(const float* kernel, float* out, cudaStream_t stream) {
  MVB_REQUIRE(kernel && out, "cell_xdense_weights: bad args");
  xdense_weights_kernel<<<72, 256, 0, stream>>>(kernel, out);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

// weights of the sparse x path: rows (tap, channel) of the x block of the TF kernel [3,3,cx+256,1024], packed columns
__global__ void xsparse_weights_kernel(const float* __restrict__ kernel, int cx, float* __restrict__ out) {
  const long long total = 9ll * cx * kGates;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i % kGates);
    const long long k = i / kGates;
    const int tap = (int)(k / cx), ch = (int)(k % cx);
    const int tile = n / BLOCK_N, gate = (n % BLOCK_N) / TILE_CH, j = n % TILE_CH;
    const int col = gate * kHidden + tile * TILE_CH + j;
    out[i] = kernel[((long long)tap * (cx + kHidden) + ch) * kGates + col];
  }
}
int cell_xsparse_weights(const float* kernel, int cx, float* out, cudaStream_t stream) {
  MVB_REQUIRE(kernel && out && cx > 0, "cell_xsparse_weights: bad args");
  xsparse_weights_kernel<<<sm_count() * 4, 256, 0, stream>>>(kernel, cx, out);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

// xs_tab[s][tap][n] = sum_ch feat[frame[s]][label[s]][ch] * Wx[tap][ch][n]   (64 scene channels).
// One block per (tap, 256-column tile, sample chunk): the weight tile [64][256] sits in shared memory, thread = column.
__global__ void __launch_bounds__(256)
xsparse_table_kernel(const float* __restrict__ scene_conv, const int* __restrict__ frame_idx,
                     const int* __restrict__ label, const float* __restrict__ Wx, float* __restrict__ tab,
                     long long NS, int hw, int chunks) {
  extern __shared__ float wsm[];                      // [64][256]
  const int tap = blockIdx.x / N_TILES, nt = blockIdx.x % N_TILES;
  for (int i = threadIdx.x; i < 64 * 256; i += 256)
    wsm[i] = Wx[((long long)tap * 64 + i / 256) * kGates + nt * 256 + (i % 256)];
  __syncthreads();
  const int col = threadIdx.x;
  for (long long s = blockIdx.y; s < NS; s += chunks) {
    const int l = label[s];
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (l >= 0 && l < hw) {
      const float4* f4 = reinterpret_cast<const float4*>(scene_conv + ((long long)frame_idx[s] * hw + l) * 64);
#pragma unroll 4
      for (int c4 = 0; c4 < 16; ++c4) {
        const float4 f = __ldg(f4 + c4);              // warp-uniform
        acc[0] = fmaf(f.x, wsm[(4 * c4 + 0) * 256 + col], acc[0]);
        acc[1] = fmaf(f.y, wsm[(4 * c4 + 1) * 256 + col], acc[1]);
        acc[2] = fmaf(f.z, wsm[(4 * c4 + 2) * 256 + col], acc[2]);
        acc[3] = fmaf(f.w, wsm[(4 * c4 + 3) * 256 + col], acc[3]);
      }
    }
    tab[(s * 9 + tap) * kGates + nt * 256 + col] = (acc[0] + acc[1]) + (acc[2] + acc[3]);
  }
}
int cell_xsparse_table(const float* scene_conv, const int* frame_idx, const int* label, const float* Wx, float* tab,
                       long long NS, int H, int W, cudaStream_t stream) {
  MVB_REQUIRE(scene_conv && frame_idx && label && Wx && tab && NS > 0, "cell_xsparse_table: bad args");
  static SmemOptIn opt;
  MVB_CHECK_CUDA(smem_opt_in(opt, xsparse_table_kernel, 64 * 256 * (int)sizeof(float)));
  const int chunks = (int)(NS < 8 ? NS : 8);
  xsparse_table_kernel<<<dim3(9 * N_TILES, chunks), 256, 64 * 256 * sizeof(float), stream>>>(
      scene_conv, frame_idx, label, Wx, tab, NS, H * W, chunks);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int cell_xfold_tables(const float* kernel, const float* biases, const float* We, const float* be, int E,
                      float* Bt, float* T2, cudaStream_t stream) {
  MVB_REQUIRE(kernel && biases && We && be && Bt && T2 && E > 0, "cell_xfold_tables: bad args");
  xfold_tables_kernel<<<234, 256, 0, stream>>>(kernel, biases, We, be, E, Bt, T2);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

// variant of the last launch_cell() of this process: planes code * 2 + multicast (tests assert which kernel ran)
static int g_last_variant = -1;
static unsigned long long g_variants_seen = 0;      // bit (format * 2 + pair): format 0 bf16x2, 1 f16f8
int cell_last_variant() { return g_last_variant; }
unsigned long long cell_variants_seen(int reset) {
  const unsigned long long v = g_variants_seen;
  if (reset) g_variants_seen = 0;
  return v;
}
static void note_variant(int fmt, int pair) {
  g_last_variant = (fmt ? kPlanesF16F8 : kBf16Planes) * 2 + pair;
  g_variants_seen |= 1ull << (fmt * 2 + pair);
}

#ifdef MVB_CELL_PROBE
static CellRing g_probe_ring = {};
// Phase profile of the cell launches since the last reset (probe build only, not part of the public header):
// out[kProbePhases] in CellProbePhase order, then weight slots, A stages and A stage bytes of the last launch.
extern "C" int mvb_cell_probe(unsigned long long* out, int reset) {
  MVB_CHECK_CUDA(cudaDeviceSynchronize());
  MVB_CHECK_CUDA(cudaMemcpyFromSymbol(out, g_cell_probe, sizeof(g_cell_probe)));
  out[kProbePhases] = g_probe_ring.b_slots;
  out[kProbePhases + 1] = g_probe_ring.a_stages;
  out[kProbePhases + 2] = g_probe_ring.a_stage_bytes;
  if (reset) {
    const unsigned long long zero[kProbePhases] = {};
    MVB_CHECK_CUDA(cudaMemcpyToSymbol(g_cell_probe, zero, sizeof(zero)));
  }
  return MVB_OK;
}
#endif

// A, B, Bh: 16-bit (bf16x2 planes, or the fp16 region of f16f8) activation rows, weight tiles of 256 rows, halves of
// them (CTA pairs); A8, B8, B8h: the same over the e4m3 region.  f16f8 only: Bq / B8q the four 32-row gate groups of
// an N tile of cell_fwd_epi_kernel, Bqh / B8qh two of them (CTA pairs).
struct CellMaps { CUtensorMap A, B, Bh, A8, B8, B8h, Bq, Bqh, B8q, B8qh; };

// Work order of a launch (CellParams::order, work_index()).  1: the four N tiles of an M tile (pair) run back to back
// on the same CTA (pair), so the tile's operand rows are re-read from L2 by the SM that fetched them.
// 0: work items strided over the CTAs.  A launch of few M tiles (the encoders and the greedy decoders of a small
// shard: 32 trajectories of 36x18 = 176 M tiles on 132 CTAs) is bound by its longest CTA instead: back to back the
// busiest CTA runs 2 x 4 items, strided ceil(704 / 132) = 6.  Strided whenever that makespan is shorter and the
// launch is small enough for its operands to stay in L2.
static int pick_order(int forced, long long units, long long ctas, int n_tiles) {
  if (forced == 0 || forced == 1) return forced;
  const long long back_to_back = ((units + ctas - 1) / ctas) * n_tiles, strided = (units * n_tiles + ctas - 1) / ctas;
  return (strided < back_to_back && units < 4 * ctas) ? 0 : 1;
}

// cell_fwd_epi_kernel (f16f8): the same choice of pair or single-CTA kernel and of work order as launch_cell
static int launch_cell_epi(const CellMaps& tm, const CellParams& prm_in, int num_sms, bool multicast,
                           cudaStream_t stream) {
  CellParams prm = prm_in;
  static SmemOptIn opt_plain, opt_mc;
  const int ra8 = (BLOCK_M + 2 * (prm.W + 2) + 7) & ~7;
  prm.ring = CellEpiCfg::ring(ra8);
  const int smem_bytes = CellEpiCfg::smem_bytes(prm.ring);
  MVB_REQUIRE(ra8 <= CellCfg<1>::MAX_RA8 && smem_bytes <= kSmemLimit && prm.ring.b_slots >= 2,
              "cell_fwd: grid width W=%d too large (A stage of %d rows: %d weight slots, %d B shared memory)",
              prm.W, ra8, prm.ring.b_slots, smem_bytes);
  CELL_PROBE(g_probe_ring = prm.ring;)
  MVB_CHECK_CUDA(smem_opt_in(opt_plain, cell_fwd_epi_kernel<false>, smem_bytes));
  MVB_CHECK_CUDA(smem_opt_in(opt_mc, cell_fwd_epi_kernel<true>, smem_bytes));
  const long long m_tiles = (prm.R + BLOCK_M - 1) / BLOCK_M;
  if (multicast && m_tiles >= 2 * (long long)num_sms) {
    prm.order = pick_order(prm_in.order, (m_tiles + 1) / 2, num_sms / 2, EW_N_TILES);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(num_sms / 2 * 2)); cfg.blockDim = dim3(EW_THREADS);
    cfg.dynamicSmemBytes = smem_bytes; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    MVB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, cell_fwd_epi_kernel<true>, tm.A, tm.Bqh, tm.A8, tm.B8qh, prm));
    count_launch(1);
    note_variant(1, 1);
    return MVB_OK;
  }
  const long long num_tiles = m_tiles * EW_N_TILES;
  const int grid = (int)(num_tiles < num_sms ? num_tiles : num_sms);
  prm.order = pick_order(prm_in.order, m_tiles, grid, EW_N_TILES);
  cell_fwd_epi_kernel<false><<<grid, EW_THREADS, smem_bytes, stream>>>(tm.A, tm.Bq, tm.A8, tm.B8q, prm);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  note_variant(1, 0);
  return MVB_OK;
}

// cell_fwd_epi_kernel runs f16f8 launches of at least this many M tiles per SM (the K=20 beam steps: over 400).  On
// the H100 it is 5 % faster there, but slower on launches of a few M tiles per SM (the greedy decoders of c3: 3 - 11),
// where each CTA's first and last tiles - its pipeline fill and the epilogue of its last tile, which nothing hides -
// weigh more.
constexpr long long kEpiWgMinTilesPerSm = 64;

template <int FMT>
static int launch_cell(const CellMaps& tm, const CellParams& prm_in, int num_sms, bool multicast, int epi_wg,
                       cudaStream_t stream) {
  CellParams prm = prm_in;
  static SmemOptIn opt_plain, opt_mc;
  // MVB_CELL_FORMAT_RINGS=0: f16f8 launches use the bf16x2 rings (two-plane A stages, 4 or 3 weight slots), the
  // layout before the rings were sized per format, for A/B runs; the results are bit-identical either way
  static const bool format_rings = [] { const char* e = getenv("MVB_CELL_FORMAT_RINGS"); return !(e && e[0] == '0'); }();
  if (FMT == 1 && (epi_wg == 1 || (epi_wg == 2 && (prm.R + BLOCK_M - 1) / BLOCK_M >= kEpiWgMinTilesPerSm * num_sms)))
    return launch_cell_epi(tm, prm, num_sms, multicast, stream);
  const int ra8 = (BLOCK_M + 2 * (prm.W + 2) + 7) & ~7;
  prm.ring = format_rings ? CellCfg<FMT>::ring(ra8) : CellCfg<0>::ring(ra8);
  const int smem_bytes = prm.ring.smem_bytes();
  MVB_REQUIRE(ra8 <= CellCfg<FMT>::MAX_RA8 && smem_bytes <= kSmemLimit && prm.ring.b_slots >= 2 &&
              prm.ring.b_slots <= kMaxBSlots && prm.ring.a_stages >= 2 && prm.ring.a_stages <= kMaxAStages,
              "cell_fwd: grid width W=%d too large (A stage of %d rows: %d weight slots, %d A stages, %d B shared memory)",
              prm.W, ra8, prm.ring.b_slots, prm.ring.a_stages, smem_bytes);
  CELL_PROBE(g_probe_ring = prm.ring;)
  MVB_CHECK_CUDA(smem_opt_in(opt_plain, cell_fwd_kernel<false, FMT>, smem_bytes));
  MVB_CHECK_CUDA(smem_opt_in(opt_mc, cell_fwd_kernel<true, FMT>, smem_bytes));
  const long long m_tiles = (prm.R + BLOCK_M - 1) / BLOCK_M;
  if (multicast && m_tiles >= 2 * (long long)num_sms) {
    prm.order = pick_order(prm_in.order, (m_tiles + 1) / 2, num_sms / 2, N_TILES);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(num_sms / 2 * 2)); cfg.blockDim = dim3(NUM_THREADS);
    cfg.dynamicSmemBytes = smem_bytes; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    MVB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, cell_fwd_kernel<true, FMT>, tm.A, tm.Bh, tm.A8, tm.B8h, prm));
    count_launch(1);
    note_variant(FMT, 1);
    return MVB_OK;
  }
  const long long num_tiles = m_tiles * N_TILES;
  const int grid = (int)(num_tiles < num_sms ? num_tiles : num_sms);
  prm.order = pick_order(prm_in.order, m_tiles, grid, N_TILES);
  cell_fwd_kernel<false, FMT><<<grid, NUM_THREADS, smem_bytes, stream>>>(tm.A, tm.B, tm.A8, tm.B8, prm);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  note_variant(FMT, 0);
  return MVB_OK;
}

// fan-out stage 2: every parent row -> its K children (c_out / h32_out hold NS * fanout sample rows)
static int fanout_children(const CellStep& s, const float* col_scale, const Grid& g, cudaStream_t stream) {
  const unsigned blocks = (unsigned)((s.NS * g.H * g.W * 32 + 255) / 256);      // a warp per parent cell
  auto children = col_scale ? fanout_children_kernel<1> : fanout_children_kernel<0>;
  children<<<blocks, 256, 0, stream>>>(s.fanout_ws, col_scale, s.xf_B, s.xf_T2, s.xf_ids, s.c_in, s.c_out, s.h32_out,
                                       s.NS, s.fanout, g, s.forget_bias);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

int cell_fwd(const CellStep& s, cudaStream_t stream) {
  const int P = s.planes & 0xFF, P_out = (s.planes >> 8) ? (s.planes >> 8) : P;
  MVB_REQUIRE(valid_planes(P) && valid_planes(P_out), "cell_fwd: planes P=%d (output planes %d) not 2 or %d", P, P_out,
              kPlanesF16F8);
  const bool mixed = P == kPlanesF16F8, fan = s.fanout > 1 || (s.fanout == 1 && !s.xh);
  const bool children_only = fan && !s.xh;     // the accumulators of these parents are in fanout_ws already
  const int x_sources = !!s.xf_B + !!s.xs_tab + !!s.xr_W;
  const long long NS = s.NS; const int H = s.H, W = s.W, cpad = s.cpad;
  MVB_REQUIRE(!mixed || !s.gates_out, "cell_fwd: the f16f8 format is an inference format (no gates_out)");
  MVB_REQUIRE(x_sources <= 1, "cell_fwd: at most one x source (x-fold, sparse or dense x)");
  MVB_REQUIRE(!s.row_map || !(s.xs_tab || s.xr_W), "cell_fwd: a row map goes with the x-fold tables or no x source");
  MVB_REQUIRE(!fan || (s.xf_B && s.c_in && s.h32_out && s.fanout_ws && !s.row_map && !s.hp_out),
              "cell_fwd: fanout=%d needs the x-fold tables, c_in, h32_out, a [R,1024] fp32 workspace and no row_map / hp_out", s.fanout);
  MVB_REQUIRE(!s.xf_B || (s.xf_T2 && s.xf_ids && H >= 3 && W >= 3), "cell_fwd: x-fold needs its tables, ids and a grid of at least 3x3");
  MVB_REQUIRE((!s.xs_tab || s.xs_label) && (!s.xr_W || s.xr_in), "cell_fwd: the sparse x path needs its labels, the dense one its input");
  MVB_REQUIRE(cpad % XPAD == 0 && cpad >= kHidden + XPAD && cpad <= kHidden + kMaxXBlock,
              "cell_fwd: cpad=%d must be a multiple of %d from %d to %d (x block of 32 to %d channels)", cpad, XPAD,
              kHidden + XPAD, kHidden + kMaxXBlock, kMaxXBlock);
  MVB_REQUIRE(!s.tiles || (s.tile_count && !fan), "cell_fwd: a work list needs its count and no fan-out");
  MVB_REQUIRE(NS > 0 && H > 0 && W > 0, "cell_fwd: bad sizes NS=%lld H=%d W=%d", NS, H, W);
  MVB_REQUIRE((s.xh || children_only) && s.w && (s.bias || s.xf_B) && s.c_out, "cell_fwd: null pointer");
  if (s.hp_out) MVB_REQUIRE(s.cpad_out % 8 == 0 && s.ch_off_out % 8 == 0, "cell_fwd: hp_out pitch/offset must be multiples of 8");
  const Grid g = make_grid(H, W);
  const long long R = NS * g.S;
  MVB_REQUIRE(R + 2LL * g.Wp + 256 < 0x7fffffffLL, "cell_fwd: too many rows (%lld) for int32 TMA coordinates", R);

  // weight-tile multicast across CTA pairs is on by default (MVB_CELL_MULTICAST=0 turns it off for A/B runs)
  static const bool multicast = [] { const char* e = getenv("MVB_CELL_MULTICAST"); return !(e && e[0] == '0'); }();
  // Large f16f8 launches run cell_fwd_epi_kernel (an epilogue warpgroup, kEpiWgMinTilesPerSm).  For A/B runs,
  // MVB_CELL_EPI_WG=1 runs it for every f16f8 launch, MVB_CELL_EPI_WG=0 (or MVB_CELL_FORMAT_RINGS=0) for none; the
  // results are bit-identical either way.  0: never, 1: always, 2: by size
  static const int epi_wg = [] {
    const char* e = getenv("MVB_CELL_EPI_WG"), *r = getenv("MVB_CELL_FORMAT_RINGS");
    if ((e && e[0] == '0') || (r && r[0] == '0')) return 0;
    return (e && e[0] == '1') ? 1 : 2;
  }();
  if (children_only) {
    const float* col_scale = mixed ? reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(s.w) +
                                                                    4ull * kGates * 9 * cpad) : nullptr;
    return fanout_children(s, col_scale, g, stream);
  }
  CellMaps tm;
  const int P16 = mixed ? 1 : kBf16Planes;      // 16-bit "planes" the A / B maps describe
  const uint32_t ra8 = (uint32_t)((BLOCK_M + 2 * (W + 2) + 7) & ~7);      // rows of an A stage (see CellCfg)
  MVB_REQUIRE(ra8 <= 256, "cell_fwd: grid width W=%d too large for the halo'd A stage (%u rows > 256)", W, ra8);
  int rc = encode_tmap_3d_bf16(&tm.A, s.xh, (uint64_t)cpad, (uint64_t)R, (uint64_t)P16,
                               (uint64_t)cpad * 2, (uint64_t)R * cpad * 2, CHUNK, ra8, P16, 128);
  if (rc) return rc;
  const uint64_t ktot = 9ull * cpad;
  rc = encode_tmap_3d_bf16(&tm.B, s.w, ktot, (uint64_t)kGates, (uint64_t)P16, ktot * 2,
                           ktot * kGates * 2, CHUNK, BLOCK_N, 1, 128);          // one plane of a tile = one slot
  if (rc) return rc;
  rc = encode_tmap_3d_bf16(&tm.Bh, s.w, ktot, (uint64_t)kGates, (uint64_t)P16, ktot * 2,
                           ktot * kGates * 2, CHUNK, BLOCK_N / 2, 1, 128);      // half of it (CTA pairs)
  if (rc) return rc;
  tm.A8 = tm.A; tm.B8 = tm.B; tm.B8h = tm.Bh;
  const float* col_scale = nullptr;
  if (mixed) {
    // [fp16 region][fp8 region: rows of 2*cpad bytes, both e4m3 planes interleaved per chunk (f8_off)]
    // ([+ 1024 fp32 column scales] after the weights)
    const uint8_t* a8 = reinterpret_cast<const uint8_t*>(s.xh) + 2ull * R * cpad;
    const uint8_t* b8 = reinterpret_cast<const uint8_t*>(s.w) + 2ull * kGates * ktot;
    rc = encode_tmap_3d_u8(&tm.A8, a8, 2ull * cpad, (uint64_t)R, 1, 2ull * cpad, 2ull * R * cpad, ROW_BYTES, ra8, 1, 128);
    if (rc) return rc;
    rc = encode_tmap_3d_u8(&tm.B8, b8, 2 * ktot, (uint64_t)kGates, 1, 2 * ktot, 2 * ktot * kGates, ROW_BYTES, BLOCK_N, 1, 128);
    if (rc) return rc;
    rc = encode_tmap_3d_u8(&tm.B8h, b8, 2 * ktot, (uint64_t)kGates, 1, 2 * ktot, 2 * ktot * kGates, ROW_BYTES, BLOCK_N / 2, 1, 128);
    if (rc) return rc;
    col_scale = reinterpret_cast<const float*>(b8 + 2ull * kGates * ktot);
  }
  if (mixed && epi_wg) {
    const uint8_t* b8 = reinterpret_cast<const uint8_t*>(s.w) + 2ull * kGates * ktot;
    // cell_fwd_epi_kernel: weight rows as [32 rows][2 halves][16 (256-column tile, gate)], a box of 32 rows x 1 half
    // x 4 gates (2 for each CTA of a pair) is one N tile of 128 columns
    const uint64_t d16[4] = {ktot, 32, 2, 16}, s16[3] = {ktot * 2, 32 * ktot * 2, 64 * ktot * 2};
    const uint64_t d8[4] = {2 * ktot, 32, 2, 16}, s8[3] = {2 * ktot, 32 * 2 * ktot, 64 * 2 * ktot};
    const uint32_t q16[4] = {CHUNK, 32, 1, 4}, q16h[4] = {CHUNK, 32, 1, 2};
    const uint32_t q8[4] = {ROW_BYTES, 32, 1, 4}, q8h[4] = {ROW_BYTES, 32, 1, 2};
    if ((rc = encode_tmap_4d_bf16(&tm.Bq, s.w, d16, s16, q16, 128))) return rc;
    if ((rc = encode_tmap_4d_bf16(&tm.Bqh, s.w, d16, s16, q16h, 128))) return rc;
    if ((rc = encode_tmap_4d_u8(&tm.B8q, b8, d8, s8, q8, 128))) return rc;
    if ((rc = encode_tmap_4d_u8(&tm.B8qh, b8, d8, s8, q8h, 128))) return rc;
  }

  CellParams prm;
  prm.bias = s.bias; prm.col_scale = col_scale; prm.c_in = s.c_in; prm.row_map = s.row_map; prm.c_out = s.c_out;
  prm.h32_out = s.h32_out; prm.gates_out = s.gates_out;
  prm.preact_out = fan ? s.fanout_ws : nullptr;      // fan-out: stage 1 stores the raw accumulators there
  prm.xf_B = s.xf_B; prm.xf_T2 = s.xf_T2; prm.xf_ids = s.xf_ids;
  prm.xs_tab = s.xs_tab; prm.xs_label = s.xs_label; prm.xr_in = s.xr_in; prm.xr_W = s.xr_W;
  prm.skip_x = x_sources;      // an x source replaces the x chunk of the K loop
  // work order: chosen per launch in launch_cell (MVB_CELL_ORDER=0|1 forces one)
  static const int order = [] { const char* e = getenv("MVB_CELL_ORDER"); return e ? atoi(e) : -1; }();
  prm.order = order;
  prm.hp_mixed = P_out == kPlanesF16F8;
  prm.hp_out = reinterpret_cast<__nv_bfloat16*>(s.hp_out);
  prm.hp_plane_stride = s.hp_plane_stride; prm.cpad_out = s.cpad_out; prm.ch_off_out = s.ch_off_out;
  prm.R = R; prm.H = H; prm.W = W; prm.cpad = cpad; prm.forget_bias = s.forget_bias;
  prm.tiles = s.tiles; prm.tile_count = s.tile_count;

  int dev = 0, num_sms = 0;
  MVB_CHECK_CUDA(cudaGetDevice(&dev));
  MVB_CHECK_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
  rc = mixed ? launch_cell<1>(tm, prm, num_sms, multicast, epi_wg, stream)
             : launch_cell<0>(tm, prm, num_sms, multicast, 0, stream);
  if (rc || !fan) return rc;
  return fanout_children(s, col_scale, g, stream);
}

// ----------------------------------------------------------------------------------
// f16f8 weight packing (see mvb_common.cuh): per packed column n a power-of-two scale 2^S with
// max|w| * 2^S in [2^13, 2^14), so that b0 = fp16(w 2^S) is a normal number for every weight down to 2^-27 of the
// column maximum, the residual b1 = w 2^S - b0 (|b1| <= 4) and b0 2^-12 (<= 4) sit in e4m3's normal range.
//   w16 [1024][9*cpad] fp16 = b0;  w8 [1024][9][2*cpad bytes] = e4m3(b1) and e4m3(b0 * 2^-12), interleaved per chunk
//   like the activation rows (f8_off);  col_scale [1024] = 2^-S
// ----------------------------------------------------------------------------------
__device__ __forceinline__ float packed_weight(const float* __restrict__ kernel, int n, int k, int cx, int cxp,
                                               int cpad) {
  const int tap = k / cpad, kcn = k - tap * cpad;
  const int tile = n / BLOCK_N, gate = (n % BLOCK_N) / TILE_CH, j = n % TILE_CH;
  const int col = gate * kHidden + tile * TILE_CH + j;
  int cin = -1;
  if (kcn >= cxp) cin = cx + (kcn - cxp);
  else if (kcn < cx) cin = kcn;
  return (cin >= 0) ? kernel[((long long)tap * (cx + kHidden) + cin) * kGates + col] : 0.f;
}

__global__ void colscale_kernel(const float* __restrict__ kernel, float* __restrict__ col_scale, int cx) {
  // one warp per packed column: max |w| over the 9 * (cx + 256) weights that feed it
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (n >= kGates) return;
  const int tile = n / BLOCK_N, gate = (n % BLOCK_N) / TILE_CH, j = n % TILE_CH;
  const int col = gate * kHidden + tile * TILE_CH + j;
  float m = 0.f;
  for (int r = lane; r < 9 * (cx + kHidden); r += 32) m = fmaxf(m, fabsf(kernel[(long long)r * kGates + col]));
  m = warp_max(m);
  if (lane == 0) {
    int e = 0;
    if (m > 0.f) frexpf(m, &e);            // m = f * 2^e, f in [0.5, 1)  ->  floor(log2 m) = e - 1
    const int S = m > 0.f ? 13 - (e - 1) : 0;
    col_scale[n] = ldexpf(1.0f, -S);
  }
}

__global__ void pack_weights_f16f8_kernel(const float* __restrict__ kernel, const float* __restrict__ biases,
                                          __half* __restrict__ w16, uint8_t* __restrict__ w8,
                                          const float* __restrict__ col_scale, float* __restrict__ bias_packed,
                                          int cx, int cxp, int cpad) {
  const long long ktot = 9LL * cpad;
  const long long total = (long long)kGates * ktot;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i / ktot);
    const int k = (int)(i - (long long)n * ktot);
    const float v = packed_weight(kernel, n, k, cx, cxp, cpad) / col_scale[n];     // exact: power of two
    const __half b0 = __float2half_rn(v);
    const float f0 = __half2float(b0);
    w16[i] = b0;
    const int tap = k / cpad, kcn = k - tap * cpad;
    uint8_t* w8row = w8 + ((long long)n * 9 + tap) * 2 * cpad;
    w8row[f8_off(kcn, 0, cpad)] = to_e4m3(v - f0);
    w8row[f8_off(kcn, 1, cpad)] = to_e4m3(f0 * (1.0f / kF8ResidualScale));
    if (k == 0) {
      const int tile = n / BLOCK_N, gate = (n % BLOCK_N) / TILE_CH, j = n % TILE_CH;
      bias_packed[n] = biases[gate * kHidden + tile * TILE_CH + j];
    }
  }
}


int pack_cell_weights(const float* kernel, const float* biases, void* w_planes, float* bias_packed,
                      int cx, int P, int comp, cudaStream_t stream) {
  MVB_REQUIRE(valid_planes(P), "pack_cell_weights: planes P=%d not 2 or %d", P, kPlanesF16F8);
  MVB_REQUIRE(cx >= 1, "pack_cell_weights: cx=%d", cx);
  const int cxp = (cx + XPAD - 1) / XPAD * XPAD;
  const int cpad = cxp + kHidden;
  if (P == kPlanesF16F8) {
    MVB_REQUIRE(!comp, "pack_cell_weights: the compensated x block exists for bf16 planes only");
    const long long total = (long long)kGates * 9 * cpad;
    __half* w16 = reinterpret_cast<__half*>(w_planes);
    uint8_t* w8 = reinterpret_cast<uint8_t*>(w_planes) + 2 * total;
    float* col_scale = reinterpret_cast<float*>(w8 + 2 * total);
    colscale_kernel<<<kGates / 8, 256, 0, stream>>>(kernel, col_scale, cx);
    pack_weights_f16f8_kernel<<<1184, 256, 0, stream>>>(kernel, biases, w16, w8, col_scale, bias_packed, cx, cxp, cpad);
    MVB_CHECK_CUDA(cudaGetLastError());
    count_launch(2);
    return MVB_OK;
  }
  MVB_REQUIRE(!comp || 4 * cx <= cxp, "pack_cell_weights: compensated x block needs 4*cx <= %d", cxp);
  pack_weights_kernel<<<1184, 256, 0, stream>>>(kernel, biases, reinterpret_cast<__nv_bfloat16*>(w_planes), bias_packed,
                                                cx, cxp, cpad, comp);
  MVB_CHECK_CUDA(cudaGetLastError());
  count_launch(1);
  return MVB_OK;
}

}  // namespace mvb
