/* coda_b200 -- C ABI of the CUDA-native CODA acquisition hot path (H100, sm_90a).
 *
 * Drop-in boundary (SURVEY.md 8b).  The reference (justinkay/coda) is pure Python/PyTorch
 * and has no FFI of its own; these entry points are what a ctypes binding inside
 * coda/coda.py would call in place of the ATen op chains on the acquisition path.  Each
 * declaration cites the reference lines it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host or the comment says "host struct";
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued, nothing synchronises;
 *   - return value: CODA_B200_OK or a negative error code, message via coda_b200_last_error();
 *   - numerical problems are reported through a device-side `flags` word (bits below) that the
 *     caller reads at its next host sync -- the reference raises RuntimeError('[NUMERIC ERROR]')
 *     from coda/util.py:17-25 at the same places;
 *   - layouts: preds [H][N][C] fp32 (coda/datasets.py:14), models `model_stride` floats apart (N*C when the
 *     shard is its own tensor; the full-task stride when it is an N-range view of a bigger slab);
 *     D (dirichlets) [H][C][C] fp32; U (un-normalised pi_hat_xi) [N][C] fp32; hard [N][H] u16;
 *     Hp = H rounded up to 32;
 *   - "rows": one row = one hypothetical (item, class) update.  Rows [0, T), T = C*(1+H), are the template rows
 *     (class-major: c*(1+H) + 0 = no model predicts c, + 1 + h = only model h predicts c); rows [T, T + n_heavy) are
 *     the heavy rows (two or more models predict the class), ITEM-major: the heavy rows of item n are
 *     T + heavy_off[n] .. T + heavy_off[n+1] - 1 in ascending class order;
 *   - built for sm_90a only.
 */
#ifndef CODA_B200_H
#define CODA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CODA_B200_VERSION 203
#define CODA_B200_NODES 256 /* quadrature nodes, coda/coda.py:79 */
#define CODA_B200_MAX_WORLD 16
#define CODA_B200_REC_WORDS 8 /* arg-max record: {bits vA, iA, cntA, bits vB, iB, bits v2A, bits v2B, 0} */

#define CODA_B200_OK 0
#define CODA_B200_EINVAL (-1)
#define CODA_B200_ECUDA (-2)

/* device-side flag bits */
#define CODA_B200_FLAG_NONFINITE_INPUT 0x01u /* NaN/Inf in preds */
#define CODA_B200_FLAG_RANGE_INPUT 0x02u     /* preds outside [0, 1]: not post-softmax scores */
#define CODA_B200_FLAG_NONFINITE_TABLE 0x04u /* util._check(pdf/cdf/integrand), coda.py:96-112 */
#define CODA_B200_FLAG_NONFINITE_PI 0x08u    /* pi_hat_xi row sum not finite */
#define CODA_B200_FLAG_NONFINITE_PBEST 0x10u /* util._check(pbest), coda.py:330 */
#define CODA_B200_FLAG_NONFINITE_EIG 0x20u   /* util._check(Pbest(beta) normalized), coda.py:115 */
#define CODA_B200_FLAG_NO_CANDIDATE 0x40u    /* the host-free loop ran out of unlabeled items */
#define CODA_B200_FLAG_XCHG_TIMEOUT 0x80u    /* a peer never arrived at an exchange (2 s) */
#define CODA_B200_FLAG_NEGATIVE_PROB 0x100u  /* util._check_prob: probability < -1e-12 (util.py:33-35) */
#define CODA_B200_FLAG_ROWSUM_WARN 0x200u    /* util._check_prob: |row sum - 1| > 1e-4 (util.py:37-39), a warning */
#define CODA_B200_FLAG_PIPELINE_TIMEOUT 0x400u /* a TMA / tensor-core pipeline stopped (pi_full_tc); the result is invalid */
#define CODA_B200_FLAG_PREDRAW_MISMATCH 0x800u /* a CODA ablation step found a candidate count the host did not predict */

typedef void* coda_stream_t;

/* ---- plumbing ---------------------------------------------------------------------- */
const char* coda_b200_last_error(void);
int coda_b200_version(void);
int coda_b200_sm_count(void);
int coda_b200_device_check(void); /* fails loudly when no sm_90 device is present */
/* cudaLimitMaxL2FetchGranularity hint (32/64/128 B) for the sector-gather kernels (per device). */
int coda_b200_set_l2_fetch_granularity(int bytes);

/* ---- N-axis shards: peer-memory exchange (SURVEY.md 8e; no reference counterpart) ------------------
 * Every shard owns a mailbox in its own HBM.  The two per-step exchanges (arg-max record, marginal sums) are
 * done INSIDE the step kernels: a rank stores its contribution straight into every peer's mailbox over
 * NVLink (P2P stores), releases a flag with system scope, and spins on its own mailbox until every peer's
 * contribution of the same epoch has landed.  Slots are double-buffered by epoch parity.  The mailbox is
 * reached through CUDA IPC (one process per GPU, torchrun) or plain peer access (one process driving all GPUs). */
typedef struct coda_xchg { /* host struct */
  int world, rank;
  void* box[CODA_B200_MAX_WORLD]; /* mailbox of every rank as addressable from THIS rank's device; box[rank] is local */
  uint64_t* epoch;                /* local, [8], zero-initialised: per-channel epoch counters [0..4) and the nanoseconds
                                     spent waiting for peers per channel [4..8) (latency + skew; bench.py prints them) */
  int H, C, rep_words;            /* fix the slot sizes (same on every rank); rep_words: int64 words of a report block */
} coda_xchg_t;
size_t coda_b200_xchg_box_bytes(int world, int H, int C, int rep_words);
int coda_b200_xchg_alloc(size_t bytes, void** box_out); /* cudaMalloc + zero fill on the current device */
int coda_b200_xchg_free(void* box);
int coda_b200_ipc_export(const void* box, void* handle64_host);
int coda_b200_ipc_open(const void* handle64_host, void** box_out);
int coda_b200_ipc_close(void* box);
int coda_b200_peer_enable(int peer_device); /* current device may load/store peer_device's memory */

/* ---- construction (coda/coda.py:172-203) --------------------------------------------- */

/* One pass over the slab: per-model argmax (coda.py:217, 263, 316), ensemble-mean pseudo
 * label (coda/util.py:13-14 + coda.py:193-194), unanimity bit (coda.py:215-219).
 * ens_out (optional) [N][C]: E[n][c] = sum_h preds[h][n][c], the un-normalised ensemble of coda/util.py:13-14.
 * Also util._check_prob (util.py:28-39) on the input: negatives, non-finite values, row sums. */
int coda_b200_scan_slab(const float* preds, int64_t model_stride, int H, int64_t N, int C, uint16_t* hard,
                        int32_t* pseudo, uint8_t* disagree, float* ens_out, uint32_t* flags, coda_stream_t stream);

/* Soft confusion sums, coda.py:42 einsum('nc,hnj->hcj').  conf_fx [H][C][C] int64 fixed point
 * (value * 2^fx_shift), ACCUMULATED into; exact and order-independent so shards can be summed. */
int coda_b200_confusion_accum(const float* preds, int64_t model_stride, const int32_t* pseudo, int H, int64_t N,
                              int C, int fx_shift, int64_t* conf_fx, coda_stream_t stream);

/* Same sums with the items visited in pseudo-label order (`order` = any permutation that groups equal
 * pseudo labels; C <= 128): register accumulation, no shared-memory atomics.  Bit-identical result. */
int coda_b200_confusion_sorted(const float* preds, int64_t model_stride, const int32_t* pseudo,
                               const int32_t* order, int H, int64_t N, int C, int fx_shift, int64_t* conf_fx,
                               coda_stream_t stream);

/* Row-normalise (coda.py:43) and build the Dirichlet prior (coda.py:46-63, 196). */
/* conf_rest (optional, compact slab): [H][C] sums every column of row (h, c) carries in addition (see below). */
int coda_b200_init_dirichlets(const int64_t* conf_fx, const int64_t* conf_rest, int H, int C, int fx_shift,
                              double prior_strength, double multiplier, int uniform_prior, float* D,
                              coda_stream_t stream);

/* ---- consensus marginals (CODA.update_pi_hat, coda.py:226-233) ------------------------ */

/* U[n][c] = sum_h sum_s D[h][c][s] preds[h][n][s]  (coda.py:227-229, `adjusted` never stored). */
int coda_b200_pi_full(const float* preds, int64_t model_stride, const float* D, int H, int64_t N, int C, float* U,
                      coda_stream_t stream);

/* The same contraction on the tensor cores (wgmma, register accumulators, bulk-TMA slab stream): both operands are cut
 * into two fp16 limbs, 3 MMAs per K = 16 chunk, accumulators folded into fp32 registers every 4 models (pi_tc.cu).
 * Usable when pi_full_tc_ok(...) != 0 (16 <= C <= 128, C % 4 == 0, model_stride % 4 == 0); `scratch` =
 * pi_full_tc_scratch_bytes(H, C) bytes (the D limbs).  A stopped pipeline sets CODA_B200_FLAG_PIPELINE_TIMEOUT. */
int coda_b200_pi_full_tc_ok(int H, int64_t N, int C, int64_t model_stride);
size_t coda_b200_pi_full_tc_scratch_bytes(int H, int C);
int coda_b200_pi_full_tc(const float* preds, int64_t model_stride, const float* D, int H, int64_t N, int C, float* U,
                         void* scratch, uint32_t* flags, coda_stream_t stream);

/* Row-normalise with the 1e-12 clamp (coda.py:230) and accumulate sum_n pi_hat_xi[n][:]
 * (coda.py:232) into pisum_fx [C] (int64 fixed point, ACCUMULATED).  xi_out may be NULL. */
int coda_b200_pi_reduce(float* U, int64_t N, int C, int fx_shift, float* xi_out, int64_t* pisum_fx, uint32_t* flags,
                        coda_stream_t stream);

/* Optional class-major shadow copy T[s][c][n] = preds[model_of_slot[s]][n][c] for S of the H models (no
 * reference counterpart: a layout for the one-float-per-(model, item) gather of the rank-1 refresh).
 * Columns are `col_stride` floats apart (>= N, a multiple of 4 so that every column is 16-byte aligned). */
int coda_b200_shadow_build(const float* preds, int64_t model_stride, int H, int64_t N, int C,
                           const int32_t* model_of_slot, int S, int64_t col_stride, float* T, coda_stream_t stream);

/* update_pi_hat after the rank-1 change of D (coda.py:319): U[n][t] += lr * sum_h preds[h][n][jvec[h]],
 * then the same normalise + column sums as pi_reduce.  The gather list (`terms`, written by the step kernels
 * below) is {nterms, majority class t' or -1} followed by nterms x {element offset, sign, item stride}: with the
 * ensemble sums E the sum over models is taken as E[n][t'] + corrections for the models that disagree with the
 * majority class t' of jvec (exact algebra, fewer gathers); E[n][t'] is the first term of the list (from the
 * shadow's class-major ensemble slot, else from the item-major ens), models with a shadow slot are read from the
 * shadow.  `ens` is not read here: the list addresses the ensemble sums itself.
 * pisum_fx was zeroed by the step kernel and is accumulated into (this shard's sums).  ctas_per_sm (1..8)
 * bounds the grid so a concurrent stream keeps SM resources.  U must be 16-byte aligned and followed by 16
 * readable bytes (C <= 128 takes a bulk-TMA pipeline that rounds the last tile's copy up). */
/* const_slot: >= 0 = the caller owns that slot of the per-device constant-memory term table (slots hold 2H terms
 * rounded up to 64; floor(3584 / that) slots exist; no two streams of one process may use the same slot of the same
 * device concurrently) -- the gather list is then read through the constant cache; -1 = shared-memory copy. */
int coda_b200_pi_rank1(const float* preds, const float* ens, int H, int64_t N, int C, const int64_t* sel, double lr,
                       int fx_shift, const int32_t* terms, float* U, int64_t* pisum_fx, uint32_t* flags,
                       int ctas_per_sm, int const_slot, coda_stream_t stream);

/* ---- 16-bit prediction slabs (the reference stores its task tensors in half precision and widens them on load,
 *      coda/datasets.py:14) -----------------------------------------------------------------------------------------
 * The _x entry points take `preds` as an untyped pointer plus its element type.  Every kernel widens the value to
 * fp32 at the load and keeps the fp32 arithmetic in the same order, so a 16-bit slab gives exactly the bits of the
 * fp32 entry points run on its fp32 widening; CODA_B200_SLAB_F32 runs the fp32 entry points' code.  Strides, offsets
 * and the shadow column stride count slab ELEMENTS. */
#define CODA_B200_SLAB_F32 0
#define CODA_B200_SLAB_F16 1
#define CODA_B200_SLAB_BF16 2
/* coda.py:193-194, 215-219, 263, 316 (see coda_b200_scan_slab) */
int coda_b200_scan_slab_x(const void* preds, int fmt, int64_t model_stride, int H, int64_t N, int C, uint16_t* hard,
                          int32_t* pseudo, uint8_t* disagree, float* ens_out, uint32_t* flags, coda_stream_t stream);
/* coda.py:42 (see coda_b200_confusion_accum / coda_b200_confusion_sorted) */
int coda_b200_confusion_accum_x(const void* preds, int fmt, int64_t model_stride, const int32_t* pseudo, int H,
                                int64_t N, int C, int fx_shift, int64_t* conf_fx, coda_stream_t stream);
int coda_b200_confusion_sorted_x(const void* preds, int fmt, int64_t model_stride, const int32_t* pseudo,
                                 const int32_t* order, int H, int64_t N, int C, int fx_shift, int64_t* conf_fx,
                                 coda_stream_t stream);
/* coda.py:227-229 (see coda_b200_pi_full / coda_b200_pi_full_tc).  For a 16-bit slab the tensor-core pass takes any
 * model stride and any 2-byte aligned view (pi_full_tc_ok_x), so it serves every shape whose fp32 widening it serves. */
int coda_b200_pi_full_x(const void* preds, int fmt, int64_t model_stride, const float* D, int H, int64_t N, int C,
                        float* U, coda_stream_t stream);
int coda_b200_pi_full_tc_ok_x(int fmt, int H, int64_t N, int C, int64_t model_stride);
int coda_b200_pi_full_tc_x(const void* preds, int fmt, int64_t model_stride, const float* D, int H, int64_t N, int C,
                           float* U, void* scratch, uint32_t* flags, coda_stream_t stream);
/* Shadow copy in the slab's own element type (see coda_b200_shadow_build); col_stride a multiple of 8 elements. */
int coda_b200_shadow_build_x(const void* preds, int fmt, int64_t model_stride, int H, int64_t N, int C,
                             const int32_t* model_of_slot, int S, int64_t col_stride, void* T, coda_stream_t stream);
/* coda.py:319 (see coda_b200_pi_rank1).  Model terms are slab elements relative to `preds`; the ensemble term (the
 * first term of a list whose header names a majority class) is read as fp32 relative to `ens_base` instead, so the
 * step struct's ens_off must be set relative to ens_base.  With CODA_B200_SLAB_F32 and ens_base == preds this is
 * coda_b200_pi_rank1. */
int coda_b200_pi_rank1_x(const void* preds, int fmt, const float* ens_base, int H, int64_t N, int C,
                         const int64_t* sel, double lr, int fx_shift, const int32_t* terms, float* U,
                         int64_t* pisum_fx, uint32_t* flags, int ctas_per_sm, int const_slot, coda_stream_t stream);

/* ---- compact slab (BASELINE.json configs[4]: M=1024, N=4e6, C=1000 is 16.4 TB dense; no reference counterpart --
 *      the reference cannot run there, coda.py:227 materialises a second slab) ----------------------------------
 * For every (h, n) the K <= 8 highest-scoring classes: ids [H][N][K] u16 (descending score) and probs [H][N][K] f32;
 * every other class gets rest = (1 - sum_j probs) / (C - K).  Models are model_stride ELEMENTS apart in both
 * arrays.  Each stage below produces what its dense twin produces on the densified slab. */
int coda_b200_scan_compact(const uint16_t* ids, const float* probs, int64_t model_stride, int H, int64_t N, int C,
                           int K, uint16_t* hard, int32_t* pseudo, uint8_t* disagree, float* ens_out, uint32_t* flags,
                           coda_stream_t stream);
/* coda_b200_scan_compact with its kernel named: 0 = the one it chooses by C, 1 = one thread per item (C <= 1599),
 * 2 = one warp per item (C <= 4096).  Both give the same bits; this lets a benchmark time one against the other. */
int coda_b200_scan_compact_kernel(const uint16_t* ids, const float* probs, int64_t model_stride, int H, int64_t N,
                                  int C, int K, uint16_t* hard, int32_t* pseudo, uint8_t* disagree, float* ens_out,
                                  uint32_t* flags, int kernel, coda_stream_t stream);
/* coda.py:42: conf[h][y][j] == conf_fx[h][y][j] + conf_rest[h][y] (both ACCUMULATED into, int64 fixed point). */
int coda_b200_confusion_compact(const uint16_t* ids, const float* probs, int64_t model_stride, const int32_t* pseudo,
                                int H, int64_t N, int C, int K, int fx_shift, int64_t* conf_fx, int64_t* conf_rest,
                                coda_stream_t stream);
/* coda.py:227-229, K < C <= 4096.  DT_scratch [H][C][C] and RS_scratch [H][C] floats are overwritten (D transposed,
 * row sums). */
int coda_b200_pi_full_compact(const uint16_t* ids, const float* probs, int64_t model_stride, const float* D, int H,
                              int64_t N, int C, int K, float* DT_scratch, float* RS_scratch, float* U,
                              coda_stream_t stream);
/* coda.py:319 (see coda_b200_pi_rank1); the gather list was built with coda_step_t.compact_k = K. */
int coda_b200_pi_rank1_compact(const uint16_t* ids, const float* probs, int64_t model_stride, const float* ens, int H,
                               int64_t N, int C, int K, const int64_t* sel, double lr, int fx_shift,
                               const int32_t* terms, float* U, int64_t* pisum_fx, uint32_t* flags,
                               coda_stream_t stream);

/* Inverted index of the compact slab: for every (model, class) the items whose top-K list holds the class, as
 * {item u32, float bits of (probs - rest)} pairs.  count: counts[h][c] (ACCUMULATED into, int64); the caller turns
 * them into offsets [H*C + 1] (exclusive prefix sums) and a cursor copy; fill: places the 8-byte entries (order
 * inside a list is not defined) and writes rest_sum[n] = sum_h rest(h, n).  N < 2^32 per shard. */
int coda_b200_compact_index_count(const uint16_t* ids, int64_t model_stride, int H, int64_t N, int C, int K,
                                  int64_t* counts, coda_stream_t stream);
int coda_b200_compact_index_fill(const uint16_t* ids, const float* probs, int64_t model_stride, int H, int64_t N, int C,
                                 int K, int64_t* cursor, void* entries, float* rest_sum, coda_stream_t stream);
/* coda.py:319 from the index:  sum_h preds[h][n][jvec[h]] = rest_sum[n] + sum over the H lists (h, jvec[h]) of
 * (probs - rest), scattered into delta [N] (int64 fixed point, zero on entry and on exit: order-independent sums),
 * then the U row pass of coda_b200_pi_rank1.  Reads H lists of about N K / C entries instead of the whole slab.
 * `terms` is only consulted for "no label applied in this step" ({0, -1}). */
int coda_b200_pi_rank1_index(const int64_t* offsets, const void* entries, const float* rest_sum, const int32_t* jvec,
                             int H, int64_t N, int C, const int64_t* sel, double lr, int fx_shift, const int32_t* terms,
                             int64_t* delta, float* U, int64_t* pisum_fx, uint32_t* flags, coda_stream_t stream);

/* ---- Beta quadrature tables (dirichlet_to_beta coda.py:14-25, compute_pbest_beta_batched
 *      coda.py:77-119, batch_update_beta coda.py:150-168) for classes [cls_lo, cls_hi) ------- */
size_t coda_b200_tables_scratch_bytes(int H, int ncls);
/* sel (optional, device): {idx, class}; when non-NULL exactly one class, sel[1], is rebuilt (host-free loop). */
/* dLb / Gb (optional, both or neither): the same tables as bf16 limbs in tensor-core operand order for
 * coda_b200_pair_rows_tc: dLb [C][Hp/32][3][256*32], Gb [C][16][4][Hp*16] bf16, zero-initialised by the caller. */
int coda_b200_beta_tables(const float* D, const float* grid_x, int H, int C, int P, double hyp_w, int cls_lo,
                          int cls_hi, const int64_t* sel, void* scratch, float* dL /*[C][H][P]*/,
                          float* G0T /*[C][P][Hp]*/, float* G1T /*[C][P][Hp]*/, float* PB /*[C][Hp]*/, void* dLb,
                          void* Gb, uint32_t* flags, coda_stream_t stream);

/* ---- hypothetical-update rows (eig_batched inner loop, coda.py:261-279) ---------------- */
/* ent_cnt[n] = distinct predicted classes of item n, heavy_cnt[n] = how many of them two or more models predict,
 * cls_heavy[c] (accumulated) = heavy rows of class c. */
int coda_b200_pair_count(const uint16_t* hard, int H, int64_t N, int C, int32_t* ent_cnt /*[N]*/,
                         int32_t* heavy_cnt /*[N]*/, int32_t* cls_heavy /*[C]*/, coda_stream_t stream);
/* Fills, per item, the entry list (ent_row / ent_cls at ent_off[n]..) and, per class, the class-major work list the
 * row kernels tile over: position q in [cls_base[c], cls_base[c+1]) = {template rows of c, heavy rows of c} with
 * zmask[q] (H-bit set of the models that predict c) and row_of[q] (the row it describes). */
int coda_b200_pair_fill(const uint16_t* hard, int H, int64_t N, int C, const int32_t* ent_off /*[N+1]*/,
                        const int32_t* heavy_off /*[N+1]*/, const int64_t* cls_base /*[C+1]*/,
                        int32_t* cls_cursor /*[C] zeroed*/, int32_t* ent_row, uint16_t* ent_cls,
                        uint32_t* zmask /*[npairs][Hp/32]*/, int32_t* row_of /*[npairs]*/,
                        uint16_t* row_cls /*[n_heavy] class of every heavy row*/, coda_stream_t stream);
/* tiles [ntiles][4] int32 = {class, first work-list position, count <= 32, 0}; processes tiles [tile_lo, tile_hi).
 * Writes gain[row] = H_before - H_after (coda.py:274-276) and, if ph_cache != NULL, the normalised
 * P(best | hypothetical) row (coda.py:271-273), row = row_of[position].  With sel != NULL the launch covers
 * [0, tile_hi - tile_lo) tiles of class sel[1] (pass the largest per-class tile count). */
int coda_b200_pair_rows(const int32_t* tiles, int tile_lo, int tile_hi, const uint32_t* zmask, const int32_t* row_of,
                        const float* dL, const float* G0T, const float* G1T, const float* PB, const float* m0,
                        const float* pi_hat, int H, float* ph_cache, float* gain, const int64_t* sel /*optional*/,
                        const int64_t* tile_off /*[C+1], with sel*/, uint32_t* flags, coda_stream_t stream);
/* The same computation on the wgmma tensor cores (Hp <= 256): tiles128 are tiles of <= 128 same-class positions,
 * operands come from the bf16 limb tables of coda_b200_beta_tables. */
int coda_b200_pair_rows_tc(const int32_t* tiles128, int tile_lo, int tile_hi, const uint32_t* zmask,
                           const int32_t* row_of, const void* dLb, const void* Gb, const float* PB, const float* m0,
                           const float* pi_hat, int H, float* ph_cache, float* gain, const int64_t* sel,
                           const int64_t* tile_off, uint32_t* flags, coda_stream_t stream);

/* ---- the per-step scoring pass (eig_batched coda.py:253-278 + _prefilter coda.py:215-219 + the arg-max of
 *      get_next_item_to_label coda.py:306/309), one kernel, item-major ---------------------------------
 * For every item: the information gain of each of its rows from gain[row] (row_gains or pair_rows wrote it; template
 * rows in gain[0..T)), then eig[n] = sum_c pi_hat_xi[n][c] * gain(n, c)  (== H_before - sum_c xi * H_after because
 * sum_c xi = 1), the candidate arg-max (first index wins) and runner-up value per block -> partials [blocks][REC_WORDS]. */
int coda_b200_eig_blocks(int64_t N, int H, int C); /* number of partial records gain_eig writes */
/* max_entries: the longest entry list (or -1 if unknown); short lists and C <= 128 take an 8-lanes-per-item kernel,
 * which reads the lists from the optional ELL copy (coda_b200_ell_build; ell_k = padded list length <= 32). */
int coda_b200_gain_eig(const float* U, int64_t N, int C, int H, const int32_t* ent_off, const int32_t* ent_row,
                       const uint16_t* ent_cls, const float* gain, const uint8_t* labeled, const uint8_t* disagree,
                       int64_t n_offset, int max_entries, const int32_t* ell_row, const uint16_t* ell_cls, int ell_k,
                       float* eig, int64_t* partials, uint32_t* flags, coda_stream_t stream);
int coda_b200_ell_build(const int32_t* ent_off, const int32_t* ent_row, const uint16_t* ent_cls, int64_t N, int K,
                        int32_t* ell_row /*[N][K], -1 = empty*/, uint16_t* ell_cls /*[N][K]*/, coda_stream_t stream);
/* gain[r] (coda.py:274-276) of ALL T + n_heavy rows from their cached rows -- the template rows (class = r / (1+H))
 * and the heavy rows (class = row_cls[r - T]) in one stream: the HBM-bound kernel of the two-kernel scoring pass
 * (row_gains, then gain_eig).  Item-major heavy rows make the per-item gains contiguous for the
 * assembly that follows. */
int coda_b200_row_gains(const float* ph_cache, const uint16_t* row_cls, int64_t n_heavy, int H, int C,
                        const float* PB, const float* m0, const float* pi_hat, float* gain, coda_stream_t stream);

/* ---- fused single-CTA step kernels: selection, label, posterior update, mixture --------------------------- */
typedef struct coda_step { /* host struct: this shard's device state */
  int H, C;
  int64_t N, n_offset;
  int fx_shift;
  float lr;
  const uint16_t* hard; /* [N][H] */
  uint8_t* labeled;     /* [N] */
  float* D;             /* [H][C][C] */
  int32_t* jvec;        /* [H] p_h(idx) of the labeled item */
  int64_t* sel;         /* {local index or -1, class} */
  /* rank-1 gather list (see coda_b200_pi_rank1) */
  int32_t* terms; /* [2 + 8H] */
  const int32_t* slot_of_model;
  int64_t shadow_off, shadow_col_stride, model_stride;
  /* ensemble sums E (the majority shortcut's first term): element offset of E[item 0][class 0] relative to preds and
   * the class stride of a class-major copy (item stride 1), or 0 for the item-major [N][C] ens (item stride C) */
  int64_t ens_off, ens_col_stride;
  int have_ens;
  int compact_k; /* > 0: the slab is in the compact top-K form, the gather list names (model, class) pairs */
  /* marginals / mixture */
  int64_t* pisum_fx;   /* [C] local sums */
  const float* PB;     /* [C][Hp] */
  float* pi_hat;       /* [C] */
  float* m0;           /* [Hp] */
  float* h_before;     /* [1] */
  int64_t* best_model; /* [1] */
  /* selection */
  const int64_t* partials; /* [nblocks][REC_WORDS] */
  int nblocks;
  const float* eig;
  int64_t* bestrec; /* [REC_WORDS] merged (global) record */
  /* host-free loop */
  const int64_t* labels_global;
  int64_t* hist_idx;
  float* hist_q;
  int32_t* hist_tie;
  int64_t hist_cap;
  int64_t* step_ctr; /* [1] */
  uint32_t* flags;
  /* host-resident slab (HostSlab): every model has a shadow slot; slots [H - n_host, H) live in pinned host memory.
   * The step kernels emit a host slot's term as {element offset into host_shadow, sign, item stride 0}, which only
   * coda_b200_host_stage resolves.  n_host = 0: no host slots (every other field below is ignored). */
  int64_t n_host;
  const void* host_shadow; /* device-visible address of the pinned slots [n_host][C][shadow_col_stride] */
  void* stage;             /* device staging columns [2 * n_host][shadow_col_stride], slab element type */
  int64_t stage_off;       /* element offset of `stage` relative to the slab base pointer pi_rank1 is given */
} coda_step_t;

/* coda.py:306/309 + oracle(idx) + coda.py:316-317 with no host in the loop: merge the block records, exchange
 * {record, p_h(candidate)} with every peer, take the global arg-max (first index; an isclose tie -- coda.py:307 --
 * is recorded in hist_tie), look the label up in labels_global, mark the item labeled, D[h][t][p_h(idx)] += lr,
 * build the rank-1 gather list, zero pisum. */
int coda_b200_step_select(const coda_step_t* st, const coda_xchg_t* x, coda_stream_t stream);
/* Host-resident slab: after step_select / step_label and before pi_rank1, copy the host-slot column of every term
 * the step kernel left unresolved (item stride 0) from mapped pinned memory into the next free staging column (cs
 * slab elements at the width `fmt`), and point the term there (offset stage_off + k * cs, item stride 1).  Term
 * count, order and signs are unchanged; every other term is untouched.  census (optional, device): += host columns
 * staged.  A fixed grid reads the term count on the device (graph-capturable); no-op when st->n_host == 0. */
int coda_b200_host_stage(const coda_step_t* st, int fmt, int64_t* census, coda_stream_t stream);
/* Page-lock `bytes` of an existing host allocation and map them for every device at the same address (the host
 * slots of a HostSlab); fails when the device address would differ.  unregister undoes it. */
int coda_b200_host_register(void* ptr, size_t bytes);
int coda_b200_host_unregister(void* ptr);
/* API path, get_next_item_to_label: merge + exchange only -> bestrec. */
int coda_b200_step_merge(const coda_step_t* st, const coda_xchg_t* x, coda_stream_t stream);
/* API path, add_label (coda.py:315-317): sel = {local idx or -1, class} given; the owner shares p_h(idx). */
int coda_b200_step_label(const coda_step_t* st, const coda_xchg_t* x, coda_stream_t stream);
/* pi_hat (coda.py:232-233; the shards' sums are exchanged and added here), P(best) vector m0 == get_pbest()
 * (coda.py:253, 325-332), H_before (coda.py:254) and argmax (coda.py:346). */
int coda_b200_step_mixture(const coda_step_t* st, const coda_xchg_t* x, coda_stream_t stream);
/* One thread: hist_best[(*step_ctr - 1) % hist_cap] = *best_model, the best model (coda.py:334-346) after the step
 * step_select counted.  Enqueued after step_mixture by the device loop that records the per-step best models. */
int coda_b200_record_best(const int64_t* best_model, const int64_t* step_ctr, int32_t* hist_best, int64_t hist_cap,
                          coda_stream_t stream);

/* tie scan (coda.py:307 torch.isclose(q, best, rtol=1e-8[, atol=1e-8]) in fp32) against the global record. */
int coda_b200_ties(const float* eig, int64_t N, const uint8_t* labeled, const uint8_t* disagree, int64_t n_offset,
                   const int64_t* best /*[REC_WORDS]*/, int cap, int64_t* tie_hdr /*[2]*/, int64_t* tie_idx,
                   float* tie_val, coda_stream_t stream);
/* every shard's report block (flags, record, tie list: rep_words int64) -> rep_all [world][rep_words] on every shard */
int coda_b200_report_gather(const int64_t* rep, int rep_words, int64_t* rep_all, const coda_xchg_t* x,
                            uint32_t* flags, coda_stream_t stream);

/* ---- competing selectors (coda/baselines/<name>.py), over the products of coda_b200_scan_slab ----------------------
 * Per-item vectors are [N] over the items of one shard (all items when there is one); `labeled` [N] u8 marks the items
 * already labeled.  A compact slab is scanned by coda_b200_scan_compact; everything below reads only the scan. */

/* ModelPicker acquisition, modelpicker.py:58-86 (the C-class loop at 74-86 with (N, H) temporaries per class).
 * For item n let Z_c be the models predicting class c, A_c = sum_{h in Z_c} p_h, Q_c = sum_{h in Z_c} p_h log2 p_h,
 * S = sum p, B = sum p log2 p (0 log 0 = 0), g = gamma:  H_c = log2(S + (g-1) A_c) - (B + (g-1) Q_c + g log2(g) A_c) /
 * (S + (g-1) A_c); a class no model predicts gives log2 S - B / S; ent[n] = mean over the C classes, accumulated in
 * fp64 per item with the groups taken in the order of their lowest model index, rounded once.  The 1e-12 clamp of
 * modelpicker.py:83 is not applied (its effect is below H * 4e-11).  ent[n] = +inf for labeled items and, when
 * mask_agreeing != 0, for items every model agrees on (modelpicker.py:64-66). */
int coda_b200_mp_entropy(const uint16_t* hard, const float* posterior /*[H]*/, int H, int64_t N, int C, double gamma,
                         const uint8_t* labeled, const uint8_t* disagree, int mask_agreeing, float* ent,
                         coda_stream_t stream);
/* Static acquisition scores from l_h = 1 - ens[n][hard[n][h]] / H (the mean-ensemble surrogate, activetesting.py:18, 33):
 * at_score[n] = sum_h l_h (activetesting.py:33-44), vma_score[n] = sum_{h < h'} |l_h - l_h'| (vma.py:18-41, the
 * H x H x |D_U| tensor of vma.py:31), both over the item's distinct predicted classes with multiplicities.
 * Either output may be NULL. */
int coda_b200_static_scores(const uint16_t* hard, const float* ens, int H, int64_t N, int C, float* at_score,
                            float* vma_score, coda_stream_t stream);
/* number of partial records of the selection calls below (per-block chunks of the item axis) */
int coda_b200_select_blocks(int64_t N);
/* Selection over the unlabeled items of N-range shards (one shard, or several per GPU or one per GPU, each with its own
 * stream).  Every shard makes the same calls in the same order; each call ends in ONE single-CTA kernel that stores this
 * shard's record into every peer's mailbox (record channel of a box sized by coda_b200_xchg_box_bytes(world, H, C, ...)),
 * waits for all of them (2 s bound, then CODA_B200_FLAG_XCHG_TIMEOUT in `flags`) and merges them in rank order, so every
 * shard holds the same global answer.  Vectors, `labeled` and `partials` are this shard's (partials: 2 * select_blocks
 * words); item indices in the outputs are global (n_offset + local).  x == NULL or world 1: one shard, no mailbox is
 * touched and `flags` is never set.
 *   select_extreme_xchg: minimum (want_max = 0, modelpicker.py:68-69) or maximum (uncertainty.py:37-38) of v over the
 *     unlabeled items and the number of items exactly equal to it: out = {float bits of the global extreme, global count
 *     of items equal to it, how many of them lie on lower ranks, how many on this rank} (vc_merge is exact, so the
 *     {value, count} does not depend on the shard count);
 *   select_kth_xchg: the k-th (ascending global index, from 0) unlabeled item equal to best[0] (modelpicker.py:70,
 *     uncertainty.py:39-43), from the partials of the select_extreme_xchg call that produced best = its out; the shard
 *     whose ties cover k picks its (k - lower)-th; out_idx = global item, -1 if there is none;
 *   random.choices(d_u_idxs, weights) (activetesting.py:45-48, vma.py:44-60), u = random.random() drawn by the caller:
 *   weighted_total_xchg: total = {sum over the shards in rank order of each shard's fp64 sum of w over its unlabeled
 *     items, unlabeled count};
 *   weighted_draw_xchg: the weights w / (float)total[0] (fp32 division, the normalisation of activetesting.py:44) and
 *     their running fp64 sum cum in index order; the first unlabeled item with cum > u * cum_total (bisect_right, the
 *     last one if none) -> out = {global position among the unlabeled items, global item, float bits of its normalised
 *     weight}.  The shards' sums are exchanged; every shard forms the grand total in rank order, target = u * grand
 *     and the owner shard, which draws inside its chunks starting from the lower ranks' running sum and position.  A
 *     shard's selection blocks and per-thread runs restart at its first item, so the fp64 partial sums group the items
 *     differently from one shard: a pick can differ from one shard only when u * total lies within ~1e-16 relative of
 *     a cumulative boundary. */
int coda_b200_select_extreme_xchg(const float* v, const uint8_t* labeled, int64_t N, int want_max, int64_t* partials,
                                  int64_t* out /*[4]*/, const coda_xchg_t* x, uint32_t* flags, coda_stream_t stream);
int coda_b200_select_kth_xchg(const float* v, const uint8_t* labeled, int64_t N, const int64_t* partials,
                              const int64_t* best /*[4]*/, int64_t k, int64_t n_offset, int64_t* out_idx /*[1]*/,
                              const coda_xchg_t* x, uint32_t* flags, coda_stream_t stream);
int coda_b200_weighted_total_xchg(const float* w, const uint8_t* labeled, int64_t N, double* partials,
                                  double* total /*[2]*/, const coda_xchg_t* x, uint32_t* flags, coda_stream_t stream);
int coda_b200_weighted_draw_xchg(const float* w, const uint8_t* labeled, int64_t N, const double* total, double u,
                                 int64_t n_offset, double* partials, int64_t* out /*[3]*/, const coda_xchg_t* x,
                                 uint32_t* flags, coda_stream_t stream);
/* add_label on shards: the shard that holds the labeled item (own = 1; exactly one) sends `bytes` from src -- its hard
 * row, or the per-model losses of its (H, C) column -- and every shard receives them in dst.  bytes + 16 must fit the
 * record slot (2 * H * 2 + 64 bytes: an H-float vector does).  x == NULL or world 1: src is copied to dst. */
int coda_b200_owner_share(const void* src, int bytes, int own, void* dst, const coda_xchg_t* x, uint32_t* flags,
                          coda_stream_t stream);

/* ---- Host-free loop of the competing selectors (one captured graph per step and shard) ----------------------------
 * Every per-step scalar lives in device memory, so one graph serves every step.  Loop words `ls` (int64, per shard,
 * identical on every shard):
 *   ls[0] labels so far (global), ls[1] steps done in this run, ls[2] stop word (0 = running, 1 = VMA's weights fell
 *   below 1e-12, 2 = ActiveTesting's total is not > 0, 3 = no item was picked), ls[3] the k of this step's k-th tie,
 *   ls[4] 1 when this step's item was drawn among several exact ties, ls[5] device-loop steps ever (history slot),
 *   ls[6] the 64-bit Philox key, ls[7] unlabeled items some model disagrees on (ModelPicker), ls[8] this step's u
 *   (the bits of a double).  Once ls[2] is set every kernel below returns at once.
 * Tie draws: Philox4x32-10 (curand_Philox4x32_10), key = ls[6], counter = {label count at the draw, purpose (0 = item
 * tie, 1 = best-model tie), 0, 0}; the item tie is drawn before the step's label is added, the best-model tie after it;
 * the j-th tie in ascending index order is taken, j = (uint64)r.x * count >> 32. */
#define CODA_B200_BL_IID 0
#define CODA_B200_BL_UNCERTAINTY 1
#define CODA_B200_BL_ACTIVETESTING 2
#define CODA_B200_BL_VMA 3
#define CODA_B200_BL_MODELPICKER 4

typedef struct coda_bl_loop { /* host struct: one shard of a competing selector's device loop */
  int method;                 /* CODA_B200_BL_* */
  int H;
  int64_t N, n_offset, n_global;
  const uint16_t* hard;       /* [N][H] this shard's hard predictions */
  const uint8_t* disagree;    /* [N] (ModelPicker) */
  uint8_t* labeled;           /* [N] */
  const int64_t* labels;      /* [n_global] the oracle's labels on this shard's device */
  const double* pre;          /* [steps] pre-drawn per step: IID position among the unlabeled items, AT / VMA u */
  int64_t* ls;                /* [16] loop words, see above */
  const int64_t* best;        /* select_extreme_xchg out [4] */
  const int64_t* pick;        /* select_kth_xchg out [1] (IID, Uncertainty, ModelPicker) / weighted_draw out [3] */
  const double* total;        /* weighted_total_xchg total [2] (AT / VMA) */
  int32_t* counts;            /* [H] loss counts (IID, Uncertainty) / correct counts (ModelPicker) */
  double* s1;                 /* [H] LURE sum_m L_m (AT / VMA) */
  double* s2;                 /* [H] LURE sum_m L_m a_m / (N - m) */
  float* post;                /* [H] ModelPicker posterior */
  float gamma;                /* ModelPicker gamma as fp32 */
  int64_t hist_cap;
  int64_t* hist_idx;          /* [hist_cap] rings, slot = ls[5] % hist_cap */
  double* hist_q;
  int32_t* hist_tie;
  int32_t* hist_best;
  int32_t* hist_best_tie;
  uint8_t* hist_loss;         /* [hist_cap][H] the step's loss bits (AT / VMA), may be NULL otherwise */
  uint32_t* flags;
} coda_bl_loop_t;

/* select_kth_xchg with k = *k read on the device; nothing (no exchange either) when *stop != 0 */
int coda_b200_select_kth_xchg_dev(const float* v, const uint8_t* labeled, int64_t N, const int64_t* partials,
                                  const int64_t* best, const int64_t* k, const int64_t* stop, int64_t n_offset,
                                  int64_t* out_idx, const coda_xchg_t* x, uint32_t* flags, coda_stream_t stream);
/* weighted_draw_xchg with u = *u read on the device; nothing (no exchange either) when *stop != 0 */
int coda_b200_weighted_draw_xchg_dev(const float* w, const uint8_t* labeled, int64_t N, const double* total,
                                     const double* u, const int64_t* stop, int64_t n_offset, double* partials,
                                     int64_t* out, const coda_xchg_t* x, uint32_t* flags, coda_stream_t stream);
/* mp_entropy with mask_agreeing = (*n_disagree > 0) read on the device */
int coda_b200_mp_entropy_dev(const uint16_t* hard, const float* posterior, int H, int64_t N, int C, double gamma,
                             const uint8_t* labeled, const uint8_t* disagree, const int64_t* n_disagree, float* ent,
                             coda_stream_t stream);
/* One thread: this step's k (IID: the pre-drawn position; Uncertainty / ModelPicker: a Philox draw among best[1]
 * ties, 0 for one tie) or u (AT / VMA: the pre-drawn u, after the stop checks on total[0] as fp32). */
int coda_b200_bl_draw(const coda_bl_loop_t* a, coda_stream_t stream);
/* One CTA: the step's item and q, its label, the labeled mark, the owner's hard row to every shard (record channel),
 * the method's sums, the best model, the history slots, then the counters advance. */
int coda_b200_bl_step(const coda_bl_loop_t* a, const coda_xchg_t* x, coda_stream_t stream);

/* ---- torch's generators on the device (run_steps(..., tie_rule="reference") of the competing selectors) -----------
 * The draws the reference makes from torch's generators, from replicas of them on every shard (csrc/bl_ref.cu):
 *   cpu_rng [625] uint32: torch's CPU generator (MT19937), the 624 state words then the position of the next word,
 *     pos = 625 - left of torch.get_rng_state() (pos = next after the first word of a twist).
 *     randperm(n)[0] = word % n, then n - 2 words dropped (n < CODA_B200_RANDPERM32_MAX: torch's 32-bit branch);
 *     randint(n) = word % n for n < 2^28, else ((word1 << 32) | word2) % n.
 *   cuda_rng [2] int64: torch's CUDA generator {seed, offset}; randint(n) (n < 2^28) = curand4(curand_init(seed, 0,
 *     offset)).x % n, then offset += 4.
 * Per step: Uncertainty and ModelPicker run bl_draw_ref in place of bl_draw; every method runs bl_best_ref right after
 * bl_step.  Every shard advances its replicas by the same global counts. */
#define CODA_B200_RANDPERM32_MAX 214748364LL /* (2^32 - 1) / 20: from here torch.randperm draws 64-bit words */
/* One warp, in place of bl_draw: this step's k (Uncertainty: randperm(best[1])[0] when best[1] > 1 items tie, else 0;
 * ModelPicker: randint(best[1]), every step) from cpu_rng. */
int coda_b200_bl_draw_ref(const coda_bl_loop_t* a, uint32_t* cpu_rng, coda_stream_t stream);
/* One warp, after bl_step of a step that committed: the best model again from the sums bl_step left, with its tie drawn
 * as the reference draws it -- randperm(ties)[0] from cpu_rng when several models tie (IID, Uncertainty, ActiveTesting,
 * VMA), randint(ties) from cuda_rng every step (ModelPicker) -- into hist_best of the step.  The unused replica may be
 * NULL. */
int coda_b200_bl_best_ref(const coda_bl_loop_t* a, uint32_t* cpu_rng, int64_t* cuda_rng, coda_stream_t stream);
/* One warp runs ops [nops][2] in order, one output each: {0, n} randperm(n)[0] (0 for n = 1) and {1, n} randint(n) from
 * cpu_rng, {2, n} randint(n) from cuda_rng. */
int coda_b200_torch_rng_run(uint32_t* cpu_rng, int64_t* cuda_rng, const int64_t* ops, int nops, int64_t* out,
                            coda_stream_t stream);

/* ---- CODA's other acquisitions in its host-free loop (q='uncertainty', q='iid', prefilter_n; coda.py:215-224, 287-295)
 * Candidates: the unlabeled items some model disagrees on, all unlabeled items when there are none (coda.py:239); as
 * the exact maximum ties of `cand` (the disagreement bits as 1.0f / 0.0f) under select_extreme_xchg(want_max = 1).
 * `pre` [rows][width] int64: per step {the candidate count n_s the host predicted, then the iid position k (width 2) or
 * the prefilter's m sample positions into the ascending candidate list (width m + 1)}; `lw` [8] int64 loop words:
 * lw[0] this step's row of pre (advanced by the commit), lw[1] the iid k, lw[2] 0 (the stop word of
 * select_kth_xchg_dev).  A commit whose global candidate count differs from pre's sets CODA_B200_FLAG_PREDRAW_MISMATCH.
 * Every commit writes what step_select writes after its arg-max: sel = {local index or -1, labels_global[item]},
 * hist_idx / hist_q / hist_tie at *step_ctr % hist_cap, then *step_ctr += 1; step_label follows. */
/* q='uncertainty': this shard's block records (the layout of the EIG assembly's, nblocks = st->nblocks of them) from a
 * static score vector; step_select then picks as for EIG. */
int coda_b200_static_records(const float* score, const uint8_t* labeled, const uint8_t* disagree, int64_t N,
                             int64_t n_offset, int nblocks, int64_t* partials, coda_stream_t stream);
/* q='iid', one thread: lw[1] = pre[lw[0]][1] (the k of select_kth_xchg_dev). */
int coda_b200_abl_draw(const int64_t* pre, int width, int64_t* lw, coda_stream_t stream);
/* q='iid', one thread: item pick[0], q = fp32(1 / best[1]), hist_tie = best[1] > 1 (the reference's random.choice). */
int coda_b200_abl_commit(const coda_step_t* st, const int64_t* best /*[4]*/, const int64_t* pick /*[1]*/,
                         const int64_t* pre, int width, int64_t* lw, coda_stream_t stream);
/* number of block records of prefilter_pick for m samples */
int coda_b200_prefilter_blocks(int m);
/* prefilter_n = m (width m + 1): each sample position -> its item on the shard that holds it (from the partials and out
 * `best` of select_extreme_xchg over cand), eig[item]; per block a record {bits(v), j << 40 | global item, bits(v2), 0}
 * over its samples j (the earliest sample position wins equal values, v2 = the best of the others). */
int coda_b200_prefilter_pick(const float* eig, const float* cand, const uint8_t* labeled, int64_t N, int64_t n_offset,
                             const int64_t* partials, const int64_t* best, const int64_t* pre, int width, int m,
                             const int64_t* lw, int64_t* recs, coda_stream_t stream);
/* One CTA: merge the block records, exchange them (record channel), commit the winner with q = its EIG and hist_tie =
 * isclose(v2, v) (coda.py:307 over the sample). */
int coda_b200_prefilter_commit(const coda_step_t* st, const int64_t* recs, int nrec, const int64_t* best,
                               const int64_t* pre, int width, int64_t* lw, const coda_xchg_t* x, coda_stream_t stream);

/* ---- isclose ties from Python's random (CODA.run_steps(..., tie_rule="reference"); coda.py:306-311) -----------------
 * `rng` [625] uint32 on every shard: a replica of Python's generator as random.getstate()[1] holds it (624 MT19937 words,
 * then the position); every shard advances its replica identically.  `pending` is one int64 word set by the deferring
 * select / prefilter commit: 1 on a step whose winner has an isclose runner-up, which then commits nothing; tie_band,
 * tie_draw, step_label_if, pf_band and pf_tie_draw return at once unless it is 1.  A tie draw commits as abl_commit
 * does, with q = the drawn item's value and hist_tie = 1.  Candidate counts must be < 2^32 (the caller checks). */
/* step_select (pick = 1), except that a step with an isclose tie commits nothing and sets *pending = 1 (else 0) */
int coda_b200_step_select_defer(const coda_step_t* st, const coda_xchg_t* x, int64_t* pending, coda_stream_t stream);
/* step_label on a pending step only */
int coda_b200_step_label_if(const coda_step_t* st, const coda_xchg_t* x, const int64_t* pending, coda_stream_t stream);
/* per selection chunk {bits(best), candidates isclose to bestrec's winner} (select_extreme_xchg's partial layout) over
 * score v (the EIG vector, or q='uncertainty''s static score) */
int coda_b200_tie_band(const float* v, const uint8_t* labeled, const uint8_t* disagree, int64_t N,
                       const int64_t* bestrec, const int64_t* pending, int64_t* partials, coda_stream_t stream);
/* One CTA: n = the band's global size (record channel), r = _randbelow(n), commit the r-th band item in ascending
 * global index order */
int coda_b200_tie_draw(const coda_step_t* st, const float* v, const uint8_t* disagree, const int64_t* partials,
                       const int64_t* pending, uint32_t* rng, int64_t* lw, const coda_xchg_t* x, coda_stream_t stream);
/* prefilter_n = m: pre row 0 = {n_s = best[1], random.sample(range(n_s), m)} and lw[0] = 0.  setsize: Lib/random.py's
 * (21, plus 4 ** ceil(log(3 m, 4)) when m > 5); pool >= min(setsize, n_s) int32, seen >= ceil(n_s / 32) zero words
 * (left zero).  n_s <= m sets CODA_B200_FLAG_PREDRAW_MISMATCH. */
int coda_b200_pf_sample(const int64_t* best, int64_t* pre, int m, int64_t setsize, uint32_t* rng, int32_t* pool,
                        uint32_t* seen, int64_t* lw, uint32_t* flags, coda_stream_t stream);
/* prefilter_commit, except that a winner with an isclose runner-up is not committed: *pending = 1 (else 0), and
 * lw[4] = bits(winner's EIG) */
int coda_b200_prefilter_commit_defer(const coda_step_t* st, const int64_t* recs, int nrec, const int64_t* best,
                                     const int64_t* pre, int width, int64_t* lw, int64_t* pending,
                                     const coda_xchg_t* x, coda_stream_t stream);
/* band_item[j] (m entries) = the global item of sample position j if this shard holds it and its EIG is isclose to
 * lw[4], else -1 */
int coda_b200_pf_band(const float* eig, const float* cand, const uint8_t* labeled, int64_t N, int64_t n_offset,
                      const int64_t* partials, const int64_t* best, const int64_t* pre, int width, int m,
                      const int64_t* lw, const int64_t* pending, int64_t* band_item, coda_stream_t stream);
/* the largest m pf_tie_draw takes with several shards at H models: its band bitmap travels in one record slot */
int coda_b200_pf_tie_max_m(int H);
/* One CTA: the band bitmap over the sample positions (OR over the shards), r = _randbelow(its size), commit the r-th
 * band position in sample order.  bits: >= ceil(m / 32) words rounded up to 16 bytes, 16-byte aligned. */
int coda_b200_pf_tie_draw(const coda_step_t* st, const int64_t* band_item, int m, const int64_t* pending,
                          uint32_t* rng, uint32_t* bits, int64_t* lw, const coda_xchg_t* x, coda_stream_t stream);
/* One warp runs ops [nops][4] on the generator `state` [625] in order: {0, n, 0, 0} -> _randbelow(n) (1 <= n < 2^32),
 * one output; {1, n, m, setsize} -> random.sample(range(n), m), m outputs.  pool / seen as for pf_sample. */
int coda_b200_pyrandom_run(uint32_t* state, const int64_t* ops, int nops, int64_t* out, int32_t* pool, uint32_t* seen,
                           coda_stream_t stream);

/* ---- scoring only the prefilter_n sample (csrc/sample.cu) ---------------------------------------------------------
 * items [m] int32: the local item of every sample position on this shard, -1 for none.  Every sampled item's eig is the
 * bits the full scoring pass (row_gains + gain_eig) gives it from the same state; other entries of eig are untouched. */
/* prefilter_pick's position -> local item resolution, written to items (-1: not on this shard / past n_s) */
int coda_b200_pf_resolve(const float* cand, const uint8_t* labeled, int64_t N, const int64_t* partials,
                         const int64_t* best, const int64_t* pre, int width, int m, const int64_t* lw, int32_t* items,
                         coda_stream_t stream);
/* a step with n_s = best[1] <= m candidates: pre row 0 = {n_s, 0 .. n_s - 1, -1 ...}, lw[0] = 0, no random draw
 * (n_s > m sets CODA_B200_FLAG_PREDRAW_MISMATCH) */
int coda_b200_pf_identity(const int64_t* best, int64_t* pre, int m, int64_t* lw, uint32_t* flags, coda_stream_t stream);
/* One CTA: the sample's heavy rows as a class-major work list.  hoff [m+1]: slot of each position's first heavy row;
 * cursor [C]: class bases (consumed by sample_fill); tiles [>= heavy/width + C][4] {class, first position, count, 0} of
 * <= width (32 SIMT, 128 tensor-core) same-class positions; tile_off [2] = {0, tile count} (pair_rows' `sel` form with
 * sel[1] = 0); nheavy [1] = the heavy-row count. */
int coda_b200_sample_plan(const int32_t* items, int m, const int32_t* ent_off, const int32_t* ent_row,
                          const uint16_t* ent_cls, const int32_t* heavy_off, int H, int C, int width, int32_t* hoff,
                          int32_t* cursor, int32_t* tiles, int64_t* tile_off, int64_t* nheavy, coda_stream_t stream);
/* masks (as pair_fill builds them), row_of (slot) and row_cls (class per slot) of the sample's heavy rows */
int coda_b200_sample_fill(const int32_t* items, int m, const uint16_t* hard, int H, int C, const int32_t* ent_off,
                          const int32_t* ent_row, const uint16_t* ent_cls, const int32_t* heavy_off, const int32_t* hoff,
                          int32_t* cursor, uint32_t* zmask, int32_t* row_of, uint16_t* row_cls, coda_stream_t stream);
/* gain [T + *nheavy]: the template rows' gains from tmpl [T][Hp], the sample rows' from scratch [cap][Hp] (row_gains'
 * arithmetic) */
int coda_b200_sample_gains(const float* tmpl, const float* scratch, const uint16_t* row_cls, int64_t cap,
                           const int64_t* nheavy, int H, int C, const float* PB, const float* m0, const float* pi_hat,
                           float* gain, coda_stream_t stream);
/* eig[items[j]] for every position j with an item: the arithmetic gain_eig uses for this C and max_entries; sets
 * CODA_B200_FLAG_NONFINITE_EIG */
int coda_b200_sample_eig(const int32_t* items, int m, const int32_t* hoff, const float* U, int C, int H,
                         const int32_t* ent_off, const int32_t* ent_row, const uint16_t* ent_cls,
                         const int32_t* heavy_off, const float* gain, int max_entries, float* eig, uint32_t* flags,
                         coda_stream_t stream);

/* ---- ModelPicker's epsilon grid search (coda_b200/eps_search.py, DESIGN.md §5b) -------------------------------------
 * A run (epsilon e, realisation r) is B steps of ModelPicker.run_steps(B, labels[pool[r]], seed = keys[e][r]) on the
 * task restricted to the P items pool[r] (global item ids), bit for bit: picks[e][r][s] is the pool position labelled at
 * step s, best[e][r][s] the best model after it, pick_tie / best_tie = 1 where either was drawn among > 1 exact ties.
 * gammas[e] = fp32((1 - eps) / eps).  All arrays are on the current device; [E][R][B] outputs are row-major. */
/* plan[5] = {runs per CTA, epsilon blocks, realisations per launch, dynamic shared bytes, scratch bytes} */
int coda_b200_mp_runs_plan(int H, int E, int P, int64_t R, int B, int64_t* plan);
/* every step of every run; one launch per `plan[2]` realisations; bit 1 of *flags: a step found no item (bad input) */
int coda_b200_mp_runs(const uint16_t* hard, const int64_t* labels, const uint8_t* disagree, int H, int C,
                      const int64_t* pool, int64_t R, int P, int B, const float* gammas, const int64_t* keys, int E,
                      void* scratch, size_t scratch_bytes, int32_t* picks, int32_t* best, uint8_t* pick_tie,
                      uint8_t* best_tie, uint32_t* flags, coda_stream_t stream);
/* labels[n] = the class most models predict for item n, the smallest class id among equal counts */
int coda_b200_majority(const uint16_t* hard, int H, int64_t N, int64_t* labels, coda_stream_t stream);
/* acc[r][h] = number of pool positions p with hard[pool[r][p]][h] == labels[pool[r][p]] */
int coda_b200_pool_accuracy(const uint16_t* hard, const int64_t* labels, int H, const int64_t* pool, int64_t R, int P,
                            int32_t* acc, coda_stream_t stream);
/* a search's pool table from one N-range piece: for k < K, out_hard[slots[k]] = hard[items[k]] (rows of H u16),
 * out_disagree[slots[k]] = disagree[items[k]], out_labels[slots[k]] = labels[items[k]].  items are local to the piece
 * (in [0, N_i)), slots are rows of the output; hard and out_hard are 16-byte aligned, all arrays on the current device.
 * K = 0 launches nothing.  Running the other entry points above on the table with pool[r][p] = the slot of position
 * (r, p) gives the bits they give on the whole [N][H] table with global item ids. */
int coda_b200_pool_gather(const uint16_t* hard, const uint8_t* disagree, const int64_t* labels, int H,
                          const int64_t* slots, const int64_t* items, int64_t K, uint16_t* out_hard,
                          uint8_t* out_disagree, int64_t* out_labels, coda_stream_t stream);

/* ---- true losses of a slab held as N-range pieces (coda/oracle.py:9-21 with coda/options.py's accuracy loss) --------
 * counts[h] = number of items n of this piece with argmax_c preds[h][n][c] == labels[n], argmax as torch.argmax decides it
 * on the device (first index of the maximum, a NaN is the maximum); a label outside [0, C) never matches.  preds is a
 * CODA_B200_SLAB_* slab [H][N][C] with models `model_stride` elements apart, read at its stored width; labels [N] int64.
 * counts [H] int64 is zeroed on `stream` first; the sums are exact, so they are the same for any split of the items. */
/* ---- module loading --------------------------------------------------------------------------------------------------
 * Load every kernel of this library into the current device's context now (*loaded_host = how many).  Under CUDA's lazy
 * loading a kernel's first launch loads its code and can wait for the kernels running on the device; shards that share
 * a GPU spin on each other inside the step kernels, so an in-process group calls this before any exchange can spin. */
int coda_b200_preload_kernels(int64_t* loaded_host);

int coda_b200_true_loss_counts(const void* preds, int fmt, int64_t model_stride, int H, int64_t N, int C,
                               const int64_t* labels, int64_t* counts, coda_stream_t stream);

/* ---- building a compact slab from a dense one (csrc/compact_build.cu) -----------------------------------------------
 * For every row (h, n) of the CODA_B200_SLAB_* slab `src` [H][N][C] (models `model_stride` elements apart, 2 <= C <=
 * 4096): ids[h][n][0..K) the K highest-scoring classes in descending score order, equal scores by ascending class (so
 * ids[h][n][0] is torch.argmax's first-index maximum), probs[h][n][0..K) their scores widened to fp32, bit for bit.
 * K in {1, 2, 3, 4, 8}, K < C; ids and probs have models `out_stride` elements apart, items K apart.  ACCUMULATED into
 * (the caller starts them at 0, i.e. +0.0 for dropped_max): dropped_max[h] = max over the rows of the (K+1)-th score
 * (as the max of its int32 bits: exact for scores >= 0), flat_rows[h] += rows whose remainder (1 - sum_j probs) *
 * fp32(1 / (C - K)) (coda_b200_scan_compact's arithmetic) is >= probs[0].  *flags gets CODA_B200_FLAG_NONFINITE_INPUT /
 * CODA_B200_FLAG_RANGE_INPUT by the dense scan's rules. */
int coda_b200_compact_build(const void* src, int fmt, int64_t model_stride, int H, int64_t N, int C, int K,
                            uint16_t* ids, float* probs, int64_t out_stride, float* dropped_max, int64_t* flat_rows,
                            uint32_t* flags, coda_stream_t stream);
/* counts[h] = number of items n with ids[h][n][0] == labels[n] (ids [H][N][K], models model_stride elements apart;
 * labels [N] int64); counts [H] int64 is zeroed on `stream` first.  For a slab built by coda_b200_compact_build these are
 * coda_b200_true_loss_counts of the dense slab. */
int coda_b200_true_loss_counts_compact(const uint16_t* ids, int64_t model_stride, int H, int64_t N, int K,
                                       const int64_t* labels, int64_t* counts, coda_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* CODA_B200_H */
