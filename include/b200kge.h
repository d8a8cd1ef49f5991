/*
 * b200kge.h — C ABI of the H100-native KGE scoring engine (libb200kge.so).
 *
 * This is the drop-in boundary for ONE path of uma-pi1/kge (LibKGE): embedding-row gather +
 * relational scorer forward (+ fused BCE/KL loss, rank/tie counting, negative-sample scoring)
 * behind KgeModel.score_spo/score_sp/score_po/score_sp_po and RelationalScorer.score_emb.
 * The reference has no FFI for this path (it is PyTorch tensor expressions); every entry point
 * below names the reference function (file:line under /root/reference) whose arithmetic it
 * replaces.  INTEGRATION.md shows the ctypes binding a LibKGE maintainer would add.
 *
 * Conventions
 *  - Plain C: raw device pointers, sizes, a cudaStream_t passed as void*.  No torch types.
 *  - All float data is fp32, row-major.  Index arrays are int64 (LibKGE collates `.long()`,
 *    train_1vsAll.py:34) and live on the device unless the name says `_host`.
 *  - A "rows view" (b200kge_rows_t) is how an embedding operand is passed: row i of the operand is
 *        base + (idx ? idx[i] : i) * ld
 *    so the same entry point serves KgeModel.score_* (base = embedding table, idx = batch indexes:
 *    the LookupEmbedder gather lookup_embedder.py:96-97 is fused) and RelationalScorer.score_emb
 *    (base = already-gathered [n,D] matrix, idx = NULL).  idx == NULL with rows == vocab is
 *    "embed_all" (lookup_embedder.py:99-112) without the table copy.
 *  - Outputs and workspace are caller-allocated; nothing is retained across calls; the library
 *    keeps no global device state and is re-entrant per stream.
 *  - Every function returns 0 on success or a negative b200kge_status; b200kge_last_error() gives a
 *    thread-local message.  CUDA allocation failures are reported with the literal text
 *    "CUDA out of memory" so LibKGE's sub-batch auto-tuner (train.py:384-413) keeps working.
 */
#ifndef B200KGE_H_
#define B200KGE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200KGE_VERSION 101

typedef void* b200kge_stream_t; /* cudaStream_t */

typedef enum {
  B200KGE_OK = 0,
  B200KGE_ERR_INVALID = -1,     /* bad argument (ValueError on the Python side)            */
  B200KGE_ERR_UNSUPPORTED = -2, /* valid but not handled by this build (e.g. D % 4 != 0)   */
  B200KGE_ERR_CUDA = -3,        /* CUDA runtime error; message holds cudaGetErrorString    */
  B200KGE_ERR_WORKSPACE = -4,   /* workspace too small; see b200kge_workspace_bytes        */
  B200KGE_ERR_NO_DEVICE = -5    /* no sm_90 device: the library never falls back to a CPU */
} b200kge_status;

/* Scorers on the path (kge/model/<name>.py). */
typedef enum {
  B200KGE_COMPLEX = 0,  /* complex.py:18-43   */
  B200KGE_DISTMULT = 1, /* distmult.py:13-25  */
  B200KGE_SIMPLE = 2,   /* simple.py:13-33    */
  B200KGE_CP = 3,       /* cp.py:13-30        */
  B200KGE_RESCAL = 4,   /* rescal.py:14-52    */
  B200KGE_TRANSE = 5,   /* transe.py:15-37    */
  B200KGE_ROTATE = 6    /* rotate.py:20-69    */
} b200kge_model;

/* `combine` of RelationalScorer.score_emb (kge_model.py:151-181) for the 1-vs-N forms. */
typedef enum {
  B200KGE_SP_ = 0, /* "sp_": out[i,j] = score(s_i, p_i, cand_j) */
  B200KGE__PO = 1  /* "_po": out[i,j] = score(cand_j, p_i, o_i) */
} b200kge_combine;

/* Which kernel family computes dot-product scorers. */
typedef enum {
  B200KGE_PREC_AUTO = 0,   /* F16X3 for dot-product scorers with 32 <= K <= 1024 and n >= 16, else fp32 SIMT */
  B200KGE_PREC_FP32 = 1,   /* CUDA-core fp32 FFMA (bit-for-bit fp32 products)                    */
  B200KGE_PREC_3XTF32 = 2, /* tcgen05 tensor cores, hi/lo split, fp32-equivalent (~3e-6 of rms)  */
  B200KGE_PREC_TF32 = 3,   /* tcgen05 single pass (~4e-3 of rms; does NOT meet the 1e-4 bar)     */
  B200KGE_PREC_TF32_BF16X2 = 4, /* tf32 hi*hi + two bf16 cross terms: 8 MMAs per 32-wide K chunk instead
                              of 12, operand error ~2^-20 (below the accumulator's)               */
  B200KGE_PREC_F16X3 = 5   /* operands split ONCE per call into row-scaled fp16 hi/lo planes (22 significant
                              bits), hi*hi + hi*lo + lo*hi on the f16 tensor pipe: 6 MMA slots per 32
                              reduction elements, no shared-memory round trip in the main loop    */
} b200kge_precision;

typedef enum {
  B200KGE_LOSS_BCE = 1, /* BCEWithLogitsKgeLoss, reduction sum, + offset  loss.py:153-159 */
  B200KGE_LOSS_KL = 2,  /* KLDivWithSoftmaxKgeLoss (CE for index labels)   loss.py:198-213 */
  /* the kinds below are row-wise losses of a block with ONE positive per row: b200kge_ns_loss only */
  B200KGE_LOSS_BCE_MEAN = 3,       /* BCEWithLogitsKgeLoss, bce_type "mean"                 loss.py:160-168 */
  B200KGE_LOSS_BCE_SELF_ADV = 4,   /* BCEWithLogitsKgeLoss, bce_type "self_adversarial"     loss.py:169-187 */
  B200KGE_LOSS_MARGIN_RANKING = 5, /* MarginRankingKgeLoss, negative-sampling pairing       loss.py:240-252 */
  B200KGE_LOSS_SOFT_MARGIN = 6,    /* SoftMarginKgeLoss                                     loss.py:216-224 */
  B200KGE_LOSS_SE = 7              /* SEKgeLoss (MSELoss, reduction sum)                    loss.py:267-274 */
} b200kge_loss;

typedef struct {
  const float* base;  /* device */
  const int64_t* idx; /* device, may be NULL */
  int64_t rows;       /* number of rows of the operand (length of idx, or table rows) */
  int64_t ld;         /* row stride in floats */
  int32_t dim;        /* row width in floats */
} b200kge_rows_t;

/* Labels of a 1-vs-N loss: exactly one of idx / dense is non-NULL.
 * idx   [n]     position of the single 1 per row (1vsAll; loss.py:105-117 makes it one-hot)
 * dense [n,ldl] label matrix (KvsAll multi-hot incl. label smoothing train_KvsAll.py:242-266,
 *               negative sampling [1,0,...] train_negative_sampling.py:128-137)            */
typedef struct {
  const int64_t* idx;
  const float* dense;
  int64_t ldl;
} b200kge_labels_t;

/* Library / device ---------------------------------------------------------------------------- */
int b200kge_version(void);
const char* b200kge_last_error(void);
/* 0 if the current device is sm_90 (H100), else B200KGE_ERR_NO_DEVICE. */
int b200kge_device_ok(void);
/* Number of kernel launches issued by this library on the calling thread since the last reset
 * (bench.py reports it as gpu_launches). */
int64_t b200kge_launch_count(int reset);

/* Profiling aid (bench.py): when enabled, the dominant pairwise kernel of every 1-vs-N call on this
 * thread is bracketed by CUDA events recorded on the stream it is launched on;
 * b200kge_profile_last_ms synchronises on the closing event and returns that kernel's duration. */
int b200kge_profile_enable(int on);
int b200kge_profile_last_ms(float* ms);

/* Bytes of device workspace sufficient for any call below with n query rows (per direction), m
 * candidate rows and entity width D.  cand_has_idx != 0 reserves room to gather an index subset
 * of candidates for the tensor-core path. */
size_t b200kge_workspace_bytes(int model, int64_t n, int64_t m, int32_t D, int cand_has_idx);

/* Row-wise triples ---------------------------------------------------------------------------- */
/* out[i] = score(s_i, p_i, o_i).  Replaces KgeModel.score_spo kge_model.py:663-680 and
 * score_emb(combine="spo") of every in-scope scorer.  TransE adds eps=1e-6 to the difference like
 * F.pairwise_distance (transe.py:18). */
int b200kge_score_spo(int model, float l_norm, const b200kge_rows_t* s, const b200kge_rows_t* p,
                      const b200kge_rows_t* o, int64_t n, float* out, b200kge_stream_t stream);

/* 1-vs-N ---------------------------------------------------------------------------------------
 * out[i*ldo + j], i < n, j < cand->rows.  `q` are the per-row entity operands (subjects for sp_,
 * objects for _po), `p` the per-row relation operands, `cand` the candidate entities (all of them,
 * a contiguous chunk, or an index subset).  Replaces KgeModel.score_sp / score_po
 * kge_model.py:682-725 and score_emb(combine in {"sp_","_po"}). */
int b200kge_score_1vsN(int model, int combine, float l_norm, int precision,
                       const b200kge_rows_t* q, const b200kge_rows_t* p,
                       const b200kge_rows_t* cand, int64_t n, float* out, int64_t ldo,
                       void* workspace, size_t workspace_bytes, b200kge_stream_t stream);

/* out is [n, 2m] = [sp_ scores | _po scores], m = cand->rows.  Replaces KgeModel.score_sp_po
 * kge_model.py:749-789 (one launch sequence, no torch.cat copy). */
int b200kge_score_sp_po(int model, float l_norm, int precision, const b200kge_rows_t* s,
                        const b200kge_rows_t* p, const b200kge_rows_t* o,
                        const b200kge_rows_t* cand, int64_t n, float* out, int64_t ldo,
                        void* workspace, size_t workspace_bytes, b200kge_stream_t stream);

/* Fused 1-vs-N score + loss: the [n,m] scores never reach HBM.
 * loss_out[0] (device float) receives the SUM-reduced loss of the block exactly as
 * KgeLoss.__call__ returns it (the caller divides by batch size, train_1vsAll.py:65);
 * row_loss_out (optional, [n]) receives the per-row terms.  Replaces score_sp/score_po followed by
 * BCEWithLogitsKgeLoss / KLDivWithSoftmaxKgeLoss (train_1vsAll.py:64-65,75-76,
 * train_KvsAll.py:275-289). */
int b200kge_score_1vsN_loss(int model, int combine, float l_norm, int precision,
                            const b200kge_rows_t* q, const b200kge_rows_t* p,
                            const b200kge_rows_t* cand, int64_t n, const b200kge_labels_t* labels,
                            int loss_kind, float offset, float* loss_out, float* row_loss_out,
                            void* workspace, size_t workspace_bytes, b200kge_stream_t stream);

/* Fused 1-vs-N score + rank/tie counting against a chunk of candidates (additive over chunks,
 * eval_entity_ranking.py:222-229,310-313).  true_score[i] is the score of row i's true answer;
 * filter (optional) is the reference's dense label chunk [n, ldf] holding +inf at known-true
 * columns (own answer zeroed, :287-290) and is SUBTRACTED from the scores before comparing
 * (:561-566).  rank/ties are int64 [n] and are ACCUMULATED INTO (caller zeroes them before the
 * first chunk).  Replaces score_sp_po + _filter_and_rank + _get_ranks_and_num_ties :533-596. */
int b200kge_score_1vsN_rank(int model, int combine, float l_norm, int precision,
                            const b200kge_rows_t* q, const b200kge_rows_t* p,
                            const b200kge_rows_t* cand, int64_t n, const float* true_score,
                            const float* filter, int64_t ldf, float rtol, float atol,
                            int64_t* rank, int64_t* ties, void* workspace, size_t workspace_bytes,
                            b200kge_stream_t stream);

/* Both directions of the ranking of one batch in ONE launch sequence: rows 0..n-1 are the sp_ queries (ranked
 * against true_score[0..n)), rows n..2n-1 the _po queries (true_score[n..2n)); rank/ties are int64 [2n] in the
 * same order and are ACCUMULATED INTO; filter (optional) is [2n, ldf] in the same row order.  This is what
 * EntityRankingJob does per chunk with score_sp_po + _filter_and_rank + _get_ranks_and_num_ties
 * (eval_entity_ranking.py:222-229,533-596) without materialising the [n, 2m] scores.  CP (whose directions read
 * different candidate columns) returns B200KGE_ERR_UNSUPPORTED: call b200kge_score_1vsN_rank per direction. */
int b200kge_rank_sp_po(int model, float l_norm, int precision, const b200kge_rows_t* s,
                       const b200kge_rows_t* p, const b200kge_rows_t* o, const b200kge_rows_t* cand,
                       int64_t n, const float* true_score, const float* filter, int64_t ldf, float rtol,
                       float atol, int64_t* rank, int64_t* ties, void* workspace, size_t workspace_bytes,
                       b200kge_stream_t stream);

/* b200kge_rank_sp_po with the filter as CSR instead of a dense [2n, m] matrix: stacked row r lists the (sorted)
 * candidate columns filter_col[filter_off[r] .. filter_off[r+1]) that hold known answers; they are excluded from the
 * counts exactly like the reference's "+inf label subtracted" (eval_entity_ranking.py:489-531,561-566), except the
 * row's own answer own_col[r] (may be NULL; :287-290).  Columns are positions in `cand`, which must be a plain
 * table or chunk (cand->idx == NULL).  The CSR is consumed inside the scoring kernels' epilogues (pre-split tensor-core
 * kernels: one cursor per thread = row; CUDA-core kernel: one forward-moving cursor per owned row); CP and the in-kernel
 * split precision modes return B200KGE_ERR_UNSUPPORTED before anything is launched — pass the dense filter to
 * b200kge_rank_sp_po instead. */
int b200kge_rank_sp_po_csr(int model, float l_norm, int precision, const b200kge_rows_t* s,
                           const b200kge_rows_t* p, const b200kge_rows_t* o, const b200kge_rows_t* cand,
                           int64_t n, const float* true_score, const int64_t* filter_off,
                           const int64_t* filter_col, const int64_t* own_col, float rtol, float atol,
                           int64_t* rank, int64_t* ties, void* workspace, size_t workspace_bytes,
                           b200kge_stream_t stream);

/* Every ranking EntityRankingJob computes for one batch (raw, _filt and, with filter_with_test, _filt_test), from ONE
 * scoring pass over the whole entity table (eval_entity_ranking.py:184-315,533-596) without materialising scores or
 * label matrices.  ent / rel are the plain tables (idx == NULL), s / p / o the batch's n index triples (device int64);
 * the candidates are all rows of ent.  Rows are stacked as in b200kge_rank_sp_po: rows 0..n-1 the sp_ queries (s, p),
 * rows n..2n-1 the _po queries (p, o) — or, with num_relations = R > 0 (reciprocal relations, rel->rows == 2R), the sp_
 * queries (o, p + R) (reciprocal_relations_model.py:85-92).  Per stacked row r:
 *   true_score[r]   the score of the row's true answer; own_col[r] that answer (o for sp_ rows, s for _po rows);
 *   F               filter_col[filter_off[r] .. filter_off[r+1]): the known answers (entity_ranking.filter_splits),
 *                   sorted and unique per row (filter_col may be NULL when F is empty);
 *   T (optional)    test_col[test_off[r] .. test_off[r+1]): the test answers NOT in F, sorted and unique per row.
 * rank / ties are int64 [Rk][2n], Rk = 2 (raw, _filt) or 3 with T (_filt_test), and are ACCUMULATED INTO.  Raw counts
 * compare every column as b200kge_rank_sp_po; _filt counts every column of F except own_col as -inf (:286-290,561-566),
 * _filt_test every column of F and T except own_col (:277-307).  own_score [2n] receives the score computed at
 * own_col[r], for the reference's tie-handling consistency check (:240-274).  Workspace: b200kge_workspace_bytes(model,
 * n, ent->rows, ent->dim, 0).  CP runs its two directions as two launches.  The in-kernel split precision modes return
 * B200KGE_ERR_UNSUPPORTED before anything is launched. */
int b200kge_rank_sp_po_eval(int model, float l_norm, int precision, const b200kge_rows_t* ent,
                            const b200kge_rows_t* rel, int64_t num_relations, const int64_t* s, const int64_t* p,
                            const int64_t* o, int64_t n, const float* true_score, const int64_t* own_col,
                            const int64_t* filter_off, const int64_t* filter_col, const int64_t* test_off,
                            const int64_t* test_col, float rtol, float atol, int64_t* rank, int64_t* ties,
                            float* own_score, void* workspace, size_t workspace_bytes, b200kge_stream_t stream);

/* b200kge_score_sp_po FUSED WITH THE ALL-GATHER of an entity-sharded table: `cand` is this rank's shard; the two
 * halves are written at out[i*ldo + j] (sp_) and out[i*ldo + col_block + j] (_po), j < cand->rows, AND at the same
 * offsets into each of the n_peers (<= 7) buffers peer_out[g] — peer-mapped device pointers to the other ranks'
 * symmetric output buffers (NVLink / NVSwitch).  With out = base + lo (lo = first global row of the shard),
 * ldo = 2 * E_total and col_block = E_total every rank's [n, 2E_total] logits matrix (kge_model.py:749-789 layout)
 * is complete once all ranks have passed a barrier: the kernel's own epilogue stores replace ncclAllGather and the
 * re-layout copy.  CP is not offered. */
int b200kge_score_sp_po_bcast(int model, float l_norm, int precision, const b200kge_rows_t* s,
                              const b200kge_rows_t* p, const b200kge_rows_t* o, const b200kge_rows_t* cand,
                              int64_t n, float* out, float* const* peer_out, int n_peers, int64_t ldo,
                              int64_t col_block, void* workspace, size_t workspace_bytes,
                              b200kge_stream_t stream);

/* Entity-sharded tables (SURVEY 8e): this rank owns global rows [lo, lo + shard->rows) of the entity table.
 * out[i, :] = shard row (idx[i] - lo) if the rank owns global id idx[i], else zeros — the contribution of this rank
 * to the query-row exchange (sum over ranks == the gathered rows, exactly: every other rank adds zeros).  One
 * kernel, no host synchronisation (the reference's LookupEmbedder.embed, lookup_embedder.py:96-97, on a
 * partitioned table). */
int b200kge_shard_gather_rows(const b200kge_rows_t* shard, int64_t lo, const int64_t* idx, int64_t n,
                              float* out, int64_t ldo, b200kge_stream_t stream);

/* Dense-score epilogues (for callers that already hold a score matrix) ------------------------ */
/* KgeLoss on a dense [n,m] score matrix: loss.py:153-159 (BCE) / :198-213 (KL).  The row-wise kinds
 * (B200KGE_LOSS_BCE_MEAN and after) return B200KGE_ERR_UNSUPPORTED: use b200kge_ns_loss. */
int b200kge_loss_dense(const float* scores, int64_t lds, int64_t n, int64_t m,
                       const b200kge_labels_t* labels, int loss_kind, float offset,
                       float* loss_out, float* row_loss_out, void* workspace,
                       size_t workspace_bytes, b200kge_stream_t stream);

/* _get_ranks_and_num_ties on a dense [n,m] score matrix (eval_entity_ranking.py:571-596), with the
 * optional filter subtraction of _filter_and_rank (:561-566).  Bit-exact integer outputs;
 * ACCUMULATES INTO rank/ties. */
int b200kge_rank_dense(const float* scores, int64_t lds, int64_t n, int64_t m,
                       const float* true_score, const float* filter, int64_t ldf, float rtol,
                       float atol, int64_t* rank, int64_t* ties, b200kge_stream_t stream);

/* Negative sampling -----------------------------------------------------------------------------
 * out[i*ldo + k] = score of triple i with slot `slot` (0=S,1=P,2=O) replaced by neg[i*K + k].
 * The gather of the sampled rows is fused with the per-negative dot/distance.  If
 * with_positive != 0, column 0 of out receives score_spo of the positive triple and negatives go
 * to columns 1..K (the [n,1+K] assembly of train_negative_sampling.py:139-148).
 * Replaces BatchNegativeSample.score sampler.py:263-344 (both `triple` and `batch`
 * implementations give the same numbers; this computes them directly). */
int b200kge_ns_score(int model, float l_norm, const b200kge_rows_t* s, const b200kge_rows_t* p,
                     const b200kge_rows_t* o, const b200kge_rows_t* slot_table, int slot,
                     const int64_t* neg, int64_t n, int64_t K, int with_positive, float* out,
                     int64_t ldo, b200kge_stream_t stream);

/* On-device uniform negative sampling: out[i*K + k] ~ U{0, ..., vocab-1}, the device counterpart of
 * KgeUniformSampler._sample (kge/util/sampler.py:588-596: torch.randint on the CPU + a host->device copy of the ids).
 * Counter-based Philox4x32-10: the result depends on (seed, offset, position) only; use a fresh `offset` per call
 * (e.g. a batch counter) for independent draws.  Positives are not filtered here: b200kge_sample_uniform_filtered
 * does that. */
int b200kge_sample_uniform(uint64_t seed, uint64_t offset, int64_t vocab, int64_t n, int64_t K, int64_t* out,
                           b200kge_stream_t stream);

/* Filtered uniform negative sampling (negative_sampling.filtering.<slot>, kge/util/sampler.py:108-128,163-196,700-752):
 * out[i*K + k] ~ U({0..vocab-1} \ P_i), i.i.d., where P_i are the values of row i's key in a filter index.  The key of
 * row i of triples [n,3] (device, int64) is (p, o) for slot 0 (S), (s, o) for slot 1 (P), (s, p) for slot 2 (O).
 * The index (device, int64) is a CSR over keys [num_keys,2] in ascending lexicographic order: the values of key j are
 * values[offsets[j] .. offsets[j+1]), ascending, distinct, in [0, vocab) — what b200kge_filter_index_build returns.
 * Counter domains: element e = i*K + k first draws x exactly as b200kge_sample_uniform does (block (e/2, offset) under
 * key seed), so every position whose x is not a positive equals b200kge_sample_uniform's output bit for bit.  A
 * positive x is replaced by the u-th non-positive id, u = floor(r * (vocab - m) / 2^64) with m = |P_i| and r the same
 * word pair of block (e/2 | 2^63, offset) under key seed, a counter the first draw never uses.  The result depends on
 * (seed, offset, i, k) and the index only.  Rows whose key is absent are unfiltered; rows with m >= vocab receive -1. */
int b200kge_sample_uniform_filtered(uint64_t seed, uint64_t offset, int64_t vocab, int64_t n, int64_t K,
                                    const int64_t* triples, int slot, const int64_t* keys, const int64_t* offsets,
                                    const int64_t* values, int64_t num_keys, int64_t* out, b200kge_stream_t stream);

/* Frequency negative sampling (negative_sampling.sampling_type: frequency; KgeFrequencySampler, kge/util/sampler.py:755-793):
 * out[i*K + k] i.i.d. with P(x) = q_x / Q, where q are the integer weights of b200kge_frequency_cdf_build (proportional to
 * the slot's training counts plus the smoothing) and cdf [vocab+1] (device, uint64) is their exclusive prefix,
 * cdf[0] = 0, cdf[vocab] = Q.  Counter domain: element e = i*K + k takes exactly the 64-bit word r of
 * b200kge_sample_uniform (word pair e & 1 of Philox block (e/2, offset) under key seed), t = floor(r * Q / 2^64), and
 * the output is the largest x with cdf[x] <= t: each id's preimage is an interval of r, so P(x) = q_x / Q to within
 * 2^-64, and an id of zero weight is never drawn.  With all q_x equal the output is b200kge_sample_uniform's. */
int b200kge_sample_frequency(uint64_t seed, uint64_t offset, int64_t vocab, const uint64_t* cdf, int64_t n, int64_t K,
                             int64_t* out, b200kge_stream_t stream);

/* Filtered frequency negative sampling (filtering.<slot> with the standard implementation, sampler.py:108-128,163-196,
 * 755-793): out[i*K + k] i.i.d. with P(y) = q_y / (Q - M_i) over the non-positives y of row i's key, M_i the weight of
 * the key's positives: the law of the reference's redraw loop.  Triples, slot and filter index as in
 * b200kge_sample_uniform_filtered; cdf as in b200kge_sample_frequency; below [nnz] (device, uint64) is
 * b200kge_frequency_filter_build's output for this cdf and index.  Counter domains: each element first takes
 * b200kge_sample_frequency's draw x, so every position whose x is not a positive equals that entry's output bit for bit.
 * A positive x is replaced by one draw u = floor(r * (Q - M_i) / 2^64), r the same word pair of block (e/2 | 2^63,
 * offset), mapped to the id holding the u-th unit of non-positive weight.  No loop's length depends on chance.  Rows
 * whose key is absent are unfiltered; rows whose positives carry all the weight (Q - M_i = 0) receive -1.  With all
 * q_x equal the output is b200kge_sample_uniform_filtered's. */
int b200kge_sample_frequency_filtered(uint64_t seed, uint64_t offset, int64_t vocab, int64_t n, int64_t K,
                                      const int64_t* triples, int slot, const int64_t* keys, const int64_t* offsets,
                                      const int64_t* values, int64_t num_keys, const uint64_t* cdf,
                                      const uint64_t* below, int64_t* out, b200kge_stream_t stream);

/* ---- Embedding dropout of the 1vsAll / KvsAll training steps ---------------------------------------------------------
 * LookupEmbedder._postprocess (lookup_embedder.py:96-105) draws a fresh element-wise Bernoulli mask per embed(idx) /
 * embed_all() call and scales kept values by 1/(1-p).  One sub-batch of 1vsAll training (train_1vsAll.py:64,75 with
 * kge_model.py:682-721) makes six independent draws, numbered as mask streams:
 *   score_sp(s, p): 0 = embed(s), 1 = embed(p), 2 = embed_all()       (entity, relation, entity table)
 *   score_po(p, o): 3 = embed_all(), 4 = embed(p), 5 = embed(o)       (entity table, relation, entity)
 * so the two directions use different masks on the candidate table and on p.  KvsAll (train_KvsAll.py:274-285) draws
 * streams 0-2 for its sp_ queries and 3-5 for its _po queries; its s_o queries (score_so(s, o), kge_model.py:727-747)
 * draw three more, after streams 6-23 of negative sampling:
 *   score_so(s, o): 24 = embed(s), 25 = embed(o), 26 = embed_all() of the relations  (entity, entity, relation table)
 *
 * Mask layout (never stored: the backward regenerates the forward's mask from the same key):
 *   element (row, k) of a draw over rows of width dim has elem = row * dim + k, where row is the GLOBAL row: the entity
 *   id for the table draws (2, 3), the relation id for 26, row_base + i for row i of the sub-batch's queries (0, 1, 4,
 *   5, 24, 25);
 *   Philox4x32-10 with key = seed (64 bits) and counter = ((stream << 46) | (elem >> 2), call), both 64-bit halves
 *   little-endian as four 32-bit words; the element takes output word elem & 3;
 *   kept iff word < floor((1 - p) * 2^32), kept value x * (1 / (1 - p)) in fp32.
 * Requirements (else B200KGE_ERR_INVALID): 0 <= p < 1; row_base >= 0; elem < 2^48 for every element of every draw. */
#define B200KGE_DROP_SP_ENT 0
#define B200KGE_DROP_SP_REL 1
#define B200KGE_DROP_SP_TABLE 2
#define B200KGE_DROP_PO_TABLE 3
#define B200KGE_DROP_PO_REL 4
#define B200KGE_DROP_PO_ENT 5
#define B200KGE_DROP_SO_S 24
#define B200KGE_DROP_SO_O 25
#define B200KGE_DROP_SO_TABLE 26

typedef struct {
  float p_ent;      /* entity_embedder.dropout   */
  float p_rel;      /* relation_embedder.dropout */
  uint64_t seed;    /* Philox key                */
  uint64_t call;    /* one value per sub-batch (e.g. from epoch, batch index, sub-batch ordinal) */
  int64_t row_base; /* global index of the sub-batch's first query row */
} b200kge_dropout_t;

/* The keep mask of one draw: out[i * dim + k] = 1 if element (row_base + i, k) of stream `mask_stream` is kept, else 0,
 * for i < rows, k < dim (uint8, device). */
int b200kge_dropout_mask(float p, uint64_t seed, uint64_t call, int mask_stream, int64_t row_base, int64_t rows,
                         int32_t dim, uint8_t* out, b200kge_stream_t stream);

/* One whole 1vsAll forward step (train_1vsAll.py:48-82) for a batch of triples [n,3] (int64,
 * row-major s,p,o).  `ent`/`rel` are the device-resident tables (idx must be NULL).
 *   num_relations = 0: loss_out[0] (device) receives  (loss(score_sp, o) + loss(score_po, s)) / n.  Fused
 *     score_sp+loss and score_po+loss against the whole entity table, both directions stacked into one launch of 2n
 *     query rows where the model allows it.
 *   num_relations = R > 0: the step of a reciprocal-relations model.  LibKGE's ReciprocalRelationsModel
 *     (reciprocal_relations_model.py:85-92) keeps 2R relation rows and answers score_po as the sp_ query (o, p + R)
 *     against the same table, so loss_out[0] receives  (loss(score_sp(s, p), o) + loss(score_sp(o, p + R), s)) / n.
 *     rel->rows must be 2 * num_relations (else B200KGE_ERR_INVALID, as for num_relations < 0).  Without dropout this
 *     is the stacked problem with the rows [n, 2n) folded as sp_ queries (o_i, p_i + R), labelled s_i — CP included,
 *     which stacks here because both halves read the table columns [D/2, D).
 *   drop == NULL: no dropout.  Otherwise the six draws above are applied to gathered copies of the query rows, the
 *     relation rows and one table copy per direction, and each direction runs the per-direction scorer on those
 *     copies.  With num_relations > 0, direction 0 draws streams 0-2 as the plain step and direction 1 draws the _po
 *     streams 3-5 (embed_all, embed(p + R), embed(o)), with the mask rows of the plain step.
 * Every model and norm.  Workspace: b200kge_train_1vsall_workspace_bytes(model, n, E, D, drop != NULL); without
 * dropout b200kge_workspace_bytes(model, n, E, D, 0) is enough for the forward. */
int b200kge_train_1vsall_forward(int model, float l_norm, int precision, const b200kge_rows_t* ent,
                                 const b200kge_rows_t* rel, int64_t num_relations, const int64_t* triples, int64_t n,
                                 int loss_kind, float offset, const b200kge_dropout_t* drop, float* loss_out,
                                 void* workspace, size_t workspace_bytes, b200kge_stream_t stream);

/* Backward of b200kge_train_1vsall_forward (loss.backward() at kge/job/train_1vsAll.py:70,81) with BCE or KL and the
 * forward's num_relations and drop: dense gradients of the entity table d_ent [E, lde] and of the relation table d_rel
 * [R, ldr] (all 2R rows for a reciprocal-relations model) of the forward's loss.  Both buffers are OVERWRITTEN (the
 * reference accumulates into .grad; add them there).  Models: the dot family (tensor-core GEMMs) and TransE (l_norm 1,
 * 2) / RotatE (l_norm 1) (CUDA-core row-gradient passes, grad_distance.cu: dQ_i = sum_j G_ij s'(Q_i - T_j),
 * dT_j = sum_i G_ij s'(T_j - Q_i)).  Recompute-based: scores, G = n dL/dz (sigmoid(z+off) - y | softmax(z) - y), two
 * split-K tensor-core GEMMs on fp16 hi/lo planes (dT = G^T Q, dQ = G T), row-wise unfold of dQ through the relation
 * fold (grad.cu); the reciprocal half unfolds into d_ent[o], d_rel[p + R].  With `drop`, each direction runs that
 * machinery on its masked copies and the table and row gradients are masked with the same draws before they are added
 * into d_ent / d_rel.  Workspace: b200kge_train_1vsall_workspace_bytes(model, n, E, D, drop != NULL). */
int b200kge_train_1vsall_backward(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                                  int64_t num_relations, const int64_t* triples, int64_t n, int loss_kind, float offset,
                                  const b200kge_dropout_t* drop, float* d_ent, int64_t lde, float* d_rel, int64_t ldr,
                                  void* workspace, size_t workspace_bytes, b200kge_stream_t stream);

/* Bytes of workspace sufficient for b200kge_train_1vsall_forward and _backward with n triples, E entities of width D,
 * plain or reciprocal, with dropout (dropout != 0) or without. */
size_t b200kge_train_1vsall_workspace_bytes(int model, int64_t n, int64_t E, int32_t D, int dropout);

/* Host-buffer form of the plain forward step (end-to-end measurement, embedding in a host-side loop):
 * copies triples_host [n,3] to the device (triples.to(device), train_1vsAll.py:59), runs
 * b200kge_train_1vsall_forward, copies the scalar back to *loss_host (.item(), :66,77) and
 * synchronises the stream. */
int b200kge_train_1vsall_forward_host(int model, float l_norm, int precision,
                                      const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                                      const int64_t* triples_host, int64_t n, int loss_kind,
                                      float offset, float* loss_host, void* workspace,
                                      size_t workspace_bytes, b200kge_stream_t stream);

/* ---- host-side label plumbing (CPU; no device involved) ------------------------------------------
 * The key -> all-values index that KvsAll training and filtered entity ranking build their label and
 * filter coordinates from, in CSR form (row offsets + column ids) — what the device epilogues take
 * instead of coord_to_sparse_tensor(...).to_dense() (kge/job/util.py:32-60).
 *
 * b200kge_kvsall_index_build replaces KvsAllIndex.__init__ (kge/indexing.py:19-55,178-194):
 *   triples [n,3] (host), key columns (key_col0, key_col1) and value column = a permutation of 0,1,2.
 *   keys_out [n,2], offsets_out [n+1], values_out [n] are caller-allocated at capacity n;
 *   *num_keys receives the number of distinct keys.  Keys ascend lexicographically (np.unique axis=0),
 *   values ascend within a key, duplicate triples keep their duplicate values — element for element
 *   the reference's _keys / _values_offset / _values. */
int b200kge_kvsall_index_build(const int64_t* triples, int64_t n, int key_col0, int key_col1,
                               int value_col, int64_t* keys_out, int64_t* offsets_out,
                               int64_t* values_out, int64_t* num_keys);

/* KvsAllIndex.get_all (kge/indexing.py:113-166) and get_sp_po_coords_from_spo_batch
 * (kge/job/util.py:6-30): for each of nq query keys [nq,2] the values of that key (none if the key
 * is absent), as CSR: offsets_out [nq+1] (offsets_out[nq] = nnz), cols_out [nnz] = value +
 * col_shift (col_shift = num_entities for the po half of a [n, 2E] label matrix).  Call with
 * cols_out = NULL to size, then again with the buffer. */
int b200kge_kvsall_lookup(const int64_t* keys, const int64_t* offsets, const int64_t* values,
                          int64_t num_keys, const int64_t* query_keys, int64_t nq,
                          int64_t col_shift, int64_t* offsets_out, int64_t* cols_out);

/* The collate step of KvsAll training for one query type (kge/job/train_KvsAll.py:116-203): example
 * ids are key indexes; queries_out [nb,2] receives their keys, offsets_out [nb+1] / cols_out [nnz]
 * their labels as CSR (cols_out = NULL to size). */
int b200kge_kvsall_gather(const int64_t* keys, const int64_t* offsets, const int64_t* values,
                          int64_t num_keys, const int64_t* examples, int64_t nb,
                          int64_t* queries_out, int64_t* offsets_out, int64_t* cols_out);

/* The filter index of b200kge_sample_uniform_filtered from a key -> values index (host arrays: the _keys, _values_offset
 * and _values of a KvsAllIndex, widened to int64; keys may come in any order and repeat, values may repeat).
 * keys_out [num_keys,2], offsets_out [num_keys+1] and values_out [offsets[num_keys] - offsets[0]] are caller-allocated
 * at those capacities.  Keys come out sorted and unique, values sorted and unique per key; keys without values are
 * dropped.  *num_keys_out receives the number of keys, *max_count the largest number of values of one key.
 * B200KGE_ERR_INVALID if the offsets decrease or a value lies outside [0, vocab). */
int b200kge_filter_index_build(const int64_t* keys, const int64_t* offsets, const int64_t* values, int64_t num_keys,
                               int64_t vocab, int64_t* keys_out, int64_t* offsets_out, int64_t* values_out,
                               int64_t* num_keys_out, int64_t* max_count);

/* The weights of frequency sampling (host arrays; KgeFrequencySampler.__init__, sampler.py:762-780 defines them as
 * w_x = counts[x] + smoothing over the slot's training counts).  The library samples from integer weights
 * q_x = round((counts[x] + smoothing) * 2^s), rounded half to even, where s >= 0 is the largest integer with
 * Q = sum q_x <= 2^62: exactly proportional to w for an integral smoothing, and with a relative error per id of at
 * most 2^-62 * Q / q_x otherwise.  cdf_out [vocab+1] receives the exclusive prefix of q (cdf_out[0] = 0, cdf_out[vocab] = Q).
 * B200KGE_ERR_INVALID for vocab <= 0, a negative count, a negative or non-finite smoothing, Q = 0 (smoothing 0 and no
 * id counted) or smoothed counts summing to more than 2^62. */
int b200kge_frequency_cdf_build(const int64_t* counts, int64_t vocab, double smoothing, uint64_t* cdf_out);

/* The per-entry table of b200kge_sample_frequency_filtered (host arrays): for every value v_j of every key of a filter
 * index (b200kge_filter_index_build's offsets / values), below_out[j - offsets[0]] = cdf[v_j] - sum_{l<j} q_{v_l}, the
 * weight of the key's non-positives below v_j.  *num_full receives the number of keys whose positives carry all the
 * weight (no negative can be drawn for them), *first_full the index of the first such key or -1.  B200KGE_ERR_INVALID
 * for a cdf that does not start at 0, decreases or ends at 0, decreasing offsets (checked before any value is read), or
 * values of a key that are not ascending, distinct and in [0, vocab). */
int b200kge_frequency_filter_build(const uint64_t* cdf, int64_t vocab, const int64_t* offsets, const int64_t* values,
                                   int64_t num_keys, uint64_t* below_out, int64_t* num_full, int64_t* first_full);

/* ---- SURVEY 8(f) rows: gradients, penalties, CSR labels -------------
 *
 * b200kge_gemm_nt: C[M,N] = A[M,K] * B[N,K]^T, fp32 in / fp32 out, computed on the f16 tensor pipe from
 * hi/lo fp16 planes split once in HBM (presplit.cu + pairwise_tc3.cu) — the building block of the
 * backward GEMMs; fp32-equivalent (operand error ~5e-7 of the result's rms).  Reductions longer than 512 run
 * split-K: 512-element segments accumulated in fp32, which bounds the tensor core's accumulator error. */
size_t b200kge_gemm_nt_workspace_bytes(int64_t M, int64_t N, int64_t K);
int b200kge_gemm_nt(const float* A, int64_t lda, const float* B, int64_t ldb, int64_t M, int64_t N,
                      int64_t K, float* C, int64_t ldc, void* workspace, size_t workspace_bytes,
                      b200kge_stream_t stream);

/* Backward of b200kge_score_1vsN over the whole entity table for the dot family (the unfused route: a job computes a
 * dense [n, E] score matrix, its loss, and autograd hands back grad_scores = dL/dscores [n, ldg]): dense gradients of
 * the entity table d_ent [E, lde] and the relation table d_rel [R, ldr], both OVERWRITTEN.  Fold of the n query rows,
 * fp16 hi/lo planes of grad_scores and of its transpose, two split-K tensor-core GEMMs (dT = G^T Q, dQ = G T) and the
 * row-wise unfold — no cuBLAS, no [n, E, D] intermediate. */
size_t b200kge_score_1vsN_backward_workspace_bytes(int model, int64_t n, int64_t E, int32_t D);
int b200kge_score_1vsN_backward(int model, int combine, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                                const int64_t* q_idx, const int64_t* p_idx, int64_t n, const float* grad_scores,
                                int64_t ldg, float* d_ent, int64_t lde, float* d_rel, int64_t ldr, void* workspace,
                                size_t workspace_bytes, b200kge_stream_t stream);

/* Backward of b200kge_score_1vsN_loss_csr / batch_size (loss_value.backward() at kge/job/train_KvsAll.py:294): dense
 * gradients d_ent [E, lde], d_rel [R, ldr] (OVERWRITTEN) of  sum_i loss(score row i, y_i) / batch_size with
 * y = (1 - eps) * count + (eps > 0 ? 1/E : 0) from the CSR labels (sorted per row; a repeated column counts as often as
 * it appears).
 *   dot family: recompute, G planes written with the label-free value everywhere and patched at the nnz listed
 *     entries, two split-K tensor-core GEMMs, unfold.
 *   TransE (l_norm 1, 2) / RotatE (l_norm 1): recompute on the CUDA-core scorer, dense fp32 G (label-free value, then
 *     each row's listed columns by the row's own thread block; KL: row log-sum-exp first), the two row-gradient passes
 *     of b200kge_train_1vsall_backward, unfold.  Other norms: B200KGE_ERR_UNSUPPORTED before any launch.
 *   l_norm is ignored by the dot family.
 * drop == NULL: no dropout, and mask_dir is ignored.  Workspace: b200kge_score_1vsN_backward_workspace_bytes (the
 * distance family: Q, dQ [n, round_up(D, 32)] each, triples [3n] and the KL row statistics [2n floats] in its n * 4 * 8
 * bytes, scores and G [n, round_up(E, 4)] each, G^T [E, round_up(n, 4)], the scorer's workspace).
 * drop != NULL: the backward of b200kge_score_1vsN_loss_csr_dropout under the same key and mask_dir (same models and
 * norms).  The masks are regenerated, and the table and row gradients of the masked copies are masked with the same
 * draws before they are added into d_ent / d_rel.  Workspace: b200kge_score_1vsN_loss_csr_dropout_workspace_bytes. */
int b200kge_score_1vsN_loss_csr_backward(int model, int combine, int mask_dir, float l_norm, const b200kge_rows_t* ent,
                                         const b200kge_rows_t* rel, const int64_t* q_idx, const int64_t* p_idx,
                                         int64_t n, const int64_t* csr_off, const int64_t* csr_col,
                                         float label_smoothing, int loss_kind, float offset, int64_t batch_size,
                                         const b200kge_dropout_t* drop, float* d_ent, int64_t lde, float* d_rel,
                                         int64_t ldr, void* workspace, size_t workspace_bytes, b200kge_stream_t stream);

/* KvsAll loss with CSR multi-hot labels (kge/job/train_KvsAll.py:242-300 without the densified label matrix):
 * row i's labels are the columns csr_col[csr_off[i] .. csr_off[i+1]) (sorted; a repeated column counts as often
 * as it appears, like duplicate triples in the reference), optionally smoothed: y = (1 - eps) * count + 1/m.
 * *loss_out = sum_i loss(score row i, y_i) (BCE with offset | KL), row_loss_out (optional) the per-row terms.
 * On the pre-split tensor-core path (dot family) ONE fused pass scores, reduces the label-free loss terms and emits
 * the nnz listed scores from its epilogue (per-thread cursor into the row's sorted segment); elsewhere the listed
 * scores come from the row-wise triple kernel.  cand must be a plain table.  With eps > 0 the row sums sum_j z_ij come
 * from Q_i . colsum(T) (dot family) or from the CUDA-core scoring pass itself (TransE, RotatE: one partial per row and
 * column chunk, no second pass over the table).  Sizes: b200kge_score_1vsN_loss_csr_workspace_bytes. */
size_t b200kge_score_1vsN_loss_csr_workspace_bytes(int model, int64_t n, int64_t m, int32_t D, int64_t nnz);
int b200kge_score_1vsN_loss_csr(int model, int combine, float l_norm, int precision,
                                  const b200kge_rows_t* q, const b200kge_rows_t* p,
                                  const b200kge_rows_t* cand, int64_t n, const int64_t* csr_off,
                                  const int64_t* csr_col, int64_t nnz, float label_smoothing, int loss_kind,
                                  float offset, float* loss_out, float* row_loss_out, void* workspace,
                                  size_t workspace_bytes, b200kge_stream_t stream);

/* KgeLoss of a negative-sampling block (kge/job/train_negative_sampling.py:126-156 with kge/util/loss.py:139-274):
 * scores [n, m] (row stride lds), one positive per row at column label_idx[i] (NULL: column 0, the layout of
 * b200kge_ns_score with with_positive = 1), every other column a negative (label 0).  Any b200kge_loss kind; `arg` is
 * the offset of the BCE kinds and the margin of B200KGE_LOSS_MARGIN_RANKING (ignored otherwise), `temperature` that of
 * B200KGE_LOSS_BCE_SELF_ADV (user.bce_self_adversarial_temperature, loss.py:64-68).  The row-wise kinds need m >= 2.
 *   *loss_out       = scale * sum_i loss_i  (fixed-order reduction: deterministic)
 *   row_loss_out[i] = loss_i                (optional)
 *   grad_out[i*ldg + c] = scale * dL_i/dz_ic  (optional, [n, m]): the margin-ranking hinge passes the gradient at
 *                     exactly 0 as torch's clamp_min does; the self-adversarial weights are treated as constants
 *                     (detached, loss.py:179-181).
 * workspace: b200kge_ns_loss_workspace_bytes(n). */
size_t b200kge_ns_loss_workspace_bytes(int64_t n);
int b200kge_ns_loss(const float* scores, int64_t lds, int64_t n, int64_t m, const int64_t* label_idx,
                    int loss_kind, float arg, float temperature, float scale, float* loss_out,
                    float* row_loss_out, float* grad_out, int64_t ldg, void* workspace,
                    size_t workspace_bytes, b200kge_stream_t stream);

/* LookupEmbedder.penalty (kge/model/embedder/lookup_embedder.py:123-177) on the rows view `rows` (the whole
 * table, or the batch's unique rows through rows->idx with their `counts`, NULL = all ones):
 *   *out = scale * sum_r counts[r] * sum_k |x_rk|^p        (complex_abs: x -> sqrt(re^2 + im^2 + 1e-14): "n3",
 *   which the reference accepts in complex space only, lookup_embedder.py:29-34)
 * scale = regularize_weight / p (unweighted) or regularize_weight / p / len(indexes) (weighted).
 * workspace: (ceil(rows / 8) + 1) floats.  Deterministic (fixed-order two-stage sum). */
int b200kge_lookup_penalty(const b200kge_rows_t* rows, const float* counts, float p, int complex_abs,
                             float scale, float* out, void* workspace, size_t workspace_bytes,
                             b200kge_stream_t stream);

/* LookupEmbedder._normalize_embeddings (:64-69): rows of weight [rows, dim] (row stride ld) scaled in place to
 * unit Lp norm (torch.nn.functional.normalize, eps 1e-12). */
int b200kge_normalize_rows(float* weight, int64_t ld, int64_t rows, int32_t dim, float p,
                             b200kge_stream_t stream);

/* b200kge_score_1vsN_loss_csr with dropout for one KvsAll query type: queries ent[q_idx], relations rel[p_idx] and the
 * candidate table ent.  `combine` is the query type's fold; `mask_dir` (B200KGE_SP_ | B200KGE__PO) selects the draws:
 * streams 0-2 (queries 0, relations 1, table 2) | 3-5 (table 3, relations 4, queries 5).  A plain model's query type
 * draws with mask_dir = combine; a reciprocal-relations model's _po query type is the sp_ fold of (q_idx = o,
 * p_idx = p + R) on the _po streams (reciprocal_relations_model.py:85-92).  The backward is
 * b200kge_score_1vsN_loss_csr_backward with the same drop and mask_dir.
 * Workspace (either call): b200kge_score_1vsN_loss_csr_dropout_workspace_bytes (the masked copies and per-direction
 * buffers, then the larger of the forward's and the backward's workspace). */
size_t b200kge_score_1vsN_loss_csr_dropout_workspace_bytes(int model, int64_t n, int64_t E, int32_t D, int64_t nnz);
int b200kge_score_1vsN_loss_csr_dropout(int model, int combine, int mask_dir, float l_norm, int precision,
                                        const b200kge_rows_t* ent, const b200kge_rows_t* rel, const int64_t* q_idx,
                                        const int64_t* p_idx, int64_t n, const int64_t* csr_off, const int64_t* csr_col,
                                        int64_t nnz, float label_smoothing, int loss_kind, float offset,
                                        const b200kge_dropout_t* drop, float* loss_out, float* row_loss_out,
                                        void* workspace, size_t workspace_bytes, b200kge_stream_t stream);

/* KvsAll's s_o query type (relation prediction: train_KvsAll.py:251-254,278-281 with score_so, kge_model.py:727-747)
 * for the dot family.  Row i is the pair (ent[s_idx[i]], ent[o_idx[i]]) scored against every relation r of rel; its
 * labels are the relation ids csr_col[csr_off[i] .. csr_off[i+1]) (sorted; a repeated id counts as often as it
 * appears).  There is no label smoothing: the reference never smooths the relation targets (train_KvsAll.py:263).
 * The pair is folded into one query row Q_i (width K = the relation width: D, D/2 for CP, D^2 for RESCAL) with
 * score(s_i, r, o_i) = Q_i . rel[r]:
 *   DistMult s*o;  ComplEx [s_re*o_re + s_im*o_im | s_re*o_im - s_im*o_re];  SimplE 1/2 [s[:h]*o[h:] | s[h:]*o[:h]];
 *   CP s[:h]*o[h:];  RESCAL Q[r*D + c] = s_r o_c (the row-major relation matrix).
 * The relation table is then the candidate table of b200kge_score_1vsN_loss_csr's steps: on the pre-split tensor-core
 * path (precision auto: 32 <= K <= 1024 and n >= 16) one fused pass scores, reduces and emits the listed scores;
 * elsewhere the listed scores come from the row-wise triple kernel on (s_i, r, o_i).
 *   *loss_out = sum_i loss(score row i, y_i) (BCE with offset | KL), row_loss_out (optional) the per-row terms.
 * TransE and RotatE return B200KGE_ERR_UNSUPPORTED before any launch; l_norm is not used.
 * drop != NULL: embedding dropout with the key's masks on streams 24 (s rows, p_ent), 25 (o rows, p_ent) and 26 (the
 * relation table, p_rel), applied to masked copies of the operands.
 * Workspace: b200kge_score_so_loss_csr_workspace_bytes(model, n, R, D, nnz, drop != NULL), R = rel->rows. */
size_t b200kge_score_so_loss_csr_workspace_bytes(int model, int64_t n, int64_t R, int32_t D, int64_t nnz, int dropout);
int b200kge_score_so_loss_csr(int model, float l_norm, int precision, const b200kge_rows_t* ent,
                              const b200kge_rows_t* rel, const int64_t* s_idx, const int64_t* o_idx, int64_t n,
                              const int64_t* csr_off, const int64_t* csr_col, int64_t nnz, int loss_kind, float offset,
                              const b200kge_dropout_t* drop, float* loss_out, float* row_loss_out, void* workspace,
                              size_t workspace_bytes, b200kge_stream_t stream);

/* Backward of b200kge_score_so_loss_csr / batch_size under the same drop: d_ent [E, lde] and d_rel [R, ldr], both
 * OVERWRITTEN.  Fold, recompute, G planes of [n, R] patched at the listed entries, dT = G^T Q stored into d_rel,
 * dQ = G rel (split-K tensor-core GEMMs, as b200kge_score_1vsN_loss_csr_backward), then the fold's VJP added
 * atomically into d_ent[s_i] and d_ent[o_i] (with dropout: masked with the forward's draws first).
 * Workspace: b200kge_score_so_loss_csr_workspace_bytes (nnz is not used by the backward). */
int b200kge_score_so_loss_csr_backward(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                                       const int64_t* s_idx, const int64_t* o_idx, int64_t n, const int64_t* csr_off,
                                       const int64_t* csr_col, int loss_kind, float offset, int64_t batch_size,
                                       const b200kge_dropout_t* drop, float* d_ent, int64_t lde, float* d_rel,
                                       int64_t ldr, void* workspace, size_t workspace_bytes, b200kge_stream_t stream);

/* ---- Embedding dropout of the negative-sampling training step ------------------------------------------------------
 * Per slot (0 = S or 2 = O; the P slot is not served) and sub-batch, train_negative_sampling.py:139-148 makes six draws,
 * numbered as mask streams 6 + 6 * slot + j (streams 12-17, the P slot's, are reserved):
 *   j = 0, 1, 2  score_spo(s, p, o) of the positive column: the s, p and o rows, mask row = row_base + i
 *   j = 3, 4, 5  the negatives' s, p and o draws:
 *     B200KGE_NS_TRIPLE (score_spo over the n K corrupted triples, sampler.py:291-306): mask row = (row_base + i) K + j'
 *                       for all three operands of triple (i, j'), the sampled entity included;
 *     B200KGE_NS_BATCH  (score_sp / score_po against the unique sampled ids, sampler.py:307-356; `all` draws the same
 *                       distribution): mask row = row_base + i for the two fixed operands, the ENTITY ID for the open
 *                       slot, so every row and repeat that samples an id shares its mask.
 * Everything else is the layout above (key, counter, threshold, scale).  Rows are global within the batch, so the masks
 * do not depend on the sub-batch size.  Requirements (else B200KGE_ERR_INVALID): those of b200kge_dropout_mask for every
 * element of every draw, i.e. (mask row + 1) * width <= 2^48 with width D for entities and the relation width (D^2 for
 * RESCAL) for relations. */
#define B200KGE_NS_TRIPLE 0
#define B200KGE_NS_BATCH 1

/* b200kge_ns_score of one slot with dropout: out [n, 1 + K] (row stride ldo) receives the masked positive in column 0 and
 * the masked negatives neg [n, K] after it.  `ent` / `rel` are the plain tables, `triples` [n, 3] the sub-batch.
 * Coverage: slots S and O; the dot family (RESCAL included), TransE l_norm 1 / 2, RotatE l_norm 1; every row width a
 * multiple of 4 (D % 8 == 0 for ComplEx, SimplE, CP and RotatE).  Anything else returns B200KGE_ERR_UNSUPPORTED before
 * a launch.  TransE adds pairwise_distance's eps to the positive and `triple` scores, not to `batch` ones (cdist). */
int b200kge_ns_score_dropout(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                             const int64_t* triples, int slot, const int64_t* neg, int64_t n, int64_t K, int impl,
                             const b200kge_dropout_t* drop, float* out, int64_t ldo, b200kge_stream_t stream);

/* Backward of one slot of a negative-sampling batch (kge/job/train_negative_sampling.py:113-164): the [n, 1+K] block of
 * the slot (column 0 = the positive triple, label 1; columns 1.. = the sampled ids neg [n,K], label 0).  ADDS into
 * d_ent [E, lde] and d_rel [R, ldr] (zero them before the first slot).  slot 0 (S) or 2 (O); TransE with l_norm 1 or 2,
 * RotatE with l_norm 1, and the dot family.  Where dL/dz comes from:
 *   grad_scores == NULL: BCE with `offset`, the loss summed and divided by batch_size; the kernel computes the gradient.
 *   grad_scores [n, 1+K] (row stride ldg): dL/dz already scaled (e.g. the grad_out of b200kge_ns_loss with
 *     scale = 1 / batch_size); offset and batch_size are not used.  The fold, per-column walk, scatter and unfold are
 *     the BCE form's; only the per-column gradient is read instead of computed — so every loss of b200kge_ns_loss
 *     trains through the same kernel (loss.backward() at train_negative_sampling.py:164).
 *   drop != NULL: the backward of b200kge_ns_score_dropout under the same key and `impl` (impl is ignored without
 *     drop); grad_scores is required (else B200KGE_ERR_INVALID).  The masks are regenerated, the gradients of the
 *     masked operands are masked and scaled again and added.  Same coverage as that forward; B200KGE_NS_BATCH (not
 *     RESCAL) also needs D <= 1024.  The positive column and `triple` run row-wise (one warp per triple); the `batch`
 *     negatives run ns_kernel / ns_backward_kernel with a mask policy (q folded once per row from the masked fixed rows,
 *     sampled rows masked by id, the fixed rows' gradient reduced per row).
 * workspace: b200kge_ns_backward_workspace_bytes(model, n, K, D, drop != NULL) bytes (K is not used; without dropout
 * n * round_up(K_folded, 32) floats are used). */
size_t b200kge_ns_backward_workspace_bytes(int model, int64_t n, int64_t K, int32_t D, int dropout);
int b200kge_ns_backward(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                        const int64_t* triples, int slot, const int64_t* neg, int64_t n, int64_t K, int impl,
                        const b200kge_dropout_t* drop, const float* grad_scores, int64_t ldg, float offset,
                        int64_t batch_size, float* d_ent, int64_t lde, float* d_rel, int64_t ldr, void* workspace,
                        size_t workspace_bytes, b200kge_stream_t stream);

/* b200kge_ns_backward with each table's gradient in the layout of LibKGE's lookup_embedder.sparse (nn.Embedding with
 * sparse=True): the operands, coverage and refusals are b200kge_ns_backward's.  Per table, `*_sparse`:
 *   0: d_ent [E, lde] / d_rel [R, ldr] is the dense gradient, ADDED into as by b200kge_ns_backward; rows / count unused.
 *   1: row-sparse.  rows receives the sorted unique rows the reference looks up for the slot, *count (device, int64) their
 *      number u, and rows 0 .. u-1 of the value block d_ent / d_rel (same leading dimension) their gradients,
 *      OVERWRITTEN; rows past u are not touched.  Entity rows: the positives' s and o and every sampled id, at most
 *      min(E, n (K + 2)); relation rows: the positives' p, at most min(R, n) (R = rel->rows, so a reciprocal-relations
 *      S slot passed as (o, p + R', s) lists p + R').  rows and the value block must hold that many rows.  A row is in
 *      the set whether or not dropout zeroes its elements; ids repeated within the slot are summed.
 * The row set costs one [V] int32 map per sparse table (flags, an exclusive scan, compaction) in the workspace; no
 * untouched row of a sparse table is read or written.  Tables of 2^31 rows or more return B200KGE_ERR_UNSUPPORTED.
 * workspace: b200kge_ns_backward_sparse_workspace_bytes(model, n, K, D, E, R, drop != NULL). */
size_t b200kge_ns_backward_sparse_workspace_bytes(int model, int64_t n, int64_t K, int32_t D, int64_t E, int64_t R,
                                                  int dropout);
int b200kge_ns_backward_sparse(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                               const int64_t* triples, int slot, const int64_t* neg, int64_t n, int64_t K, int impl,
                               const b200kge_dropout_t* drop, const float* grad_scores, int64_t ldg, float offset,
                               int64_t batch_size, int ent_sparse, int64_t* ent_rows, int64_t* ent_count, float* d_ent,
                               int64_t lde, int rel_sparse, int64_t* rel_rows, int64_t* rel_count, float* d_rel,
                               int64_t ldr, void* workspace, size_t workspace_bytes, b200kge_stream_t stream);

/* Backward of the P slot of a negative-sampling batch (relation negatives; train_negative_sampling.py:139-164 with
 * sampler.py:263-356 through score_so): row i of the [n, 1+K] block scores (s_i, r, o_i) for r = p_i (column 0) and for
 * the K sampled relation ids neg [n, K].  grad_scores [n, 1+K] (row stride ldg) is dL/dz, required for every loss (BCE
 * included: the grad_out of b200kge_ns_loss with scale = 1 / batch_size).
 * The score depends on (i, r) only, so G is first summed exactly into C [n, R] with C[i, r] = the sum of row i's
 * columns whose id is r; the backward is then the all-relations backward with weights C:
 *   dot family (ComplEx, DistMult, SimplE, CP, RESCAL): the s_o fold Q [n, K_r], d_rel = C^T Q and dQ = C rel on the
 *     split-K tensor-core GEMMs, the s_o unfold into the rows s_i and o_i;
 *   TransE (l_norm 1, 2) and RotatE (l_norm 1): the VJP of the row score over the nonzero C[i, r] on the CUDA cores,
 *     one block per row for the entity rows and one per (relation, chunk of rows) for the relation rows.
 * No per-sample contribution is added atomically into the relation table.  Per table, `*_sparse`:
 *   0: d_ent [E, lde] / d_rel [R, ldr] is the dense gradient, ADDED into; rows / count unused.
 *   1: row-sparse, as b200kge_ns_backward_sparse: rows receives the sorted unique rows the reference looks up for the
 *      slot, *count (device, int64) their number u, and rows 0 .. u-1 of the value block their gradients, OVERWRITTEN.
 *      Entity rows: the positives' s and o, at most min(E, 2n); relation rows: the positives' p and every sampled id,
 *      at most min(R, n (K + 1)).  (With the reference's `implementation: all` score_so looks up every relation row:
 *      pass rel_sparse = 0 and read the dense gradient as the values of all R rows.)
 * Ids must lie in their tables.  Other models and norms, R > B200KGE_NS_P_MAX_RELATIONS and tables of 2^31 rows or
 * more return B200KGE_ERR_UNSUPPORTED before any launch; there is no dropout form.
 * workspace: b200kge_ns_p_backward_workspace_bytes(model, n, K, D, E, R): C [n, R] floats, four [n] id vectors, the
 * row-set maps, and the dot family's fold and GEMM operands (about 2 n R + R K_r + 3 n K_r floats beyond C) or the
 * distance family's relation partials (at most max(R, 4096) K_r floats).  0 for R > B200KGE_NS_P_MAX_RELATIONS. */
#define B200KGE_NS_P_MAX_RELATIONS 4096
size_t b200kge_ns_p_backward_workspace_bytes(int model, int64_t n, int64_t K, int32_t D, int64_t E, int64_t R);
int b200kge_ns_p_backward(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                          const int64_t* triples, const int64_t* neg, int64_t n, int64_t K, const float* grad_scores,
                          int64_t ldg, int ent_sparse, int64_t* ent_rows, int64_t* ent_count, float* d_ent, int64_t lde,
                          int rel_sparse, int64_t* rel_rows, int64_t* rel_count, float* d_rel, int64_t ldr,
                          void* workspace, size_t workspace_bytes, b200kge_stream_t stream);

/* ---- Shared negative sampling (negative_sampling.shared: True) -------------------------------------------------------
 * Every row of a batch draws its K negatives for slot 0 (S) or 2 (O) from the same num_unique = U' distinct entity ids
 * unique [U'] (KgeUniformSampler._sample_shared, sampler.py:597-698).  Column 1 + c of row i holds the sample
 * j = c < U ? c : repeat[c - U] (repeat [K - U], indexes into [0, U)), and the id unique[u(i, c)] with
 *   drop == NULL ("naive", U = U'):          u = j                                        (sampler.py:412-463)
 *   drop [n] ("default", U = U' - 1):        u = (j == drop[i]) ? U : j, drop[i] in [0, U] (sampler.py:503-578)
 * drop is the sub-batch's slice of the batch's drop_index; unique and repeat are the batch's.  Every column's score is
 * a score against one of the U' shared rows, so the slot is the dense problem Z [n, U'] (row i's fixed pair against
 * unique[u]) plus a gather of its columns, and its backward is a dense backward with the block's gradient summed per
 * shared id:  C[i, u] = sum over the columns c with u(i, c) = u of G[i, 1 + c].
 * impl: B200KGE_NS_TRIPLE or B200KGE_NS_BATCH (the reference's `batch` and `all`).  It matters to TransE, whose `triple`
 * scores go through F.pairwise_distance and add its eps = 1e-6 to the difference (transe.py:18): folded into the query as
 * s + p + eps (O slot) or o - p - eps (S slot); `batch` scores are cdist, without eps.  The positive column is
 * score_spo, with eps, in every case.  Coverage: the dot family, TransE (l_norm 1, 2), RotatE (l_norm 1), a folded
 * width of at most 1024, tables of fewer than 2^31 rows; anything else returns B200KGE_ERR_UNSUPPORTED before a launch.
 * Requirements (else B200KGE_ERR_INVALID): U >= 1 when K > U, K >= U, ids inside their tables. */

/* The [n, 1 + K] block of one slot into out (row stride ldo >= 1 + K): column 0 the positive triple (score_spo), columns
 * 1.. the assembled negatives.  Z is the 1-vs-N scorer against the gathered shared rows (the pre-split tensor-core path
 * where `precision` and the shape allow it, else the CUDA-core scorer), written to z_out [n, ldz >= U'] when z_out is
 * not NULL (b200kge_ns_shared_backward needs it for TransE l_norm 2).
 * workspace: b200kge_ns_shared_score_workspace_bytes(model, n, U', D). */
size_t b200kge_ns_shared_score_workspace_bytes(int model, int64_t n, int64_t num_unique, int32_t D);
int b200kge_ns_shared_score(int model, float l_norm, int precision, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                            const int64_t* triples, int slot, const int64_t* unique, int64_t num_unique,
                            const int64_t* repeat, const int64_t* drop, int64_t n, int64_t K, int impl, float* out,
                            int64_t ldo, float* z_out, int64_t ldz, void* workspace, size_t workspace_bytes,
                            b200kge_stream_t stream);

/* Backward of b200kge_ns_shared_score's block: grad_scores [n, 1 + K] (row stride ldg) is dL/dz, e.g. the grad_out of
 * b200kge_ns_loss with scale = 1 / batch_size.  C is summed from it per row, in column order, without atomics; then
 *   dot family: the query fold Q, the shared rows T gathered, dT = C^T Q and dQ = C T on the split-K tensor-core GEMMs
 *     (the backward block with C as its gradient), dT ADDED into the U' distinct rows unique[u], dQ unfolded;
 *   TransE (l_norm 1, 2), RotatE (l_norm 1): the distance row-gradient passes with weights C (divided by z for
 *     l_norm 2: z [n, ldz] is the z_out of the forward, required there), the same adds and unfold;
 * and the positive column's VJP per row.  No per-sample contribution is added atomically into the shared rows.
 * Per table, `*_sparse` as b200kge_ns_p_backward (0: dense, ADDED into; 1: row-sparse, rows / *count / the first *count
 * value rows OVERWRITTEN) with the rows the reference looks up for the slot: entities the positives' s and o plus
 * every shared id (B200KGE_NS_BATCH: score_sp / score_po(..., unique)) or the shared ids the sub-batch's rows use
 * (B200KGE_NS_TRIPLE), at most min(E, 2n + U'); relations the positives' p, at most min(R, n).  (`implementation: all`
 * looks up every entity row: pass ent_sparse = 0.)
 * workspace: b200kge_ns_shared_backward_workspace_bytes(model, n, U', D, E, R). */
size_t b200kge_ns_shared_backward_workspace_bytes(int model, int64_t n, int64_t num_unique, int32_t D, int64_t E,
                                                  int64_t R);
int b200kge_ns_shared_backward(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                               const int64_t* triples, int slot, const int64_t* unique, int64_t num_unique,
                               const int64_t* repeat, const int64_t* drop, int64_t n, int64_t K, int impl,
                               const float* z, int64_t ldz, const float* grad_scores, int64_t ldg, int ent_sparse,
                               int64_t* ent_rows, int64_t* ent_count, float* d_ent, int64_t lde, int rel_sparse,
                               int64_t* rel_rows, int64_t* rel_count, float* d_rel, int64_t ldr, void* workspace,
                               size_t workspace_bytes, b200kge_stream_t stream);

/* ---- Optimizer steps: torch.optim.Adagrad and torch.optim.SparseAdam (torch 2.11) on one fp32 parameter ----------------
 * param and its state tensors are [rows, dim], contiguous.  The gradient is
 *   dense      (grad_rows == NULL): grad [rows, dim], contiguous; nnz and coalesced are unused;
 *   row-sparse (a torch.sparse_coo_tensor with one sparse dimension): grad_rows [nnz] row ids and grad [nnz, dim] their
 *              value rows.  coalesced != 0 promises sorted unique ids (torch's is_coalesced()): the block is read in
 *              place and no workspace is needed.  Otherwise ids may repeat in any order; their rows are summed (in
 *              any order, with atomics) into a [min(rows, nnz), dim] block of the workspace first, over the row set of
 *              the ids (rowset.cu); tables of 2^31 rows or more then return B200KGE_ERR_UNSUPPORTED.
 * Rows not in a sparse gradient are neither read nor written.  Every operation rounds to nearest in the order written
 * below, with a single rounding exactly where torch's compiled kernels use an FMA (fma(...) below); with a dense or
 * coalesced gradient the result is then torch's bit for bit, as far as torch's kernels keep that rounding.
 * The caller computes the scalars in double precision, as torch does, and passes them rounded to float.
 * workspace: b200kge_optim_step_workspace_bytes(rows, dim, nnz, coalesced) (0 for a coalesced gradient; pass
 * coalesced = 1 for a dense one).  NULL operands, negative sizes and a short workspace are refused before any launch. */
size_t b200kge_optim_step_workspace_bytes(int64_t rows, int64_t dim, int64_t nnz, int coalesced);

/* One parameter of torch.optim.Adagrad.step() (adagrad.py), after the caller has incremented the step and computed
 * clr = lr / (1 + (step - 1) lr_decay).  Dense: g' = fma(weight_decay, p, g) when weight_decay != 0,
 * sum = fma(g', g', sum), then
 *   foreach_order != 0 (_multi_tensor_adagrad, torch's default on CUDA):  p = p + (g' (-clr)) / (sqrt(sum) + eps)
 *   foreach_order == 0 (_single_tensor_adagrad: foreach=False, or a group with a sparse gradient on the device):
 *                                                                        p = fma(g' / (sqrt(sum) + eps), -clr, p)
 * Row-sparse, per row of the coalesced gradient, value v: sum = sum + v v, p = p + (-clr) (v / (sqrt(sum) + eps)),
 * every operation rounded on its own; weight_decay != 0 is refused
 * (B200KGE_ERR_INVALID, torch's "weight_decay option is not compatible with sparse gradients"). */
int b200kge_adagrad_step(float* param, float* state_sum, int64_t rows, int64_t dim, const float* grad,
                         const int64_t* grad_rows, int64_t nnz, int coalesced, int foreach_order, float clr, float eps,
                         float weight_decay, void* workspace, size_t workspace_bytes, b200kge_stream_t stream);

/* One parameter of torch.optim.SparseAdam.step() (_functional.sparse_adam) with the step t already incremented and
 * step_size = lr sqrt(1 - beta2^t) / (1 - beta1^t).  one_minus_beta1 / one_minus_beta2 are 1 - beta computed in double,
 * as torch's scalars are.  Per row of the coalesced gradient, value v:
 *   m_u = (v - m)(1 - beta1), m += m_u;  q_u = (v v - q)(1 - beta2), q += q_u;
 *   p += (-step_size) ((m_u + m_old) / (sqrt(q_u + q_old) + eps))
 * with m = exp_avg, q = exp_avg_sq.  A dense gradient (grad_rows == NULL) is refused (B200KGE_ERR_INVALID). */
int b200kge_sparse_adam_step(float* param, float* exp_avg, float* exp_avg_sq, int64_t rows, int64_t dim,
                             const float* grad, const int64_t* grad_rows, int64_t nnz, int coalesced,
                             float one_minus_beta1, float one_minus_beta2, float eps, float step_size, void* workspace,
                             size_t workspace_bytes, b200kge_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200KGE_H_ */
