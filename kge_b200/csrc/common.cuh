// common.cuh — shared host/device helpers of libb200kge (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "../../include/b200kge.h"

namespace b200kge {

// ---------------------------------------------------------------------------------------------
// Host-side error plumbing (capi.cu owns the storage).
void set_error(const char* fmt, ...);
void count_launch(int n = 1);
int check_cuda(cudaError_t e, const char* what);
// profiling brackets around the dominant kernel (no-ops unless b200kge_profile_enable(1))
void profile_begin(cudaStream_t st);
void profile_end(cudaStream_t st);

#define B2K_CUDA(expr)                                             \
  do {                                                             \
    int _s = ::b200kge::check_cuda((expr), #expr);                 \
    if (_s != 0) return _s;                                        \
  } while (0)

#define B2K_LAUNCH_CHECK(name)                                     \
  do {                                                             \
    ::b200kge::count_launch();                                     \
    int _s = ::b200kge::check_cuda(cudaGetLastError(), name);      \
    if (_s != 0) return _s;                                        \
  } while (0)

// ---------------------------------------------------------------------------------------------
// Device view of b200kge_rows_t.
struct Rows {
  const float* base;
  const int64_t* idx;
  int64_t rows;
  int64_t ld;
  int dim;
  __host__ __device__ __forceinline__ const float* row(int64_t i) const {
    return base + (idx ? idx[i] : i) * ld;
  }
};

inline Rows to_rows(const b200kge_rows_t* r) {
  Rows v;
  v.base = r->base; v.idx = r->idx; v.rows = r->rows; v.ld = r->ld; v.dim = r->dim;
  return v;
}

// How a pair (query row, candidate row) is reduced over the feature dimension.
enum PairOp : int {
  PAIR_DOT = 0,      // sum q*t                          (ComplEx, DistMult, SimplE, CP, RESCAL)
  PAIR_L1 = 1,       // -sum |q-t|                       (TransE l_norm=1)
  PAIR_L2 = 2,       // -sqrt(sum (q-t)^2)               (TransE l_norm=2)
  PAIR_LP = 3,       // -(sum |q-t|^p)^(1/p)             (TransE other p)
  PAIR_CMOD_L1 = 4,  // -sum_k |q_k - t_k| complex       (RotatE l_norm=1)
  PAIR_CMOD_LP = 5   // -(sum_k |q_k-t_k|^p)^(1/p)       (RotatE other p)
};

// Folded problem: score(i, j) = pair(Q[i, 0:K], cand_j[col_off : col_off+K]).
struct Folded {
  int pair_op;
  int K;        // reduction length in floats (complex pair ops: K = 2h, re at k, im at k+h)
  int col_off;  // first candidate column used
};

__host__ __device__ inline int relation_dim(int model, int D) {
  if (model == B200KGE_CP || model == B200KGE_ROTATE) return D / 2;
  if (model == B200KGE_RESCAL) return D * D;
  return D;
}

// ---------------------------------------------------------------------------------------------
// Epilogues.  A kernel computes x = score(row, col) for a tile and hands every valid element to
// one of these functors; per-row state lives in registers and is flushed once per (row, chunk).
enum EpiKind : int { EPI_STORE = 0, EPI_BCE = 1, EPI_KL = 2, EPI_RANK = 3, EPI_RANK_EVAL = 4, EPI_BCE_ZSUM = 5, EPI_KL_ZSUM = 6 };

// EPI_BCE_ZSUM / EPI_KL_ZSUM (CUDA-core kernel only): the BCE / KL epilogue plus the row's plain score sum sum_j z_ij,
// which label smoothing of the CSR-label losses needs (the distance family has no Q . colsum(T) identity for it)
__host__ __device__ constexpr int epi_loss_base(int kind) {
  return kind == EPI_BCE_ZSUM ? EPI_BCE : (kind == EPI_KL_ZSUM ? EPI_KL : kind);
}

struct FinalizeArgs;
struct EpiParams {
  // EPI_STORE
  float* out;
  int64_t ldo;
  // losses
  const int64_t* label_idx;
  const float* label_dense;
  int64_t ldl;
  float offset;
  float* part;        // [n][nchunks][F] partial row states
  int nchunks;
  // rank
  const float* true_score;
  const float* filter;
  int64_t ldf;
  float rtol, atol;
  unsigned long long* rank;
  unsigned long long* ties;
  // row remapping for the fused sp_po launch: logical query row r (0..2n) maps to output row
  // r % n_rows_out and column block (r / n_rows_out) * col_block
  int64_t n_rows_out;
  int64_t col_block;
  // EPI_STORE, GEMM use (pairwise_tc3.cu split-K): add into `out` (zeroed by the caller) instead of overwriting it
  int accumulate_out;
  // CSR side input (SURVEY 8f-2): row r lists the sorted columns csr_col[csr_off[r] .. csr_off[r+1]) (duplicates
  // allowed).  Losses: the raw scores at the listed columns are written to csr_out[t] (t = position in csr_col) —
  // the multi-hot label terms are then sums over nnz values, no [n, m] label matrix exists (train_KvsAll.py:242-266);
  // with csr_extra the score of column 0 of row r goes to csr_out[csr_nnz + r] (KL: lse_i - z_i0 comes back from
  // the one-hot-at-0 pass).  Rank: listed columns are filtered (score -> -inf, eval_entity_ranking.py:561-566)
  // except the row's own answer csr_skip[r] (:287-290).  Candidate columns must be table rows (cand.idx == NULL).
  const int64_t* csr_off;
  const int64_t* csr_col;
  float* csr_out;
  int64_t csr_nnz;
  int csr_extra;
  const int64_t* csr_skip;
  // EPI_STORE fused with the all-gather of an entity-sharded table (SURVEY 8e): every score is also stored, at the
  // same offset, into the symmetric output buffers of the n_peers other ranks (peer-mapped pointers over
  // NVLink / NVSwitch) — the shard's logits land in place in everybody's [n, 2E] matrix, no NCCL all-gather, no
  // re-layout copy
  float* out_peer[7];
  int n_peers;
  int store_vec4;      // set by launch_pairwise_simt: every destination row start is 16-byte aligned
  // EPI_RANK_EVAL (all rankings of EntityRankingJob from one pass, eval_entity_ranking.py:277-313): csr_off / csr_col
  // list the known answers F of each row and csr_skip its own answer; csr2_off / csr2_col (optional) the test answers
  // not in F.  Both lists are sorted and unique per row.  rank / ties hold n_rank rows of rank_ld counters (raw,
  // _filt[, _filt_test]); own_score[r] receives the score at column csr_skip[r].
  const int64_t* csr2_off;
  const int64_t* csr2_col;
  int64_t rank_ld;
  int n_rank;
  float* own_score;
  // EPI_BCE_ZSUM / EPI_KL_ZSUM: zsum_part[row * nchunks + chunk] = the chunk's sum of the row's scores
  float* zsum_part;
};

// lower bound of `key` in the sorted segment col[lo, hi)
__device__ __forceinline__ int64_t csr_lower_bound(const int64_t* __restrict__ col, int64_t lo, int64_t hi, int64_t key) {
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (__ldg(col + mid) < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

#define B2K_NEG_HUGE (-3.0e38f)

__device__ __forceinline__ float softplus_f(float z) {
  // max(z,0) + log1p(exp(-|z|)), matching torch's BCEWithLogits formulation (loss.py:150)
  // branch-free (a data-dependent branch here diverges per element and cost +40 % kernel time):
  // log1p(e) ~= e for tiny e (where 1+e would round to 1), else log(1+e); both arms are already
  // computed, so the compiler emits a select.
  const float e = __expf(-fabsf(z));
  const float lg = __logf(1.0f + e);
  const float l = (e < 1e-5f) ? e : lg;
  return fmaxf(z, 0.0f) + l;
}

template <int KIND> struct RowState {};

template <> struct RowState<EPI_STORE> {
  static constexpr int F = 0;
  __device__ __forceinline__ void init() {}
};

// BCE: a = sum softplus(z), b = sum y*z            loss.py:153-159
template <> struct RowState<EPI_BCE> {
  static constexpr int F = 2;
  float a, b;
  __device__ __forceinline__ void init() { a = 0.f; b = 0.f; }
  __device__ __forceinline__ void combine(const RowState& o) { a += o.a; b += o.b; }
};

// KL / CE: online (m, s) for logsumexp, plus label sums   loss.py:198-213
//   y_sum = sum y, yx = sum y*x, ylogy = sum y*log(y)
template <> struct RowState<EPI_KL> {
  static constexpr int F = 5;
  float m, s, y_sum, yx, ylogy;
  __device__ __forceinline__ void init() { m = B2K_NEG_HUGE; s = 0.f; y_sum = 0.f; yx = 0.f; ylogy = 0.f; }
  __device__ __forceinline__ void combine(const RowState& o) {
    float mn = fmaxf(m, o.m);
    s = s * __expf(m - mn) + o.s * __expf(o.m - mn);
    m = mn;
    y_sum += o.y_sum; yx += o.yx; ylogy += o.ylogy;
  }
};

// the loss state of BASE plus the plain score sum
template <int BASE> struct RowStateZsum : RowState<BASE> {
  float zs;
  __device__ __forceinline__ void init() { RowState<BASE>::init(); zs = 0.f; }
  __device__ __forceinline__ void combine(const RowStateZsum& o) { RowState<BASE>::combine(o); zs += o.zs; }
};
template <> struct RowState<EPI_BCE_ZSUM> : RowStateZsum<EPI_BCE> {};
template <> struct RowState<EPI_KL_ZSUM> : RowStateZsum<EPI_KL> {};

// rank / ties counters     eval_entity_ranking.py:571-596
template <> struct RowState<EPI_RANK> {
  static constexpr int F = 0;
  unsigned int greater, close;
  __device__ __forceinline__ void init() { greater = 0u; close = 0u; }
  __device__ __forceinline__ void combine(const RowState& o) { greater += o.greater; close += o.close; }
};

// EPI_RANK_EVAL: every ranking of one row (eval_entity_ranking.py:277-313).  The row state holds the raw counts over all
// columns, which the flush adds to every ranking; the listed columns of a tile correct the filtered rankings right away
// (RankFix).  Both are integers, so the sums are exact whatever their order.
template <> struct RowState<EPI_RANK_EVAL> {
  static constexpr int F = 0;
  unsigned int greater, close;
  __device__ __forceinline__ void init() { greater = 0u; close = 0u; }
  __device__ __forceinline__ void combine(const RowState& o) { greater += o.greater; close += o.close; }
};

// torch.isclose(x, t, rtol, atol) for fp32 operands (equal_nan=False), evaluated in fp32 exactly
// as ATen does: (x == t) | (isfinite(|x-t|) & (|x-t| <= atol + |rtol*t|)).
__device__ __forceinline__ bool isclose_f(float x, float t, float rtol, float atol) {
  float allowed = __fadd_rn(atol, fabsf(__fmul_rn(rtol, t)));
  float actual = fabsf(__fsub_rn(x, t));
  return (x == t) || (isfinite(actual) && actual <= allowed);
}

// The corrections of one row's listed columns within one tile: a filtered column becomes score - inf = -inf (:565-566),
// which is never greater and is close iff the true score is -inf, so each listed column swaps its raw contribution for
// that one.  f* correct _filt and _filt_test (columns of F), t* _filt_test only (test answers not in F).
struct RankFix {
  unsigned int fg, fc, tg, tc;     // greater counts taken out; close counts put in minus taken out (wrap-around)
  __device__ __forceinline__ RankFix() : fg(0u), fc(0u), tg(0u), tc(0u) {}
  __device__ __forceinline__ void add(bool test, float x, float t, float rtol, float atol) {
    if (isnan(x)) x = -INFINITY;
    const bool c = isclose_f(x, t, rtol, atol);
    const unsigned int gt = (!c && x > t) ? 1u : 0u;
    const unsigned int dcl = (t == -INFINITY ? 1u : 0u) - (c ? 1u : 0u);
    if (test) { tg += gt; tc += dcl; }
    else      { fg += gt; fc += dcl; }
  }
  // rank / ties rows 1 (_filt) and 2 (_filt_test) as signed deltas: the 64-bit sums wrap back to the exact counts once
  // the flushes of the raw counts have landed
  __device__ __forceinline__ void commit(const EpiParams& P, int64_t row) const {
    const long long g1 = -(long long)fg, c1 = (long long)(int)fc;
    if (g1) atomicAdd(P.rank + P.rank_ld + row, (unsigned long long)g1);
    if (c1) atomicAdd(P.ties + P.rank_ld + row, (unsigned long long)c1);
    if (P.n_rank > 2) {
      const long long g2 = g1 - (long long)tg, c2 = c1 + (long long)(int)tc;
      if (g2) atomicAdd(P.rank + 2 * P.rank_ld + row, (unsigned long long)g2);
      if (c2) atomicAdd(P.ties + 2 * P.rank_ld + row, (unsigned long long)c2);
    }
  }
};

template <int KIND>
__device__ __forceinline__ void epi_elem(const EpiParams& P, RowState<KIND>& st, int64_t row,
                                         int64_t col, float x, float row_aux) {
  if constexpr (KIND == EPI_STORE) {
    int64_t r = row, cb = 0;
    if (P.n_rows_out > 0 && row >= P.n_rows_out) { r = row - P.n_rows_out; cb = P.col_block; }
    const int64_t at = r * P.ldo + cb + col;
    P.out[at] = x;
    for (int g = 0; g < P.n_peers; ++g) P.out_peer[g][at] = x;
  } else if constexpr (KIND == EPI_BCE) {
    float z = x + P.offset;
    st.a += softplus_f(z);
    if (P.label_dense) {
      st.b = fmaf(P.label_dense[row * P.ldl + col], z, st.b);
    } else if (col == (int64_t)__float_as_int(row_aux)) {
      st.b += z;
    }
  } else if constexpr (KIND == EPI_KL) {
    float mn = fmaxf(st.m, x);
    st.s = st.s * __expf(st.m - mn) + __expf(x - mn);
    st.m = mn;
    if (P.label_dense) {
      float y = P.label_dense[row * P.ldl + col];
      if (y != 0.f) {
        st.y_sum += y;
        st.yx = fmaf(y, x, st.yx);
        st.ylogy = fmaf(y, __logf(y), st.ylogy);
      }
    } else if (col == (int64_t)__float_as_int(row_aux)) {
      st.y_sum += 1.0f;
      st.yx += x;
    }
  } else if constexpr (KIND == EPI_RANK) {
    float v = x;
    if (P.filter) v = __fsub_rn(v, P.filter[row * P.ldf + col]);   // :561-566
    if (isnan(v)) v = -INFINITY;                                    // :583-584
    bool c = isclose_f(v, row_aux, P.rtol, P.atol);
    st.close += c ? 1u : 0u;
    st.greater += (!c && v > row_aux) ? 1u : 0u;
  } else if constexpr (KIND == EPI_RANK_EVAL) {            // raw counts; the lists are corrected per tile
    const float v = isnan(x) ? -INFINITY : x;
    const bool c = isclose_f(v, row_aux, P.rtol, P.atol);
    st.close += c ? 1u : 0u;
    st.greater += (!c && v > row_aux) ? 1u : 0u;
  } else if constexpr (KIND == EPI_BCE_ZSUM || KIND == EPI_KL_ZSUM) {
    epi_elem<epi_loss_base(KIND)>(P, st, row, col, x, row_aux);
    st.zs += x;
  }
}

// Per-row auxiliary scalar loaded once per (thread,row): label index (as int bits; rows are
// < 2^31 candidates per call) or the NaN-cleaned true score.
template <int KIND>
__device__ __forceinline__ float epi_row_aux(const EpiParams& P, int64_t row) {
  if constexpr (epi_loss_base(KIND) == EPI_BCE || epi_loss_base(KIND) == EPI_KL) {
    return P.label_idx ? __int_as_float((int)P.label_idx[row]) : __int_as_float(-1);
  } else if constexpr (KIND == EPI_RANK || KIND == EPI_RANK_EVAL) {
    float t = P.true_score[row];
    return isnan(t) ? -INFINITY : t;                                // :585-586
  } else {
    return 0.f;
  }
}

template <int KIND>
__device__ __forceinline__ void epi_flush(const EpiParams& P, const RowState<KIND>& st,
                                          int64_t row, int chunk) {
  if constexpr (KIND == EPI_BCE) {
    float* p = P.part + (row * P.nchunks + chunk) * 2;
    p[0] = st.a; p[1] = st.b;
  } else if constexpr (KIND == EPI_KL) {
    float* p = P.part + (row * P.nchunks + chunk) * 5;
    p[0] = st.m; p[1] = st.s; p[2] = st.y_sum; p[3] = st.yx; p[4] = st.ylogy;
  } else if constexpr (KIND == EPI_RANK) {
    // integer atomics: order-independent, hence bit-exact
    if (st.greater) atomicAdd(P.rank + row, (unsigned long long)st.greater);
    if (st.close) atomicAdd(P.ties + row, (unsigned long long)st.close);
  } else if constexpr (KIND == EPI_RANK_EVAL) {
    // the raw counts enter every ranking; the listed columns' corrections were committed per tile (RankFix)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (k >= P.n_rank) break;
      if (st.greater) atomicAdd(P.rank + k * P.rank_ld + row, (unsigned long long)st.greater);
      if (st.close) atomicAdd(P.ties + k * P.rank_ld + row, (unsigned long long)st.close);
    }
  } else if constexpr (KIND == EPI_BCE_ZSUM || KIND == EPI_KL_ZSUM) {
    epi_flush<epi_loss_base(KIND)>(P, st, row, chunk);
    P.zsum_part[row * P.nchunks + chunk] = st.zs;
  }
}

// Combine the states of the `width` (power of two <= 32) adjacent lanes that share a row.
template <int KIND>
__device__ __forceinline__ void epi_lane_reduce(RowState<KIND>& st, int width) {
  if constexpr (KIND != EPI_STORE) {
    constexpr int W = sizeof(RowState<KIND>) / 4;
    for (int off = width >> 1; off > 0; off >>= 1) {
      RowState<KIND> o;
      uint32_t* src = reinterpret_cast<uint32_t*>(&st);
      uint32_t* dst = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int w = 0; w < W; ++w) dst[w] = __shfl_xor_sync(0xffffffffu, src[w], off);
      st.combine(o);
    }
  }
}


// ---------------------------------------------------------------------------------------------
// Deterministic finaliser of the fused losses: partial[n][nchunks][F] -> row loss -> scalar.
// Fixed reduction order at every level (lanes over chunks -> shuffle tree, rows per warp in
// order, warps per block in order, blocks in index order by the last block): the result does not
// depend on scheduling.
struct FinalizeArgs {
  const float* part;
  int nchunks;
  int64_t n;
  float* loss_out;
  float* row_loss_out;
  float scale;
  int accumulate;
  unsigned int* ticket;   // zero-initialised counter for the last-block-done protocol
  float* block_sums;      // [gridDim.x] scratch
};

template <int LOSS>
__device__ __forceinline__ float finalize_row(const float* __restrict__ part, int nchunks, int64_t r) {
  if constexpr (LOSS == B200KGE_LOSS_BCE) {
    float a = 0.f, b = 0.f;
    for (int c = 0; c < nchunks; ++c) {
      const float* p = part + (r * nchunks + c) * 2;
      a += p[0]; b += p[1];
    }
    return a - b;                       // sum softplus(z) - sum y*z
  } else {
    RowState<EPI_KL> st;
    st.init();
    for (int c = 0; c < nchunks; ++c) {
      const float* p = part + (r * nchunks + c) * 5;
      RowState<EPI_KL> o;
      o.m = p[0]; o.s = p[1]; o.y_sum = p[2]; o.yx = p[3]; o.ylogy = p[4];
      st.combine(o);
    }
    const float lse = st.m + logf(st.s);
    // KLDiv(log_softmax(x), y / max(||y||_1, 1e-12)), reduction sum   loss.py:209-213
    const float yc = fmaxf(st.y_sum, 1e-12f);
    const float w = st.y_sum / yc;
    return (st.y_sum > 0.f) ? (st.ylogy / yc - w * logf(yc) - st.yx / yc + lse * w) : 0.f;
  }
}


// ---------------------------------------------------------------------------------------------
// Internal kernels' host launchers (one per .cu file).
int launch_fold_queries(int model, int combine, const Rows& q, const Rows& p, int64_t n,
                        int64_t row0, float* Q, int64_t ldq, cudaStream_t st);
// s_o fold of the dot family (fold.cu): Q [n, ldq] with score(s_i, r, o_i) = Q_i . rel[r][0 : relation_dim(model, D)]
int launch_fold_so(int model, const Rows& s, const Rows& o, int64_t n, float* Q, int64_t ldq, cudaStream_t st);
// its VJP: dQ row i ADDED into dS[s_dst[i]] and dO[o_dst[i]] (a NULL index array: row i)
int launch_unfold_so(int model, const Rows& s, const Rows& o, int64_t n, const float* dQ, int64_t ldq, float* dS,
                     int64_t lds, const int64_t* s_dst, float* dO, int64_t ldo, const int64_t* o_dst, cudaStream_t st);
// one launch: unpack triples [n,3], fold sp_ rows (0..n) and _po rows (n..2n) into Q, write the
// stacked labels [o ; s] and zero the finalisation ticket.  num_rel > 0 (reciprocal relations): rows n..2n fold
// (o, p + num_rel) with the sp_ fold instead
int launch_prep_1vsall(int model, const Rows& ent, const Rows& rel, const int64_t* triples, int64_t n,
                       float* Q, int64_t ldq, int64_t* labels2n, unsigned int* ticket, cudaStream_t st,
                       int64_t num_rel = 0);
int launch_gather_rows(const Rows& src, int col_off, int K, float* dst, int64_t ldd,
                       cudaStream_t st);
int launch_pairwise_simt(int epi_kind, int pair_op, float l_norm, const float* Q, int64_t ldq,
                         int64_t nq, const Rows& cand, int col_off, int K, const EpiParams& P,
                         cudaStream_t st);
int pairwise_simt_nchunks(int64_t nq, int64_t m);
// tensor-core path: returns B200KGE_ERR_UNSUPPORTED if the shape cannot be served.
bool tc_supported(int pair_op, int K, const Rows& cand, int col_off);
int tc_nchunks(int64_t nq, int64_t m);
int launch_pairwise_tc(int epi_kind, int passes, const float* Q, int64_t ldq,
                       int64_t nq, const float* T, int64_t ldt, int64_t m, int K,
                       const EpiParams& P, cudaStream_t st);
// scratch: >= 1024 bytes of device memory (128 block sums + ticket); ticket_zeroed: the caller already
// zeroed the ticket word at scratch+512 on this stream (else a 4-byte memset is enqueued)
int launch_loss_finalize(int loss_kind, const float* part, int nchunks, int64_t n, float* loss_out,
                         float* row_loss_out, float scale, int accumulate, void* scratch,
                         int ticket_zeroed, cudaStream_t st);
int launch_spo(int model, float l_norm, const Rows& s, const Rows& p, const Rows& o, int64_t n,
               float* out, int64_t out_stride, cudaStream_t st);
int launch_ns(int model, float l_norm, const Rows& s, const Rows& p, const Rows& o,
              const Rows& table, int slot, const int64_t* neg, int64_t n, int64_t K, float* out,
              int64_t ldo, int col0, cudaStream_t st);
int launch_sample_uniform(uint64_t seed, uint64_t offset, int64_t vocab, int64_t total, int64_t* out, cudaStream_t st);
// launch_sample_uniform's draws with the positives of each row's key replaced (b200kge_sample_uniform_filtered)
int launch_sample_uniform_filtered(uint64_t seed, uint64_t offset, int64_t vocab, int64_t n, int64_t K,
                                   const int64_t* triples, int slot, const int64_t* keys, const int64_t* offsets,
                                   const int64_t* values, int64_t num_keys, int64_t* out, cudaStream_t st);
// frequency-weighted draws over cdf[0..vocab] (b200kge_sample_frequency / _filtered)
int launch_sample_frequency(uint64_t seed, uint64_t offset, int64_t vocab, const uint64_t* cdf, int64_t total,
                            int64_t* out, cudaStream_t st);
int launch_sample_frequency_filtered(uint64_t seed, uint64_t offset, int64_t vocab, int64_t n, int64_t K,
                                     const int64_t* triples, int slot, const int64_t* keys, const int64_t* offsets,
                                     const int64_t* values, int64_t num_keys, const uint64_t* cdf,
                                     const uint64_t* below, int64_t* out, cudaStream_t st);
int launch_loss_dense(int loss_kind, const float* scores, int64_t lds, int64_t n, int64_t m,
                      const EpiParams& P, cudaStream_t st);
int loss_dense_nchunks(int64_t m);
int launch_rank_dense(const float* scores, int64_t lds, int64_t n, int64_t m, const EpiParams& P,
                      cudaStream_t st);

// Dropout masks (dropout.cu; layout in include/b200kge.h): one draw = one (stream, key).  Element (r, k) of a draw over
// rows [row_base, row_base + rows) is kept iff its Philox word is below `thresh`; kept values are scaled by `scale`.
struct DropMask {
  uint64_t seed, call;
  uint64_t thresh;      // floor((1 - p) * 2^32); 2^32 keeps everything
  float scale;          // 1 / (1 - p)
  int stream;
  int64_t row_base;
};
int launch_dropout_mask(const DropMask& m, int64_t rows, int dim, uint8_t* out, cudaStream_t st);
// dst[i, k] = mask(row_base + i, k) * src.row(i)[k]   (i < src.rows, k < src.dim)
int launch_dropout_gather(const DropMask& m, const Rows& src, float* dst, int64_t ldd, cudaStream_t st);
// dst[r, k] += mask(row_base + r, k) * src[r, k] for r < rows, k in [c0, c1) (row width `dim` keys the mask)
int launch_dropout_add_cols(const DropMask& m, const float* src, int64_t lds, int64_t rows, int dim, int c0, int c1,
                            float* dst, int64_t ldd, cudaStream_t st);
// dst[idx[i], k] += mask(row_base + i, k) * src[i, k]   (atomic: rows of idx may repeat)
int launch_dropout_scatter(const DropMask& m, const float* src, int64_t lds, int64_t rows, int dim, const int64_t* idx,
                           float* dst, int64_t ldd, cudaStream_t st);
// tri[3 i + j] = i: the triples under which the row-wise unfold writes row i's gradient into row i of [n, D] buffers
int launch_identity_triples(int64_t n, int64_t* tri, cudaStream_t st);

// ns_kernel with dropout on the `batch` negatives (rowwise.cu): the fixed rows of triples [n, 3] (entity, draw ma;
// relation, draw mp) masked at mask row row_base + i, each sampled row by its entity id (draw mt); scores into
// out[i * ldo + col0 + k].  ent / rel are the plain tables.
int launch_ns_masked(int model, float l_norm, const Rows& ent, const Rows& rel, const int64_t* triples, int slot,
                     const int64_t* neg, int64_t n, int64_t K, const DropMask& ma, const DropMask& mp, const DropMask& mt,
                     float* out, int64_t ldo, int col0, cudaStream_t st);
// ns_backward_kernel with the same masks (grad.cu): a and p are [n, D] / [n, Dr] masked copies of the fixed rows (plain
// rows, row i of the sub-batch), so the fold and the unfold run unchanged and the row gradients land in dA / dP
// (OVERWRITTEN); the sampled rows' gradients are masked and scattered into d_ent (pe: into row pe[e]).  Columns 1..K of
// G only.
int launch_ns_backward_masked(int model, float l_norm, const Rows& a, const Rows& p, const Rows& table, int slot,
                              const int64_t* neg, int64_t n, int64_t K, const DropMask& mt, const float* G, int64_t ldg,
                              float* d_ent, int64_t lde, float* dQ, int64_t ldq, int64_t* tri_ws, float* dA, float* dP,
                              cudaStream_t st, const int32_t* pe = nullptr);
// Dropout of one negative-sampling slot (ns_dropout.cu): the entity and relation draws' key and rate (stream and
// row_base are set per draw) and the sub-batch's first global row.
struct NsDropKeys {
  DropMask ent, rel;
  int64_t row_base;
};
// G == NULL: scores of the [n, 1+K] block into out (positive in column 0); else the backward of that block with
// grad_scores G, ADDED into d_ent / d_rel.  impl: B200KGE_NS_TRIPLE | B200KGE_NS_BATCH.
// workspace: ns_dropout_workspace_bytes (the backward of the `batch` negatives only; the rest needs none).  pe / pr (both
// or neither): row maps of the backward, as launch_ns_backward's.
size_t ns_dropout_workspace_bytes(int model, int64_t n, int32_t D);
int launch_ns_dropout(int model, float l_norm, const Rows& ent, const Rows& rel, const int64_t* triples, int slot,
                      const int64_t* neg, int64_t n, int64_t K, int impl, const NsDropKeys& keys, const float* G,
                      int64_t ldg, float* out, int64_t ldo, float* d_ent, int64_t lde, float* d_rel, int64_t ldr,
                      void* workspace, size_t workspace_bytes, cudaStream_t st, const int32_t* pe = nullptr,
                      const int32_t* pr = nullptr);

// Row set of a row-sparse table gradient (rowset.cu).  ids[i * stride], i < count: one list of looked-up rows.
struct IdList {
  const int64_t* ids;
  int64_t count, stride;
};
// workspace of launch_row_set over V rows: the [V] int32 row map first, then per-tile counts
size_t row_set_workspace_bytes(int64_t V);
// The sorted unique ids of the lists into rows[0 .. u) and u into *count (device); the map at the start of the workspace
// gets map[id] = the id's row in [0, u) for every listed id (other entries undefined); the first u rows of vals [*, ld]
// are zeroed.
int launch_row_set(int64_t V, const IdList* lists, int nlists, void* workspace, int64_t* rows, int64_t* count,
                   float* vals, int64_t ld, cudaStream_t st);
// map[id] = id for id < V at the start of the workspace: a dense table through the row-mapped kernels
int launch_identity_map(int64_t V, void* workspace, cudaStream_t st);

// Negative-sampling P slot (ns_p.cu), operands as b200kge_ns_p_backward; arguments already checked.
// C [n, ldc] with C[i, r] = the sum of G[i, c] over the columns c of row i whose id (p_i, then neg[i, :]) is r
int launch_ns_p_collapse(const int64_t* triples, const int64_t* neg, int64_t n, int64_t K, const float* G, int64_t ldg,
                         int64_t R, float* C, int64_t ldc, cudaStream_t st);
// s_idx, o_idx = the triples' s and o; s_dst, o_dst = pe[s], pe[o] (pe NULL: s, o)
int launch_ns_p_unpack(const int64_t* triples, int64_t n, const int32_t* pe, int64_t* s_idx, int64_t* o_idx,
                       int64_t* s_dst, int64_t* o_dst, cudaStream_t st);
// chunks of rows of the distance family's relation pass: its partials take ns_p_parts(n, R) * R * rel.dim floats
int ns_p_parts(int64_t n, int64_t R);
// TransE (l_norm 1, 2), RotatE (l_norm 1) with weights C (scaled in place for L2): d s_i, d o_i ADDED into rows
// s_dst[i], o_dst[i] of d_ent; the relation gradient as ns_p_parts(n, R) partials [R, rel.dim] STORED into parts
int launch_ns_p_distance(int model, float l_norm, const Rows& E, const Rows& Rl, const int64_t* s_idx,
                         const int64_t* o_idx, int64_t n, float* C, int64_t ldc, float* d_ent, int64_t lde,
                         const int64_t* s_dst, const int64_t* o_dst, float* parts, cudaStream_t st);
// out[j] += sum over the nparts partials (rows ldp apart, partials part_stride apart) of relation row rows[j], for
// j < *count; rows / count NULL: out[r] += ... for every r < R
int launch_ns_p_rel_add(const float* parts, int64_t ldp, int64_t part_stride, int nparts, int64_t R, int Dr,
                        const int64_t* rows, const int64_t* count, float* out, int64_t ldo, cudaStream_t st);

// Shared negative sampling (ns_shared.cu), operands as b200kge_ns_shared_score / _backward; arguments already checked.
// U = the shared samples before the repeats, nu = U' = the unique ids (U + 1 with drop, else U).
// out[i, 1 + c] = Z[i, u(i, c)] for c < K
int launch_ns_shared_assemble(const float* Z, int64_t ldz, int64_t n, int64_t K, int64_t U, const int64_t* repeat,
                              const int64_t* drop, float* out, int64_t ldo, cudaStream_t st);
// C [n, ldc] with C[i, u] = the sum of G[i, 1 + c] over the columns c with u(i, c) = u, in column order
int launch_ns_shared_collapse(const float* G, int64_t ldg, int64_t n, int64_t K, int64_t U, int64_t nu,
                              const int64_t* repeat, const int64_t* drop, float* C, int64_t ldc, cudaStream_t st);
// used[u] = unique[u] where some row of the sub-batch uses it (default type: drop [n]), else *fill; cnt: [nu] ints of
// scratch
int launch_ns_shared_used(const int64_t* unique, int64_t nu, const int64_t* drop, int64_t n, const int64_t* fill,
                          int* cnt, int64_t* used, cudaStream_t st);
// Q[i, k] += eps for k < D
int launch_ns_shared_eps(float* Q, int64_t ldq, int64_t n, int D, float eps, cudaStream_t st);
// d_ent[pe ? pe[unique[u]] : unique[u], col_off + k] += dT[u, k] for u < nu, k < K
int launch_ns_shared_row_add(const float* dT, int64_t ldt, int64_t nu, int K, const int64_t* unique, const int32_t* pe,
                             float* d_ent, int64_t lde, int col_off, cudaStream_t st);

// Optimizer steps (optim.cu), operands as b200kge_adagrad_step / b200kge_sparse_adam_step; arguments already checked.
size_t optim_step_workspace_bytes(int64_t rows, int64_t dim, int64_t nnz, int coalesced);
int launch_adagrad_step(float* param, float* state_sum, int64_t rows, int64_t dim, const float* grad,
                        const int64_t* grad_rows, int64_t nnz, int coalesced, int foreach_order, float clr, float eps,
                        float weight_decay, void* workspace, cudaStream_t st);
int launch_sparse_adam_step(float* param, float* exp_avg, float* exp_avg_sq, int64_t rows, int64_t dim,
                            const float* grad, const int64_t* grad_rows, int64_t nnz, int coalesced,
                            float one_minus_beta1, float one_minus_beta2, float eps, float step_size, void* workspace,
                            cudaStream_t st);

}  // namespace b200kge
