// capi.cu — extern "C" entry points of libb200kge (see include/b200kge.h for the contract).
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include "fold.cuh"
#include "tc_common.cuh"

namespace b200kge {

static thread_local char g_err[512] = "";
static thread_local int64_t g_launches = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches += n; }

int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return 0;
  if (e == cudaErrorMemoryAllocation)
    set_error("CUDA out of memory (%s)", what);  // literal matched by LibKGE train.py:384-413
  else
    set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return B200KGE_ERR_CUDA;
}

static thread_local int g_prof_on = 0;
static thread_local cudaEvent_t g_ev0 = nullptr, g_ev1 = nullptr;
static thread_local int g_prof_valid = 0;

void profile_begin(cudaStream_t st) {
  if (!g_prof_on) return;
  if (!g_ev0) { cudaEventCreate(&g_ev0); cudaEventCreate(&g_ev1); }
  cudaEventRecord(g_ev0, st);
}
void profile_end(cudaStream_t st) {
  if (!g_prof_on || !g_ev0) return;
  cudaEventRecord(g_ev1, st);
  g_prof_valid = 1;
}

namespace {

// bump allocator over the caller's workspace
struct Arena {
  uint8_t* base;
  size_t cap, off;
  void* take(size_t bytes) {
    size_t a = (off + 255) & ~size_t(255);
    if (a + bytes > cap) return nullptr;
    off = a + bytes;
    return base + a;
  }
};

inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

int validate_model(int model, const Rows& ent_like, const Rows& rel_like) {
  if (model < 0 || model > B200KGE_ROTATE) { set_error("unknown model %d", model); return B200KGE_ERR_INVALID; }
  const int D = ent_like.dim;
  if (D <= 0) { set_error("entity dim must be positive"); return B200KGE_ERR_INVALID; }
  if ((model == B200KGE_COMPLEX || model == B200KGE_SIMPLE || model == B200KGE_CP || model == B200KGE_ROTATE) && (D & 1)) {
    set_error("model %d requires embeddings of even dimensionality (got %d)", model, D);
    return B200KGE_ERR_INVALID;
  }
  const int want = relation_dim(model, D);
  if (rel_like.dim != want) {
    set_error("relation dim %d does not match model %d with entity dim %d (expected %d)", rel_like.dim, model, D, want);
    return B200KGE_ERR_INVALID;
  }
  return 0;
}

int validate_norm(int model, float l_norm) {
  if ((model == B200KGE_TRANSE || model == B200KGE_ROTATE) && !(l_norm > 0.f && l_norm < 1e30f)) {
    set_error("l_norm must be a positive finite number (got %g)", (double)l_norm);
    return B200KGE_ERR_INVALID;
  }
  return 0;
}

// ent / rel of the entry points that take whole tables: present, plain (idx == NULL), a model and norm they fit
int check_tables(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel) {
  if (!ent || !rel) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (ent->idx || rel->idx) { set_error("ent/rel must be plain tables (idx == NULL)"); return B200KGE_ERR_INVALID; }
  int rc = validate_model(model, to_rows(ent), to_rows(rel));
  return rc ? rc : validate_norm(model, l_norm);
}

int check_loss_kind(int loss_kind) {
  if (loss_kind != B200KGE_LOSS_BCE && loss_kind != B200KGE_LOSS_KL) { set_error("unknown loss kind %d", loss_kind); return B200KGE_ERR_INVALID; }
  return 0;
}

int check_grad_ld(const b200kge_rows_t* ent, int64_t lde, const b200kge_rows_t* rel, int64_t ldr) {
  if (lde < ent->dim || ldr < rel->dim) { set_error("gradient leading dimensions are smaller than the table widths"); return B200KGE_ERR_INVALID; }
  return 0;
}

EpiParams empty_epi() {
  EpiParams P;
  memset(&P, 0, sizeof(P));
  return P;
}

bool take_planes(Arena& ws, SplitSet& S) {
  S.hi = ws.take((size_t)S.rows * S.Kp * 2);
  S.lo = ws.take((size_t)S.rows * S.Kp * 2);
  S.inv_scale = (float*)ws.take((size_t)S.rows_pad * 4);
  return S.hi && S.lo && S.inv_scale;
}
size_t planes_bytes(int64_t rows, int64_t rows_pad, int64_t Kp) {
  return 2 * ((size_t)rows * Kp * 2 + 256) + (size_t)rows_pad * 4 + 256;
}

// C[M,N] = A B^T on planes: A = "queries" (rows M), B = "table" (rows N, inv_scale padded to N+32)
// Long reductions are split into 512-element segments accumulated in fp32 (C is zeroed here first).
int gemm_planes(const SplitSet& A, const SplitSet& B, float* C, int64_t ldc, cudaStream_t st) {
  EpiParams P = empty_epi();
  P.out = C; P.ldo = ldc;
  if (A.Kp > 512) {
    P.accumulate_out = 1;
    cudaError_t e = cudaMemset2DAsync(C, (size_t)ldc * 4, 0, (size_t)B.rows * 4, (size_t)A.rows, st);
    if (e != cudaSuccess) return check_cuda(e, "cudaMemset2DAsync(gemm output)");
  }
  return launch_pairwise_tc3(EPI_STORE, A, B, P, st);
}

// One direction (or the stacked sp+po pair) of a 1-vs-N problem, with any epilogue.
struct Block {
  int model, combine;     // combine of the first n rows; stacked => second n rows use the other one
  const Rows* q0; const Rows* q1;  // per-row entity operands of the two halves (q1 null if not stacked)
  const Rows* p;
  const Rows* cand;
  int64_t n;
  const float* Qpre = nullptr;   // already-folded queries [nq, round_up(K,32)] (skips the fold launches)
  bool same_fold = false;        // stacked halves BOTH use `combine` (the reciprocal-relations step)
};

// The block's folded queries [nq, ldq]: B.Qpre, or both halves folded into the workspace.
int fold_block(const Block& B, int64_t ldq, Arena& ws, cudaStream_t st, const float** Q) {
  *Q = B.Qpre;
  if (*Q) return 0;
  const int64_t n = B.n;
  float* Qw = (float*)ws.take((size_t)(B.q1 ? 2 * n : n) * ldq * 4);
  if (!Qw) { set_error("workspace too small for folded queries"); return B200KGE_ERR_WORKSPACE; }
  int rc = launch_fold_queries(B.model, B.combine, *B.q0, *B.p, n, 0, Qw, ldq, st);
  if (rc) return rc;
  if (B.q1 && (rc = launch_fold_queries(B.model, B.same_fold ? B.combine : 1 - B.combine, *B.q1, *B.p, n, n, Qw, ldq, st)))
    return rc;
  *Q = Qw;
  return 0;
}

// The scorer's nch chunks per row, and for the BCE/KL epilogues their loss partials [nq, nch, F].
int take_partials(int epi_kind, int64_t nq, int nch, EpiParams& P, Arena& ws, int* nchunks_out, float** part_out) {
  const int loss_epi = epi_loss_base(epi_kind);
  if (loss_epi == EPI_BCE || loss_epi == EPI_KL) {
    const int F = (loss_epi == EPI_BCE) ? 2 : 5;
    P.part = (float*)ws.take((size_t)nq * nch * F * 4);
    if (!P.part) { set_error("workspace too small for loss partials"); return B200KGE_ERR_WORKSPACE; }
    if (part_out) *part_out = P.part;
  }
  P.nchunks = nch;
  if (nchunks_out) *nchunks_out = nch;
  return 0;
}

// nchunks_out / part_out (optional): number of per-row partial chunks and the partial buffer the loss
// epilogues wrote (input of launch_loss_finalize).
int run_block(const Block& B, float l_norm, int precision, int epi_kind, EpiParams P, Arena& ws,
              cudaStream_t st, int* nchunks_out, float** part_out = nullptr) {
  const int64_t n = B.n, nq = B.q1 ? 2 * n : n, m = B.cand->rows;
  const int D = B.q0->dim;
  Folded f0 = folded_problem(B.model, B.combine, D, l_norm);
  Folded f1 = f0;
  if (B.q1 && !B.same_fold) f1 = folded_problem(B.model, 1 - B.combine, D, l_norm);
  const bool cols_differ = B.q1 && (f0.col_off != f1.col_off);   // CP: halves read different columns
  const int K = f0.K;
  const int64_t ldq = round_up(K, 32);

  // Path selection depends on the model, K, the table and the PER-DIRECTION row count n only — never on whether
  // the two directions are stacked — so score_sp / score_po / score_sp_po / the fused forms of one batch all run
  // the same arithmetic (EntityRankingJob compares them, eval_entity_ranking.py:192-203,242-274).
  //   AUTO    -> F16X3 (pre-split fp16 planes, pairwise_tc.cu) for dot-product scorers with 32 <= K <= 1024 and
  //              n >= 16; fp32 SIMT otherwise (beyond K = 1024 the tensor core's fp32 accumulator error, which
  //              grows with the reduction length — 2.8e-4 of rms at K = 14541 — leaves too little margin)
  //   TF32_BF16X2 / 3XTF32 / TF32 -> pairwise_tc.cu (in-kernel split of raw fp32 tiles; needs TMA-able tables)
  int tc_kind = 0;       // 0 SIMT, 1 in-kernel split (pairwise_tc.cu), 3 pre-split planes
  if (f0.pair_op == PAIR_DOT && precision != B200KGE_PREC_FP32 && !cols_differ) {
    if (precision == B200KGE_PREC_AUTO) {
      if (K >= 32 && K <= 1024 && n >= 16 && m < (1ll << 31)) tc_kind = 3;
    } else if (precision == B200KGE_PREC_F16X3) {
      if (K < 16 || m >= (1ll << 31)) { set_error("the pre-split tensor-core path needs K >= 16"); return B200KGE_ERR_UNSUPPORTED; }
      tc_kind = 3;
    } else {
      if (!tc_supported(f0.pair_op, K, *B.cand, f0.col_off)) { set_error("tensor-core path needs K>=32, 16-byte aligned tables with ld%%4==0"); return B200KGE_ERR_UNSUPPORTED; }
      tc_kind = 1;
    }
  } else if (precision != B200KGE_PREC_AUTO && precision != B200KGE_PREC_FP32) {
    if (f0.pair_op != PAIR_DOT) { set_error("tensor-core precision modes apply to dot-product scorers only"); return B200KGE_ERR_UNSUPPORTED; }
  }

  if (epi_kind == EPI_RANK_EVAL) {
    // every ranking in one pass: the pre-split tensor-core kernel and the CUDA-core kernel; CP runs per direction below
    if (B.cand->idx || tc_kind == 1) {
      set_error("the evaluation ranking runs on the pre-split tensor-core or the CUDA-core kernel over a plain table");
      return B200KGE_ERR_UNSUPPORTED;
    }
  } else if (P.csr_off && (cols_differ || B.cand->idx || tc_kind == 1 || (tc_kind == 0 && epi_kind != EPI_RANK))) {
    // CSR side inputs: the pre-split tensor-core epilogue (losses and rank) and the CUDA-core kernel's rank epilogue.
    // Nothing has been launched or taken from the workspace yet: callers fall back to their dense / composed form.
    set_error("this CSR side input is not consumed by the kernel serving this call (losses: pre-split tensor-core path; "
              "rank: that path or the CUDA-core kernel; plain candidate table)");
    return B200KGE_ERR_UNSUPPORTED;
  }

  if (cols_differ) {
    // run the two halves as separate blocks (CP reads different candidate columns per direction)
    Block h0 = B; h0.q1 = nullptr;
    Block h1 = B; h1.q0 = B.q1; h1.q1 = nullptr; h1.combine = 1 - B.combine;
    EpiParams P0 = P, P1 = P;
    P0.n_rows_out = 0; P1.n_rows_out = 0;
    if (epi_kind == EPI_STORE) { P1.out = P.out + P.col_block; }
    else if (epi_kind == EPI_RANK_EVAL) {
      // the second half's rows of every per-row operand (CSR row offsets included: they index the shared col arrays)
      P1.true_score += n; P1.csr_skip += n; P1.csr_off += n; P1.own_score += n; P1.rank += n; P1.ties += n;
      if (P1.csr2_off) P1.csr2_off += n;
    }
    else { set_error("stacked fused epilogues are not available for CP"); return B200KGE_ERR_UNSUPPORTED; }
    int rc = run_block(h0, l_norm, precision, epi_kind, P0, ws, st, nchunks_out);
    if (rc) return rc;
    return run_block(h1, l_norm, precision, epi_kind, P1, ws, st, nchunks_out);
  }

  const float* Q = nullptr;
  int rc = fold_block(B, ldq, ws, st, &Q);
  if (rc) return rc;
  if (tc_kind == 3) {
    // pre-split fp16 path (presplit.cu + pairwise_tc.cu): one launch derives the hi/lo planes of the folded queries
    // and of the (gathered) candidate rows, one launch scores them.
    const int Kp = (int)round_up(K, 64);
    SplitSet SQ{Q, ldq, nullptr, 0, nq, nq, K, Kp, nullptr, nullptr, nullptr};
    SplitSet ST{B.cand->base, B.cand->ld, B.cand->idx, f0.col_off, m, m + 32, K, Kp, nullptr, nullptr, nullptr};
    if (!take_planes(ws, SQ) || !take_planes(ws, ST)) {
      set_error("workspace too small for the pre-split operand planes");
      return B200KGE_ERR_WORKSPACE;
    }
    if ((rc = take_partials(epi_kind, nq, tc_nchunks(nq, m), P, ws, nchunks_out, part_out))) return rc;
    if ((rc = launch_presplit(ST, SQ, st))) return rc;
    return launch_pairwise_tc3(epi_kind, SQ, ST, P, st);
  }
  if (tc_kind == 1) {
    const int passes = (precision == B200KGE_PREC_TF32) ? 1 : (precision == B200KGE_PREC_3XTF32 ? 3 : 2);
    const float* T = B.cand->base + f0.col_off;
    int64_t ldt = B.cand->ld;
    if (B.cand->idx) {
      float* G = (float*)ws.take((size_t)m * ldq * 4);
      if (!G) { set_error("workspace too small to gather the candidate subset"); return B200KGE_ERR_WORKSPACE; }
      if ((rc = launch_gather_rows(*B.cand, f0.col_off, K, G, ldq, st))) return rc;
      T = G; ldt = ldq;
    }
    if ((rc = take_partials(epi_kind, nq, tc_nchunks(nq, m), P, ws, nchunks_out, part_out))) return rc;
    return launch_pairwise_tc(epi_kind, passes, Q, ldq, nq, T, ldt, m, K, P, st);
  }
  if ((rc = take_partials(epi_kind, nq, pairwise_simt_nchunks(nq, m), P, ws, nchunks_out, part_out))) return rc;
  return launch_pairwise_simt(epi_kind, f0.pair_op, l_norm, Q, ldq, nq, *B.cand, f0.col_off, K, P, st);
}

int check_1vsN_args(int model, int combine, const b200kge_rows_t* q, const b200kge_rows_t* p,
                    const b200kge_rows_t* cand, int64_t n) {
  if (!q || !p || !cand) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (combine != B200KGE_SP_ && combine != B200KGE__PO) {
    set_error("cannot handle combine=%d", combine);   // ValueError in kge_model.py:211
    return B200KGE_ERR_INVALID;
  }
  if (n < 0 || q->rows < n || p->rows < n) { set_error("operand has fewer than n=%lld rows", (long long)n); return B200KGE_ERR_INVALID; }
  if (cand->dim != q->dim) { set_error("candidate dim %d != query entity dim %d", cand->dim, q->dim); return B200KGE_ERR_INVALID; }
  return validate_model(model, to_rows(q), to_rows(p));
}

__global__ void unpack_triples_kernel(const int64_t* __restrict__ tri, int64_t n, int64_t* s, int64_t* p,
                                      int64_t* o, int64_t* labels2n) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) {
    const int64_t a = tri[3 * i], b = tri[3 * i + 1], c = tri[3 * i + 2];
    s[i] = a; p[i] = b; o[i] = c;
    labels2n[i] = c;       // sp_ rows are labelled with the object      train_1vsAll.py:64-65
    labels2n[n + i] = a;   // _po rows are labelled with the subject     train_1vsAll.py:75-76
  }
}

// s/p/o and the [2n] labels of [n, 3] triples into the caller's buffers; S, O (rows of E) and P (rows of R) index them
int unpack_triples(const int64_t* triples, int64_t n, int64_t* sidx, int64_t* pidx, int64_t* oidx, int64_t* lab,
                   const Rows& E, const Rows& R, Rows& S, Rows& O, Rows& P, cudaStream_t st) {
  unpack_triples_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(triples, n, sidx, pidx, oidx, lab);
  B2K_LAUNCH_CHECK("unpack_triples_kernel");
  S = E; S.idx = sidx; S.rows = n;
  O = E; O.idx = oidx; O.rows = n;
  P = R; P.idx = pidx; P.rows = n;
  return 0;
}

__global__ void pack_triples_kernel(const int64_t* __restrict__ q, const int64_t* __restrict__ p, int64_t n, int combine,
                                    int64_t* __restrict__ tri) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  tri[3 * i + 1] = p[i];
  tri[3 * i + (combine == B200KGE_SP_ ? 0 : 2)] = q[i];
  tri[3 * i + (combine == B200KGE_SP_ ? 2 : 0)] = 0;
}

// out[i] = idx[i] + off: the reciprocal relation rows p + num_relations (reciprocal_relations_model.py:90)
__global__ void offset_index_kernel(const int64_t* __restrict__ idx, int64_t n, int64_t off, int64_t* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = idx[i] + off;
}

// rel must hold the 2R rows of a reciprocal-relations base model
int check_reciprocal(const b200kge_rows_t* rel, int64_t num_rel) {
  if (num_rel <= 0 || rel->rows != 2 * num_rel) {
    set_error("reciprocal relations need rel->rows == 2 * num_relations (got %lld rows, num_relations %lld)",
              (long long)rel->rows, (long long)num_rel);
    return B200KGE_ERR_INVALID;
  }
  return 0;
}

__global__ void __launch_bounds__(128)
shard_gather_rows_kernel(Rows shard, int64_t lo, const int64_t* __restrict__ idx, float* __restrict__ out, int64_t ldo) {
  const int64_t i = blockIdx.x;
  const int64_t g = idx[i] - lo;
  const bool mine = g >= 0 && g < shard.rows;
  const float* __restrict__ src = shard.base + (mine ? g : 0) * shard.ld;
  float* __restrict__ dst = out + i * ldo;
  for (int k = threadIdx.x; k < shard.dim; k += blockDim.x) dst[k] = mine ? src[k] : 0.f;
}

}  // namespace
}  // namespace b200kge

using namespace b200kge;

extern "C" {

int b200kge_version(void) { return B200KGE_VERSION; }
const char* b200kge_last_error(void) { return g_err; }
int64_t b200kge_launch_count(int reset) {
  int64_t v = g_launches;
  if (reset) g_launches = 0;
  return v;
}

int b200kge_profile_enable(int on) { g_prof_on = on; g_prof_valid = 0; return 0; }
int b200kge_profile_last_ms(float* ms) {
  if (!ms) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (!g_prof_valid) { set_error("no profiled kernel yet"); return B200KGE_ERR_INVALID; }
  B2K_CUDA(cudaEventSynchronize(g_ev1));
  B2K_CUDA(cudaEventElapsedTime(ms, g_ev0, g_ev1));
  return 0;
}

int b200kge_device_ok(void) {
  int dev = 0, major = 0, minor = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) {
    cudaGetLastError();
    set_error("no CUDA device available: libb200kge has no CPU fallback");
    return B200KGE_ERR_NO_DEVICE;
  }
  if (major != 9 || minor != 0) {
    set_error("device compute capability %d.%d is not sm_90 (H100)", major, minor);
    return B200KGE_ERR_NO_DEVICE;
  }
  return 0;
}

size_t b200kge_workspace_bytes(int model, int64_t n, int64_t m, int32_t D, int cand_has_idx) {
  (void)model;
  const int64_t ldq = round_up(D, 32);
  const int64_t nq = 2 * n;
  size_t b = 0;
  b += 2 * ((size_t)nq * ldq * 4 + 256);                 // Qhi/Qlo (or Q)
  if (cand_has_idx) b += (size_t)m * ldq * 4 + 256;      // gathered candidate subset
  int64_t nch = pairwise_simt_nchunks(nq, m);
  if (nch < 320) nch = 320;                              // tensor-core kernels: <= 2 * #SMs chunks per row
  b += (size_t)nq * nch * 5 * 4 + 256;                   // loss partials
  b += (size_t)n * 3 * 8 + (size_t)n * 5 * 8 + 4096;     // host entry: triples, s/p/o, labels, scalar, finaliser scratch
  { // pre-split fp16 planes + row scales (the default tensor-core path)
    const int64_t Kp = round_up(D, 64);
    b += 2 * ((size_t)nq * Kp * 2 + 256) + 2 * ((size_t)m * Kp * 2 + 256) + (size_t)(nq + m + 32) * 4 + 512;
  }
  return b + 4096;
}

int b200kge_score_spo(int model, float l_norm, const b200kge_rows_t* s, const b200kge_rows_t* p,
                      const b200kge_rows_t* o, int64_t n, float* out, b200kge_stream_t stream) {
  if (!s || !p || !o || (!out && n > 0)) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  int rc = validate_model(model, to_rows(s), to_rows(p)); if (rc) return rc;
  if ((rc = validate_norm(model, l_norm))) return rc;
  if (s->rows < n || p->rows < n || o->rows < n) { set_error("operand has fewer than n rows"); return B200KGE_ERR_INVALID; }
  return launch_spo(model, l_norm, to_rows(s), to_rows(p), to_rows(o), n, out, 1, (cudaStream_t)stream);
}

int b200kge_score_1vsN(int model, int combine, float l_norm, int precision,
                       const b200kge_rows_t* q, const b200kge_rows_t* p,
                       const b200kge_rows_t* cand, int64_t n, float* out, int64_t ldo,
                       void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  int rc = check_1vsN_args(model, combine, q, p, cand, n); if (rc) return rc;
  if ((rc = validate_norm(model, l_norm))) return rc;
  Rows Q = to_rows(q), Pr = to_rows(p), C = to_rows(cand);
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  EpiParams P = empty_epi();
  P.out = out; P.ldo = ldo;
  Block B{model, combine, &Q, nullptr, &Pr, &C, n};
  return run_block(B, l_norm, precision, EPI_STORE, P, ws, (cudaStream_t)stream, nullptr);
}

int b200kge_score_sp_po(int model, float l_norm, int precision, const b200kge_rows_t* s,
                        const b200kge_rows_t* p, const b200kge_rows_t* o,
                        const b200kge_rows_t* cand, int64_t n, float* out, int64_t ldo,
                        void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  int rc = check_1vsN_args(model, B200KGE_SP_, s, p, cand, n); if (rc) return rc;
  if ((rc = check_1vsN_args(model, B200KGE__PO, o, p, cand, n))) return rc;
  if ((rc = validate_norm(model, l_norm))) return rc;
  Rows Sr = to_rows(s), Pr = to_rows(p), Or = to_rows(o), C = to_rows(cand);
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  EpiParams P = empty_epi();
  P.out = out; P.ldo = ldo; P.n_rows_out = n; P.col_block = cand->rows;
  Block B{model, B200KGE_SP_, &Sr, &Or, &Pr, &C, n};
  return run_block(B, l_norm, precision, EPI_STORE, P, ws, (cudaStream_t)stream, nullptr);
}

int b200kge_score_sp_po_bcast(int model, float l_norm, int precision, const b200kge_rows_t* s,
                              const b200kge_rows_t* p, const b200kge_rows_t* o, const b200kge_rows_t* cand,
                              int64_t n, float* out, float* const* peer_out, int n_peers, int64_t ldo,
                              int64_t col_block, void* workspace, size_t workspace_bytes,
                              b200kge_stream_t stream) {
  int rc = check_1vsN_args(model, B200KGE_SP_, s, p, cand, n); if (rc) return rc;
  if ((rc = check_1vsN_args(model, B200KGE__PO, o, p, cand, n))) return rc;
  if ((rc = validate_norm(model, l_norm))) return rc;
  if (n_peers < 0 || n_peers > 7 || (n_peers > 0 && !peer_out)) { set_error("0..7 peer buffers"); return B200KGE_ERR_INVALID; }
  if (col_block < cand->rows) { set_error("col_block smaller than the number of candidates"); return B200KGE_ERR_INVALID; }
  Rows Sr = to_rows(s), Pr = to_rows(p), Or = to_rows(o), C = to_rows(cand);
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  EpiParams P = empty_epi();
  P.out = out; P.ldo = ldo; P.n_rows_out = n; P.col_block = col_block;
  P.n_peers = n_peers;
  for (int g = 0; g < n_peers; ++g) P.out_peer[g] = peer_out[g];
  if (model == B200KGE_CP) { set_error("the broadcast store is not offered for CP"); return B200KGE_ERR_UNSUPPORTED; }
  Block B{model, B200KGE_SP_, &Sr, &Or, &Pr, &C, n};
  return run_block(B, l_norm, precision, EPI_STORE, P, ws, (cudaStream_t)stream, nullptr);
}

int b200kge_score_1vsN_loss(int model, int combine, float l_norm, int precision,
                            const b200kge_rows_t* q, const b200kge_rows_t* p,
                            const b200kge_rows_t* cand, int64_t n, const b200kge_labels_t* labels,
                            int loss_kind, float offset, float* loss_out, float* row_loss_out,
                            void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  int rc = check_1vsN_args(model, combine, q, p, cand, n); if (rc) return rc;
  if ((rc = validate_norm(model, l_norm))) return rc;
  if (!labels || (!labels->idx) == (!labels->dense)) { set_error("exactly one of labels.idx / labels.dense must be given"); return B200KGE_ERR_INVALID; }
  if ((rc = check_loss_kind(loss_kind))) return rc;
  if (!loss_out) { set_error("loss_out is null"); return B200KGE_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  Rows Q = to_rows(q), Pr = to_rows(p), C = to_rows(cand);
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  EpiParams P = empty_epi();
  P.label_idx = labels->idx; P.label_dense = labels->dense; P.ldl = labels->ldl;
  P.offset = (loss_kind == B200KGE_LOSS_BCE) ? offset : 0.f;
  Block B{model, combine, &Q, nullptr, &Pr, &C, n};
  int nch = 0;
  const int epi = (loss_kind == B200KGE_LOSS_BCE) ? EPI_BCE : EPI_KL;
  float* part = nullptr;
  rc = run_block(B, l_norm, precision, epi, P, ws, st, &nch, &part);
  if (rc) return rc;
  if (n == 0 || C.rows == 0) { B2K_CUDA(cudaMemsetAsync(loss_out, 0, 4, st)); return 0; }
  void* scratch = ws.take(1024);
  if (!scratch) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  return launch_loss_finalize(loss_kind, part, nch, n, loss_out, row_loss_out, 1.0f, 0, scratch, 0, st);
}

int b200kge_score_1vsN_rank(int model, int combine, float l_norm, int precision,
                            const b200kge_rows_t* q, const b200kge_rows_t* p,
                            const b200kge_rows_t* cand, int64_t n, const float* true_score,
                            const float* filter, int64_t ldf, float rtol, float atol,
                            int64_t* rank, int64_t* ties, void* workspace, size_t workspace_bytes,
                            b200kge_stream_t stream) {
  int rc = check_1vsN_args(model, combine, q, p, cand, n); if (rc) return rc;
  if ((rc = validate_norm(model, l_norm))) return rc;
  if (!true_score || !rank || !ties) { set_error("null rank operand"); return B200KGE_ERR_INVALID; }
  Rows Q = to_rows(q), Pr = to_rows(p), C = to_rows(cand);
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  EpiParams P = empty_epi();
  P.true_score = true_score; P.filter = filter; P.ldf = ldf; P.rtol = rtol; P.atol = atol;
  P.rank = reinterpret_cast<unsigned long long*>(rank);
  P.ties = reinterpret_cast<unsigned long long*>(ties);
  Block B{model, combine, &Q, nullptr, &Pr, &C, n};
  return run_block(B, l_norm, precision, EPI_RANK, P, ws, (cudaStream_t)stream, nullptr);
}

int b200kge_rank_sp_po(int model, float l_norm, int precision, const b200kge_rows_t* s,
                       const b200kge_rows_t* p, const b200kge_rows_t* o, const b200kge_rows_t* cand,
                       int64_t n, const float* true_score, const float* filter, int64_t ldf, float rtol,
                       float atol, int64_t* rank, int64_t* ties, void* workspace, size_t workspace_bytes,
                       b200kge_stream_t stream) {
  int rc = check_1vsN_args(model, B200KGE_SP_, s, p, cand, n); if (rc) return rc;
  if ((rc = check_1vsN_args(model, B200KGE__PO, o, p, cand, n))) return rc;
  if ((rc = validate_norm(model, l_norm))) return rc;
  if (!true_score || !rank || !ties) { set_error("null rank operand"); return B200KGE_ERR_INVALID; }
  Rows Sr = to_rows(s), Pr = to_rows(p), Or = to_rows(o), C = to_rows(cand);
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  EpiParams P = empty_epi();
  P.true_score = true_score; P.filter = filter; P.ldf = ldf; P.rtol = rtol; P.atol = atol;
  P.rank = reinterpret_cast<unsigned long long*>(rank);
  P.ties = reinterpret_cast<unsigned long long*>(ties);
  Block B{model, B200KGE_SP_, &Sr, &Or, &Pr, &C, n};
  return run_block(B, l_norm, precision, EPI_RANK, P, ws, (cudaStream_t)stream, nullptr);
}

int b200kge_rank_sp_po_csr(int model, float l_norm, int precision, const b200kge_rows_t* s,
                           const b200kge_rows_t* p, const b200kge_rows_t* o, const b200kge_rows_t* cand,
                           int64_t n, const float* true_score, const int64_t* filter_off,
                           const int64_t* filter_col, const int64_t* own_col, float rtol, float atol,
                           int64_t* rank, int64_t* ties, void* workspace, size_t workspace_bytes,
                           b200kge_stream_t stream) {
  int rc = check_1vsN_args(model, B200KGE_SP_, s, p, cand, n); if (rc) return rc;
  if ((rc = check_1vsN_args(model, B200KGE__PO, o, p, cand, n))) return rc;
  if ((rc = validate_norm(model, l_norm))) return rc;
  if (!true_score || !rank || !ties || !filter_off) { set_error("null rank operand"); return B200KGE_ERR_INVALID; }
  Rows Sr = to_rows(s), Pr = to_rows(p), Or = to_rows(o), C = to_rows(cand);
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  EpiParams P = empty_epi();
  P.true_score = true_score; P.rtol = rtol; P.atol = atol;
  P.rank = reinterpret_cast<unsigned long long*>(rank);
  P.ties = reinterpret_cast<unsigned long long*>(ties);
  P.csr_off = filter_off; P.csr_col = filter_col; P.csr_skip = own_col;
  Block B{model, B200KGE_SP_, &Sr, &Or, &Pr, &C, n};
  return run_block(B, l_norm, precision, EPI_RANK, P, ws, (cudaStream_t)stream, nullptr);
}

int b200kge_rank_sp_po_eval(int model, float l_norm, int precision, const b200kge_rows_t* ent,
                            const b200kge_rows_t* rel, int64_t num_relations, const int64_t* s, const int64_t* p,
                            const int64_t* o, int64_t n, const float* true_score, const int64_t* own_col,
                            const int64_t* filter_off, const int64_t* filter_col, const int64_t* test_off,
                            const int64_t* test_col, float rtol, float atol, int64_t* rank, int64_t* ties,
                            float* own_score, void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  if (!s || !p || !o || !true_score || !own_col || !filter_off || !rank || !ties || !own_score) {
    set_error("null rank operand");
    return B200KGE_ERR_INVALID;
  }
  if (n < 0) { set_error("negative batch size"); return B200KGE_ERR_INVALID; }
  if (num_relations < 0) { set_error("num_relations must be >= 0"); return B200KGE_ERR_INVALID; }
  int rc = check_tables(model, l_norm, ent, rel); if (rc) return rc;
  if (num_relations > 0 && (rc = check_reciprocal(rel, num_relations))) return rc;
  if (precision == B200KGE_PREC_TF32 || precision == B200KGE_PREC_3XTF32 || precision == B200KGE_PREC_TF32_BF16X2) {
    set_error("the evaluation ranking does not run the in-kernel split precision modes");
    return B200KGE_ERR_UNSUPPORTED;
  }
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const Rows E = to_rows(ent), R = to_rows(rel);
  Rows S = E, O = E, Pr = R;
  S.idx = s; S.rows = n; O.idx = o; O.rows = n; Pr.idx = p; Pr.rows = n;
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  EpiParams P = empty_epi();
  P.true_score = true_score; P.rtol = rtol; P.atol = atol;
  P.rank = reinterpret_cast<unsigned long long*>(rank);
  P.ties = reinterpret_cast<unsigned long long*>(ties);
  P.csr_off = filter_off; P.csr_col = filter_col; P.csr_skip = own_col;
  P.csr2_off = test_off; P.csr2_col = test_col;
  P.rank_ld = 2 * n; P.n_rank = test_off ? 3 : 2;
  P.own_score = own_score;
  Block B{model, B200KGE_SP_, &S, &O, &Pr, &E, n};
  if (num_relations > 0) {
    // reciprocal relations: rows n..2n-1 are the sp_ queries (o, p + R) (reciprocal_relations_model.py:85-92), folded
    // here with the sp_ fold; both halves then read the same table columns, so CP stacks too
    const Folded f = folded_problem(model, B200KGE_SP_, E.dim, l_norm);
    const int64_t ldq = round_up(f.K, 32);
    float* Q = (float*)ws.take((size_t)2 * n * ldq * 4);
    int64_t* p2 = (int64_t*)ws.take((size_t)n * 8);
    if (!Q || !p2) { set_error("workspace too small for folded queries"); return B200KGE_ERR_WORKSPACE; }
    offset_index_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, n, num_relations, p2);
    B2K_LAUNCH_CHECK("offset_index_kernel");
    Rows P2 = R; P2.idx = p2; P2.rows = n;
    if ((rc = launch_fold_queries(model, B200KGE_SP_, S, Pr, n, 0, Q, ldq, st))) return rc;
    if ((rc = launch_fold_queries(model, B200KGE_SP_, O, P2, n, n, Q, ldq, st))) return rc;
    B.Qpre = Q;
    B.same_fold = true;
  }
  return run_block(B, l_norm, precision, EPI_RANK_EVAL, P, ws, st, nullptr);
}

int b200kge_shard_gather_rows(const b200kge_rows_t* shard, int64_t lo, const int64_t* idx, int64_t n,
                              float* out, int64_t ldo, b200kge_stream_t stream) {
  if (!shard || (!idx && n > 0) || (!out && n > 0)) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (shard->idx) { set_error("shard must be a plain table (idx == NULL)"); return B200KGE_ERR_INVALID; }
  if (ldo < shard->dim) { set_error("output row stride smaller than the row width"); return B200KGE_ERR_INVALID; }
  if (n <= 0) return 0;
  shard_gather_rows_kernel<<<(unsigned)n, 128, 0, (cudaStream_t)stream>>>(to_rows(shard), lo, idx, out, ldo);
  B2K_LAUNCH_CHECK("shard_gather_rows_kernel");
  return 0;
}

int b200kge_loss_dense(const float* scores, int64_t lds, int64_t n, int64_t m,
                       const b200kge_labels_t* labels, int loss_kind, float offset,
                       float* loss_out, float* row_loss_out, void* workspace,
                       size_t workspace_bytes, b200kge_stream_t stream) {
  if (!scores || !labels || !loss_out) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if ((!labels->idx) == (!labels->dense)) { set_error("exactly one of labels.idx / labels.dense must be given"); return B200KGE_ERR_INVALID; }
  if (loss_kind >= B200KGE_LOSS_BCE_MEAN && loss_kind <= B200KGE_LOSS_SE) { set_error("loss kind %d is row-wise with one positive per row: use b200kge_ns_loss", loss_kind); return B200KGE_ERR_UNSUPPORTED; }
  int rc = check_loss_kind(loss_kind); if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0 || m == 0) { B2K_CUDA(cudaMemsetAsync(loss_out, 0, 4, st)); return 0; }
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  const int nch = loss_dense_nchunks(m);
  const int F = (loss_kind == B200KGE_LOSS_BCE) ? 2 : 5;
  EpiParams P = empty_epi();
  P.label_idx = labels->idx; P.label_dense = labels->dense; P.ldl = labels->ldl;
  P.offset = (loss_kind == B200KGE_LOSS_BCE) ? offset : 0.f;
  P.nchunks = nch;
  P.part = (float*)ws.take((size_t)n * nch * F * 4);
  if (!P.part) { set_error("workspace too small for loss partials (need %zu bytes)", (size_t)n * nch * F * 4); return B200KGE_ERR_WORKSPACE; }
  void* scratch = ws.take(1024);
  if (!scratch) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  if ((rc = launch_loss_dense(loss_kind, scores, lds, n, m, P, st))) return rc;
  return launch_loss_finalize(loss_kind, P.part, nch, n, loss_out, row_loss_out, 1.0f, 0, scratch, 0, st);
}

int b200kge_rank_dense(const float* scores, int64_t lds, int64_t n, int64_t m,
                       const float* true_score, const float* filter, int64_t ldf, float rtol,
                       float atol, int64_t* rank, int64_t* ties, b200kge_stream_t stream) {
  if (!scores || !true_score || !rank || !ties) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  EpiParams P = empty_epi();
  P.true_score = true_score; P.filter = filter; P.ldf = ldf; P.rtol = rtol; P.atol = atol;
  P.rank = reinterpret_cast<unsigned long long*>(rank);
  P.ties = reinterpret_cast<unsigned long long*>(ties);
  return launch_rank_dense(scores, lds, n, m, P, (cudaStream_t)stream);
}

int b200kge_ns_score(int model, float l_norm, const b200kge_rows_t* s, const b200kge_rows_t* p,
                     const b200kge_rows_t* o, const b200kge_rows_t* slot_table, int slot,
                     const int64_t* neg, int64_t n, int64_t K, int with_positive, float* out,
                     int64_t ldo, b200kge_stream_t stream) {
  if (n == 0 || (K == 0 && !with_positive)) return 0;          // nothing to score
  if (!s || !p || !o || !slot_table || (!neg && n * K > 0) || !out) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (slot < 0 || slot > 2) { set_error("slot must be 0 (S), 1 (P) or 2 (O)"); return B200KGE_ERR_INVALID; }
  int rc = validate_model(model, to_rows(s), to_rows(p)); if (rc) return rc;
  if ((rc = validate_norm(model, l_norm))) return rc;
  if (slot_table->idx) { set_error("slot_table must be a plain table (idx == NULL)"); return B200KGE_ERR_INVALID; }
  if (slot_table->dim != (slot == 1 ? p->dim : s->dim)) { set_error("slot_table width does not match the slot"); return B200KGE_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const int col0 = with_positive ? 1 : 0;
  if (with_positive) {
    rc = launch_spo(model, l_norm, to_rows(s), to_rows(p), to_rows(o), n, out, ldo, st);
    if (rc) return rc;
  }
  return launch_ns(model, l_norm, to_rows(s), to_rows(p), to_rows(o), to_rows(slot_table), slot, neg, n, K,
                   out, ldo, col0, st);
}

int b200kge_sample_uniform(uint64_t seed, uint64_t offset, int64_t vocab, int64_t n, int64_t K, int64_t* out,
                           b200kge_stream_t stream) {
  if (vocab <= 0) { set_error("vocabulary size must be positive"); return B200KGE_ERR_INVALID; }
  if (n < 0 || K < 0 || (!out && n * K > 0)) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  return launch_sample_uniform(seed, offset, vocab, n * K, out, (cudaStream_t)stream);
}

int b200kge_sample_uniform_filtered(uint64_t seed, uint64_t offset, int64_t vocab, int64_t n, int64_t K,
                                    const int64_t* triples, int slot, const int64_t* keys, const int64_t* offsets,
                                    const int64_t* values, int64_t num_keys, int64_t* out, b200kge_stream_t stream) {
  if (vocab <= 0) { set_error("vocabulary size must be positive"); return B200KGE_ERR_INVALID; }
  if (slot < 0 || slot > 2) { set_error("slot must be 0 (S), 1 (P) or 2 (O)"); return B200KGE_ERR_INVALID; }
  if (n < 0 || K < 0 || num_keys < 0) { set_error("negative size"); return B200KGE_ERR_INVALID; }
  if (n * K > 0 && (!out || !triples || (num_keys > 0 && (!keys || !offsets || !values)))) {
    set_error("null operand");
    return B200KGE_ERR_INVALID;
  }
  return launch_sample_uniform_filtered(seed, offset, vocab, n, K, triples, slot, keys, offsets, values, num_keys, out,
                                        (cudaStream_t)stream);
}

int b200kge_sample_frequency(uint64_t seed, uint64_t offset, int64_t vocab, const uint64_t* cdf, int64_t n, int64_t K,
                             int64_t* out, b200kge_stream_t stream) {
  if (vocab <= 0) { set_error("vocabulary size must be positive"); return B200KGE_ERR_INVALID; }
  if (n < 0 || K < 0) { set_error("negative size"); return B200KGE_ERR_INVALID; }
  if (n * K > 0 && (!out || !cdf)) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  return launch_sample_frequency(seed, offset, vocab, cdf, n * K, out, (cudaStream_t)stream);
}

int b200kge_sample_frequency_filtered(uint64_t seed, uint64_t offset, int64_t vocab, int64_t n, int64_t K,
                                      const int64_t* triples, int slot, const int64_t* keys, const int64_t* offsets,
                                      const int64_t* values, int64_t num_keys, const uint64_t* cdf,
                                      const uint64_t* below, int64_t* out, b200kge_stream_t stream) {
  if (vocab <= 0) { set_error("vocabulary size must be positive"); return B200KGE_ERR_INVALID; }
  if (slot < 0 || slot > 2) { set_error("slot must be 0 (S), 1 (P) or 2 (O)"); return B200KGE_ERR_INVALID; }
  if (n < 0 || K < 0 || num_keys < 0) { set_error("negative size"); return B200KGE_ERR_INVALID; }
  if (n * K > 0 && (!out || !triples || !cdf || (num_keys > 0 && (!keys || !offsets || !values || !below)))) {
    set_error("null operand");
    return B200KGE_ERR_INVALID;
  }
  return launch_sample_frequency_filtered(seed, offset, vocab, n, K, triples, slot, keys, offsets, values, num_keys, cdf,
                                          below, out, (cudaStream_t)stream);
}

// The 1vsAll step without dropout on validated arguments, n > 0.  num_rel > 0: the reciprocal-relations step (rows
// n..2n are the sp_ queries (o, p + num_rel), label s)
static int train_1vsall_forward_impl(int model, float l_norm, int precision, const b200kge_rows_t* ent,
                                     const b200kge_rows_t* rel, const int64_t* triples, int64_t n, int loss_kind,
                                     float offset, float* loss_out, void* workspace, size_t workspace_bytes,
                                     cudaStream_t st, int64_t num_rel) {
  int rc;
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  Rows E = to_rows(ent), R = to_rows(rel);
  const int epi = (loss_kind == B200KGE_LOSS_BCE) ? EPI_BCE : EPI_KL;
  const float scale = 1.0f / (float)n;       // "/ batch_size"   train_1vsAll.py:65,76
  // reciprocal: both halves are sp_ queries
  Folded f0 = folded_problem(model, B200KGE_SP_, E.dim, l_norm),
         f1 = folded_problem(model, num_rel > 0 ? B200KGE_SP_ : B200KGE__PO, E.dim, l_norm);
  // Pre-split tensor-core path (dot family except CP, whose directions read different table columns — CP joins in
  // the reciprocal step): the whole step is THREE launches — prologue (gather + both folds + operand split of queries
  // and table + labels), the scorer with the loss reduction in its epilogue, and the fixed-order finaliser.
  const int K = f0.K;
  const bool presplit = f0.col_off == f1.col_off && f0.pair_op == PAIR_DOT && (model != B200KGE_CP || num_rel > 0) &&
                        (precision == B200KGE_PREC_AUTO || precision == B200KGE_PREC_F16X3) && K >= 32 && K <= 1024 &&
                        n >= 16 && E.rows < (1ll << 31) &&
                        ((size_t)round_up(K, 64) + (model == B200KGE_RESCAL ? E.dim : 0)) * 4 <= 48 * 1024;
  if (presplit) {
    const int64_t nq = 2 * n, m = E.rows;
    const int Kp = (int)round_up(K, 64);
    SplitSet SQ{nullptr, 0, nullptr, 0, nq, nq, K, Kp, nullptr, nullptr, nullptr};
    SplitSet ST{E.base, E.ld, nullptr, f0.col_off, m, m + 32, K, Kp, nullptr, nullptr, nullptr};
    const bool planes = take_planes(ws, SQ) && take_planes(ws, ST);
    int64_t* lab = (int64_t*)ws.take((size_t)n * 2 * 8);
    uint8_t* scratch = (uint8_t*)ws.take(1024);
    const int nch = tc_nchunks(nq, m);
    const int F = (loss_kind == B200KGE_LOSS_BCE) ? 2 : 5;
    float* part = (float*)ws.take((size_t)nq * nch * F * 4);
    if (!planes || !lab || !scratch || !part) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
    unsigned int* ticket = reinterpret_cast<unsigned int*>(scratch + 512);
    if ((rc = launch_prep_split_1vsall(model, E, R, triples, n, SQ, ST, lab, ticket, st, num_rel))) return rc;
    EpiParams P = empty_epi();
    P.label_idx = lab;
    P.offset = (loss_kind == B200KGE_LOSS_BCE) ? offset : 0.f;
    P.part = part; P.nchunks = nch;
    if ((rc = launch_pairwise_tc3(epi, SQ, ST, P, st))) return rc;
    return launch_loss_finalize(loss_kind, part, nch, nq, loss_out, nullptr, scale, 0, scratch, 1, st);
  }
  if (f0.col_off == f1.col_off) {
    // sp_ and _po rows stacked into ONE problem of 2n query rows against the same table:
    // prologue (unpack + both folds + labels) = 1 launch, scoring + loss + finalisation = 1 launch
    const int64_t ldq = round_up(f0.K, 32);
    float* Q = (float*)ws.take((size_t)(2 * n) * ldq * 4);
    int64_t* lab = (int64_t*)ws.take((size_t)n * 2 * 8);
    uint8_t* scratch = (uint8_t*)ws.take(1024);      // finaliser scratch: block sums + ticket (+512)
    if (!Q || !lab || !scratch) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
    rc = launch_prep_1vsall(model, E, R, triples, n, Q, ldq, lab, reinterpret_cast<unsigned int*>(scratch + 512), st,
                            num_rel);
    if (rc) return rc;
    Rows S = E; S.idx = lab; S.rows = n;           // placeholders: operands are pre-folded
    Rows Pr = R; Pr.idx = lab; Pr.rows = n;
    EpiParams P = empty_epi();
    P.label_idx = lab;
    P.offset = (loss_kind == B200KGE_LOSS_BCE) ? offset : 0.f;
    Block B{model, B200KGE_SP_, &S, &S, &Pr, &E, n};
    B.Qpre = Q;
    B.same_fold = num_rel > 0;
    int nch = 0;
    float* part = nullptr;
    rc = run_block(B, l_norm, precision, epi, P, ws, st, &nch, &part);
    if (rc) return rc;
    return launch_loss_finalize(loss_kind, part, nch, 2 * n, loss_out, nullptr, scale, 0, scratch, 1, st);
  }
  int64_t* sidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* pidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* oidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* lab = (int64_t*)ws.take((size_t)n * 2 * 8);
  if (!sidx || !pidx || !oidx || !lab) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  Rows S, O, Pr;
  if ((rc = unpack_triples(triples, n, sidx, pidx, oidx, lab, E, R, S, O, Pr, st))) return rc;
  EpiParams P = empty_epi();
  P.label_idx = lab;
  P.offset = (loss_kind == B200KGE_LOSS_BCE) ? offset : 0.f;
  for (int dir = 0; dir < 2; ++dir) {   // CP: the two directions read different table columns
    Arena w2 = ws;
    EpiParams Pd = P;
    Pd.label_idx = lab + dir * n;
    Block B{model, dir, dir == 0 ? &S : &O, nullptr, &Pr, &E, n};
    int nch = 0;
    float* part = nullptr;
    rc = run_block(B, l_norm, precision, epi, Pd, w2, st, &nch, &part);
    if (rc) return rc;
    void* scratch = w2.take(1024);
    if (!scratch) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
    rc = launch_loss_finalize(loss_kind, part, nch, n, loss_out, nullptr, scale, dir, scratch, 0, st);
    if (rc) return rc;
  }
  return 0;
}

int b200kge_train_1vsall_forward_host(int model, float l_norm, int precision,
                                      const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                                      const int64_t* triples_host, int64_t n, int loss_kind,
                                      float offset, float* loss_host, void* workspace,
                                      size_t workspace_bytes, b200kge_stream_t stream) {
  if (!triples_host || !loss_host) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (n <= 0) { *loss_host = 0.f; return 0; }
  cudaStream_t st = (cudaStream_t)stream;
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  int64_t* tri = (int64_t*)ws.take((size_t)n * 3 * 8);
  float* loss_dev = (float*)ws.take(256);
  if (!tri || !loss_dev) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  // triples.to(device)   train_1vsAll.py:59
  B2K_CUDA(cudaMemcpyAsync(tri, triples_host, (size_t)n * 3 * 8, cudaMemcpyHostToDevice, st));
  size_t used = (ws.off + 255) & ~size_t(255);
  int rc = b200kge_train_1vsall_forward(model, l_norm, precision, ent, rel, 0, tri, n, loss_kind, offset, nullptr,
                                        loss_dev, ws.base + used, workspace_bytes - used, stream);
  if (rc) return rc;
  // .item()   train_1vsAll.py:66,77
  B2K_CUDA(cudaMemcpyAsync(loss_host, loss_dev, 4, cudaMemcpyDeviceToHost, st));
  B2K_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"

// ==================================================================================================
// Pre-split fp16 GEMM, the analytic backward of the 1vsAll step for the dot family (grad.cu), penalties, row
// normalisation, negative-sampling backward, CSR-label losses: SURVEY 8f rows.
namespace {

// Where dL/dz of a backward comes from: one-hot labels lab [nq] (1vsAll, scaled 1/n), the CSR labels of a KvsAll
// query type (target a * y + b, scaled inv_batch), or the caller's dense G [nq, ldg] (autograd through a dense score
// matrix).  lab also serves as the placeholder index vector of the pre-folded operands.
struct GradSpec {
  const int64_t* lab = nullptr;
  int loss_kind = B200KGE_LOSS_BCE;
  float offset = 0.f;
  const int64_t* csr_off = nullptr;
  const int64_t* csr_col = nullptr;
  float csr_a = 1.f, csr_b = 0.f, inv_batch = 0.f;
  const float* G = nullptr;
  int64_t ldg = 0;
};

// the CSR labels of a KvsAll query type over m candidates, label smoothing as in KvsAll (y (1 - ls) + ls / m)
GradSpec csr_grad(const int64_t* q_idx, const int64_t* csr_off, const int64_t* csr_col, float label_smoothing, int64_t m,
                  int64_t batch_size, int loss_kind, float offset) {
  GradSpec g;
  g.lab = q_idx;
  g.loss_kind = loss_kind; g.offset = offset;
  g.csr_off = csr_off; g.csr_col = csr_col;
  g.csr_a = 1.0f - label_smoothing; g.csr_b = label_smoothing > 0.f ? 1.0f / (float)m : 0.f;
  g.inv_batch = 1.0f / (float)batch_size;
  return g;
}

// One block of the backward up to dQ: nq folded query rows Q [nq, ldq] against the candidate columns [off, off+K)
// of the entity table; stores dT into those columns of d_ent and dQ [nq, ldq] into the caller's buffer.  dir as in
// launch_unfold.
int backward_block(int model, const Rows& E, const Rows& R, int64_t n, int dir, bool same_fold, const float* Q,
                   int64_t ldq, int col_off, int K, const GradSpec& g, float* d_ent, int64_t lde, float* dQ, Arena ws,
                   cudaStream_t st) {
  const int64_t nq = dir < 0 ? 2 * n : n, m = E.rows;
  const int64_t ldz = round_up(m, 4), Ep = round_up(m, 64), Np = round_up(nq, 64);
  const int64_t ldE = round_up(m, 4), ldN = round_up(nq, 4);
  int rc;
  SplitSet SG{nullptr, 0, nullptr, 0, nq, nq, (int)m, (int)Ep, nullptr, nullptr, nullptr};
  SplitSet SGT{nullptr, 0, nullptr, 0, m, m, (int)nq, (int)Np, nullptr, nullptr, nullptr};
  if (g.G) {
    // planes of G and of its transpose, row scaled
    float* Gt = (float*)ws.take((size_t)m * ldN * 4);
    if (!Gt) { set_error("workspace too small for the transposed gradient"); return B200KGE_ERR_WORKSPACE; }
    if ((rc = launch_transpose(g.G, g.ldg, nq, m, Gt, ldN, st))) return rc;
    SG.src = g.G; SG.ld = g.ldg;
    SGT.src = Gt; SGT.ld = ldN;
    if (!take_planes(ws, SG) || !take_planes(ws, SGT)) { set_error("workspace too small for the gradient planes"); return B200KGE_ERR_WORKSPACE; }
    if ((rc = launch_presplit(SGT, SG, st))) return rc;
  } else {
    // 1. scores through the validated scorer (plain-store epilogue)
    float* z = (float*)ws.take((size_t)nq * ldz * 4);
    if (!z) { set_error("workspace too small for the score matrix"); return B200KGE_ERR_WORKSPACE; }
    {
      Rows S = E; S.idx = g.lab; S.rows = n;      // placeholders: operands are pre-folded
      Rows Pr = R; Pr.idx = g.lab; Pr.rows = n;
      EpiParams P = empty_epi();
      P.out = z; P.ldo = ldz;
      Block B{model, dir <= 0 ? B200KGE_SP_ : B200KGE__PO, &S, dir < 0 ? &S : nullptr, &Pr, &E, n};
      B.Qpre = Q;
      B.same_fold = same_fold;
      if ((rc = run_block(B, 1.0f, B200KGE_PREC_AUTO, EPI_STORE, P, ws, st, nullptr))) return rc;
    }
    // 2. G = sigmoid(z + off) - y as planes, both layouts
    if (!take_planes(ws, SG) || !take_planes(ws, SGT)) { set_error("workspace too small for the gradient planes"); return B200KGE_ERR_WORKSPACE; }
    float* row_stat = nullptr;
    if (g.loss_kind == B200KGE_LOSS_KL) {
      row_stat = (float*)ws.take((size_t)nq * 2 * 4);
      if (!row_stat) { set_error("workspace too small for the row statistics"); return B200KGE_ERR_WORKSPACE; }
    }
    const float off = g.loss_kind == B200KGE_LOSS_KL ? 0.f : g.offset;
    if (g.csr_off)
      rc = launch_grad_planes_csr(z, ldz, nq, m, g.csr_off, g.csr_col, g.csr_a, g.csr_b, row_stat, off, g.inv_batch,
                                  SG.hi, SG.lo, Ep, SGT.hi, SGT.lo, Np, SG.inv_scale, SGT.inv_scale, st);
    else
      rc = launch_grad_planes(z, ldz, nq, m, g.lab, nullptr, 0, row_stat, off, 1.0f / (float)n, SG.hi, SG.lo, Ep,
                              SGT.hi, SGT.lo, Np, SG.inv_scale, SGT.inv_scale, st);
    if (rc) return rc;
  }
  // 3. transposed operands T^T [K, E] and Q^T [K, nq], then their planes
  float* Tt = (float*)ws.take((size_t)K * ldE * 4);
  float* Qt = (float*)ws.take((size_t)K * ldN * 4);
  if (!Tt || !Qt) { set_error("workspace too small for the transposed operands"); return B200KGE_ERR_WORKSPACE; }
  if ((rc = launch_transpose(E.base + col_off, E.ld, m, K, Tt, ldE, st))) return rc;
  if ((rc = launch_transpose(Q, ldq, nq, K, Qt, ldN, st))) return rc;
  SplitSet STt{Tt, ldE, nullptr, 0, K, K + 32, (int)m, (int)Ep, nullptr, nullptr, nullptr};
  SplitSet SQt{Qt, ldN, nullptr, 0, K, K + 32, (int)nq, (int)Np, nullptr, nullptr, nullptr};
  if (!take_planes(ws, STt) || !take_planes(ws, SQt)) { set_error("workspace too small for the operand planes"); return B200KGE_ERR_WORKSPACE; }
  if ((rc = launch_presplit(STt, SQt, st))) return rc;
  // 4. dT = G^T Q -> entity-table gradient columns [off, off+K) (overwrites);  dQ = G T
  if ((rc = gemm_planes(SGT, SQt, d_ent + col_off, lde, st))) return rc;
  return gemm_planes(SG, STt, dQ, ldq, st);
  // 5. (caller) unfold dQ into the rows of the batch — after EVERY block has stored its dT columns
}

// The two row-gradient passes of the distance family (grad_distance.cu) with weights W = dL/dz [nq, m]: Wt = W^T,
// dQ [nq, ldq] from the queries Q against the table T, dT [m, ldt] from T against Q.  Each pass reads its weights
// transposed ([column, row]): the other pass's orientation.
int distance_rowgrads(int pair_op, const float* Q, int64_t ldq, int64_t nq, const Rows& T, int K, const float* W,
                      int64_t ldw, float* Wt, float* dQ, float* dT, int64_t ldt, cudaStream_t st) {
  const int64_t m = T.rows, ldN = round_up(nq, 4);
  int rc;
  if ((rc = launch_transpose(W, ldw, nq, m, Wt, ldN, st))) return rc;
  if ((rc = launch_pair_rowgrad(pair_op, Q, ldq, nq, T.base, T.ld, m, K, Wt, ldN, dQ, ldq, st))) return rc;
  return launch_pair_rowgrad(pair_op, T.base, T.ld, m, Q, ldq, nq, K, W, ldw, dT, ldt, st);
}

// The distance-family backward of the pre-folded queries B.Qpre (nq rows) against the plain table B.cand, one-hot or
// CSR labels: scores by the CUDA-core scorer, the KL row statistics, dense G, then both row-gradient passes into dQ
// and dT.  The caller unfolds dQ.
int distance_backward(const Block& B, float l_norm, const GradSpec& g, float* dQ, float* dT, int64_t ldt, Arena& ws,
                      cudaStream_t st) {
  const Folded f = folded_problem(B.model, B.combine, B.cand->dim, l_norm);
  const int64_t nq = B.q1 ? 2 * B.n : B.n, m = B.cand->rows, ldz = round_up(m, 4), ldN = round_up(nq, 4);
  const bool kl = g.loss_kind == B200KGE_LOSS_KL;
  float* z = (float*)ws.take((size_t)nq * ldz * 4);
  float* G = (float*)ws.take((size_t)nq * ldz * 4);
  float* Gt = (float*)ws.take((size_t)m * ldN * 4);
  float* row_stat = kl ? (float*)ws.take((size_t)nq * 2 * 4) : nullptr;
  if (!z || !G || !Gt || (kl && !row_stat)) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  EpiParams P = empty_epi();
  P.out = z; P.ldo = ldz;
  int rc;
  if ((rc = run_block(B, l_norm, B200KGE_PREC_AUTO, EPI_STORE, P, ws, st, nullptr))) return rc;
  const int64_t* lab = g.csr_off ? nullptr : g.lab;       // CSR: only the log-sum-exp, grad_csr_kernel has the label mass
  if (kl && (rc = launch_row_lse(z, ldz, nq, m, lab, row_stat, st))) return rc;
  if (g.csr_off)
    rc = launch_grad_csr(z, ldz, nq, m, g.csr_off, g.csr_col, g.csr_a, g.csr_b, row_stat, kl ? 0.f : g.offset,
                         g.inv_batch, f.pair_op == PAIR_L2, G, ldz, st);
  else
    rc = launch_grad_dense(z, ldz, nq, m, g.lab, row_stat, kl ? 0.f : g.offset, 1.0f / (float)B.n,
                           f.pair_op == PAIR_L2, G, ldz, st);
  if (rc) return rc;
  return distance_rowgrads(f.pair_op, B.Qpre, round_up(f.K, 32), nq, *B.cand, f.K, G, ldz, Gt, dQ, dT, ldt, st);
}

// the distance-family backward covers these pairings only
int check_distance_pair(int pair_op) {
  if (pair_op != PAIR_L1 && pair_op != PAIR_L2 && pair_op != PAIR_CMOD_L1) {
    set_error("the distance-family backward covers l_norm 1 and 2 (TransE) and 1 (RotatE)");
    return B200KGE_ERR_UNSUPPORTED;
  }
  return 0;
}

// Buffers of the CSR-label loss steps below: the label-free pass's label vector, the listed entries' selections and
// scores (tot = nnz, plus n for KL's column-0 scores), the per-row terms and the finaliser's scalar and scratch.
struct CsrBufs {
  int64_t *lab, *qsel, *psel, *esel;
  float *zpos, *fused, *rows, *total;
  void* scratch;
};
bool take_csr_bufs(Arena& ws, int64_t n, int64_t nnz, int loss_kind, float* row_loss_out, CsrBufs& b) {
  const int64_t tot = nnz + (loss_kind == B200KGE_LOSS_KL ? n : 0);
  b.lab = (int64_t*)ws.take((size_t)n * 8);
  b.qsel = (int64_t*)ws.take((size_t)tot * 8 + 8);
  b.psel = (int64_t*)ws.take((size_t)tot * 8 + 8);
  b.esel = (int64_t*)ws.take((size_t)tot * 8 + 8);
  b.zpos = (float*)ws.take((size_t)tot * 4 + 8);
  b.fused = (float*)ws.take((size_t)n * 4);
  b.rows = row_loss_out ? row_loss_out : (float*)ws.take((size_t)n * 4);
  b.total = (float*)ws.take(256);
  b.scratch = ws.take(1024);
  return b.lab && b.qsel && b.psel && b.esel && b.zpos && b.fused && b.rows && b.total && b.scratch;
}

// Steps 1 and 2 of a CSR-label KvsAll loss (b200kge_score_1vsN_loss_csr, b200kge_score_so_loss_csr) for the n query
// rows of block B against its candidate table: b.fused[i] = the label-free row term, b.zpos = the scores of the listed
// columns (and of column 0 for KL).  `roles` places the row-wise triple kernel's operands (row i of q and p, the
// listed row of cand) as (s, p, o): B200KGE_SP_ (q, p, cand), B200KGE__PO (cand, p, q), ROLES_SO (q, cand, p).
constexpr int ROLES_SO = 2;
int csr_loss_terms(const Block& B, int model, int roles, float l_norm, int precision, const Rows& q, const Rows& p,
                   const Rows& cand, const int64_t* csr_off, const int64_t* csr_col, int64_t nnz, int loss_kind,
                   float offset, float* zsum, const CsrBufs& b, const Arena& ws, cudaStream_t st) {
  const int64_t n = B.n, tot = nnz + (loss_kind == B200KGE_LOSS_KL ? n : 0);
  int rc;
  // 1. label-free fused pass: BCE with no label (index -1) -> sum_j softplus;  KL with the one-hot label at
  //    column 0 -> lse_i - z_i0.  On the pre-split tensor-core path the SAME pass also emits the scores of the listed
  //    columns (and z_i0) from its epilogue (per-thread cursor into the row's sorted CSR segment, tc_common.cuh):
  //    DRAM traffic = table + queries + nnz * 12 bytes.
  B2K_CUDA(cudaMemsetAsync(b.lab, loss_kind == B200KGE_LOSS_BCE ? 0xFF : 0, (size_t)n * 8, st));
  bool emitted = false;
  {
    // zsum (label smoothing of the distance family): the CUDA-core pass also sums each row's scores
    const int epi = (loss_kind == B200KGE_LOSS_BCE) ? (zsum ? EPI_BCE_ZSUM : EPI_BCE) : (zsum ? EPI_KL_ZSUM : EPI_KL);
    for (int attempt = 0; attempt < 2; ++attempt) {
      EpiParams P = empty_epi();
      P.label_idx = b.lab;
      P.offset = (loss_kind == B200KGE_LOSS_BCE) ? offset : 0.f;
      P.zsum_part = zsum;
      if (attempt == 0) {
        P.csr_off = csr_off; P.csr_col = csr_col; P.csr_out = b.zpos; P.csr_nnz = nnz;
        P.csr_extra = (loss_kind == B200KGE_LOSS_KL) ? 1 : 0;
      }
      int nch = 0;
      float* part = nullptr;
      Arena w2 = ws;
      rc = run_block(B, l_norm, precision, epi, P, w2, st, &nch, &part);
      if (rc == B200KGE_ERR_UNSUPPORTED && attempt == 0) continue;      // not the pre-split path: compose below
      if (rc) return rc;
      emitted = (attempt == 0);
      if ((rc = launch_loss_finalize(loss_kind, part, nch, n, b.total, b.fused, 1.0f, 0, b.scratch, 0, st))) return rc;
      break;
    }
  }
  // 2. otherwise: scores of the listed columns (and of column 0 for KL) through the row-wise triple kernel
  if (!emitted) {
    if ((rc = launch_csr_expand(csr_off, csr_col, n, nnz, loss_kind == B200KGE_LOSS_KL ? 1 : 0, q.idx, p.idx, b.qsel,
                                b.psel, b.esel, st))) return rc;
    if (tot > 0) {
      Rows Qs = q; Qs.idx = b.qsel; Qs.rows = tot;
      Rows Ps = p; Ps.idx = b.psel; Ps.rows = tot;
      Rows Cs = cand; Cs.idx = b.esel; Cs.rows = tot;
      if (roles == B200KGE_SP_)      rc = launch_spo(model, l_norm, Qs, Ps, Cs, tot, b.zpos, 1, st);
      else if (roles == B200KGE__PO) rc = launch_spo(model, l_norm, Cs, Ps, Qs, tot, b.zpos, 1, st);
      else                           rc = launch_spo(model, l_norm, Qs, Cs, Ps, tot, b.zpos, 1, st);
      if (rc) return rc;
    }
  }
  return 0;
}

// Step 4: the per-row combination with labels y = a * count + b over m candidates, and the scalar
int csr_loss_rows(int loss_kind, const int64_t* csr_off, const int64_t* csr_col, int64_t n, int64_t nnz, int64_t m,
                  float label_smoothing, float offset, const float* zsum, int zch, const CsrBufs& b, float* loss_out,
                  cudaStream_t st) {
  const float a = 1.0f - label_smoothing, c = label_smoothing > 0.f ? 1.0f / (float)m : 0.f;
  int rc;
  if ((rc = launch_csr_rows(loss_kind, csr_off, csr_col, b.zpos, n, nnz, b.fused, zsum, zch, a, c, (float)m,
                            loss_kind == B200KGE_LOSS_BCE ? offset : 0.f, b.rows, st))) return rc;
  return launch_rows_sum(b.rows, n, 1.0f, loss_out, st);
}

size_t backward_block_bytes(int64_t nq, int64_t m, int64_t K, int64_t ldq) {
  const int64_t Ep = round_up(m, 64), Np = round_up(nq, 64);
  size_t b = (size_t)nq * round_up(m, 4) * 4 + 256;
  b += b200kge_workspace_bytes(0, nq, m, (int32_t)K, 0);
  b += planes_bytes(nq, nq, Ep) + planes_bytes(m, m, Np);
  b += (size_t)K * round_up(m, 4) * 4 + (size_t)K * round_up(nq, 4) * 4 + 2 * (size_t)nq * ldq * 4 + (size_t)nq * 8 + 5 * 256;
  b += planes_bytes(K, K + 32, Ep) + planes_bytes(K, K + 32, Np);
  return b;
}

}  // namespace

extern "C" {

size_t b200kge_gemm_nt_workspace_bytes(int64_t M, int64_t N, int64_t K) {
  const int64_t Kp = round_up(K, 64);
  return planes_bytes(M, M, Kp) + planes_bytes(N, N + 32, Kp) + 1024;
}

int b200kge_gemm_nt(const float* A, int64_t lda, const float* B, int64_t ldb, int64_t M, int64_t N, int64_t K,
                      float* C, int64_t ldc, void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  if (!A || !B || !C) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (M < 0 || N < 0 || K <= 0 || N >= (1ll << 31)) { set_error("bad GEMM shape"); return B200KGE_ERR_INVALID; }
  if (M == 0 || N == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  const int Kp = (int)round_up(K, 64);
  SplitSet SA{A, lda, nullptr, 0, M, M, (int)K, Kp, nullptr, nullptr, nullptr};
  SplitSet SB{B, ldb, nullptr, 0, N, N + 32, (int)K, Kp, nullptr, nullptr, nullptr};
  if (!take_planes(ws, SA) || !take_planes(ws, SB)) { set_error("workspace too small for the operand planes"); return B200KGE_ERR_WORKSPACE; }
  int rc = launch_presplit(SB, SA, st);
  if (rc) return rc;
  return gemm_planes(SA, SB, C, ldc, st);
}

// the workspace of train_1vsall_backward_impl
static size_t train_1vsall_backward_bytes(int model, int64_t n, int64_t E, int32_t D) {
  const int64_t K = (model == B200KGE_CP) ? D / 2 : D;
  const int64_t nq = 2 * n, ldq = round_up(K, 32);
  if (model == B200KGE_TRANSE || model == B200KGE_ROTATE)   // Q, dQ, labels, z, G, G^T, z^T, row stats + scorer workspace
    return 2 * (size_t)nq * ldq * 4 + (size_t)nq * 8 + 2 * (size_t)nq * round_up(E, 4) * 4 + 2 * (size_t)E * round_up(nq, 4) * 4 +
           (size_t)nq * 8 + 16 * 256 + b200kge_workspace_bytes(model, n, E, D, 0);
  return (size_t)nq * ldq * 4 + (size_t)n * 5 * 8 + 4096 + backward_block_bytes(nq, E, K, ldq);
}

// The backward of train_1vsall_forward_impl on validated arguments.  num_rel > 0: the reciprocal-relations step
static int train_1vsall_backward_impl(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                                      const int64_t* triples, int64_t n, int loss_kind, float offset, float* d_ent,
                                      int64_t lde, float* d_rel, int64_t ldr, void* workspace, size_t workspace_bytes,
                                      cudaStream_t st, int64_t num_rel) {
  int rc;
  Rows E = to_rows(ent), R = to_rows(rel);
  B2K_CUDA(cudaMemsetAsync(d_rel, 0, (size_t)R.rows * ldr * 4, st));
  if (n <= 0) { B2K_CUDA(cudaMemsetAsync(d_ent, 0, (size_t)E.rows * lde * 4, st)); return 0; }
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  if (model == B200KGE_TRANSE || model == B200KGE_ROTATE) {
    Folded f = folded_problem(model, B200KGE_SP_, E.dim, l_norm);
    if ((rc = check_distance_pair(f.pair_op))) return rc;
    const int64_t nq = 2 * n, ldq = round_up(f.K, 32);
    float* Q = (float*)ws.take((size_t)nq * ldq * 4);
    float* dQ = (float*)ws.take((size_t)nq * ldq * 4);
    int64_t* lab = (int64_t*)ws.take((size_t)nq * 8);
    if (!Q || !dQ || !lab) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
    if ((rc = launch_prep_1vsall(model, E, R, triples, n, Q, ldq, lab, nullptr, st, num_rel))) return rc;
    Rows S = E; S.idx = lab; S.rows = n;      // placeholders: operands are pre-folded
    Rows Pr = R; Pr.idx = lab; Pr.rows = n;
    Block B{model, B200KGE_SP_, &S, &S, &Pr, &E, n};
    B.Qpre = Q;
    B.same_fold = num_rel > 0;
    GradSpec g;
    g.lab = lab; g.loss_kind = loss_kind; g.offset = offset;
    if ((rc = distance_backward(B, l_norm, g, dQ, d_ent, lde, ws, st))) return rc;
    return launch_unfold_distance(model, E, R, triples, n, -1, dQ, ldq, d_ent, lde, d_rel, ldr, st, num_rel);
  }
  Folded f0 = folded_problem(model, B200KGE_SP_, E.dim, 1.0f),
         f1 = folded_problem(model, num_rel > 0 ? B200KGE_SP_ : B200KGE__PO, E.dim, 1.0f);
  const int64_t ldq = round_up(f0.K, 32);
  GradSpec g;
  g.loss_kind = loss_kind; g.offset = offset;
  if (f0.col_off == f1.col_off) {
    float* Q = (float*)ws.take((size_t)(2 * n) * ldq * 4);
    int64_t* lab = (int64_t*)ws.take((size_t)n * 2 * 8);
    if (!Q || !lab) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
    float* dQ = (float*)ws.take((size_t)(2 * n) * ldq * 4);
    if (!dQ) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
    if ((rc = launch_prep_1vsall(model, E, R, triples, n, Q, ldq, lab, nullptr, st, num_rel))) return rc;
    // reciprocal CP: the table GEMM stores columns [h, D) only; the unfold adds the rows' [0, h) into zeros
    if (f0.col_off > 0) B2K_CUDA(cudaMemset2DAsync(d_ent, (size_t)lde * 4, 0, (size_t)f0.col_off * 4, (size_t)E.rows, st));
    g.lab = lab;
    if ((rc = backward_block(model, E, R, n, -1, num_rel > 0, Q, ldq, f0.col_off, f0.K, g, d_ent, lde, dQ, ws, st))) return rc;
    return launch_unfold(model, E, R, triples, n, -1, dQ, ldq, d_ent, lde, d_rel, ldr, st, num_rel);
  }
  // CP: the two directions pair with different halves of the candidate columns
  int64_t* sidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* pidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* oidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* lab = (int64_t*)ws.take((size_t)n * 2 * 8);
  float* Q = (float*)ws.take((size_t)n * ldq * 4);
  float* dQ2 = (float*)ws.take((size_t)(2 * n) * ldq * 4);
  if (!sidx || !pidx || !oidx || !lab || !Q || !dQ2) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  Rows S, O, Pr;
  if ((rc = unpack_triples(triples, n, sidx, pidx, oidx, lab, E, R, S, O, Pr, st))) return rc;
  for (int dir = 0; dir < 2; ++dir) {
    const Folded& f = dir == 0 ? f0 : f1;
    if ((rc = launch_fold_queries(model, dir, dir == 0 ? S : O, Pr, n, 0, Q, ldq, st))) return rc;
    g.lab = lab + dir * n;
    if ((rc = backward_block(model, E, R, n, dir, false, Q, ldq, f.col_off, f.K, g, d_ent, lde,
                             dQ2 + (size_t)dir * n * ldq, ws, st))) return rc;
  }
  // both halves of the dense column gradient are stored: now add the batch rows' own gradients
  for (int dir = 0; dir < 2; ++dir)
    if ((rc = launch_unfold(model, E, R, triples, n, dir, dQ2 + (size_t)dir * n * ldq, ldq, d_ent, lde, d_rel, ldr, st))) return rc;
  return 0;
}

size_t b200kge_score_1vsN_backward_workspace_bytes(int model, int64_t n, int64_t E, int32_t D) {
  const int64_t K = (model == B200KGE_CP) ? D / 2 : D;
  const int64_t ldq = round_up(K, 32);
  // distance family: Q, dQ, triples [3n] + the KL row statistics of the CSR-label backward [2n floats] (n * 4 * 8 bytes),
  // z + W (L2) or z + G (CSR labels), W^T / G^T, scorer workspace
  if (model == B200KGE_TRANSE || model == B200KGE_ROTATE)
    return 2 * (size_t)n * ldq * 4 + (size_t)n * 4 * 8 + 2 * (size_t)n * round_up(E, 4) * 4 + (size_t)E * round_up(n, 4) * 4 +
           16 * 256 + b200kge_workspace_bytes(model, n, E, D, 0);
  return 2 * (size_t)n * ldq * 4 + (size_t)n * 4 * 8 + (size_t)E * round_up(n, 4) * 4 + 8192 + backward_block_bytes(n, E, K, ldq);
}

int b200kge_score_1vsN_backward(int model, int combine, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                                const int64_t* q_idx, const int64_t* p_idx, int64_t n, const float* grad_scores,
                                int64_t ldg, float* d_ent, int64_t lde, float* d_rel, int64_t ldr, void* workspace,
                                size_t workspace_bytes, b200kge_stream_t stream) {
  if (!q_idx || !p_idx || !grad_scores || !d_ent || !d_rel) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (combine != B200KGE_SP_ && combine != B200KGE__PO) { set_error("cannot handle combine=%d", combine); return B200KGE_ERR_INVALID; }
  int rc = check_tables(model, l_norm, ent, rel); if (rc) return rc;
  if ((rc = check_grad_ld(ent, lde, rel, ldr))) return rc;
  if (ldg < ent->rows) { set_error("grad_scores is narrower than the entity table"); return B200KGE_ERR_INVALID; }
  const bool distance = (model == B200KGE_TRANSE || model == B200KGE_ROTATE);
  cudaStream_t st = (cudaStream_t)stream;
  Rows E = to_rows(ent), R = to_rows(rel);
  Folded f = folded_problem(model, combine, E.dim, l_norm);
  if (distance && (rc = check_distance_pair(f.pair_op))) return rc;
  B2K_CUDA(cudaMemsetAsync(d_rel, 0, (size_t)R.rows * ldr * 4, st));
  B2K_CUDA(cudaMemsetAsync(d_ent, 0, (size_t)E.rows * lde * 4, st));
  if (n <= 0) return 0;
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  const int64_t ldq = round_up(f.K, 32);
  float* Q = (float*)ws.take((size_t)n * ldq * 4);
  float* dQ = (float*)ws.take((size_t)n * ldq * 4);
  int64_t* tri = (int64_t*)ws.take((size_t)n * 3 * 8);
  if (!Q || !dQ || !tri) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  // the unfold works on [n,3] triples: (q, p, .) for sp_, (., p, q) for _po
  pack_triples_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(q_idx, p_idx, n, combine, tri);
  B2K_LAUNCH_CHECK("pack_triples_kernel");
  Rows A = E; A.idx = q_idx; A.rows = n;
  Rows Pr = R; Pr.idx = p_idx; Pr.rows = n;
  if ((rc = launch_fold_queries(model, combine, A, Pr, n, 0, Q, ldq, st))) return rc;
  if (distance) {
    // W = dL/dscores (L2: divided by the recomputed scores), then the two row-gradient passes
    const int64_t m = E.rows, ldz = round_up(m, 4), ldN = round_up(n, 4);
    const float* W = grad_scores;
    int64_t ldw = ldg;
    if (f.pair_op == PAIR_L2) {
      float* z = (float*)ws.take((size_t)n * ldz * 4);
      float* Wd = (float*)ws.take((size_t)n * ldz * 4);
      if (!z || !Wd) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
      EpiParams P = empty_epi();
      P.out = z; P.ldo = ldz;
      Block B{model, combine, &A, nullptr, &Pr, &E, n};
      B.Qpre = Q;
      if ((rc = run_block(B, l_norm, B200KGE_PREC_AUTO, EPI_STORE, P, ws, st, nullptr))) return rc;
      if ((rc = launch_div_scores(grad_scores, ldg, z, ldz, n, m, Wd, ldz, st))) return rc;
      W = Wd; ldw = ldz;
    }
    float* Wt = (float*)ws.take((size_t)m * ldN * 4);
    if (!Wt) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
    if ((rc = distance_rowgrads(f.pair_op, Q, ldq, n, E, f.K, W, ldw, Wt, dQ, d_ent, lde, st))) return rc;
    return launch_unfold_distance(model, E, R, tri, n, combine, dQ, ldq, d_ent, lde, d_rel, ldr, st);
  }
  GradSpec g;
  g.G = grad_scores; g.ldg = ldg;
  if ((rc = backward_block(model, E, R, n, combine, false, Q, ldq, f.col_off, f.K, g, d_ent, lde, dQ, ws, st))) return rc;
  return launch_unfold(model, E, R, tri, n, combine, dQ, ldq, d_ent, lde, d_rel, ldr, st);
}

int b200kge_lookup_penalty(const b200kge_rows_t* rows, const float* counts, float p, int complex_abs, float scale,
                             float* out, void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  if (!rows || !out) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (!(p > 0.f)) { set_error("p must be positive (got %g)", (double)p); return B200KGE_ERR_INVALID; }
  if (complex_abs && (rows->dim & 1)) { set_error("complex-space penalty needs an even embedding width"); return B200KGE_ERR_INVALID; }
  return launch_penalty(to_rows(rows), counts, p, complex_abs, scale, (float*)workspace, workspace_bytes / 4, out,
                        (cudaStream_t)stream);
}

int b200kge_normalize_rows(float* weight, int64_t ld, int64_t rows, int32_t dim, float p, b200kge_stream_t stream) {
  if (!weight && rows > 0) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  return launch_normalize_rows(weight, ld, rows, dim, p, (cudaStream_t)stream);
}


size_t b200kge_ns_loss_workspace_bytes(int64_t n) { return (size_t)n * 2 * 4 + 256 + 1024; }

int b200kge_ns_loss(const float* scores, int64_t lds, int64_t n, int64_t m, const int64_t* label_idx,
                    int loss_kind, float arg, float temperature, float scale, float* loss_out,
                    float* row_loss_out, float* grad_out, int64_t ldg, void* workspace,
                    size_t workspace_bytes, b200kge_stream_t stream) {
  if ((!scores && n * m > 0) || !loss_out) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (loss_kind < B200KGE_LOSS_BCE || loss_kind > B200KGE_LOSS_SE) { set_error("unknown loss kind %d", loss_kind); return B200KGE_ERR_INVALID; }
  if (n > 0 && m < (loss_kind >= B200KGE_LOSS_BCE_MEAN && loss_kind <= B200KGE_LOSS_MARGIN_RANKING ? 2 : 1)) {
    set_error("loss kind %d needs a positive and at least one negative per row (m = %lld)", loss_kind, (long long)m);
    return B200KGE_ERR_INVALID;
  }
  if (lds < m || (grad_out && ldg < m)) { set_error("row stride smaller than the row width"); return B200KGE_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) { B2K_CUDA(cudaMemsetAsync(loss_out, 0, 4, st)); return 0; }
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  float* part = (float*)ws.take((size_t)n * 2 * 4);
  void* scratch = ws.take(1024);
  if (!part || !scratch) { set_error("workspace too small (need b200kge_ns_loss_workspace_bytes(n) = %zu bytes)", b200kge_ns_loss_workspace_bytes(n)); return B200KGE_ERR_WORKSPACE; }
  int rc = launch_ns_loss(loss_kind, scores, lds, n, m, label_idx, arg, temperature, scale, part, grad_out, ldg, st);
  if (rc) return rc;
  return launch_loss_finalize(B200KGE_LOSS_BCE, part, 1, n, loss_out, row_loss_out, scale, 0, scratch, 0, st);
}


size_t b200kge_score_1vsN_loss_csr_workspace_bytes(int model, int64_t n, int64_t m, int32_t D, int64_t nnz) {
  const int64_t ldq = round_up(D, 32), tot = nnz + n;
  size_t b = b200kge_workspace_bytes(model, n, m, D, 0);
  b += (size_t)n * 8 + 3 * ((size_t)tot * 8 + 256) + (size_t)tot * 4 + 4 * ((size_t)n * 4 + 256) + 2048;
  b += (size_t)n * ldq * 4 + ((size_t)((m + 1023) / 1024) + 1) * ldq * 4 + 512;
  if (model == B200KGE_TRANSE || model == B200KGE_ROTATE)    // label smoothing: the scorer's partial row score sums
    b += (size_t)n * pairwise_simt_nchunks(n, m) * 4 + 256;
  return b;
}

int b200kge_score_1vsN_loss_csr(int model, int combine, float l_norm, int precision, const b200kge_rows_t* q,
                                  const b200kge_rows_t* p, const b200kge_rows_t* cand, int64_t n,
                                  const int64_t* csr_off, const int64_t* csr_col, int64_t nnz, float label_smoothing,
                                  int loss_kind, float offset, float* loss_out, float* row_loss_out, void* workspace,
                                  size_t workspace_bytes, b200kge_stream_t stream) {
  int rc = check_1vsN_args(model, combine, q, p, cand, n); if (rc) return rc;
  if ((rc = validate_norm(model, l_norm))) return rc;
  if (!csr_off || (!csr_col && nnz > 0) || !loss_out || nnz < 0) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (cand->idx) { set_error("CSR labels address the columns of a plain candidate table (cand.idx must be NULL)"); return B200KGE_ERR_INVALID; }
  if ((rc = check_loss_kind(loss_kind))) return rc;
  if (!(label_smoothing >= 0.f && label_smoothing < 1.f)) { set_error("label_smoothing must be in [0, 1)"); return B200KGE_ERR_INVALID; }
  const bool dot = model <= B200KGE_RESCAL;
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0 || cand->rows == 0) { B2K_CUDA(cudaMemsetAsync(loss_out, 0, 4, st)); return 0; }
  Rows Q = to_rows(q), Pr = to_rows(p), C = to_rows(cand);
  const int64_t m = C.rows;
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  CsrBufs cb;
  const bool bufs = take_csr_bufs(ws, n, nnz, loss_kind, row_loss_out, cb);
  // label smoothing needs sum_j z_ij: the distance family's CUDA-core pass below sums it per row and column chunk
  const bool zsum_fused = label_smoothing > 0.f && !dot;
  const int zch = zsum_fused ? pairwise_simt_nchunks(n, m) : 1;
  float* zsum = zsum_fused ? (float*)ws.take((size_t)n * zch * 4) : nullptr;
  if (!bufs || (zsum_fused && !zsum)) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  Block B{model, combine, &Q, nullptr, &Pr, &C, n};
  if ((rc = csr_loss_terms(B, model, combine, l_norm, precision, Q, Pr, C, csr_off, csr_col, nnz, loss_kind, offset, zsum,
                           cb, ws, st))) return rc;
  // 3. label smoothing: sum_j z_ij = Q_i . colsum(T)   (dot family)
  if (label_smoothing > 0.f && dot) {
    Folded f = folded_problem(model, combine, Q.dim, l_norm);
    const int64_t ldq = round_up(f.K, 32);
    float* Qf = (float*)ws.take((size_t)n * ldq * 4);
    float* cs = (float*)ws.take(((size_t)((m + 1023) / 1024) + 1) * ldq * 4);
    zsum = (float*)ws.take((size_t)n * 4);
    if (!Qf || !cs || !zsum) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
    if ((rc = launch_fold_queries(model, combine, Q, Pr, n, 0, Qf, ldq, st))) return rc;
    if ((rc = launch_row_score_sums(Qf, ldq, n, C.base + f.col_off, C.ld, m, f.K, cs, zsum, st))) return rc;
  }
  return csr_loss_rows(loss_kind, csr_off, csr_col, n, nnz, m, label_smoothing, offset, zsum, zch, cb, loss_out, st);
}

}  // extern "C"

// ==================================================================================================
// Embedding dropout for the 1vsAll and KvsAll training steps (layout: include/b200kge.h, kernels: dropout.cu).  Each
// direction gathers masked copies of its query rows, relation rows and candidate table into the workspace and runs the
// existing per-direction machinery on them as plain operands (idx = NULL).  The backward hands the unfold identity
// triples, so row i's gradient lands in row i of [n, D] buffers, and then adds the masked table gradient and scatters
// the masked row gradients into d_ent / d_rel: two directions that read the same table columns under different masks
// contribute the SUM of their masked dT.
namespace {

int validate_dropout(const b200kge_dropout_t* d, int64_t n, int64_t E, int D, int Dr) {
  if (!d) { set_error("null dropout key"); return B200KGE_ERR_INVALID; }
  if (!(d->p_ent >= 0.f && d->p_ent < 1.f) || !(d->p_rel >= 0.f && d->p_rel < 1.f)) {
    set_error("dropout rates must lie in [0, 1) (got %g, %g)", (double)d->p_ent, (double)d->p_rel);
    return B200KGE_ERR_INVALID;
  }
  const double lim = 281474976710656.0;    // 2^48: elem >> 2 must fit below the stream bits of the counter
  if (d->row_base < 0 || (double)(d->row_base + n) * D > lim || (double)(d->row_base + n) * Dr > lim ||
      (double)E * D > lim) {
    set_error("dropout rows out of range: row_base >= 0 and row * dim + k < 2^48 are required");
    return B200KGE_ERR_INVALID;
  }
  return 0;
}

DropMask drop_mask(float p, uint64_t seed, uint64_t call, int stream, int64_t row_base) {
  DropMask m;
  m.seed = seed; m.call = call; m.stream = stream; m.row_base = row_base;
  m.thresh = (uint64_t)floor((1.0 - (double)p) * 4294967296.0);
  m.scale = (float)(1.0 / (1.0 - (double)p));
  return m;
}

// the three draws of one direction: query entity rows, relation rows, candidate table
struct DirMasks { DropMask q, r, t; };
DirMasks dir_masks(const b200kge_dropout_t& d, int dir) {
  DirMasks m;
  m.q = drop_mask(d.p_ent, d.seed, d.call, dir == 0 ? B200KGE_DROP_SP_ENT : B200KGE_DROP_PO_ENT, d.row_base);
  m.r = drop_mask(d.p_rel, d.seed, d.call, dir == 0 ? B200KGE_DROP_SP_REL : B200KGE_DROP_PO_REL, d.row_base);
  m.t = drop_mask(d.p_ent, d.seed, d.call, dir == 0 ? B200KGE_DROP_SP_TABLE : B200KGE_DROP_PO_TABLE, 0);
  return m;
}

// masked copies of one direction's operands: Qm [n, D], Pm [n, Dr], Tm [E, D] (row strides = widths)
struct MaskedOps { float *Qm, *Pm, *Tm; };
bool take_masked(Arena& ws, int64_t n, int64_t E, int D, int Dr, MaskedOps& o) {
  o.Qm = (float*)ws.take((size_t)n * D * 4);
  o.Pm = (float*)ws.take((size_t)n * Dr * 4);
  o.Tm = (float*)ws.take((size_t)E * D * 4);
  return o.Qm && o.Pm && o.Tm;
}
int gather_masked(const DirMasks& m, const Rows& E, const Rows& R, const int64_t* q_idx, const int64_t* p_idx, int64_t n,
                  const MaskedOps& o, Rows& Qr, Rows& Pr, Rows& Tr, cudaStream_t st) {
  Rows qs = E; qs.idx = q_idx; qs.rows = n;
  Rows ps = R; ps.idx = p_idx; ps.rows = n;
  Rows ts = E; ts.idx = nullptr;
  int rc;
  if ((rc = launch_dropout_gather(m.q, qs, o.Qm, E.dim, st))) return rc;
  if ((rc = launch_dropout_gather(m.r, ps, o.Pm, R.dim, st))) return rc;
  if ((rc = launch_dropout_gather(m.t, ts, o.Tm, E.dim, st))) return rc;
  Qr = Rows{o.Qm, nullptr, n, E.dim, E.dim};
  Pr = Rows{o.Pm, nullptr, n, R.dim, R.dim};
  Tr = Rows{o.Tm, nullptr, E.rows, E.dim, E.dim};
  return 0;
}

size_t masked_bytes(int model, int64_t n, int64_t E, int32_t D) {
  const int64_t Dr = relation_dim(model, D), ldq = round_up(D, 32);
  return 2 * ((size_t)E * D * 4 + 256)                       // Tm, dT
         + 2 * ((size_t)n * D * 4 + (size_t)n * Dr * 4 + 512)  // Qm, Pm, dQe, dPr
         + 2 * ((size_t)n * ldq * 4 + 256)                     // Q, dQ
         + (size_t)n * 10 * 8 + 5 * 256                        // s/p/o, labels [2n], identity triples [3n]
         + (size_t)n * 2 * 4 + 4096;                           // KL row statistics, scalars
}

// the per-direction buffers of the backward
struct BackBufs { MaskedOps o; float *Q, *dQ, *dT, *dQe, *dPr; int64_t* tri; };
bool take_back(Arena& ws, int64_t n, int64_t E, int D, int Dr, int64_t ldq, BackBufs& b) {
  if (!take_masked(ws, n, E, D, Dr, b.o)) return false;
  b.Q = (float*)ws.take((size_t)n * ldq * 4);
  b.dQ = (float*)ws.take((size_t)n * ldq * 4);
  b.dT = (float*)ws.take((size_t)E * D * 4);
  b.dQe = (float*)ws.take((size_t)n * D * 4);
  b.dPr = (float*)ws.take((size_t)n * Dr * 4);
  b.tri = (int64_t*)ws.take((size_t)n * 3 * 8);
  return b.Q && b.dQ && b.dT && b.dQe && b.dPr && b.tri;
}

// One direction of the masked backward: gather, fold, dT and dQ (tensor-core GEMMs or the distance row-gradient
// passes), unfold into the per-row buffers, then d_ent[:, cols] += mask_t * dT, d_ent[q] += mask_q * dQe,
// d_rel[p] += mask_r * dPr.  `dir` is the fold (query type); `mask_dir` picks the draws (they differ for the
// reciprocal direction: sp_ fold, _po draws).
int dropout_backward_dir(int model, float l_norm, int dir, int mask_dir, const Rows& E, const Rows& R, const int64_t* q_idx,
                         const int64_t* p_idx, int64_t n, const b200kge_dropout_t& d, const GradSpec& g,
                         const BackBufs& b, Arena ws, float* d_ent, int64_t lde, float* d_rel, int64_t ldr, cudaStream_t st) {
  const DirMasks m = dir_masks(d, mask_dir);
  const Folded f = folded_problem(model, dir, E.dim, l_norm);
  const int64_t ldq = round_up(f.K, 32), mE = E.rows;
  const int D = E.dim, Dr = R.dim;
  Rows Qr, Pr, Tr;
  int rc = gather_masked(m, E, R, q_idx, p_idx, n, b.o, Qr, Pr, Tr, st);
  if (rc) return rc;
  if ((rc = launch_fold_queries(model, dir, Qr, Pr, n, 0, b.Q, ldq, st))) return rc;
  B2K_CUDA(cudaMemsetAsync(b.dQe, 0, (size_t)n * D * 4, st));
  B2K_CUDA(cudaMemsetAsync(b.dPr, 0, (size_t)n * Dr * 4, st));
  if (f.pair_op == PAIR_DOT) {
    if ((rc = backward_block(model, Tr, Pr, n, dir, false, b.Q, ldq, f.col_off, f.K, g, b.dT, D, b.dQ, ws, st))) return rc;
    if ((rc = launch_unfold(model, Qr, Pr, b.tri, n, dir, b.dQ, ldq, b.dQe, D, b.dPr, Dr, st))) return rc;
  } else {
    Block B{model, dir, &Qr, nullptr, &Pr, &Tr, n};
    B.Qpre = b.Q;
    if ((rc = distance_backward(B, l_norm, g, b.dQ, b.dT, D, ws, st))) return rc;
    if ((rc = launch_unfold_distance(model, Qr, Pr, b.tri, n, dir, b.dQ, ldq, b.dQe, D, b.dPr, Dr, st))) return rc;
  }
  if ((rc = launch_dropout_add_cols(m.t, b.dT, D, mE, D, f.col_off, f.col_off + f.K, d_ent, lde, st))) return rc;
  if ((rc = launch_dropout_scatter(m.q, b.dQe, D, n, D, q_idx, d_ent, lde, st))) return rc;
  return launch_dropout_scatter(m.r, b.dPr, Dr, n, Dr, p_idx, d_rel, ldr, st);
}

Arena rest_of(const Arena& ws) {
  const size_t used = (ws.off + 255) & ~size_t(255);
  return Arena{ws.base + used, used < ws.cap ? ws.cap - used : 0, 0};
}

}  // namespace

extern "C" {

int b200kge_dropout_mask(float p, uint64_t seed, uint64_t call, int mask_stream, int64_t row_base, int64_t rows,
                         int32_t dim, uint8_t* out, b200kge_stream_t stream) {
  if (!out && rows > 0 && dim > 0) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (rows < 0 || dim < 0 || mask_stream < 0 || mask_stream >= (1 << 18)) { set_error("bad mask shape or stream"); return B200KGE_ERR_INVALID; }
  b200kge_dropout_t d{p, 0.f, seed, call, row_base};
  int rc = validate_dropout(&d, rows, 0, dim, 0); if (rc) return rc;
  return launch_dropout_mask(drop_mask(p, seed, call, mask_stream, row_base), rows, dim, out, (cudaStream_t)stream);
}

// The 1vsAll step under embedding dropout on validated arguments, n > 0; the masks of direction dir are drawn on dir's
// streams.  num_rel > 0: the reciprocal-relations step (reciprocal_relations_model.py:85-92): both directions are sp_
// queries against the table; the second one, (o, p + R) labelled s, is score_po and draws its masks on the _po streams
// in the reference's call order (embed_all: B200KGE_DROP_PO_TABLE, embed(p + R): B200KGE_DROP_PO_REL, embed(o):
// B200KGE_DROP_PO_ENT).
static int train_1vsall_forward_dropout_impl(int model, float l_norm, int precision, const b200kge_rows_t* ent,
                                             const b200kge_rows_t* rel, const int64_t* triples, int64_t n,
                                             int loss_kind, float offset, const b200kge_dropout_t* drop,
                                             float* loss_out, void* workspace, size_t workspace_bytes,
                                             cudaStream_t st, int64_t num_rel) {
  int rc;
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  Rows E = to_rows(ent), R = to_rows(rel);
  int64_t* sidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* pidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* oidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* pinv = num_rel > 0 ? (int64_t*)ws.take((size_t)n * 8) : nullptr;
  int64_t* lab = (int64_t*)ws.take((size_t)n * 2 * 8);
  float* dir_loss = (float*)ws.take(256);
  MaskedOps o;
  if (!sidx || !pidx || !oidx || (num_rel > 0 && !pinv) || !lab || !dir_loss ||
      !take_masked(ws, n, E.rows, E.dim, R.dim, o)) {
    set_error("workspace too small (see b200kge_train_1vsall_workspace_bytes)");
    return B200KGE_ERR_WORKSPACE;
  }
  Rows S, O, P;
  if ((rc = unpack_triples(triples, n, sidx, pidx, oidx, lab, E, R, S, O, P, st))) return rc;
  if (num_rel > 0) {
    offset_index_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(pidx, n, num_rel, pinv);
    B2K_LAUNCH_CHECK("offset_index_kernel");
  }
  const Arena rest = rest_of(ws);
  for (int dir = 0; dir < 2; ++dir) {
    Rows Qr, Pr, Tr;
    if ((rc = gather_masked(dir_masks(*drop, dir), E, R, dir == 0 ? sidx : oidx, dir == 1 && pinv ? pinv : pidx, n, o,
                            Qr, Pr, Tr, st))) return rc;
    const b200kge_rows_t q{Qr.base, nullptr, n, Qr.ld, Qr.dim}, p{Pr.base, nullptr, n, Pr.ld, Pr.dim},
        c{Tr.base, nullptr, Tr.rows, Tr.ld, Tr.dim};
    const b200kge_labels_t labels{lab + dir * n, nullptr, 0};
    if ((rc = b200kge_score_1vsN_loss(model, num_rel > 0 ? B200KGE_SP_ : dir, l_norm, precision, &q, &p, &c, n, &labels,
                                      loss_kind, offset, dir_loss + dir, nullptr, rest.base, rest.cap, st))) return rc;
  }
  return launch_rows_sum(dir_loss, 2, 1.0f / (float)n, loss_out, st);    // (loss_sp + loss_po) / n
}

// the backward of train_1vsall_forward_dropout_impl, on validated arguments
static int train_1vsall_backward_dropout_impl(int model, float l_norm, const b200kge_rows_t* ent,
                                              const b200kge_rows_t* rel, const int64_t* triples, int64_t n,
                                              int loss_kind, float offset, const b200kge_dropout_t* drop, float* d_ent,
                                              int64_t lde, float* d_rel, int64_t ldr, void* workspace,
                                              size_t workspace_bytes, cudaStream_t st, int64_t num_rel) {
  int rc;
  const Folded f = folded_problem(model, B200KGE_SP_, ent->dim, l_norm);
  if (f.pair_op != PAIR_DOT && (rc = check_distance_pair(f.pair_op))) return rc;
  Rows E = to_rows(ent), R = to_rows(rel);
  B2K_CUDA(cudaMemsetAsync(d_rel, 0, (size_t)R.rows * ldr * 4, st));
  B2K_CUDA(cudaMemsetAsync(d_ent, 0, (size_t)E.rows * lde * 4, st));
  if (n <= 0) return 0;
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  int64_t* sidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* pidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* oidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* pinv = num_rel > 0 ? (int64_t*)ws.take((size_t)n * 8) : nullptr;
  int64_t* lab = (int64_t*)ws.take((size_t)n * 2 * 8);
  BackBufs b;
  if (!sidx || !pidx || !oidx || (num_rel > 0 && !pinv) || !lab ||
      !take_back(ws, n, E.rows, E.dim, R.dim, round_up(f.K, 32), b)) {
    set_error("workspace too small (see b200kge_train_1vsall_workspace_bytes)");
    return B200KGE_ERR_WORKSPACE;
  }
  Rows S, O, P;
  if ((rc = unpack_triples(triples, n, sidx, pidx, oidx, lab, E, R, S, O, P, st))) return rc;
  if (num_rel > 0) {
    offset_index_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(pidx, n, num_rel, pinv);
    B2K_LAUNCH_CHECK("offset_index_kernel");
  }
  if ((rc = launch_identity_triples(n, b.tri, st))) return rc;
  const Arena rest = rest_of(ws);
  GradSpec g;
  g.loss_kind = loss_kind; g.offset = offset;
  for (int dir = 0; dir < 2; ++dir) {
    g.lab = lab + dir * n;
    if ((rc = dropout_backward_dir(model, l_norm, num_rel > 0 ? B200KGE_SP_ : dir, dir, E, R, dir == 0 ? sidx : oidx,
                                   dir == 1 && pinv ? pinv : pidx, n, *drop, g, b, rest, d_ent, lde, d_rel, ldr, st)))
      return rc;
  }
  return 0;
}

// rel holds the 2 * num_rel rows of a reciprocal-relations base model; num_rel = 0 is the plain model
int b200kge_train_1vsall_forward(int model, float l_norm, int precision, const b200kge_rows_t* ent,
                                 const b200kge_rows_t* rel, int64_t num_relations, const int64_t* triples, int64_t n,
                                 int loss_kind, float offset, const b200kge_dropout_t* drop, float* loss_out,
                                 void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  if (!ent || !rel || !triples || !loss_out) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  int rc;
  if (num_relations != 0 && (rc = check_reciprocal(rel, num_relations))) return rc;
  if ((rc = check_tables(model, l_norm, ent, rel))) return rc;
  if ((rc = check_loss_kind(loss_kind))) return rc;
  if (drop && (rc = validate_dropout(drop, n > 0 ? n : 0, ent->rows, ent->dim, rel->dim))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0) { B2K_CUDA(cudaMemsetAsync(loss_out, 0, 4, st)); return 0; }
  if (drop)
    return train_1vsall_forward_dropout_impl(model, l_norm, precision, ent, rel, triples, n, loss_kind, offset, drop,
                                             loss_out, workspace, workspace_bytes, st, num_relations);
  return train_1vsall_forward_impl(model, l_norm, precision, ent, rel, triples, n, loss_kind, offset, loss_out,
                                   workspace, workspace_bytes, st, num_relations);
}

int b200kge_train_1vsall_backward(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                                  int64_t num_relations, const int64_t* triples, int64_t n, int loss_kind, float offset,
                                  const b200kge_dropout_t* drop, float* d_ent, int64_t lde, float* d_rel, int64_t ldr,
                                  void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  if (!ent || !rel || !triples || !d_ent || !d_rel) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  int rc;
  if (num_relations != 0 && (rc = check_reciprocal(rel, num_relations))) return rc;
  if ((rc = check_tables(model, l_norm, ent, rel))) return rc;
  if ((rc = check_loss_kind(loss_kind))) return rc;
  if ((rc = check_grad_ld(ent, lde, rel, ldr))) return rc;
  if (drop && (rc = validate_dropout(drop, n > 0 ? n : 0, ent->rows, ent->dim, rel->dim))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (drop)
    return train_1vsall_backward_dropout_impl(model, l_norm, ent, rel, triples, n, loss_kind, offset, drop, d_ent, lde,
                                              d_rel, ldr, workspace, workspace_bytes, st, num_relations);
  return train_1vsall_backward_impl(model, l_norm, ent, rel, triples, n, loss_kind, offset, d_ent, lde, d_rel, ldr,
                                    workspace, workspace_bytes, st, num_relations);
}

size_t b200kge_train_1vsall_workspace_bytes(int model, int64_t n, int64_t E, int32_t D, int dropout) {
  const size_t fwd = b200kge_workspace_bytes(model, n, E, D, 0);
  if (dropout) {
    // the masked copies and per-direction buffers, the larger of one direction's forward and backward, the p + R index
    const size_t dir = b200kge_score_1vsN_backward_workspace_bytes(model, n, E, D) + (size_t)n * 2 * 4 + 1024;
    return masked_bytes(model, n, E, D) + (dir > fwd ? dir : fwd) + (size_t)n * 8 + 256;
  }
  const size_t bwd = train_1vsall_backward_bytes(model, n, E, D);
  return fwd > bwd ? fwd : bwd;
}

size_t b200kge_score_1vsN_loss_csr_dropout_workspace_bytes(int model, int64_t n, int64_t E, int32_t D, int64_t nnz) {
  const size_t fwd = b200kge_score_1vsN_loss_csr_workspace_bytes(model, n, E, D, nnz);
  const size_t bwd = b200kge_score_1vsN_backward_workspace_bytes(model, n, E, D) + 1024;
  return masked_bytes(model, n, E, D) + (fwd > bwd ? fwd : bwd);
}

int b200kge_score_1vsN_loss_csr_dropout(int model, int combine, int mask_dir, float l_norm, int precision,
                                        const b200kge_rows_t* ent, const b200kge_rows_t* rel, const int64_t* q_idx,
                                        const int64_t* p_idx, int64_t n, const int64_t* csr_off, const int64_t* csr_col,
                                        int64_t nnz, float label_smoothing, int loss_kind, float offset,
                                        const b200kge_dropout_t* drop, float* loss_out, float* row_loss_out,
                                        void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  if ((!q_idx && n > 0) || (!p_idx && n > 0) || !loss_out) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (combine != B200KGE_SP_ && combine != B200KGE__PO) { set_error("cannot handle combine=%d", combine); return B200KGE_ERR_INVALID; }
  if (mask_dir != B200KGE_SP_ && mask_dir != B200KGE__PO) { set_error("bad mask direction %d", mask_dir); return B200KGE_ERR_INVALID; }
  // l_norm is checked by b200kge_score_1vsN_loss_csr below
  int rc = check_tables(model, 1.0f, ent, rel); if (rc) return rc;
  if ((rc = validate_dropout(drop, n > 0 ? n : 0, ent->rows, ent->dim, rel->dim))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0) { B2K_CUDA(cudaMemsetAsync(loss_out, 0, 4, st)); return 0; }
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  Rows E = to_rows(ent), R = to_rows(rel);
  MaskedOps o;
  if (!take_masked(ws, n, E.rows, E.dim, R.dim, o)) {
    set_error("workspace too small (see b200kge_score_1vsN_loss_csr_dropout_workspace_bytes)");
    return B200KGE_ERR_WORKSPACE;
  }
  Rows Qr, Pr, Tr;
  if ((rc = gather_masked(dir_masks(*drop, mask_dir), E, R, q_idx, p_idx, n, o, Qr, Pr, Tr, st))) return rc;
  const b200kge_rows_t q{Qr.base, nullptr, n, Qr.ld, Qr.dim}, p{Pr.base, nullptr, n, Pr.ld, Pr.dim},
      c{Tr.base, nullptr, Tr.rows, Tr.ld, Tr.dim};
  const Arena rest = rest_of(ws);
  return b200kge_score_1vsN_loss_csr(model, combine, l_norm, precision, &q, &p, &c, n, csr_off, csr_col, nnz,
                                     label_smoothing, loss_kind, offset, loss_out, row_loss_out, rest.base, rest.cap,
                                     stream);
}

int b200kge_score_1vsN_loss_csr_backward(int model, int combine, int mask_dir, float l_norm, const b200kge_rows_t* ent,
                                         const b200kge_rows_t* rel, const int64_t* q_idx, const int64_t* p_idx,
                                         int64_t n, const int64_t* csr_off, const int64_t* csr_col,
                                         float label_smoothing, int loss_kind, float offset, int64_t batch_size,
                                         const b200kge_dropout_t* drop, float* d_ent, int64_t lde, float* d_rel,
                                         int64_t ldr, void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  if (!q_idx || !p_idx || !csr_off || !d_ent || !d_rel) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (combine != B200KGE_SP_ && combine != B200KGE__PO) { set_error("cannot handle combine=%d", combine); return B200KGE_ERR_INVALID; }
  if (drop && mask_dir != B200KGE_SP_ && mask_dir != B200KGE__PO) { set_error("bad mask direction %d", mask_dir); return B200KGE_ERR_INVALID; }
  int rc = check_tables(model, l_norm, ent, rel); if (rc) return rc;
  const bool distance = (model == B200KGE_TRANSE || model == B200KGE_ROTATE);
  if (!distance) l_norm = 1.0f;                                           // the dot family folds with l_norm 1
  const Folded f = folded_problem(model, combine, ent->dim, l_norm);
  if (distance && (rc = check_distance_pair(f.pair_op))) return rc;
  if ((rc = check_loss_kind(loss_kind))) return rc;
  if (batch_size <= 0 || !(label_smoothing >= 0.f && label_smoothing < 1.f)) { set_error("bad batch_size / label_smoothing"); return B200KGE_ERR_INVALID; }
  if ((rc = check_grad_ld(ent, lde, rel, ldr))) return rc;
  if (drop && (rc = validate_dropout(drop, n > 0 ? n : 0, ent->rows, ent->dim, rel->dim))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Rows E = to_rows(ent), R = to_rows(rel);
  B2K_CUDA(cudaMemsetAsync(d_rel, 0, (size_t)R.rows * ldr * 4, st));
  B2K_CUDA(cudaMemsetAsync(d_ent, 0, (size_t)E.rows * lde * 4, st));
  if (n <= 0) return 0;
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  const int64_t ldq = round_up(f.K, 32);
  const GradSpec g = csr_grad(q_idx, csr_off, csr_col, label_smoothing, E.rows, batch_size, loss_kind, offset);
  if (drop) {
    BackBufs b;
    if (!take_back(ws, n, E.rows, E.dim, R.dim, ldq, b)) {
      set_error("workspace too small (see b200kge_score_1vsN_loss_csr_dropout_workspace_bytes)");
      return B200KGE_ERR_WORKSPACE;
    }
    if ((rc = launch_identity_triples(n, b.tri, st))) return rc;
    return dropout_backward_dir(model, l_norm, combine, mask_dir, E, R, q_idx, p_idx, n, *drop, g, b, rest_of(ws), d_ent,
                                lde, d_rel, ldr, st);
  }
  float* Q = (float*)ws.take((size_t)n * ldq * 4);
  float* dQ = (float*)ws.take((size_t)n * ldq * 4);
  int64_t* tri = (int64_t*)ws.take((size_t)n * 3 * 8);
  if (!Q || !dQ || !tri) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  pack_triples_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(q_idx, p_idx, n, combine, tri);
  B2K_LAUNCH_CHECK("pack_triples_kernel");
  Rows A = E; A.idx = q_idx; A.rows = n;
  Rows Pr = R; Pr.idx = p_idx; Pr.rows = n;
  if ((rc = launch_fold_queries(model, combine, A, Pr, n, 0, Q, ldq, st))) return rc;
  if (distance) {
    Block B{model, combine, &A, nullptr, &Pr, &E, n};
    B.Qpre = Q;
    if ((rc = distance_backward(B, l_norm, g, dQ, d_ent, lde, ws, st))) return rc;
    return launch_unfold_distance(model, E, R, tri, n, combine, dQ, ldq, d_ent, lde, d_rel, ldr, st);
  }
  if ((rc = backward_block(model, E, R, n, combine, false, Q, ldq, f.col_off, f.K, g, d_ent, lde, dQ, ws, st))) return rc;
  return launch_unfold(model, E, R, tri, n, combine, dQ, ldq, d_ent, lde, d_rel, ldr, st);
}

}  // extern "C"

// ==================================================================================================
// KvsAll's s_o query type (relation prediction, train_KvsAll.py:251-254,278-281 with kge_model.py:727-747): every (s, o)
// pair scored against the whole relation table.  The s_o fold (fold.cu) turns the pair into one query row
// Q_i = fold_so(s_i, o_i) with score(s_i, r, o_i) = Q_i . rel[r], so the relation table is the candidate table of a
// plain dot-product block (the DistMult pair problem of width K = relation_dim): the CSR-label loss steps and the
// backward block of the entity query types run on it unchanged, and the unfold is the fold's VJP.
namespace {

int check_so_args(int model, const b200kge_rows_t* ent, const b200kge_rows_t* rel, const int64_t* s_idx,
                  const int64_t* o_idx, int64_t n, const int64_t* csr_off, int loss_kind) {
  if (!ent || !rel || ((!s_idx || !o_idx) && n > 0) || !csr_off) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (n < 0) { set_error("negative n"); return B200KGE_ERR_INVALID; }
  int rc = check_tables(model, 1.0f, ent, rel); if (rc) return rc;
  if (model == B200KGE_TRANSE || model == B200KGE_ROTATE) {
    set_error("the s_o query type covers the dot family (ComplEx, DistMult, SimplE, CP, RESCAL)");
    return B200KGE_ERR_UNSUPPORTED;
  }
  return check_loss_kind(loss_kind);
}

// the three s_o draws (include/b200kge.h): embed(s), embed(o) at mask rows row_base + i, embed_all() of the relations
struct SoMasks { DropMask s, o, t; };
SoMasks so_masks(const b200kge_dropout_t& d) {
  return SoMasks{drop_mask(d.p_ent, d.seed, d.call, B200KGE_DROP_SO_S, d.row_base),
                 drop_mask(d.p_ent, d.seed, d.call, B200KGE_DROP_SO_O, d.row_base),
                 drop_mask(d.p_rel, d.seed, d.call, B200KGE_DROP_SO_TABLE, 0)};
}

int validate_so_dropout(const b200kge_dropout_t* drop, int64_t n, const b200kge_rows_t* ent, const b200kge_rows_t* rel) {
  int rc = validate_dropout(drop, n, ent->rows, ent->dim, rel->dim);
  return rc ? rc : validate_dropout(drop, n, rel->rows, rel->dim, rel->dim);    // the relation table draw
}

// masked copies Sm, Om [n, D] and Tm [R, K] (row strides = widths)
struct SoMasked { float *Sm, *Om, *Tm; };
bool take_so_masked(Arena& ws, int64_t n, const Rows& E, const Rows& R, SoMasked& m) {
  m.Sm = (float*)ws.take((size_t)n * E.dim * 4);
  m.Om = (float*)ws.take((size_t)n * E.dim * 4);
  m.Tm = (float*)ws.take((size_t)R.rows * R.dim * 4);
  return m.Sm && m.Om && m.Tm;
}
int gather_so_masked(const SoMasks& k, const Rows& E, const Rows& R, const int64_t* s_idx, const int64_t* o_idx,
                     int64_t n, const SoMasked& m, Rows& S, Rows& O, Rows& T, cudaStream_t st) {
  Rows ss = E; ss.idx = s_idx; ss.rows = n;
  Rows os = E; os.idx = o_idx; os.rows = n;
  int rc;
  if ((rc = launch_dropout_gather(k.s, ss, m.Sm, E.dim, st))) return rc;
  if ((rc = launch_dropout_gather(k.o, os, m.Om, E.dim, st))) return rc;
  if ((rc = launch_dropout_gather(k.t, R, m.Tm, R.dim, st))) return rc;
  S = Rows{m.Sm, nullptr, n, E.dim, E.dim};
  O = Rows{m.Om, nullptr, n, E.dim, E.dim};
  T = Rows{m.Tm, nullptr, R.rows, R.dim, R.dim};
  return 0;
}

size_t so_masked_bytes(int64_t n, int64_t R, int32_t D, int64_t K) {
  return 2 * (2 * (size_t)n * D * 4 + (size_t)R * K * 4 + 3 * 256);    // Sm, Om, Tm and their gradients
}

// The s_o loss on validated operands, n > 0: S, O the pair rows (index views of the entity table or masked copies),
// T the relation table (or its masked copy)
int so_loss_impl(int model, int precision, const Rows& S, const Rows& O, const Rows& T, int64_t n, const int64_t* csr_off,
                 const int64_t* csr_col, int64_t nnz, int loss_kind, float offset, float* loss_out, float* row_loss_out,
                 Arena ws, cudaStream_t st) {
  const int64_t ldq = round_up(T.dim, 32);
  float* Q = (float*)ws.take((size_t)n * ldq * 4);
  CsrBufs cb;
  if (!Q || !take_csr_bufs(ws, n, nnz, loss_kind, row_loss_out, cb)) {
    set_error("workspace too small (see b200kge_score_so_loss_csr_workspace_bytes)");
    return B200KGE_ERR_WORKSPACE;
  }
  int rc;
  if ((rc = launch_fold_so(model, S, O, n, Q, ldq, st))) return rc;
  // the pre-folded rows against the relation table: a plain dot-product block of width K (placeholder operands)
  Rows ph{nullptr, nullptr, n, T.dim, T.dim};
  Block B{B200KGE_DISTMULT, B200KGE_SP_, &ph, nullptr, &ph, &T, n};
  B.Qpre = Q;
  if ((rc = csr_loss_terms(B, model, ROLES_SO, 1.0f, precision, S, O, T, csr_off, csr_col, nnz, loss_kind, offset,
                           nullptr, cb, ws, st))) return rc;
  return csr_loss_rows(loss_kind, csr_off, csr_col, n, nnz, T.rows, 0.f, offset, nullptr, 1, cb, loss_out, st);
}

// Its backward: d_T [R, ldt] OVERWRITTEN with dT = G^T Q, the pair rows' gradients ADDED into dS[s_dst[i]], dO[o_dst[i]]
int so_backward_impl(int model, const Rows& S, const Rows& O, const Rows& T, int64_t n, const int64_t* csr_off,
                     const int64_t* csr_col, int loss_kind, float offset, int64_t batch_size, float* dS, int64_t lds,
                     const int64_t* s_dst, float* dO, int64_t ldo, const int64_t* o_dst, float* dT, int64_t ldt,
                     Arena ws, cudaStream_t st) {
  const int K = T.dim;
  const int64_t ldq = round_up(K, 32);
  float* Q = (float*)ws.take((size_t)n * ldq * 4);
  float* dQ = (float*)ws.take((size_t)n * ldq * 4);
  if (!Q || !dQ) { set_error("workspace too small (see b200kge_score_so_loss_csr_workspace_bytes)"); return B200KGE_ERR_WORKSPACE; }
  int rc;
  if ((rc = launch_fold_so(model, S, O, n, Q, ldq, st))) return rc;
  // no label smoothing: the reference never smooths the relation targets (train_KvsAll.py:263)
  const GradSpec g = csr_grad(nullptr, csr_off, csr_col, 0.f, T.rows, batch_size, loss_kind, offset);
  if ((rc = backward_block(B200KGE_DISTMULT, T, T, n, B200KGE_SP_, false, Q, ldq, 0, K, g, dT, ldt, dQ, ws, st))) return rc;
  return launch_unfold_so(model, S, O, n, dQ, ldq, dS, lds, s_dst, dO, ldo, o_dst, st);
}

}  // namespace

extern "C" {

size_t b200kge_score_so_loss_csr_workspace_bytes(int model, int64_t n, int64_t R, int32_t D, int64_t nnz, int dropout) {
  const int64_t K = relation_dim(model, D), ldq = round_up(K, 32), tot = nnz + n;
  const size_t fwd = (size_t)n * ldq * 4 + b200kge_workspace_bytes(B200KGE_DISTMULT, n, R, (int32_t)K, 0) +
                     (size_t)n * 8 + 3 * ((size_t)tot * 8 + 256) + (size_t)tot * 4 + 3 * ((size_t)n * 4 + 256) + 2048;
  const size_t bwd = 2 * ((size_t)n * ldq * 4 + 256) + backward_block_bytes(n, R, K, ldq) + 1024;
  return (fwd > bwd ? fwd : bwd) + (dropout ? so_masked_bytes(n, R, D, K) : 0);
}

int b200kge_score_so_loss_csr(int model, float l_norm, int precision, const b200kge_rows_t* ent,
                              const b200kge_rows_t* rel, const int64_t* s_idx, const int64_t* o_idx, int64_t n,
                              const int64_t* csr_off, const int64_t* csr_col, int64_t nnz, int loss_kind, float offset,
                              const b200kge_dropout_t* drop, float* loss_out, float* row_loss_out, void* workspace,
                              size_t workspace_bytes, b200kge_stream_t stream) {
  (void)l_norm;                                  // the dot family scores without a norm
  int rc = check_so_args(model, ent, rel, s_idx, o_idx, n, csr_off, loss_kind); if (rc) return rc;
  if ((!csr_col && nnz > 0) || !loss_out || nnz < 0) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (drop && (rc = validate_so_dropout(drop, n, ent, rel))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0 || rel->rows == 0) { B2K_CUDA(cudaMemsetAsync(loss_out, 0, 4, st)); return 0; }
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  const Rows E = to_rows(ent), R = to_rows(rel);
  if (!drop) {
    Rows S = E; S.idx = s_idx; S.rows = n;
    Rows O = E; O.idx = o_idx; O.rows = n;
    return so_loss_impl(model, precision, S, O, R, n, csr_off, csr_col, nnz, loss_kind, offset, loss_out, row_loss_out,
                        ws, st);
  }
  SoMasked m;
  if (!take_so_masked(ws, n, E, R, m)) {
    set_error("workspace too small (see b200kge_score_so_loss_csr_workspace_bytes)");
    return B200KGE_ERR_WORKSPACE;
  }
  Rows S, O, T;
  if ((rc = gather_so_masked(so_masks(*drop), E, R, s_idx, o_idx, n, m, S, O, T, st))) return rc;
  return so_loss_impl(model, precision, S, O, T, n, csr_off, csr_col, nnz, loss_kind, offset, loss_out, row_loss_out,
                      rest_of(ws), st);
}

int b200kge_score_so_loss_csr_backward(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                                       const int64_t* s_idx, const int64_t* o_idx, int64_t n, const int64_t* csr_off,
                                       const int64_t* csr_col, int loss_kind, float offset, int64_t batch_size,
                                       const b200kge_dropout_t* drop, float* d_ent, int64_t lde, float* d_rel,
                                       int64_t ldr, void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  (void)l_norm;
  int rc = check_so_args(model, ent, rel, s_idx, o_idx, n, csr_off, loss_kind); if (rc) return rc;
  if (!d_ent || !d_rel) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (batch_size <= 0) { set_error("batch_size must be positive"); return B200KGE_ERR_INVALID; }
  if ((rc = check_grad_ld(ent, lde, rel, ldr))) return rc;
  if (drop && (rc = validate_so_dropout(drop, n, ent, rel))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const Rows E = to_rows(ent), R = to_rows(rel);
  B2K_CUDA(cudaMemsetAsync(d_ent, 0, (size_t)E.rows * lde * 4, st));
  B2K_CUDA(cudaMemsetAsync(d_rel, 0, (size_t)R.rows * ldr * 4, st));
  if (n == 0 || R.rows == 0) return 0;
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  if (!drop) {
    Rows S = E; S.idx = s_idx; S.rows = n;
    Rows O = E; O.idx = o_idx; O.rows = n;
    return so_backward_impl(model, S, O, R, n, csr_off, csr_col, loss_kind, offset, batch_size, d_ent, lde, s_idx, d_ent,
                            lde, o_idx, d_rel, ldr, ws, st);
  }
  // the masked copies' gradients land in row i of dSm / dOm and in dTm; then masked with the same draws and added
  SoMasked m;
  float* dSm = (float*)ws.take((size_t)n * E.dim * 4);
  float* dOm = (float*)ws.take((size_t)n * E.dim * 4);
  float* dTm = (float*)ws.take((size_t)R.rows * R.dim * 4);
  if (!take_so_masked(ws, n, E, R, m) || !dSm || !dOm || !dTm) {
    set_error("workspace too small (see b200kge_score_so_loss_csr_workspace_bytes)");
    return B200KGE_ERR_WORKSPACE;
  }
  const SoMasks k = so_masks(*drop);
  Rows S, O, T;
  if ((rc = gather_so_masked(k, E, R, s_idx, o_idx, n, m, S, O, T, st))) return rc;
  B2K_CUDA(cudaMemsetAsync(dSm, 0, (size_t)n * E.dim * 4, st));
  B2K_CUDA(cudaMemsetAsync(dOm, 0, (size_t)n * E.dim * 4, st));
  if ((rc = so_backward_impl(model, S, O, T, n, csr_off, csr_col, loss_kind, offset, batch_size, dSm, E.dim, nullptr, dOm,
                             E.dim, nullptr, dTm, R.dim, rest_of(ws), st))) return rc;
  if ((rc = launch_dropout_add_cols(k.t, dTm, R.dim, R.rows, R.dim, 0, R.dim, d_rel, ldr, st))) return rc;
  if ((rc = launch_dropout_scatter(k.s, dSm, E.dim, n, E.dim, s_idx, d_ent, lde, st))) return rc;
  return launch_dropout_scatter(k.o, dOm, E.dim, n, E.dim, o_idx, d_ent, lde, st);
}

}  // extern "C"

// ==================================================================================================
// Embedding dropout of one negative-sampling slot (layout: include/b200kge.h, kernels: ns_dropout.cu).
namespace {

int validate_ns_dropout(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                        const int64_t* triples, int slot, const int64_t* neg, int64_t n, int64_t K, int impl,
                        const b200kge_dropout_t* drop) {
  if ((!triples && n > 0) || (!neg && n * K > 0)) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (n < 0 || K < 0) { set_error("negative sizes"); return B200KGE_ERR_INVALID; }
  int rc = check_tables(model, l_norm, ent, rel); if (rc) return rc;
  if (impl != B200KGE_NS_TRIPLE && impl != B200KGE_NS_BATCH) { set_error("impl must be B200KGE_NS_TRIPLE or B200KGE_NS_BATCH"); return B200KGE_ERR_INVALID; }
  if (slot != 0 && slot != 2) { set_error("negative-sampling dropout covers the S and O slots"); return B200KGE_ERR_UNSUPPORTED; }
  if ((model == B200KGE_TRANSE && l_norm != 1.0f && l_norm != 2.0f) || (model == B200KGE_ROTATE && l_norm != 1.0f)) {
    set_error("negative-sampling dropout covers l_norm 1 and 2 (TransE) / 1 (RotatE)");
    return B200KGE_ERR_UNSUPPORTED;
  }
  const int D = ent->dim;
  const bool halves = model == B200KGE_COMPLEX || model == B200KGE_SIMPLE || model == B200KGE_CP || model == B200KGE_ROTATE;
  if (D % (halves ? 8 : 4) != 0) {
    set_error("negative-sampling dropout needs D %% %d == 0 (got %d)", halves ? 8 : 4, D);
    return B200KGE_ERR_UNSUPPORTED;
  }
  if (!drop) { set_error("null dropout key"); return B200KGE_ERR_INVALID; }
  if (impl == B200KGE_NS_BATCH && model != B200KGE_RESCAL && D > 1024) {
    set_error("negative-sampling dropout with `batch` covers D <= 1024 (got %d)", D);
    return B200KGE_ERR_UNSUPPORTED;
  }
  if ((rc = validate_dropout(drop, n, ent->rows, D, rel->dim))) return rc;
  // `triple` mask rows reach (row_base + n) K - 1: bound them in double, before any int64 product can overflow
  const double lim = 281474976710656.0;    // 2^48
  const double top = ((double)drop->row_base + (double)n) * (double)(K > 0 ? K : 1);
  if (impl == B200KGE_NS_TRIPLE && (top * ent->dim > lim || top * rel->dim > lim)) {
    set_error("dropout rows out of range: row * dim + k < 2^48 is required");
    return B200KGE_ERR_INVALID;
  }
  return 0;
}

NsDropKeys ns_drop_keys(const b200kge_dropout_t& d) {
  NsDropKeys k;
  k.ent = drop_mask(d.p_ent, d.seed, d.call, 0, 0);
  k.rel = drop_mask(d.p_rel, d.seed, d.call, 0, 0);
  k.row_base = d.row_base;
  return k;
}

}  // namespace

extern "C" {

int b200kge_ns_score_dropout(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                             const int64_t* triples, int slot, const int64_t* neg, int64_t n, int64_t K, int impl,
                             const b200kge_dropout_t* drop, float* out, int64_t ldo, b200kge_stream_t stream) {
  int rc = validate_ns_dropout(model, l_norm, ent, rel, triples, slot, neg, n, K, impl, drop); if (rc) return rc;
  if (n == 0) return 0;
  if (!out) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (ldo < K + 1) { set_error("out is narrower than the 1 + K columns of the block"); return B200KGE_ERR_INVALID; }
  return launch_ns_dropout(model, l_norm, to_rows(ent), to_rows(rel), triples, slot, neg, n, K, impl, ns_drop_keys(*drop),
                           nullptr, 0, out, ldo, nullptr, 0, nullptr, 0, nullptr, 0, (cudaStream_t)stream);
}

size_t b200kge_ns_backward_workspace_bytes(int model, int64_t n, int64_t K, int32_t D, int dropout) {
  (void)K;
  if (dropout) return (n > 0 && D > 0) ? ns_dropout_workspace_bytes(model, n, D) : 0;
  return (size_t)n * (D + 32) * 4 + 1024;    // dQ [n, round_up(K_folded, 32)] floats
}

int b200kge_ns_backward(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                        const int64_t* triples, int slot, const int64_t* neg, int64_t n, int64_t K, int impl,
                        const b200kge_dropout_t* drop, const float* grad_scores, int64_t ldg, float offset,
                        int64_t batch_size, float* d_ent, int64_t lde, float* d_rel, int64_t ldr, void* workspace,
                        size_t workspace_bytes, b200kge_stream_t stream) {
  int rc;
  if (drop) {
    if ((rc = validate_ns_dropout(model, l_norm, ent, rel, triples, slot, neg, n, K, impl, drop))) return rc;
    if (n == 0) return 0;
  }
  // dropout has no in-kernel BCE form: it needs grad_scores
  if (!triples || (!neg && n * K > 0) || (drop && !grad_scores) || !d_ent || !d_rel) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if ((rc = check_tables(model, l_norm, ent, rel))) return rc;
  if (!grad_scores && batch_size <= 0) { set_error("batch_size must be positive"); return B200KGE_ERR_INVALID; }
  if (grad_scores && ldg < K + 1) { set_error("grad_scores is narrower than the 1 + K columns of the block"); return B200KGE_ERR_INVALID; }
  if ((rc = check_grad_ld(ent, lde, rel, ldr))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Rows E = to_rows(ent), R = to_rows(rel);
  if (drop)
    return launch_ns_dropout(model, l_norm, E, R, triples, slot, neg, n, K, impl, ns_drop_keys(*drop), grad_scores, ldg,
                             nullptr, 0, d_ent, lde, d_rel, ldr, workspace, workspace_bytes, st);
  const int64_t ldq = round_up(folded_problem(model, B200KGE_SP_, E.dim, l_norm).K, 32);
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  float* dQ = (float*)ws.take((size_t)n * ldq * 4);
  if (!dQ && n > 0) { set_error("workspace too small (need n * round_up(K,32) floats)"); return B200KGE_ERR_WORKSPACE; }
  // BCE: dL/dz computed in the kernel from the offset, scaled 1 / batch_size; else read from grad_scores
  return launch_ns_backward(model, l_norm, E, R, triples, slot, neg, n, K, grad_scores ? 0.f : offset,
                            grad_scores ? 1.f : 1.0f / (float)batch_size, grad_scores, grad_scores ? ldg : 0, d_ent, lde,
                            d_rel, ldr, dQ, ldq, st);
}

size_t b200kge_ns_backward_sparse_workspace_bytes(int model, int64_t n, int64_t K, int32_t D, int64_t E, int64_t R,
                                                  int dropout) {
  if (n < 0 || K < 0 || D <= 0 || E < 0 || R < 0) return 0;
  return row_set_workspace_bytes(E) + row_set_workspace_bytes(R) +
         round_up((int64_t)b200kge_ns_backward_workspace_bytes(model, n, K, D, dropout), 256);
}

int b200kge_ns_backward_sparse(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                               const int64_t* triples, int slot, const int64_t* neg, int64_t n, int64_t K, int impl,
                               const b200kge_dropout_t* drop, const float* grad_scores, int64_t ldg, float offset,
                               int64_t batch_size, int ent_sparse, int64_t* ent_rows, int64_t* ent_count, float* d_ent,
                               int64_t lde, int rel_sparse, int64_t* rel_rows, int64_t* rel_count, float* d_rel,
                               int64_t ldr, void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  int rc;
  if (drop && (rc = validate_ns_dropout(model, l_norm, ent, rel, triples, slot, neg, n, K, impl, drop))) return rc;
  if (!triples || (!neg && n * K > 0) || (drop && !grad_scores) || !d_ent || !d_rel || (ent_sparse && (!ent_rows || !ent_count)) ||
      (rel_sparse && (!rel_rows || !rel_count))) {
    set_error("null operand");
    return B200KGE_ERR_INVALID;
  }
  if (n < 0 || K < 0) { set_error("negative sizes"); return B200KGE_ERR_INVALID; }
  if ((rc = check_tables(model, l_norm, ent, rel))) return rc;
  if (!grad_scores && batch_size <= 0) { set_error("batch_size must be positive"); return B200KGE_ERR_INVALID; }
  if (grad_scores && ldg < K + 1) { set_error("grad_scores is narrower than the 1 + K columns of the block"); return B200KGE_ERR_INVALID; }
  if ((rc = check_grad_ld(ent, lde, rel, ldr))) return rc;
  // the coverage of the gradient kernels, refused before the row sets are built
  if (slot != 0 && slot != 2) { set_error("the fused negative-sampling backward covers the S and O slots"); return B200KGE_ERR_UNSUPPORTED; }
  if ((model == B200KGE_TRANSE && l_norm != 1.0f && l_norm != 2.0f) || (model == B200KGE_ROTATE && l_norm != 1.0f)) {
    set_error("the negative-sampling backward covers l_norm 1 and 2 (TransE) / 1 (RotatE)");
    return B200KGE_ERR_UNSUPPORTED;
  }
  const int kf = folded_problem(model, B200KGE_SP_, ent->dim, l_norm).K;
  if (kf > 1024) { set_error("embedding width %d exceeds the backward kernel's limit of 1024", kf); return B200KGE_ERR_UNSUPPORTED; }
  if ((K + 64) / 64 > 65535) { set_error("too many negatives per row (%lld)", (long long)K); return B200KGE_ERR_UNSUPPORTED; }
  if (ent->rows > INT32_MAX || rel->rows > INT32_MAX) { set_error("the row maps cover tables of fewer than 2^31 rows"); return B200KGE_ERR_UNSUPPORTED; }
  const size_t need = b200kge_ns_backward_sparse_workspace_bytes(model, n, K, ent->dim, ent->rows, rel->rows, drop != nullptr);
  if (!workspace || workspace_bytes < need) { set_error("workspace too small (see b200kge_ns_backward_sparse_workspace_bytes)"); return B200KGE_ERR_WORKSPACE; }
  cudaStream_t st = (cudaStream_t)stream;
  Rows E = to_rows(ent), R = to_rows(rel);
  uint8_t* ws_e = (uint8_t*)workspace;
  uint8_t* ws_r = ws_e + row_set_workspace_bytes(E.rows);
  uint8_t* ws_ns = ws_r + row_set_workspace_bytes(R.rows);
  const size_t ns_bytes = workspace_bytes - (size_t)(ws_ns - ws_e);
  // the rows the reference looks up for the slot: the positives' s, o and every sampled id; the positives' p
  const IdList le[3] = {{triples, n, 3}, {triples + 2, n, 3}, {neg, n * K, 1}};
  const IdList lr[1] = {{triples + 1, n, 3}};
  if ((rc = ent_sparse ? launch_row_set(E.rows, le, 3, ws_e, ent_rows, ent_count, d_ent, lde, st)
                       : launch_identity_map(E.rows, ws_e, st))) return rc;
  if ((rc = rel_sparse ? launch_row_set(R.rows, lr, 1, ws_r, rel_rows, rel_count, d_rel, ldr, st)
                       : launch_identity_map(R.rows, ws_r, st))) return rc;
  if (n == 0) return 0;
  const int32_t* pe = (const int32_t*)ws_e;
  const int32_t* pr = (const int32_t*)ws_r;
  if (drop)
    return launch_ns_dropout(model, l_norm, E, R, triples, slot, neg, n, K, impl, ns_drop_keys(*drop), grad_scores, ldg,
                             nullptr, 0, d_ent, lde, d_rel, ldr, ws_ns, ns_bytes, st, pe, pr);
  const int64_t ldq = round_up(folded_problem(model, B200KGE_SP_, E.dim, l_norm).K, 32);
  return launch_ns_backward(model, l_norm, E, R, triples, slot, neg, n, K, grad_scores ? 0.f : offset,
                            grad_scores ? 1.f : 1.0f / (float)batch_size, grad_scores, grad_scores ? ldg : 0, d_ent, lde,
                            d_rel, ldr, (float*)ws_ns, ldq, st, pe, pr);
}

size_t b200kge_ns_p_backward_workspace_bytes(int model, int64_t n, int64_t K, int32_t D, int64_t E, int64_t R) {
  if (n < 0 || K < 0 || D <= 0 || E < 0 || R < 0 || R > B200KGE_NS_P_MAX_RELATIONS) return 0;
  const int64_t Kr = relation_dim(model, D), ldc = round_up(R > 0 ? R : 1, 4);
  // row-set maps, C, s / o ids and destination rows
  size_t b = row_set_workspace_bytes(E) + row_set_workspace_bytes(R) + (size_t)n * ldc * 4 + 4 * ((size_t)n * 8 + 256) + 4 * 256;
  if (model == B200KGE_TRANSE || model == B200KGE_ROTATE)
    return b + (size_t)ns_p_parts(n, R) * R * Kr * 4 + 256;
  const int64_t ldq = round_up(Kr, 32);
  // Q, dQ, dT [R, ldq], the backward block
  return b + 2 * ((size_t)n * ldq * 4 + 256) + (size_t)R * ldq * 4 + 256 + backward_block_bytes(n, R, Kr, ldq);
}

int b200kge_ns_p_backward(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                          const int64_t* triples, const int64_t* neg, int64_t n, int64_t K, const float* grad_scores,
                          int64_t ldg, int ent_sparse, int64_t* ent_rows, int64_t* ent_count, float* d_ent, int64_t lde,
                          int rel_sparse, int64_t* rel_rows, int64_t* rel_count, float* d_rel, int64_t ldr,
                          void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  if (!triples || (!neg && n * K > 0) || !grad_scores || !d_ent || !d_rel || (ent_sparse && (!ent_rows || !ent_count)) ||
      (rel_sparse && (!rel_rows || !rel_count))) {
    set_error("null operand");
    return B200KGE_ERR_INVALID;
  }
  if (n < 0 || K < 0) { set_error("negative sizes"); return B200KGE_ERR_INVALID; }
  int rc = check_tables(model, l_norm, ent, rel); if (rc) return rc;
  if (ldg < K + 1) { set_error("grad_scores is narrower than the 1 + K columns of the block"); return B200KGE_ERR_INVALID; }
  if ((rc = check_grad_ld(ent, lde, rel, ldr))) return rc;
  const bool distance = model == B200KGE_TRANSE || model == B200KGE_ROTATE;
  if ((model == B200KGE_TRANSE && l_norm != 1.0f && l_norm != 2.0f) || (model == B200KGE_ROTATE && l_norm != 1.0f)) {
    set_error("the P-slot backward covers l_norm 1 and 2 (TransE) / 1 (RotatE)");
    return B200KGE_ERR_UNSUPPORTED;
  }
  if (rel->rows > B200KGE_NS_P_MAX_RELATIONS) {
    set_error("the P-slot backward covers up to %d relations (got %lld)", B200KGE_NS_P_MAX_RELATIONS, (long long)rel->rows);
    return B200KGE_ERR_UNSUPPORTED;
  }
  if (ent->rows > INT32_MAX) { set_error("the row maps cover tables of fewer than 2^31 rows"); return B200KGE_ERR_UNSUPPORTED; }
  const size_t need = b200kge_ns_p_backward_workspace_bytes(model, n, K, ent->dim, ent->rows, rel->rows);
  if (!workspace || workspace_bytes < need) { set_error("workspace too small (see b200kge_ns_p_backward_workspace_bytes)"); return B200KGE_ERR_WORKSPACE; }
  cudaStream_t st = (cudaStream_t)stream;
  const Rows E = to_rows(ent), Rl = to_rows(rel);
  uint8_t* ws_e = (uint8_t*)workspace;
  uint8_t* ws_r = ws_e + row_set_workspace_bytes(E.rows);
  uint8_t* ws_rest = ws_r + row_set_workspace_bytes(Rl.rows);
  // the rows score_so looks up: the positives' s and o; the positives' p and every sampled id
  const IdList le[2] = {{triples, n, 3}, {triples + 2, n, 3}};
  const IdList lr[2] = {{triples + 1, n, 3}, {neg, n * K, 1}};
  if (ent_sparse && (rc = launch_row_set(E.rows, le, 2, ws_e, ent_rows, ent_count, d_ent, lde, st))) return rc;
  if (rel_sparse && (rc = launch_row_set(Rl.rows, lr, 2, ws_r, rel_rows, rel_count, d_rel, ldr, st))) return rc;
  if (n == 0 || Rl.rows == 0) return 0;
  Arena ws{ws_rest, workspace_bytes - (size_t)(ws_rest - ws_e), 0};
  const int64_t R = Rl.rows, Kr = Rl.dim, ldc = round_up(R, 4);
  float* Cw = (float*)ws.take((size_t)n * ldc * 4);
  int64_t* s_idx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* o_idx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* s_dst = (int64_t*)ws.take((size_t)n * 8);
  int64_t* o_dst = (int64_t*)ws.take((size_t)n * 8);
  if (!Cw || !s_idx || !o_idx || !s_dst || !o_dst) { set_error("workspace too small (see b200kge_ns_p_backward_workspace_bytes)"); return B200KGE_ERR_WORKSPACE; }
  if ((rc = launch_ns_p_unpack(triples, n, ent_sparse ? (const int32_t*)ws_e : nullptr, s_idx, o_idx, s_dst, o_dst, st))) return rc;
  if ((rc = launch_ns_p_collapse(triples, neg, n, K, grad_scores, ldg, R, Cw, ldc, st))) return rc;
  const int64_t* rows = rel_sparse ? rel_rows : nullptr;
  const int64_t* count = rel_sparse ? rel_count : nullptr;
  if (distance) {
    const int P = ns_p_parts(n, R);
    float* parts = (float*)ws.take((size_t)P * R * Kr * 4);
    if (!parts) { set_error("workspace too small (see b200kge_ns_p_backward_workspace_bytes)"); return B200KGE_ERR_WORKSPACE; }
    if ((rc = launch_ns_p_distance(model, l_norm, E, Rl, s_idx, o_idx, n, Cw, ldc, d_ent, lde, s_dst, o_dst, parts, st))) return rc;
    return launch_ns_p_rel_add(parts, Kr, R * Kr, P, R, (int)Kr, rows, count, d_rel, ldr, st);
  }
  // dot family: the s_o fold against the relation table, C as the dense gradient of the block
  const int64_t ldq = round_up(Kr, 32);
  float* Q = (float*)ws.take((size_t)n * ldq * 4);
  float* dQ = (float*)ws.take((size_t)n * ldq * 4);
  float* dT = (float*)ws.take((size_t)R * ldq * 4);
  if (!Q || !dQ || !dT) { set_error("workspace too small (see b200kge_ns_p_backward_workspace_bytes)"); return B200KGE_ERR_WORKSPACE; }
  Rows S = E; S.idx = s_idx; S.rows = n;
  Rows O = E; O.idx = o_idx; O.rows = n;
  if ((rc = launch_fold_so(model, S, O, n, Q, ldq, st))) return rc;
  GradSpec g;
  g.G = Cw; g.ldg = ldc;
  if ((rc = backward_block(B200KGE_DISTMULT, Rl, Rl, n, B200KGE_SP_, false, Q, ldq, 0, (int)Kr, g, dT, ldq, dQ, ws, st))) return rc;
  if ((rc = launch_ns_p_rel_add(dT, ldq, 0, 1, R, (int)Kr, rows, count, d_rel, ldr, st))) return rc;
  return launch_unfold_so(model, S, O, n, dQ, ldq, d_ent, lde, s_dst, d_ent, lde, o_dst, st);
}

// The checks shared by the two shared-sampling entry points; *U = the shared samples before the repeats
static int check_ns_shared(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                           const int64_t* triples, int slot, const int64_t* unique, int64_t num_unique,
                           const int64_t* repeat, const int64_t* drop, int64_t n, int64_t K, int impl, int64_t* U) {
  if (!triples && n > 0) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (n < 0 || K < 0 || num_unique < 0) { set_error("negative sizes"); return B200KGE_ERR_INVALID; }
  int rc = check_tables(model, l_norm, ent, rel); if (rc) return rc;
  if (impl != B200KGE_NS_TRIPLE && impl != B200KGE_NS_BATCH) { set_error("unknown implementation %d", impl); return B200KGE_ERR_INVALID; }
  *U = drop ? num_unique - 1 : num_unique;
  if (*U < 0 || *U > K || (*U == 0 && K > 0)) {
    set_error("%lld unique ids do not fit %lld samples per row (%s)", (long long)num_unique, (long long)K,
              drop ? "default: U + 1 ids, 1 <= U <= K" : "naive: 1 <= U <= K");
    return B200KGE_ERR_INVALID;
  }
  if ((!unique && num_unique > 0) || (!repeat && K > *U)) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (slot != 0 && slot != 2) { set_error("shared negative sampling covers the S and O slots"); return B200KGE_ERR_UNSUPPORTED; }
  if ((model == B200KGE_TRANSE && l_norm != 1.0f && l_norm != 2.0f) || (model == B200KGE_ROTATE && l_norm != 1.0f)) {
    set_error("shared negative sampling covers l_norm 1 and 2 (TransE) / 1 (RotatE)");
    return B200KGE_ERR_UNSUPPORTED;
  }
  const int kf = folded_problem(model, B200KGE_SP_, ent->dim, l_norm).K;
  if (kf > 1024) { set_error("embedding width %d exceeds the backward kernel's limit of 1024", kf); return B200KGE_ERR_UNSUPPORTED; }
  if (ent->rows > INT32_MAX || rel->rows > INT32_MAX) { set_error("shared negative sampling covers tables of fewer than 2^31 rows"); return B200KGE_ERR_UNSUPPORTED; }
  return 0;
}

// The slot's folded queries Q [n, ldq] (O slot: sp_ of (s, p); S slot: _po of (o, p)), with pairwise_distance's eps for
// TransE's `triple` scores: (s + p) - o' + eps = (s + p + eps) - o',  s' + p - o + eps = s' - (o - p - eps)
static int ns_shared_queries(int model, int slot, int impl, const Rows& E, const Rows& Rl, const int64_t* triples,
                             int64_t n, Arena& ws, Rows& S, Rows& P, Rows& O, float** Q, int64_t ldq, cudaStream_t st) {
  int64_t* sidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* pidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* oidx = (int64_t*)ws.take((size_t)n * 8);
  int64_t* lab = (int64_t*)ws.take((size_t)n * 16);
  *Q = (float*)ws.take((size_t)n * ldq * 4);
  if (!sidx || !pidx || !oidx || !lab || !*Q) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  int rc = unpack_triples(triples, n, sidx, pidx, oidx, lab, E, Rl, S, O, P, st); if (rc) return rc;
  const bool sp = slot == 2;
  if ((rc = launch_fold_queries(model, sp ? B200KGE_SP_ : B200KGE__PO, sp ? S : O, P, n, 0, *Q, ldq, st))) return rc;
  if (model == B200KGE_TRANSE && impl == B200KGE_NS_TRIPLE)
    return launch_ns_shared_eps(*Q, ldq, n, E.dim, sp ? 1e-6f : -1e-6f, st);
  return 0;
}

size_t b200kge_ns_shared_score_workspace_bytes(int model, int64_t n, int64_t num_unique, int32_t D) {
  if (n < 0 || num_unique < 0 || D <= 0) return 0;
  const int64_t ldq = round_up(D, 32), ldz = round_up(num_unique > 0 ? num_unique : 1, 4);
  // s, p, o, labels, Q, Z, the scorer's workspace
  return 5 * ((size_t)n * 8 + 256) + (size_t)n * ldq * 4 + 256 + (size_t)n * ldz * 4 + 256 +
         b200kge_workspace_bytes(model, n, num_unique, D, 1);
}

int b200kge_ns_shared_score(int model, float l_norm, int precision, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                            const int64_t* triples, int slot, const int64_t* unique, int64_t num_unique,
                            const int64_t* repeat, const int64_t* drop, int64_t n, int64_t K, int impl, float* out,
                            int64_t ldo, float* z_out, int64_t ldz, void* workspace, size_t workspace_bytes,
                            b200kge_stream_t stream) {
  int64_t U = 0;
  int rc = check_ns_shared(model, l_norm, ent, rel, triples, slot, unique, num_unique, repeat, drop, n, K, impl, &U);
  if (rc) return rc;
  if (!out && n > 0) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (ldo < K + 1) { set_error("out is narrower than the 1 + K columns of the block"); return B200KGE_ERR_INVALID; }
  if (z_out && ldz < num_unique) { set_error("z_out is narrower than the %lld unique ids", (long long)num_unique); return B200KGE_ERR_INVALID; }
  const Folded f = folded_problem(model, slot == 2 ? B200KGE_SP_ : B200KGE__PO, ent->dim, l_norm);
  if (precision != B200KGE_PREC_AUTO && precision != B200KGE_PREC_FP32 &&
      (precision != B200KGE_PREC_F16X3 || f.pair_op != PAIR_DOT || f.K < 16)) {
    set_error("shared negative sampling scores at precision auto, fp32 or (dot family, K >= 16) f16x3");
    return B200KGE_ERR_UNSUPPORTED;
  }
  if (!workspace || workspace_bytes < b200kge_ns_shared_score_workspace_bytes(model, n, num_unique, ent->dim)) {
    set_error("workspace too small (see b200kge_ns_shared_score_workspace_bytes)");
    return B200KGE_ERR_WORKSPACE;
  }
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const Rows E = to_rows(ent), Rl = to_rows(rel);
  Arena ws{(uint8_t*)workspace, workspace_bytes, 0};
  Rows S, P, O;
  float* Q = nullptr;
  const int64_t ldq = round_up(f.K, 32);
  if ((rc = ns_shared_queries(model, slot, impl, E, Rl, triples, n, ws, S, P, O, &Q, ldq, st))) return rc;
  // column 0: score_spo of the positive (train_negative_sampling.py:141-143)
  if ((rc = launch_spo(model, l_norm, S, P, O, n, out, ldo, st))) return rc;
  if (K == 0) return 0;
  float* Z = z_out;
  if (!Z) {
    ldz = round_up(num_unique, 4);
    if (!(Z = (float*)ws.take((size_t)n * ldz * 4))) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  }
  // Z = score_sp(s, p, unique) / score_po(p, o, unique) (sampler.py:347-356)
  Rows cand = E; cand.idx = unique; cand.rows = num_unique;
  EpiParams Pz = empty_epi();
  Pz.out = Z; Pz.ldo = ldz;
  Block B{model, slot == 2 ? B200KGE_SP_ : B200KGE__PO, slot == 2 ? &S : &O, nullptr, &P, &cand, n};
  B.Qpre = Q;
  if ((rc = run_block(B, l_norm, precision, EPI_STORE, Pz, ws, st, nullptr))) return rc;
  return launch_ns_shared_assemble(Z, ldz, n, K, U, repeat, drop, out, ldo, st);
}

size_t b200kge_ns_shared_backward_workspace_bytes(int model, int64_t n, int64_t num_unique, int32_t D, int64_t E,
                                                  int64_t R) {
  if (n < 0 || num_unique < 0 || D <= 0 || E < 0 || R < 0) return 0;
  const int64_t nu = num_unique > 0 ? num_unique : 1, ldq = round_up(D, 32), ldc = round_up(nu, 4);
  // row-set maps; s, p, o, labels, Q; used ids and drop counts; C; dQ of the shared columns and of the positive;
  // T and dT of the shared rows
  size_t b = row_set_workspace_bytes(E) + row_set_workspace_bytes(R) + 5 * ((size_t)n * 8 + 256) +
             (size_t)n * ldq * 4 + 256 + (size_t)nu * 12 + 512 + (size_t)n * ldc * 4 + 256 +
             2 * ((size_t)n * ldq * 4 + 256) + 2 * ((size_t)nu * ldq * 4 + 256);
  if (model == B200KGE_TRANSE || model == B200KGE_ROTATE) return b + (size_t)nu * round_up(n, 4) * 4 + 256;   // C^T
  return b + backward_block_bytes(n, nu, D, ldq);
}

int b200kge_ns_shared_backward(int model, float l_norm, const b200kge_rows_t* ent, const b200kge_rows_t* rel,
                               const int64_t* triples, int slot, const int64_t* unique, int64_t num_unique,
                               const int64_t* repeat, const int64_t* drop, int64_t n, int64_t K, int impl,
                               const float* z, int64_t ldz, const float* grad_scores, int64_t ldg, int ent_sparse,
                               int64_t* ent_rows, int64_t* ent_count, float* d_ent, int64_t lde, int rel_sparse,
                               int64_t* rel_rows, int64_t* rel_count, float* d_rel, int64_t ldr, void* workspace,
                               size_t workspace_bytes, b200kge_stream_t stream) {
  int64_t U = 0;
  int rc = check_ns_shared(model, l_norm, ent, rel, triples, slot, unique, num_unique, repeat, drop, n, K, impl, &U);
  if (rc) return rc;
  if ((!grad_scores && n > 0) || !d_ent || !d_rel || (ent_sparse && (!ent_rows || !ent_count)) ||
      (rel_sparse && (!rel_rows || !rel_count))) {
    set_error("null operand");
    return B200KGE_ERR_INVALID;
  }
  if (ldg < K + 1) { set_error("grad_scores is narrower than the 1 + K columns of the block"); return B200KGE_ERR_INVALID; }
  if ((rc = check_grad_ld(ent, lde, rel, ldr))) return rc;
  const Folded f = folded_problem(model, slot == 2 ? B200KGE_SP_ : B200KGE__PO, ent->dim, l_norm);
  if (f.pair_op == PAIR_L2 && K > 0 && (!z || ldz < num_unique)) {
    set_error("TransE l_norm 2 needs the forward's scores z [n, >= %lld]", (long long)num_unique);
    return B200KGE_ERR_INVALID;
  }
  const size_t need = b200kge_ns_shared_backward_workspace_bytes(model, n, num_unique, ent->dim, ent->rows, rel->rows);
  if (!workspace || workspace_bytes < need) { set_error("workspace too small (see b200kge_ns_shared_backward_workspace_bytes)"); return B200KGE_ERR_WORKSPACE; }
  cudaStream_t st = (cudaStream_t)stream;
  const Rows E = to_rows(ent), Rl = to_rows(rel);
  uint8_t* ws_e = (uint8_t*)workspace;
  uint8_t* ws_r = ws_e + row_set_workspace_bytes(E.rows);
  uint8_t* ws_rest = ws_r + row_set_workspace_bytes(Rl.rows);
  Arena ws{ws_rest, workspace_bytes - (size_t)(ws_rest - ws_e), 0};
  const int64_t nu = num_unique;
  int64_t* used = (int64_t*)ws.take((size_t)(nu > 0 ? nu : 1) * 8);
  int* cnt = (int*)ws.take((size_t)(nu > 0 ? nu : 1) * 4);
  if (!used || !cnt) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  // the rows the reference looks up for the slot: the positives' s, o and the shared ids (`batch`: all of them, as
  // score_sp / score_po(..., unique) embeds them; `triple`: those the sub-batch's rows use); the positives' p
  const int64_t* ids = unique;
  if (ent_sparse && impl == B200KGE_NS_TRIPLE && drop && n > 0) {     // naive: every row uses every shared id
    if ((rc = launch_ns_shared_used(unique, nu, drop, n, triples, cnt, used, st))) return rc;
    ids = used;
  }
  const IdList le[3] = {{triples, n, 3}, {triples + 2, n, 3}, {ids, n > 0 ? nu : 0, 1}};
  const IdList lr[1] = {{triples + 1, n, 3}};
  const bool mapped = ent_sparse || rel_sparse;
  if (mapped && (rc = ent_sparse ? launch_row_set(E.rows, le, 3, ws_e, ent_rows, ent_count, d_ent, lde, st)
                                 : launch_identity_map(E.rows, ws_e, st))) return rc;
  if (mapped && (rc = rel_sparse ? launch_row_set(Rl.rows, lr, 1, ws_r, rel_rows, rel_count, d_rel, ldr, st)
                                 : launch_identity_map(Rl.rows, ws_r, st))) return rc;
  if (n == 0) return 0;
  const int32_t* pe = mapped ? (const int32_t*)ws_e : nullptr;
  const int32_t* pr = mapped ? (const int32_t*)ws_r : nullptr;
  Rows S, P, O;
  float* Q = nullptr;
  const int64_t ldq = round_up(f.K, 32), ldc = round_up(nu > 0 ? nu : 1, 4);
  if ((rc = ns_shared_queries(model, slot, impl, E, Rl, triples, n, ws, S, P, O, &Q, ldq, st))) return rc;
  float* dQp = (float*)ws.take((size_t)n * ldq * 4);
  if (!dQp) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  // the positive column (G[:, 0]) through the row-wise kernel, unfolded into its rows
  if ((rc = launch_ns_backward(model, l_norm, E, Rl, triples, slot, nullptr, n, 0, 0.f, 1.f, grad_scores, ldg, d_ent, lde,
                               d_rel, ldr, dQp, ldq, st, pe, pr))) return rc;
  if (K == 0) return 0;
  float* C = (float*)ws.take((size_t)n * ldc * 4);
  float* dQ = (float*)ws.take((size_t)n * ldq * 4);
  float* T = (float*)ws.take((size_t)nu * ldq * 4);
  float* dT = (float*)ws.take((size_t)nu * ldq * 4);
  if (!C || !dQ || !T || !dT) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
  if ((rc = launch_ns_shared_collapse(grad_scores, ldg, n, K, U, nu, repeat, drop, C, ldc, st))) return rc;
  Rows cand = E; cand.idx = unique; cand.rows = nu;
  if ((rc = launch_gather_rows(cand, f.col_off, f.K, T, ldq, st))) return rc;
  const Rows Tr{T, nullptr, nu, ldq, f.K};
  const int dir = slot == 2 ? 0 : 1;
  if (model == B200KGE_TRANSE || model == B200KGE_ROTATE) {
    float* Ct = (float*)ws.take((size_t)nu * round_up(n, 4) * 4);
    if (!Ct) { set_error("workspace too small"); return B200KGE_ERR_WORKSPACE; }
    if (f.pair_op == PAIR_L2 && (rc = launch_div_scores(C, ldc, z, ldz, n, nu, C, ldc, st))) return rc;
    if ((rc = distance_rowgrads(f.pair_op, Q, ldq, n, Tr, f.K, C, ldc, Ct, dQ, dT, ldq, st))) return rc;
    if ((rc = launch_ns_shared_row_add(dT, ldq, nu, f.K, unique, pe, d_ent, lde, f.col_off, st))) return rc;
    return launch_unfold_distance(model, E, Rl, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, st, 0, pe, pr);
  }
  GradSpec g;
  g.G = C; g.ldg = ldc;
  if ((rc = backward_block(B200KGE_DISTMULT, Tr, Rl, n, B200KGE_SP_, false, Q, ldq, 0, f.K, g, dT, ldq, dQ, ws, st))) return rc;
  if ((rc = launch_ns_shared_row_add(dT, ldq, nu, f.K, unique, pe, d_ent, lde, f.col_off, st))) return rc;
  return launch_unfold(model, E, Rl, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, st, 0, pe, pr);
}


// The checks shared by the two optimizer steps: operands, sizes and the workspace of a row-sparse gradient
static int check_optim_step(const float* param, const float* state0, const float* state1, int64_t rows, int64_t dim,
                            const float* grad, const int64_t* grad_rows, int64_t nnz, int coalesced, void* workspace,
                            size_t workspace_bytes) {
  if (rows < 0 || dim <= 0 || (grad_rows && nnz < 0)) { set_error("negative sizes"); return B200KGE_ERR_INVALID; }
  const bool any = grad_rows ? nnz > 0 : rows > 0;
  if (!param || !state0 || !state1 || (any && !grad)) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (!grad_rows) return 0;
  if (!coalesced && rows > INT32_MAX) { set_error("the row map covers tables of fewer than 2^31 rows"); return B200KGE_ERR_UNSUPPORTED; }
  const size_t need = b200kge_optim_step_workspace_bytes(rows, dim, nnz, coalesced);
  if (need && (!workspace || workspace_bytes < need)) {
    set_error("workspace too small (need b200kge_optim_step_workspace_bytes = %zu bytes)", need);
    return B200KGE_ERR_WORKSPACE;
  }
  return 0;
}

size_t b200kge_optim_step_workspace_bytes(int64_t rows, int64_t dim, int64_t nnz, int coalesced) {
  return optim_step_workspace_bytes(rows, dim, nnz, coalesced);
}

int b200kge_adagrad_step(float* param, float* state_sum, int64_t rows, int64_t dim, const float* grad,
                         const int64_t* grad_rows, int64_t nnz, int coalesced, int foreach_order, float clr, float eps,
                         float weight_decay, void* workspace, size_t workspace_bytes, b200kge_stream_t stream) {
  int rc = check_optim_step(param, state_sum, state_sum, rows, dim, grad, grad_rows, nnz, coalesced, workspace,
                            workspace_bytes);
  if (rc) return rc;
  if (grad_rows && weight_decay != 0.f) {
    set_error("weight_decay option is not compatible with sparse gradients");
    return B200KGE_ERR_INVALID;
  }
  return launch_adagrad_step(param, state_sum, rows, dim, grad, grad_rows, nnz, coalesced, foreach_order, clr, eps,
                             weight_decay, workspace, (cudaStream_t)stream);
}

int b200kge_sparse_adam_step(float* param, float* exp_avg, float* exp_avg_sq, int64_t rows, int64_t dim,
                             const float* grad, const int64_t* grad_rows, int64_t nnz, int coalesced,
                             float one_minus_beta1, float one_minus_beta2, float eps, float step_size, void* workspace,
                             size_t workspace_bytes, b200kge_stream_t stream) {
  if (!grad_rows) {
    set_error("SparseAdam does not support dense gradients, please consider Adam instead");
    return B200KGE_ERR_INVALID;
  }
  int rc = check_optim_step(param, exp_avg, exp_avg_sq, rows, dim, grad, grad_rows, nnz, coalesced, workspace,
                            workspace_bytes);
  if (rc) return rc;
  return launch_sparse_adam_step(param, exp_avg, exp_avg_sq, rows, dim, grad, grad_rows, nnz, coalesced,
                                 one_minus_beta1, one_minus_beta2, eps, step_size, workspace, (cudaStream_t)stream);
}

}  // extern "C"
