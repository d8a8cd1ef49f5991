// fold.cu — prologue kernels: fused embedding-row gather + relation folding.
//
// Every in-scope scorer's 1-vs-N form factors as  score(i, j) = pair(Q_i, cand_j[cols])  where Q_i
// depends only on the per-row operands (subject-or-object row, relation row).  This kernel
// gathers those rows by index straight from the embedding tables (LookupEmbedder.embed,
// lookup_embedder.py:96-97) and builds Q without materialising the gathered rows or the
// reference's concatenated operands (complex.py:26-32).  Folds (SURVEY.md section 7):
//   ComplEx  sp_: [s_re*p_re - s_im*p_im | s_im*p_re + s_re*p_im]   _po: [p_re*o_re + p_im*o_im | p_re*o_im - p_im*o_re]
//   DistMult a*p
//   SimplE   sp_: 1/2 [s_t*p_b | s_h*p_f]                           _po: 1/2 [o_t*p_f | o_h*p_b]
//   CP       sp_: s[:h]*p  (vs cand[:, h:])                          _po: o[h:]*p (vs cand[:, :h])
//   RESCAL   sp_: s^T M_p                                            _po: M_p o
//   TransE   sp_: s + p                                              _po: o - p
//   RotatE   sp_: s * e^{i theta}                                    _po: conj(e^{i theta}) * o
#include "fold.cuh"

namespace b200kge {

template <int MODEL>
__global__ void __launch_bounds__(128)
fold_kernel(int combine, Rows qa, Rows pr, int64_t row0, float* __restrict__ Q, int64_t ldq, int K) {
  const int64_t i = blockIdx.x;
  const float* __restrict__ a = qa.row(i);
  const float* __restrict__ p = pr.row(i);
  const int D = qa.dim;
  const int h = D >> 1;
  const int64_t obase = (row0 + i) * ldq;
  const bool sp = (combine == B200KGE_SP_);

  if constexpr (MODEL == B200KGE_RESCAL) {
    extern __shared__ float sh[];
    for (int k = threadIdx.x; k < D; k += blockDim.x) sh[k] = a[k];
    __syncthreads();
    fold_rescal_block(sp, sh, p, D, [&](int k, float v) { Q[obase + k] = v; });
  } else {
    for (int k = threadIdx.x; k < K; k += blockDim.x)
      Q[obase + k] = fold_element<MODEL>(sp, a, p, k, h);
  }
  // zero the padding columns [K, ldq) so padded K-chunks contribute nothing
  for (int64_t k = K + threadIdx.x; k < ldq; k += blockDim.x) Q[obase + k] = 0.f;
}

// One launch for a whole 1vsAll step's prologue: block b < n folds (s_b, p_b) for the sp_ direction
// into Q row b and labels it with o_b; block n+b folds (o_b, p_b) for _po into Q row n+b, label s_b
// (train_1vsAll.py:59-65,75-76).  Replaces unpack + two fold launches.
// RECIP (reciprocal relations, reciprocal_relations_model.py:85-92): block n+b folds (o_b, p_b + num_rel) with the sp_
// fold instead, label s_b — both halves are sp_ queries against the same table columns.
template <int MODEL, bool RECIP>
__global__ void __launch_bounds__(128)
prep_1vsall_kernel(Rows ent, Rows rel, const int64_t* __restrict__ tri, int64_t n, float* __restrict__ Q,
                   int64_t ldq, int64_t* __restrict__ labels2n, unsigned int* ticket, int K, int64_t num_rel) {
  const int64_t b = blockIdx.x;
  const bool first = b < n;
  const bool sp = RECIP || first;
  const int64_t i = first ? b : b - n;
  const int64_t si = tri[3 * i], pi = tri[3 * i + 1], oi = tri[3 * i + 2];
  const float* __restrict__ a = ent.base + (first ? si : oi) * ent.ld;
  const float* __restrict__ p = rel.base + (RECIP && !first ? pi + num_rel : pi) * rel.ld;
  const int D = ent.dim, h = D >> 1;
  const int64_t obase = b * ldq;
  if (threadIdx.x == 0) {
    labels2n[b] = first ? oi : si;
    if (b == 0 && ticket) *ticket = 0u;
  }
  if constexpr (MODEL == B200KGE_RESCAL) {
    extern __shared__ float sh[];
    for (int k = threadIdx.x; k < D; k += blockDim.x) sh[k] = a[k];
    __syncthreads();
    fold_rescal_block(sp, sh, p, D, [&](int k, float v) { Q[obase + k] = v; });
  } else {
    for (int k = threadIdx.x; k < K; k += blockDim.x) Q[obase + k] = fold_element<MODEL>(sp, a, p, k, h);
  }
  for (int64_t k = K + threadIdx.x; k < ldq; k += blockDim.x) Q[obase + k] = 0.f;
}

int launch_prep_1vsall(int model, const Rows& ent, const Rows& rel, const int64_t* triples, int64_t n,
                       float* Q, int64_t ldq, int64_t* labels2n, unsigned int* ticket, cudaStream_t st,
                       int64_t num_rel) {
  if (n == 0) return 0;
  const int D = ent.dim;
  const int K = (model == B200KGE_CP) ? D / 2 : D;
  dim3 grid((unsigned)(2 * n)), block(128);
#define B2K_PREP(M, SM) case M: prep_1vsall_kernel<M, false><<<grid, block, SM, st>>>(ent, rel, triples, n, Q, ldq, labels2n, ticket, K, 0); break;
#define B2K_PREP_R(M, SM) case M: prep_1vsall_kernel<M, true><<<grid, block, SM, st>>>(ent, rel, triples, n, Q, ldq, labels2n, ticket, K, num_rel); break;
  if (num_rel > 0) {
    // reciprocal: CP joins the stacked problem (both halves read the table columns [h, D))
    switch (model) {
      B2K_PREP_R(B200KGE_COMPLEX, 0) B2K_PREP_R(B200KGE_DISTMULT, 0) B2K_PREP_R(B200KGE_SIMPLE, 0) B2K_PREP_R(B200KGE_CP, 0)
      B2K_PREP_R(B200KGE_RESCAL, D * sizeof(float)) B2K_PREP_R(B200KGE_TRANSE, 0) B2K_PREP_R(B200KGE_ROTATE, 0)
      default: set_error("model %d has no stacked 1vsAll prologue", model); return B200KGE_ERR_INVALID;
    }
  } else {
    switch (model) {
      B2K_PREP(B200KGE_COMPLEX, 0) B2K_PREP(B200KGE_DISTMULT, 0) B2K_PREP(B200KGE_SIMPLE, 0)
      B2K_PREP(B200KGE_RESCAL, D * sizeof(float)) B2K_PREP(B200KGE_TRANSE, 0) B2K_PREP(B200KGE_ROTATE, 0)
      default: set_error("model %d has no stacked 1vsAll prologue", model); return B200KGE_ERR_INVALID;
    }
  }
#undef B2K_PREP
#undef B2K_PREP_R
  B2K_LAUNCH_CHECK("prep_1vsall_kernel");
  return 0;
}

int launch_fold_queries(int model, int combine, const Rows& q, const Rows& p, int64_t n,
                        int64_t row0, float* Q, int64_t ldq, cudaStream_t st) {
  if (n == 0) return 0;
  const int D = q.dim;
  int K = D;
  if (model == B200KGE_CP) K = D / 2;
  dim3 grid((unsigned)n), block(128);
  switch (model) {
    case B200KGE_COMPLEX:
      fold_kernel<B200KGE_COMPLEX><<<grid, block, 0, st>>>(combine, q, p, row0, Q, ldq, K); break;
    case B200KGE_DISTMULT:
      fold_kernel<B200KGE_DISTMULT><<<grid, block, 0, st>>>(combine, q, p, row0, Q, ldq, K); break;
    case B200KGE_SIMPLE:
      fold_kernel<B200KGE_SIMPLE><<<grid, block, 0, st>>>(combine, q, p, row0, Q, ldq, K); break;
    case B200KGE_CP:
      fold_kernel<B200KGE_CP><<<grid, block, 0, st>>>(combine, q, p, row0, Q, ldq, K); break;
    case B200KGE_RESCAL:
      fold_kernel<B200KGE_RESCAL><<<grid, block, D * sizeof(float), st>>>(combine, q, p, row0, Q, ldq, K); break;
    case B200KGE_TRANSE:
      fold_kernel<B200KGE_TRANSE><<<grid, block, 0, st>>>(combine, q, p, row0, Q, ldq, K); break;
    case B200KGE_ROTATE:
      fold_kernel<B200KGE_ROTATE><<<grid, block, 0, st>>>(combine, q, p, row0, Q, ldq, K); break;
    default:
      set_error("unknown model %d", model);
      return B200KGE_ERR_INVALID;
  }
  B2K_LAUNCH_CHECK("fold_kernel");
  return 0;
}

// s_o fold (relation prediction): Q row i such that score(s_i, r, o_i) = Q_i . rel[r][0:K] for every relation r.
//   DistMult s*o   ComplEx [s_re*o_re + s_im*o_im | s_re*o_im - s_im*o_re]   SimplE 1/2 [s_h*o_t | s_t*o_h]
//   CP s[:h]*o[h:] (K = h)   RESCAL Q[r*D + c] = s_r o_c (K = D^2, the row-major p.view(D, D) of rescal.py)
template <int MODEL>
__global__ void __launch_bounds__(128)
fold_so_kernel(Rows S, Rows O, float* __restrict__ Q, int64_t ldq, int K) {
  const int64_t i = blockIdx.x;
  const float* __restrict__ s = S.row(i);
  const float* __restrict__ o = O.row(i);
  const int D = S.dim, h = D >> 1;
  float* __restrict__ q = Q + i * ldq;
  if constexpr (MODEL == B200KGE_RESCAL) {
    for (int e = threadIdx.x; e < K; e += blockDim.x) {
      const int r = e / D;
      q[e] = s[r] * o[e - r * D];
    }
  } else {
    for (int k = threadIdx.x; k < K; k += blockDim.x) q[k] = fold_so_element<MODEL>(s, o, k, h);
  }
  for (int64_t k = K + threadIdx.x; k < ldq; k += blockDim.x) q[k] = 0.f;
}

// The VJP of fold_so_kernel: row i's dQ [K] ADDED (atomically: pairs share entities) into dS[s_dst[i]] and
// dO[o_dst[i]] (NULL index: row i).
template <int MODEL>
__global__ void __launch_bounds__(128)
unfold_so_kernel(Rows S, Rows O, const float* __restrict__ dQ, int64_t ldq, float* __restrict__ dS, int64_t lds,
                 const int64_t* __restrict__ s_dst, float* __restrict__ dO, int64_t ldo,
                 const int64_t* __restrict__ o_dst) {
  const int64_t i = blockIdx.x;
  const float* __restrict__ s = S.row(i);
  const float* __restrict__ o = O.row(i);
  const float* __restrict__ g = dQ + i * ldq;
  float* ds = dS + (s_dst ? s_dst[i] : i) * lds;
  float* dO_row = dO + (o_dst ? o_dst[i] : i) * ldo;
  const int D = S.dim, h = D >> 1;
  if constexpr (MODEL == B200KGE_RESCAL) {
    // d_s[r] = sum_c dQ[r, c] o_c: one warp per r;  d_o[c] = sum_r dQ[r, c] s_r: one thread per c
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    for (int r = warp; r < D; r += nw) {
      float acc = 0.f;
      for (int c = lane; c < D; c += 32) acc = fmaf(g[(int64_t)r * D + c], o[c], acc);
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
      if (lane == 0) atomicAdd(ds + r, acc);
    }
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
      float acc = 0.f;
      for (int r = 0; r < D; ++r) acc = fmaf(g[(int64_t)r * D + c], s[r], acc);
      atomicAdd(dO_row + c, acc);
    }
  } else {
    for (int k = threadIdx.x; k < D; k += blockDim.x) {
      if constexpr (MODEL == B200KGE_CP) {      // s[:h] pairs with o[h:]
        if (k < h) atomicAdd(ds + k, g[k] * o[k + h]);
        else       atomicAdd(dO_row + k, g[k - h] * s[k - h]);
      } else {
        float gs, go;
        if constexpr (MODEL == B200KGE_COMPLEX) {
          const int kk = (k < h) ? k : k - h;
          const float g_re = g[kk], g_im = g[kk + h];
          if (k < h) { gs = g_re * o[k] + g_im * o[k + h];  go = g_re * s[k] - g_im * s[k + h]; }
          else       { gs = g_re * o[k] - g_im * o[kk];     go = g_re * s[k] + g_im * s[kk]; }
        } else if constexpr (MODEL == B200KGE_DISTMULT) {
          gs = g[k] * o[k]; go = g[k] * s[k];
        } else {  // SIMPLE
          const int pk = (k < h) ? k + h : k - h;   // the partner column of k in the other half
          gs = 0.5f * g[k] * o[pk]; go = 0.5f * g[pk] * s[pk];
        }
        atomicAdd(ds + k, gs);
        atomicAdd(dO_row + k, go);
      }
    }
  }
}

int launch_fold_so(int model, const Rows& s, const Rows& o, int64_t n, float* Q, int64_t ldq, cudaStream_t st) {
  if (n == 0) return 0;
  const int K = relation_dim(model, s.dim);
#define B2K_FOLD_SO(M) case M: fold_so_kernel<M><<<(unsigned)n, 128, 0, st>>>(s, o, Q, ldq, K); break;
  switch (model) {
    B2K_FOLD_SO(B200KGE_COMPLEX) B2K_FOLD_SO(B200KGE_DISTMULT) B2K_FOLD_SO(B200KGE_SIMPLE) B2K_FOLD_SO(B200KGE_CP)
    B2K_FOLD_SO(B200KGE_RESCAL)
    default: set_error("the s_o fold covers the dot family only (model %d)", model); return B200KGE_ERR_UNSUPPORTED;
  }
#undef B2K_FOLD_SO
  B2K_LAUNCH_CHECK("fold_so_kernel");
  return 0;
}

int launch_unfold_so(int model, const Rows& s, const Rows& o, int64_t n, const float* dQ, int64_t ldq, float* dS,
                     int64_t lds, const int64_t* s_dst, float* dO, int64_t ldo, const int64_t* o_dst, cudaStream_t st) {
  if (n == 0) return 0;
#define B2K_UNFOLD_SO(M) case M: unfold_so_kernel<M><<<(unsigned)n, 128, 0, st>>>(s, o, dQ, ldq, dS, lds, s_dst, dO, ldo, o_dst); break;
  switch (model) {
    B2K_UNFOLD_SO(B200KGE_COMPLEX) B2K_UNFOLD_SO(B200KGE_DISTMULT) B2K_UNFOLD_SO(B200KGE_SIMPLE) B2K_UNFOLD_SO(B200KGE_CP)
    B2K_UNFOLD_SO(B200KGE_RESCAL)
    default: set_error("the s_o unfold covers the dot family only (model %d)", model); return B200KGE_ERR_UNSUPPORTED;
  }
#undef B2K_UNFOLD_SO
  B2K_LAUNCH_CHECK("unfold_so_kernel");
  return 0;
}

// Gather candidate rows (index subset) into a dense [m, ldd] block holding only the K columns the
// pair op reads; used by the tensor-core path, whose TMA loads need a regular 2-D table.
__global__ void __launch_bounds__(256)
gather_rows_kernel(Rows src, int col_off, int K, float* __restrict__ dst, int64_t ldd) {
  const int64_t r = blockIdx.x;
  const float* __restrict__ s = src.row(r) + col_off;
  for (int k = threadIdx.x; k < ldd; k += blockDim.x) dst[r * ldd + k] = (k < K) ? s[k] : 0.f;
}

int launch_gather_rows(const Rows& src, int col_off, int K, float* dst, int64_t ldd,
                       cudaStream_t st) {
  if (src.rows == 0) return 0;
  gather_rows_kernel<<<(unsigned)src.rows, 256, 0, st>>>(src, col_off, K, dst, ldd);
  B2K_LAUNCH_CHECK("gather_rows_kernel");
  return 0;
}

}  // namespace b200kge
