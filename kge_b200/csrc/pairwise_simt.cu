// pairwise_simt.cu — CUDA-core 1-vs-N scoring kernel (fp32 FFMA/FADD pipes, no tensor cores).
//
// score(i, j) = pair(Q_i, cand_j[col_off : col_off+K]) for a [128 x 128] tile per CTA, 8x8 register
// micro-tile per thread, K streamed through shared memory in 16-float chunks (register-prefetch
// double buffering), fused with the STORE / BCE / KL / RANK epilogues of common.cuh (distance family: also BCE / KL
// with the row's score sum, for label smoothing of the CSR-label losses).
//
// This is THE kernel for the distance family — TransE (transe.py:20-35, cdist without matmul) and
// RotatE (rotate.py:42-65, which materialises [n,E,D/2] intermediates in the reference) — whose
// inner op is sub/abs/add (or complex modulus), i.e. CUDA-core work with no tensor-core form.  It
// also serves dot-product scorers in exact-fp32 mode (B200KGE_PREC_FP32) and for shapes the
// tensor-core kernel does not take (tiny n, unaligned tables).
#include "common.cuh"

namespace b200kge {

namespace {

constexpr int BM = 128, BN = 128, BK = 16, LDS_ = BM + 4, NT = 256;

template <int PAIR>
__device__ __forceinline__ void pair_step(float (&acc)[8][8], const float (&a)[8], const float (&b)[8],
                                          const float (&a2)[8], const float (&b2)[8], float p) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if constexpr (PAIR == PAIR_DOT) {
        acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      } else if constexpr (PAIR == PAIR_L1) {
        acc[i][j] += fabsf(a[i] - b[j]);
      } else if constexpr (PAIR == PAIR_L2) {
        float d = a[i] - b[j];
        acc[i][j] = fmaf(d, d, acc[i][j]);
      } else if constexpr (PAIR == PAIR_LP) {
        acc[i][j] += __powf(fabsf(a[i] - b[j]), p);
      } else {
        float dre = a[i] - b[j];
        float dim = a2[i] - b2[j];
        float m2 = fmaf(dim, dim, dre * dre);
        if constexpr (PAIR == PAIR_CMOD_L1) {
          float r;
          asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(m2));
          acc[i][j] += r;
        } else {
          acc[i][j] += __powf(m2, 0.5f * p);
        }
      }
    }
  }
}

template <int PAIR>
__device__ __forceinline__ float pair_finish(float acc, float p) {
  if constexpr (PAIR == PAIR_DOT) return acc;
  else if constexpr (PAIR == PAIR_L1 || PAIR == PAIR_CMOD_L1) return -acc;
  else if constexpr (PAIR == PAIR_L2) return -sqrtf(acc);
  else return -powf(acc, 1.0f / p);
}

// One thread fetches 8 consecutive floats of one tile row for the current K chunk.
template <bool VEC>
__device__ __forceinline__ void fetch8(const float* __restrict__ rowp, bool row_ok, int k, int kmax,
                                       float (&r)[8]) {
  if (VEC) {
    if (row_ok && k + 8 <= kmax) {
      float4 u = __ldg(reinterpret_cast<const float4*>(rowp + k));
      float4 v = __ldg(reinterpret_cast<const float4*>(rowp + k + 4));
      r[0] = u.x; r[1] = u.y; r[2] = u.z; r[3] = u.w; r[4] = v.x; r[5] = v.y; r[6] = v.z; r[7] = v.w;
      return;
    }
  }
#pragma unroll
  for (int c = 0; c < 8; ++c) r[c] = (row_ok && k + c < kmax) ? __ldg(rowp + k + c) : 0.f;
}

// EPI_RANK_EVAL after the raw counts of a tile (the tensor-core form is tc_common.cuh: rank_eval_row).  The thread holds
// columns col0 + 4 tx + 64 (j >> 2) + (j & 3) of the row, acc[j] their unfinished scores, t the NaN-cleaned true score.
// One binary search per list, row and tile: the lists are short, and forward-moving cursors for two lists would cost
// 32 registers.
template <int PAIR>
__device__ __forceinline__ void rank_eval_tile(const EpiParams& P, const float (&acc)[8], float p_norm, int64_t row,
                                               int64_t col0, int64_t m, int tx, float t) {
  const int64_t lim = col0 + BN < m ? col0 + BN : m;
  const int64_t own = __ldg(P.csr_skip + row);
  auto holds = [&](int64_t cj) { return (((int)(cj - col0) & 63) >> 2) == tx; };
  auto pick = [&](int64_t cj) {
    const int rel = (int)(cj - col0), j = (rel >> 6) * 4 + (rel & 3);
    float x = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (i == j) x = acc[i];
    return pair_finish<PAIR>(x, p_norm);
  };
  if (own >= col0 && own < lim && holds(own)) P.own_score[row] = pick(own);
  RankFix fix;
#pragma unroll
  for (int list = 0; list < 2; ++list) {
    const int64_t* __restrict__ off = list ? P.csr2_off : P.csr_off;
    const int64_t* __restrict__ col = list ? P.csr2_col : P.csr_col;
    if (!off) continue;
    const int64_t end = __ldg(off + row + 1);
    for (int64_t cur = csr_lower_bound(col, __ldg(off + row), end, col0); cur < end; ++cur) {
      const int64_t cj = __ldg(col + cur);
      if (cj >= lim) break;
      if (holds(cj) && cj != own) fix.add(list == 1, pick(cj), t, P.rtol, P.atol);
    }
  }
  fix.commit(P, row);
}

// CSR: the ranking epilogue with a CSR filter is its own instantiation — its 16 cursor registers would otherwise cost the
// plain rank kernel its second resident CTA (168 vs <= 128 registers: 5.83 -> 6.59 ms on the cfg5 shard).
template <int PAIR, int EPI, bool VEC, bool CSR = false>
__global__ void __launch_bounds__(NT)   // (NT, 2) was measured: spills in the fused epilogues, no net gain
pairwise_simt_kernel(const float* __restrict__ Q, int64_t ldq, int64_t nq, Rows cand, int col_off,
                     int K, float p_norm, int col_tiles, EpiParams P) {
  __shared__ __align__(16) float As[2][BK][LDS_];
  __shared__ __align__(16) float Bs[2][BK][LDS_];
  constexpr bool CMOD = (PAIR == PAIR_CMOD_L1 || PAIR == PAIR_CMOD_LP);

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t row0 = (int64_t)blockIdx.y * BM;
  const int64_t m = cand.rows;

  // this CTA's range of column tiles (chunk = blockIdx.x of gridDim.x)
  const int nch = gridDim.x, ch = blockIdx.x;
  const int tbase = col_tiles / nch, trem = col_tiles % nch;
  const int t0 = ch * tbase + (ch < trem ? ch : trem);
  const int t1 = t0 + tbase + (ch < trem ? 1 : 0);

  // loader role: row lr of the tile, half lh (floats [lh*8, lh*8+8) of the chunk)
  const int lr = tid >> 1, lh = tid & 1;
  const bool a_ok = (row0 + lr) < nq;
  const float* __restrict__ arow = Q + (a_ok ? (row0 + lr) : 0) * ldq;

  // complex pair ops: chunk = 8 re (slots 0..7) + 8 im (slots 8..15); reduction runs over h = K/2
  const int h = K >> 1;
  const int kspan = CMOD ? h : K;
  const int kstep = CMOD ? 8 : BK;
  const int nk = (kspan + kstep - 1) / kstep;
  auto chunk_k = [&](int kt) { return CMOD ? (lh ? h + kt * 8 : kt * 8) : (kt * BK + lh * 8); };
  const int kmax = CMOD ? (lh ? K : h) : K;

  // per-row epilogue state lives across all tiles of the chunk
  RowState<EPI> st[8];
  float aux[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    st[i].init();
    const int64_t row = row0 + ty * 4 + 64 * (i >> 2) + (i & 3);
    aux[i] = (row < nq) ? epi_row_aux<EPI>(P, row) : 0.f;
  }
  // CSR ranking filter (SURVEY 8f-2): per owned row a cursor into its sorted segment of known answers; the CTA visits
  // its column tiles in increasing order, so each cursor only moves forward (one binary search at the first tile, then
  // ~one L1-resident load per row and tile)
  int ccur[CSR ? 8 : 1], cend[CSR ? 8 : 1];          // nnz < 2^31 (checked by the launcher)
  if constexpr (CSR) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int64_t row = row0 + ty * 4 + 64 * (i >> 2) + (i & 3);
      ccur[i] = 0; cend[i] = 0;
      if (row < nq) {
        cend[i] = (int)__ldg(P.csr_off + row + 1);
        ccur[i] = (int)csr_lower_bound(P.csr_col, __ldg(P.csr_off + row), (int64_t)cend[i], (int64_t)t0 * BN);
      }
    }
  }

  for (int tile = t0; tile < t1; ++tile) {
    const int64_t col0 = (int64_t)tile * BN;
    const bool b_ok = (col0 + lr) < m;
    const float* __restrict__ brow = (b_ok ? cand.row(col0 + lr) : cand.base) + col_off;

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    float ra[8], rb[8];
    fetch8<VEC>(arow, a_ok, chunk_k(0), kmax, ra);
    fetch8<VEC>(brow, b_ok, chunk_k(0), kmax, rb);
    __syncthreads();  // previous tile's readers are done with buffer 0
#pragma unroll
    for (int c = 0; c < 8; ++c) { As[0][lh * 8 + c][lr] = ra[c]; Bs[0][lh * 8 + c][lr] = rb[c]; }
    __syncthreads();

    for (int kt = 0; kt < nk; ++kt) {
      const int cur = kt & 1;
      const bool more = (kt + 1) < nk;
      if (more) {
        fetch8<VEC>(arow, a_ok, chunk_k(kt + 1), kmax, ra);
        fetch8<VEC>(brow, b_ok, chunk_k(kt + 1), kmax, rb);
      }
      constexpr int KK = CMOD ? 8 : BK;
#pragma unroll
      for (int kk = 0; kk < KK; ++kk) {
        float a[8], b[8], a2[8], b2[8];
#pragma unroll
        for (int ii = 0; ii < 2; ++ii) {
          float4 v = *reinterpret_cast<const float4*>(&As[cur][kk][ty * 4 + 64 * ii]);
          a[ii * 4 + 0] = v.x; a[ii * 4 + 1] = v.y; a[ii * 4 + 2] = v.z; a[ii * 4 + 3] = v.w;
          float4 w = *reinterpret_cast<const float4*>(&Bs[cur][kk][tx * 4 + 64 * ii]);
          b[ii * 4 + 0] = w.x; b[ii * 4 + 1] = w.y; b[ii * 4 + 2] = w.z; b[ii * 4 + 3] = w.w;
          if constexpr (CMOD) {
            float4 v2 = *reinterpret_cast<const float4*>(&As[cur][kk + 8][ty * 4 + 64 * ii]);
            a2[ii * 4 + 0] = v2.x; a2[ii * 4 + 1] = v2.y; a2[ii * 4 + 2] = v2.z; a2[ii * 4 + 3] = v2.w;
            float4 w2 = *reinterpret_cast<const float4*>(&Bs[cur][kk + 8][tx * 4 + 64 * ii]);
            b2[ii * 4 + 0] = w2.x; b2[ii * 4 + 1] = w2.y; b2[ii * 4 + 2] = w2.z; b2[ii * 4 + 3] = w2.w;
          }
        }
        pair_step<PAIR>(acc, a, b, a2, b2, p_norm);
      }
      if (more) {
#pragma unroll
        for (int c = 0; c < 8; ++c) { As[cur ^ 1][lh * 8 + c][lr] = ra[c]; Bs[cur ^ 1][lh * 8 + c][lr] = rb[c]; }
      }
      __syncthreads();
    }

    // ---- tile epilogue: thread owns rows ty*4 + 64*ii + r, cols tx*4 + 64*jj + c --------------
    if constexpr (EPI == EPI_STORE) {
      if (P.store_vec4) {
        // 16-byte stores: the 4 consecutive columns a thread owns go out as one float4, so a half-warp writes 256
        // contiguous bytes of one output row (the scalar form writes 4-byte words 16 bytes apart — tolerable into
        // local HBM behind L2, ruinous for the peer stores of the fused all-gather over NVLink)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int64_t row = row0 + ty * 4 + 64 * (i >> 2) + (i & 3);
          if (row >= nq) continue;
          int64_t r = row, cb = 0;
          if (P.n_rows_out > 0 && row >= P.n_rows_out) { r = row - P.n_rows_out; cb = P.col_block; }
#pragma unroll
          for (int jj = 0; jj < 2; ++jj) {
            const int64_t col = col0 + tx * 4 + 64 * jj;
            if (col >= m) continue;
            const float4 v = make_float4(pair_finish<PAIR>(acc[i][jj * 4 + 0], p_norm), pair_finish<PAIR>(acc[i][jj * 4 + 1], p_norm),
                                         pair_finish<PAIR>(acc[i][jj * 4 + 2], p_norm), pair_finish<PAIR>(acc[i][jj * 4 + 3], p_norm));
            const int64_t at = r * P.ldo + cb + col;
            if (col + 3 < m) {
              *reinterpret_cast<float4*>(P.out + at) = v;
              for (int g = 0; g < P.n_peers; ++g) *reinterpret_cast<float4*>(P.out_peer[g] + at) = v;
            } else {
              const float vv[4] = {v.x, v.y, v.z, v.w};
              for (int c = 0; c < 4 && col + c < m; ++c) {
                P.out[at + c] = vv[c];
                for (int g = 0; g < P.n_peers; ++g) P.out_peer[g][at + c] = vv[c];
              }
            }
          }
        }
        continue;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int64_t row = row0 + ty * 4 + 64 * (i >> 2) + (i & 3);
      const bool row_ok = row < nq;
      unsigned filtered = 0u;          // bit j: element (i, j) is a known answer of this row (rank filter)
      if constexpr (CSR) {
        if (ccur[i] < cend[i]) {
          const int64_t own = P.csr_skip ? __ldg(P.csr_skip + row) : -1;
          int64_t cj = __ldg(P.csr_col + ccur[i]);
          while (cj < col0 + BN) {                       // listed columns inside this tile
            const int rel = (int)(cj - col0), jj = rel >> 6, c4 = rel & 63;
            if ((c4 >> 2) == tx && cj != own) filtered |= 1u << (jj * 4 + (c4 & 3));
            if (++ccur[i] >= cend[i]) break;
            cj = __ldg(P.csr_col + ccur[i]);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int64_t col = col0 + tx * 4 + 64 * (j >> 2) + (j & 3);
        float x = pair_finish<PAIR>(acc[i][j], p_norm);
        if constexpr (CSR) {
          if (filtered & (1u << j)) x = -INFINITY;       // eval_entity_ranking.py:561-566: score - inf
        }
        if (row_ok && col < m) epi_elem<EPI>(P, st[i], row, col, x, aux[i]);
      }
      if constexpr (EPI == EPI_RANK_EVAL) {
        if (row_ok) rank_eval_tile<PAIR>(P, acc[i], p_norm, row, col0, m, tx, aux[i]);
      }
    }
  }

  if constexpr (EPI != EPI_STORE) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int64_t row = row0 + ty * 4 + 64 * (i >> 2) + (i & 3);
      epi_lane_reduce<EPI>(st[i], 16);
      if (tx == 0 && row < nq) epi_flush<EPI>(P, st[i], row, ch);
    }
  }
}

template <int PAIR, int EPI>
int launch_pe(bool vec, dim3 grid, cudaStream_t st, const float* Q, int64_t ldq, int64_t nq,
              const Rows& cand, int col_off, int K, float p, const EpiParams& P) {
  const int col_tiles = (int)((cand.rows + BN - 1) / BN);
  if constexpr (EPI == EPI_RANK) {
    if (P.csr_off) {
      if (P.csr_nnz >= (1ll << 31)) { set_error("CSR filter too long for the CUDA-core rank epilogue"); return B200KGE_ERR_UNSUPPORTED; }
      profile_begin(st);
      if (vec) pairwise_simt_kernel<PAIR, EPI, true, true><<<grid, NT, 0, st>>>(Q, ldq, nq, cand, col_off, K, p, col_tiles, P);
      else     pairwise_simt_kernel<PAIR, EPI, false, true><<<grid, NT, 0, st>>>(Q, ldq, nq, cand, col_off, K, p, col_tiles, P);
      profile_end(st);
      B2K_LAUNCH_CHECK("pairwise_simt_kernel");
      return 0;
    }
  }
  profile_begin(st);
  if (vec) pairwise_simt_kernel<PAIR, EPI, true><<<grid, NT, 0, st>>>(Q, ldq, nq, cand, col_off, K, p, col_tiles, P);
  else     pairwise_simt_kernel<PAIR, EPI, false><<<grid, NT, 0, st>>>(Q, ldq, nq, cand, col_off, K, p, col_tiles, P);
  profile_end(st);
  B2K_LAUNCH_CHECK("pairwise_simt_kernel");
  return 0;
}

template <int PAIR>
int launch_p(int epi, bool vec, dim3 grid, cudaStream_t st, const float* Q, int64_t ldq, int64_t nq,
             const Rows& cand, int col_off, int K, float p, const EpiParams& P) {
  switch (epi) {
    case EPI_STORE: return launch_pe<PAIR, EPI_STORE>(vec, grid, st, Q, ldq, nq, cand, col_off, K, p, P);
    case EPI_BCE:   return launch_pe<PAIR, EPI_BCE>(vec, grid, st, Q, ldq, nq, cand, col_off, K, p, P);
    case EPI_KL:    return launch_pe<PAIR, EPI_KL>(vec, grid, st, Q, ldq, nq, cand, col_off, K, p, P);
    case EPI_RANK:  return launch_pe<PAIR, EPI_RANK>(vec, grid, st, Q, ldq, nq, cand, col_off, K, p, P);
    case EPI_RANK_EVAL: return launch_pe<PAIR, EPI_RANK_EVAL>(vec, grid, st, Q, ldq, nq, cand, col_off, K, p, P);
  }
  if constexpr (PAIR != PAIR_DOT) {      // the dot family sums its scores as Q . colsum(T) instead
    switch (epi) {
      case EPI_BCE_ZSUM: return launch_pe<PAIR, EPI_BCE_ZSUM>(vec, grid, st, Q, ldq, nq, cand, col_off, K, p, P);
      case EPI_KL_ZSUM:  return launch_pe<PAIR, EPI_KL_ZSUM>(vec, grid, st, Q, ldq, nq, cand, col_off, K, p, P);
    }
  }
  set_error("bad epilogue kind %d", epi);
  return B200KGE_ERR_INVALID;
}

}  // namespace

// Number of column chunks (= CTAs along x): enough CTAs to fill the GPU a few times over, but
// bounded so that the per-(row, chunk) partial buffers of the fused losses stay small.
int pairwise_simt_nchunks(int64_t nq, int64_t m) {
  const int64_t ct = (m + BN - 1) / BN, rt = (nq + BM - 1) / BM;
  int64_t want = (132 * 6 + rt - 1) / (rt > 0 ? rt : 1);
  if (want < 1) want = 1;
  return (int)(want < ct ? want : ct);
}

int launch_pairwise_simt(int epi_kind, int pair_op, float l_norm, const float* Q, int64_t ldq,
                         int64_t nq, const Rows& cand, int col_off, int K, const EpiParams& P,
                         cudaStream_t st) {
  if (nq == 0 || cand.rows == 0) return 0;
  const int64_t ct = pairwise_simt_nchunks(nq, cand.rows), rt = (nq + BM - 1) / BM;
  if (rt > 65535) { set_error("too many query rows for one launch (%lld)", (long long)nq); return B200KGE_ERR_UNSUPPORTED; }
  dim3 grid((unsigned)ct, (unsigned)rt);
  const bool cm = (pair_op == PAIR_CMOD_L1 || pair_op == PAIR_CMOD_LP);
  bool vec = (ldq % 4 == 0) && (cand.ld % 4 == 0) && (col_off % 4 == 0) &&
             ((reinterpret_cast<uintptr_t>(Q) & 15) == 0) &&
             ((reinterpret_cast<uintptr_t>(cand.base) & 15) == 0) && (!cm || ((K / 2) % 4 == 0));
  EpiParams Pv = P;
  if (epi_kind == EPI_STORE) {
    // float4 stores need 16-byte aligned row starts in every destination
    bool ok = (P.ldo % 4 == 0) && (P.col_block % 4 == 0) && ((reinterpret_cast<uintptr_t>(P.out) & 15) == 0);
    for (int g = 0; g < P.n_peers; ++g) ok = ok && ((reinterpret_cast<uintptr_t>(P.out_peer[g]) & 15) == 0);
    Pv.store_vec4 = ok ? 1 : 0;
  }
  switch (pair_op) {
    case PAIR_DOT:     return launch_p<PAIR_DOT>(epi_kind, vec, grid, st, Q, ldq, nq, cand, col_off, K, l_norm, Pv);
    case PAIR_L1:      return launch_p<PAIR_L1>(epi_kind, vec, grid, st, Q, ldq, nq, cand, col_off, K, l_norm, Pv);
    case PAIR_L2:      return launch_p<PAIR_L2>(epi_kind, vec, grid, st, Q, ldq, nq, cand, col_off, K, l_norm, Pv);
    case PAIR_LP:      return launch_p<PAIR_LP>(epi_kind, vec, grid, st, Q, ldq, nq, cand, col_off, K, l_norm, Pv);
    case PAIR_CMOD_L1: return launch_p<PAIR_CMOD_L1>(epi_kind, vec, grid, st, Q, ldq, nq, cand, col_off, K, l_norm, Pv);
    case PAIR_CMOD_LP: return launch_p<PAIR_CMOD_LP>(epi_kind, vec, grid, st, Q, ldq, nq, cand, col_off, K, l_norm, Pv);
  }
  set_error("bad pair op %d", pair_op);
  return B200KGE_ERR_INVALID;
}

}  // namespace b200kge
