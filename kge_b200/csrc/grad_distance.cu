// grad_distance.cu — SURVEY §8 f-1 for the distance family: backward of the 1-vs-N scores of TransE (L1, L2;
// transe.py:20-35) and RotatE (L1 of complex moduli; rotate.py:42-65) through the folded form score(i, j) = pair(Q_i, T_j).
//
// Every pair op here is a function of the difference d = q - t, so with s'(d) = d pair / d q:
//   dQ_i = sum_j G_ij s'(Q_i - T_j)            dT_j = sum_i G_ij s'(T_j - Q_i)        (s' is odd in d)
// i.e. ONE kernel, "row gradient": dA[r, :] = sum_c W[r, c] * s'(A_r - B_c), called with (A, B, W) = (Q, T, G) and
// with (T, Q, G^T).  No tensor cores (sign / normalise per element, like the forward: CUDA-core bound).
//   L1      s = -sum_k |d_k|             s'_k = -sign(d_k)
//   L2      s = -||d||                   s'_k = -d_k / ||d|| = d_k / s        (G is pre-divided by the stored score s)
//   CMOD L1 s = -sum_k |d_k| (complex)   s'_(re,im),k = -(d_re, d_im)_k / |d_k|   (0 if |d_k| = 0)
// G = n dL/dz comes from grad_dense_kernel (BCE: sigmoid(z + off) - y; KL: w softmax(z) - y / sum y), fp32, dense, or
// from grad_csr_kernel for the CSR labels of KvsAll (dL/dz / batch_size).
//
// Tiling: a CTA owns 64 rows of A x one 64-float chunk of the reduction axis (grid.y; every element of the axis is
// independent) and walks ALL columns in shared-memory tiles of 64, so dA is written once, without atomics.  A thread
// holds a 4-row x 4-element register tile: per column ONE 16-byte shared load of 4 weights (W arrives TRANSPOSED,
// [column, row], so the tile fill is coalesced and conflict-free) and one of 4 B elements feed 16 element updates
// (L1: sub, xor-sign, compare, predicated add).  First version (16 rows x 16 lanes, 5 scalar shared loads per 4
// updates): 16.6 ms (dQ, 128 CTAs) + 6.3 ms (dT) at n = 1024, E = 14 541, D = 512 — shared-memory bound.
#include "common.cuh"

namespace b200kge {

namespace {

constexpr int RG_ROWS = 64;    // rows of A per CTA (16 thread rows x 4)
constexpr int RG_CT = 64;      // columns per shared-memory tile
constexpr int RG_KC = 64;      // floats of the reduction axis per CTA (CMOD: 32 complex elements = 32 re + 32 im)

// float x in [0, 64) of the CTA's chunk -> offset inside a row (or -1).  Plain: element e0 + x.  CMOD: groups of four
// (re_e, re_e+1, im_e, im_e+1) so a thread's float4 holds two complex elements.
template <bool CMOD>
__device__ __forceinline__ int chunk_offset(int x, int e0, int span, int h) {
  if (CMOD) {
    const int e = e0 + (x >> 2) * 2 + (x & 1);
    return e < span ? ((x & 2) ? h + e : e) : -1;
  }
  const int e = e0 + x;
  return e < span ? e : -1;
}

template <int PAIR>
__global__ void __launch_bounds__(256)
pair_rowgrad_kernel(const float* __restrict__ A, int64_t lda, int64_t ra, const float* __restrict__ B, int64_t ldb,
                    int64_t rb, int K, const float* __restrict__ Wt, int64_t ldwt, float* __restrict__ dA,
                    int64_t ldda) {
  __shared__ __align__(16) float Bs[RG_CT][RG_KC + 4];
  __shared__ __align__(16) float Ws[RG_CT][RG_ROWS];
  constexpr bool CMOD = (PAIR == PAIR_CMOD_L1);
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int h = K >> 1, span = CMOD ? h : K;
  const int e0 = blockIdx.y * (CMOD ? RG_KC / 2 : RG_KC);
  const int64_t row0 = (int64_t)blockIdx.x * RG_ROWS;
  float a[4][4], acc[4][4];
  int offs[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) offs[j] = chunk_offset<CMOD>(tx * 4 + j, e0, span, h);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t row = row0 + ty * 4 + i;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      a[i][j] = (row < ra && offs[j] >= 0) ? __ldg(A + row * lda + offs[j]) : 0.f;
      acc[i][j] = 0.f;
    }
  }
  const int fx = tid & 63, fr = tid >> 6;              // tile fills: 4 tile rows per pass
  const int foff = chunk_offset<CMOD>(fx, e0, span, h);
  for (int64_t c0 = 0; c0 < rb; c0 += RG_CT) {
    __syncthreads();
#pragma unroll 4
    for (int c = fr; c < RG_CT; c += 4) {
      const int64_t col = c0 + c;
      Bs[c][fx] = (col < rb && foff >= 0) ? __ldg(B + col * ldb + foff) : 0.f;
      Ws[c][fx] = (col < rb && row0 + fx < ra) ? __ldg(Wt + col * ldwt + row0 + fx) : 0.f;
    }
    __syncthreads();
#pragma unroll 2
    for (int c = 0; c < RG_CT; ++c) {
      const float4 w4 = *reinterpret_cast<const float4*>(&Ws[c][ty * 4]);
      const float4 b4 = *reinterpret_cast<const float4*>(&Bs[c][tx * 4]);
      const float w[4] = {w4.x, w4.y, w4.z, w4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if constexpr (PAIR == PAIR_L1) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float d = a[i][j] - b[j];
            const float ws = __uint_as_float(__float_as_uint(w[i]) ^ (__float_as_uint(d) & 0x80000000u));   // w sign(d)
            if (d != 0.f) acc[i][j] -= ws;
          }
        } else if constexpr (PAIR == PAIR_L2) {
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(w[i], a[i][j] - b[j], acc[i][j]);     // w holds G / score
        } else {
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const float dre = a[i][j] - b[j], dim = a[i][2 + j] - b[2 + j];
            const float m2 = fmaf(dim, dim, dre * dre);
            const float wi = (m2 > 0.f) ? w[i] * rsqrtf(m2) : 0.f;
            acc[i][j] = fmaf(-wi, dre, acc[i][j]);
            acc[i][2 + j] = fmaf(-wi, dim, acc[i][2 + j]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t row = row0 + ty * 4 + i;
    if (row >= ra) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (offs[j] >= 0) dA[row * ldda + offs[j]] = acc[i][j];
  }
}

// G[i, e] = n dL/dz_ie for one-hot labels (1vsAll): BCE sigmoid(z + off) - y | KL softmax(z) - y  (row_stat[2i] = lse_i),
// times inv_n; div_z: divided by the score itself (L2: d(-||d||)/dq = d / score; 0 where the score is 0).
// grid = (ceil(E / 256), nq)
__global__ void __launch_bounds__(256)
grad_dense_kernel(const float* __restrict__ z, int64_t ldz, int64_t E, const int64_t* __restrict__ label_idx,
                  const float* __restrict__ row_stat, float offset, float inv_n, int div_z, float* __restrict__ G,
                  int64_t ldg) {
  const int64_t i = blockIdx.y, e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const float zv = z[i * ldz + e], x = zv + offset;
  const float y = (label_idx[i] == e) ? 1.f : 0.f;
  float g;
  if (row_stat) {
    const float ys = row_stat[2 * i + 1], yc = fmaxf(ys, 1e-12f);
    g = (ys / yc) * expf(x - row_stat[2 * i]) - y / yc;
  } else {
    g = 1.0f / (1.0f + expf(-x)) - y;
  }
  g *= inv_n;
  if (div_z) g = (zv != 0.f) ? g / zv : 0.f;
  G[i * ldg + e] = g;
}

// G for the CSR labels of a KvsAll query type (train_KvsAll.py:242-266), the fp32 counterpart of grad.cu's CSR planes:
// y_ie = a c_ie + b with c_ie the multiplicity of column e in row i's sorted segment col[off[i], off[i+1]).
//   BCE  sigmoid(z + off) - y          KL  w softmax(z) - y / yc,  Y = a nnz_i + b E, yc = max(Y, 1e-12), w = Y / yc
// (row_stat[2i] = lse_i), times inv_n; div_z as in grad_dense_kernel.  One block per row: the label-free value (y = b)
// everywhere, then, after the block barrier, the row's listed columns overwritten by the same block — no atomics and
// no [n, E] label matrix.  A row with no labels and no smoothing gets sigmoid(z + off) (BCE) or 0 (KL), as on the
// tensor-core path.  grid = nq
__global__ void __launch_bounds__(256)
grad_csr_kernel(const float* __restrict__ z, int64_t ldz, int64_t E, const int64_t* __restrict__ off,
                const int64_t* __restrict__ col, float a, float b, const float* __restrict__ row_stat, float offset,
                float inv_n, int div_z, float* __restrict__ G, int64_t ldg) {
  const int64_t i = blockIdx.x, t0 = off[i], t1 = off[i + 1];
  const float* __restrict__ zr = z + i * ldz;
  float* __restrict__ gr = G + i * ldg;
  const float ys = a * (float)(t1 - t0) + b * (float)E, yc = fmaxf(ys, 1e-12f);
  auto grad = [&](float zv, float y) {
    const float x = zv + offset;
    float g = row_stat ? (ys / yc) * expf(x - row_stat[2 * i]) - y / yc : 1.0f / (1.0f + expf(-x)) - y;
    g *= inv_n;
    return div_z ? ((zv != 0.f) ? g / zv : 0.f) : g;
  };
  for (int64_t e = threadIdx.x; e < E; e += blockDim.x) gr[e] = grad(zr[e], b);
  __syncthreads();
  for (int64_t t = t0 + threadIdx.x; t < t1; t += blockDim.x) {
    if (t > t0 && col[t] == col[t - 1]) continue;             // a run of equal columns is handled by its first entry
    int64_t c = 1;
    while (t + c < t1 && col[t + c] == col[t]) ++c;
    const int64_t e = col[t];
    gr[e] = grad(zr[e], a * (float)c + b);
  }
}

// W[i, e] = g[i, e] / z[i, e] (0 where z = 0): the L2 pair op's chain factor for a given dL/dscores.  grid = (ceil(E/256), n)
__global__ void __launch_bounds__(256)
div_scores_kernel(const float* __restrict__ g, int64_t ldg, const float* __restrict__ z, int64_t ldz, int64_t E,
                  float* __restrict__ W, int64_t ldw) {
  const int64_t i = blockIdx.y, e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const float zv = z[i * ldz + e];
  W[i * ldw + e] = (zv != 0.f) ? g[i * ldg + e] / zv : 0.f;
}

template <int PAIR>
int launch_rowgrad_t(const float* A, int64_t lda, int64_t ra, const float* B, int64_t ldb, int64_t rb, int K, const float* Wt,
                     int64_t ldwt, float* dA, int64_t ldda, cudaStream_t st) {
  if (ra == 0 || rb == 0 || K == 0) return 0;
  const int span = (PAIR == PAIR_CMOD_L1) ? K / 2 : K, epc = (PAIR == PAIR_CMOD_L1) ? RG_KC / 2 : RG_KC;
  dim3 grid((unsigned)((ra + RG_ROWS - 1) / RG_ROWS), (unsigned)((span + epc - 1) / epc));
  pair_rowgrad_kernel<PAIR><<<grid, 256, 0, st>>>(A, lda, ra, B, ldb, rb, K, Wt, ldwt, dA, ldda);
  B2K_LAUNCH_CHECK("pair_rowgrad_kernel");
  return 0;
}

}  // namespace

int launch_pair_rowgrad(int pair_op, const float* A, int64_t lda, int64_t ra, const float* B, int64_t ldb, int64_t rb, int K,
                        const float* Wt, int64_t ldwt, float* dA, int64_t ldda, cudaStream_t st) {
  switch (pair_op) {
    case PAIR_L1:      return launch_rowgrad_t<PAIR_L1>(A, lda, ra, B, ldb, rb, K, Wt, ldwt, dA, ldda, st);
    case PAIR_L2:      return launch_rowgrad_t<PAIR_L2>(A, lda, ra, B, ldb, rb, K, Wt, ldwt, dA, ldda, st);
    case PAIR_CMOD_L1: return launch_rowgrad_t<PAIR_CMOD_L1>(A, lda, ra, B, ldb, rb, K, Wt, ldwt, dA, ldda, st);
  }
  set_error("the distance-family backward covers L1, L2 (TransE) and the L1 of complex moduli (RotatE)");
  return B200KGE_ERR_UNSUPPORTED;
}

int launch_div_scores(const float* g, int64_t ldg, const float* z, int64_t ldz, int64_t n, int64_t E, float* W, int64_t ldw,
                      cudaStream_t st) {
  if (n == 0 || E == 0) return 0;
  if (n > 65535) { set_error("too many rows for one launch (%lld)", (long long)n); return B200KGE_ERR_UNSUPPORTED; }
  dim3 grid((unsigned)((E + 255) / 256), (unsigned)n);
  div_scores_kernel<<<grid, 256, 0, st>>>(g, ldg, z, ldz, E, W, ldw);
  B2K_LAUNCH_CHECK("div_scores_kernel");
  return 0;
}

int launch_grad_dense(const float* z, int64_t ldz, int64_t nq, int64_t E, const int64_t* label_idx, const float* row_stat,
                      float offset, float inv_n, int div_z, float* G, int64_t ldg, cudaStream_t st) {
  if (nq == 0 || E == 0) return 0;
  if (nq > 65535) { set_error("too many rows for one launch (%lld)", (long long)nq); return B200KGE_ERR_UNSUPPORTED; }
  dim3 grid((unsigned)((E + 255) / 256), (unsigned)nq);
  grad_dense_kernel<<<grid, 256, 0, st>>>(z, ldz, E, label_idx, row_stat, offset, inv_n, div_z, G, ldg);
  B2K_LAUNCH_CHECK("grad_dense_kernel");
  return 0;
}

int launch_grad_csr(const float* z, int64_t ldz, int64_t nq, int64_t E, const int64_t* csr_off, const int64_t* csr_col,
                    float a, float b, const float* row_stat, float offset, float inv_n, int div_z, float* G, int64_t ldg,
                    cudaStream_t st) {
  if (nq == 0 || E == 0) return 0;
  grad_csr_kernel<<<(unsigned)nq, 256, 0, st>>>(z, ldz, E, csr_off, csr_col, a, b, row_stat, offset, inv_n, div_z, G, ldg);
  B2K_LAUNCH_CHECK("grad_csr_kernel");
  return 0;
}

}  // namespace b200kge
