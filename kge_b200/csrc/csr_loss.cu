// csr_loss.cu — SURVEY §8 f-2, device half: KvsAll losses with CSR multi-hot labels — no [n, E] label matrix is
// built or read.  The label-free part comes from the fused scorer; the scores of the listed columns are emitted by
// the same pass's epilogue on the pre-split tensor-core path (tc_common.cuh, per-thread cursor into the row's sorted
// CSR segment) or, for the CUDA-core families, by the row-wise triple kernel; the row kernels below combine them.
//
// With labels y_ij = a * c_ij + b  (c_ij = multiplicity of column j in row i's CSR segment, a = 1 - eps,
// b = eps > 0 ? 1/E : 0; train_KvsAll.py:242-266) both losses split into a label-free part, which the fused
// scorer already produces per row, and a sparse part that needs the scores of the listed columns only:
//   BCE  (loss.py:153-159)   L_i = sum_j softplus(z_ij + off)  -  a * sum_csr (z + off)  -  b * sum_j (z_ij + off)
//   KL   (loss.py:198-213)   L_i = sum_j yh log yh  -  (a * sum_csr z + b * sum_j z_ij) / Y  +  lse_i,
//                            Y = a * nnz_i + b * E,  yh = y / Y   (rows with Y = 0 contribute nothing)
// sum_j softplus: fused BCE kernel with no label (index -1).  lse_i: fused KL kernel with the one-hot label at
// column 0 returns lse_i - z_i0, and z_i0 rides along with the listed columns.  The listed scores come from the
// row-wise triple kernel (gather + dot per CSR entry: nnz * D work).  sum_j z_ij (label smoothing only) is
// Q_i . colsum(T) for the dot family; the distance family's CUDA-core scorer sums it in the same pass that reduces the
// label-free terms (EPI_BCE_ZSUM / EPI_KL_ZSUM, one partial per row and column chunk).
#include "common.cuh"

namespace b200kge {

namespace {

// one thread per row: expand the row's CSR segment into (query row, relation row, entity) selections for the
// row-wise scorer; with `extra`, entry nnz + i scores row i against entity 0.
__global__ void __launch_bounds__(256)
csr_expand_kernel(const int64_t* __restrict__ off, const int64_t* __restrict__ col, int64_t n, int64_t nnz, int extra,
                  const int64_t* __restrict__ q_idx, const int64_t* __restrict__ p_idx, int64_t* __restrict__ qsel,
                  int64_t* __restrict__ psel, int64_t* __restrict__ esel) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t qi = q_idx ? q_idx[i] : i, pi = p_idx ? p_idx[i] : i;
  for (int64_t t = off[i]; t < off[i + 1]; ++t) { qsel[t] = qi; psel[t] = pi; esel[t] = col[t]; }
  if (extra) { qsel[nnz + i] = qi; psel[nnz + i] = pi; esel[nnz + i] = 0; }
}

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// one warp per row: combine the fused kernel's per-row term with the sparse label terms.
//   fused[i]: BCE -> sum_j softplus(z + off);  KL -> lse_i - z_i0.   zsum may be null (no smoothing); else row i's
//   sum_j z_ij in zch partial sums zsum[i * zch ..] (the CUDA-core scorer's chunks; 1 for the dot family's Q . colsum).
template <int LOSS>
__global__ void __launch_bounds__(256)
csr_rows_kernel(const int64_t* __restrict__ off, const int64_t* __restrict__ col, const float* __restrict__ zpos,
                int64_t n, int64_t nnz, const float* __restrict__ fused, const float* __restrict__ zsum, int zch, float a,
                float b, float E, float offset, float* __restrict__ row_loss) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= n) return;
  const int64_t t0 = off[i], t1 = off[i + 1];
  float B = 0.f, ylogy = 0.f, distinct = 0.f;
  for (int64_t t = t0 + lane; t < t1; t += 32) {
    B += zpos[t];
    if (LOSS == B200KGE_LOSS_KL && (t == t0 || col[t] != col[t - 1])) {     // start of a run of equal columns
      int64_t c = 1;
      while (t + c < t1 && col[t + c] == col[t]) ++c;
      const float y = a * (float)c + b;
      ylogy += y * logf(y);
      distinct += 1.f;
    }
  }
  B = wsum(B);
  const float cnt = (float)(t1 - t0);
  float zs = 0.f;
  if (zsum) {
    for (int c = lane; c < zch; c += 32) zs += zsum[i * zch + c];
    zs = wsum(zs);
  }
  float L;
  if (LOSS == B200KGE_LOSS_BCE) {
    L = fused[i] - a * (B + cnt * offset) - b * (zs + E * offset);
  } else {
    ylogy = wsum(ylogy);
    distinct = wsum(distinct);
    const float Y = a * cnt + b * E;
    if (Y > 0.f) {
      const float rest = (b > 0.f) ? (E - distinct) * b * logf(b) : 0.f;
      const float lse = fused[i] + zpos[nnz + i];
      L = (ylogy + rest) / Y - logf(Y) - (a * B + b * zs) / Y + lse;
    } else {
      L = 0.f;
    }
  }
  if (lane == 0) row_loss[i] = L;
}

// deterministic scalar sum of n row terms by one block (fixed order)
__global__ void __launch_bounds__(256)
rows_sum_kernel(const float* __restrict__ rows, int64_t n, float scale, float* __restrict__ out) {
  __shared__ float red[8];
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) acc += rows[i];
  acc = wsum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w];
    *out = t * scale;
  }
}

// column sums of T[E, K] (row stride ld): partial[chunk][k] over CS_ROWS-row chunks, then summed in order
constexpr int CS_ROWS = 1024;
__global__ void __launch_bounds__(256)
colsum_partial_kernel(const float* __restrict__ T, int64_t ld, int64_t E, int K, float* __restrict__ partial, int Kpad) {
  __shared__ float red[8][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int k = blockIdx.x * 32 + lane;
  const int64_t r0 = (int64_t)blockIdx.y * CS_ROWS;
  float acc = 0.f;
  if (k < K)
    for (int64_t r = r0 + warp; r < r0 + CS_ROWS && r < E; r += 8) acc += __ldg(T + r * ld + k);
  red[warp][lane] = acc;
  __syncthreads();
  if (warp == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][lane];
    if (k < K) partial[(int64_t)blockIdx.y * Kpad + k] = t;
  }
}
__global__ void __launch_bounds__(256)
colsum_final_kernel(const float* __restrict__ partial, int nchunks, int K, int Kpad, float* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  float t = 0.f;
  for (int c = 0; c < nchunks; ++c) t += partial[(int64_t)c * Kpad + k];
  out[k] = t;
}
// zsum[i] = Q[i, :K] . cs   (one warp per row)
__global__ void __launch_bounds__(256)
rowdot_kernel(const float* __restrict__ Q, int64_t ldq, int64_t n, int K, const float* __restrict__ cs,
              float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= n) return;
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) acc = fmaf(Q[i * ldq + k], cs[k], acc);
  acc = wsum(acc);
  if (lane == 0) out[i] = acc;
}

}  // namespace

int launch_csr_expand(const int64_t* off, const int64_t* col, int64_t n, int64_t nnz, int extra, const int64_t* q_idx,
                      const int64_t* p_idx, int64_t* qsel, int64_t* psel, int64_t* esel, cudaStream_t st) {
  if (n == 0) return 0;
  csr_expand_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(off, col, n, nnz, extra, q_idx, p_idx, qsel, psel, esel);
  B2K_LAUNCH_CHECK("csr_expand_kernel");
  return 0;
}

int launch_csr_rows(int loss_kind, const int64_t* off, const int64_t* col, const float* zpos, int64_t n, int64_t nnz,
                    const float* fused, const float* zsum, int zsum_chunks, float a, float b, float E, float offset,
                    float* row_loss, cudaStream_t st) {
  if (n == 0) return 0;
  const unsigned blocks = (unsigned)((n + 7) / 8);
  if (loss_kind == B200KGE_LOSS_BCE)
    csr_rows_kernel<B200KGE_LOSS_BCE><<<blocks, 256, 0, st>>>(off, col, zpos, n, nnz, fused, zsum, zsum_chunks, a, b, E,
                                                              offset, row_loss);
  else
    csr_rows_kernel<B200KGE_LOSS_KL><<<blocks, 256, 0, st>>>(off, col, zpos, n, nnz, fused, zsum, zsum_chunks, a, b, E,
                                                             offset, row_loss);
  B2K_LAUNCH_CHECK("csr_rows_kernel");
  return 0;
}

int launch_rows_sum(const float* rows, int64_t n, float scale, float* out, cudaStream_t st) {
  rows_sum_kernel<<<1, 256, 0, st>>>(rows, n, scale, out);
  B2K_LAUNCH_CHECK("rows_sum_kernel");
  return 0;
}

// zsum[i] = sum_j Q_i . T_j = Q_i . colsum(T); scratch: (ceil(E / 1024) + 1) * round_up(K, 32) floats
int launch_row_score_sums(const float* Q, int64_t ldq, int64_t n, const float* T, int64_t ldt, int64_t E, int K,
                          float* scratch, float* zsum, cudaStream_t st) {
  if (n == 0 || E == 0) return 0;
  const int Kpad = (K + 31) / 32 * 32;
  const int nch = (int)((E + CS_ROWS - 1) / CS_ROWS);
  float* partial = scratch;
  float* cs = scratch + (size_t)nch * Kpad;
  dim3 grid((unsigned)(Kpad / 32), (unsigned)nch);
  colsum_partial_kernel<<<grid, 256, 0, st>>>(T, ldt, E, K, partial, Kpad);
  B2K_LAUNCH_CHECK("colsum_partial_kernel");
  colsum_final_kernel<<<(unsigned)((K + 255) / 256), 256, 0, st>>>(partial, nch, K, Kpad, cs);
  B2K_LAUNCH_CHECK("colsum_final_kernel");
  rowdot_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(Q, ldq, n, K, cs, zsum);
  B2K_LAUNCH_CHECK("rowdot_kernel");
  return 0;
}

}  // namespace b200kge
