// dropout.cu — embedding dropout of LookupEmbedder._postprocess (lookup_embedder.py:96-105) for the 1vsAll and KvsAll
// training steps, without storing a mask.
//
// Element e = row * dim + k of draw `stream` is a pure function of (seed, call, stream, row, k): Philox4x32-10 with key
// `seed` and counter ((stream << 46) | (e >> 2), call) gives four words, word e & 3 belongs to e, and the element is
// kept iff that word is below floor((1 - p) * 2^32).  The forward gathers masked copies of the operands; the backward
// regenerates the same words from the same key to mask the gradients.  One thread serves one Philox block, i.e. four
// consecutive elements (they may straddle a row boundary when dim % 4 != 0).
#include "fold.cuh"
#include "philox.cuh"

namespace b200kge {

namespace {

// Calls f(local row, column, keep) for the elements of Philox block `blockIdx.x * blockDim.x + threadIdx.x` (counted
// from the first block touching the draw) that lie inside rows [row_base, row_base + rows) x [0, dim).
template <class F>
__device__ __forceinline__ void for_mask_block(const DropMask& m, int64_t rows, int dim, F&& f) {
  const uint64_t e_lo = (uint64_t)m.row_base * (uint64_t)dim, e_hi = e_lo + (uint64_t)rows * (uint64_t)dim;
  const uint64_t g = (e_lo >> 2) + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint64_t e = g << 2;
  if (e >= e_hi) return;
  uint32_t w[4] = {(uint32_t)(((uint64_t)m.stream << 46) | g), (uint32_t)((((uint64_t)m.stream << 46) | g) >> 32),
                   (uint32_t)m.call, (uint32_t)(m.call >> 32)};
  philox4x32_10(w, m.seed);
  int64_t r = (int64_t)(e / (uint64_t)dim);
  int k = (int)(e - (uint64_t)r * dim);
#pragma unroll
  for (int j = 0; j < 4; ++j, ++e) {
    if (e >= e_lo && e < e_hi) f(r - m.row_base, k, (uint64_t)w[j] < m.thresh);
    if (++k == dim) { k = 0; ++r; }
  }
}

inline unsigned mask_grid(const DropMask& m, int64_t rows, int dim) {
  const uint64_t e_lo = (uint64_t)m.row_base * (uint64_t)dim, e_hi = e_lo + (uint64_t)rows * (uint64_t)dim;
  const uint64_t blocks = ((e_hi - 1) >> 2) - (e_lo >> 2) + 1;
  return (unsigned)((blocks + 255) / 256);
}

__global__ void __launch_bounds__(256)
dropout_mask_kernel(DropMask m, int64_t rows, int dim, uint8_t* __restrict__ out) {
  for_mask_block(m, rows, dim, [&](int64_t i, int k, bool keep) { out[i * dim + k] = keep ? 1 : 0; });
}

__global__ void __launch_bounds__(256)
dropout_gather_kernel(DropMask m, Rows src, float* __restrict__ dst, int64_t ldd) {
  for_mask_block(m, src.rows, src.dim, [&](int64_t i, int k, bool keep) {
    dst[i * ldd + k] = keep ? src.row(i)[k] * m.scale : 0.f;
  });
}

__global__ void __launch_bounds__(256)
dropout_add_cols_kernel(DropMask m, const float* __restrict__ src, int64_t lds, int64_t rows, int dim, int c0, int c1,
                        float* __restrict__ dst, int64_t ldd) {
  for_mask_block(m, rows, dim, [&](int64_t r, int k, bool keep) {
    if (keep && k >= c0 && k < c1) dst[r * ldd + k] += src[r * lds + k] * m.scale;
  });
}

__global__ void __launch_bounds__(256)
dropout_scatter_kernel(DropMask m, const float* __restrict__ src, int64_t lds, int64_t rows, int dim,
                       const int64_t* __restrict__ idx, float* __restrict__ dst, int64_t ldd) {
  for_mask_block(m, rows, dim, [&](int64_t i, int k, bool keep) {
    if (keep) atomicAdd(dst + idx[i] * ldd + k, src[i * lds + k] * m.scale);
  });
}

__global__ void identity_triples_kernel(int64_t n, int64_t* __restrict__ tri) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) { tri[3 * i] = i; tri[3 * i + 1] = i; tri[3 * i + 2] = i; }
}

}  // namespace

int launch_dropout_mask(const DropMask& m, int64_t rows, int dim, uint8_t* out, cudaStream_t st) {
  if (rows <= 0 || dim <= 0) return 0;
  dropout_mask_kernel<<<mask_grid(m, rows, dim), 256, 0, st>>>(m, rows, dim, out);
  B2K_LAUNCH_CHECK("dropout_mask_kernel");
  return 0;
}

int launch_dropout_gather(const DropMask& m, const Rows& src, float* dst, int64_t ldd, cudaStream_t st) {
  if (src.rows <= 0 || src.dim <= 0) return 0;
  dropout_gather_kernel<<<mask_grid(m, src.rows, src.dim), 256, 0, st>>>(m, src, dst, ldd);
  B2K_LAUNCH_CHECK("dropout_gather_kernel");
  return 0;
}

int launch_dropout_add_cols(const DropMask& m, const float* src, int64_t lds, int64_t rows, int dim, int c0, int c1,
                            float* dst, int64_t ldd, cudaStream_t st) {
  if (rows <= 0 || dim <= 0 || c1 <= c0) return 0;
  dropout_add_cols_kernel<<<mask_grid(m, rows, dim), 256, 0, st>>>(m, src, lds, rows, dim, c0, c1, dst, ldd);
  B2K_LAUNCH_CHECK("dropout_add_cols_kernel");
  return 0;
}

int launch_dropout_scatter(const DropMask& m, const float* src, int64_t lds, int64_t rows, int dim, const int64_t* idx,
                           float* dst, int64_t ldd, cudaStream_t st) {
  if (rows <= 0 || dim <= 0) return 0;
  dropout_scatter_kernel<<<mask_grid(m, rows, dim), 256, 0, st>>>(m, src, lds, rows, dim, idx, dst, ldd);
  B2K_LAUNCH_CHECK("dropout_scatter_kernel");
  return 0;
}

int launch_identity_triples(int64_t n, int64_t* tri, cudaStream_t st) {
  if (n <= 0) return 0;
  identity_triples_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, tri);
  B2K_LAUNCH_CHECK("identity_triples_kernel");
  return 0;
}

}  // namespace b200kge
