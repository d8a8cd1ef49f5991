// grad.cu — SURVEY §8 f-1: device pieces of the backward of the fused 1vsAll step for the dot family, of the
// negative-sampling step, and the penalty / normalisation row kernels.  Checked on the GPU by
// tests/test_gpu_backward.py and tests/test_gpu_jobs.py::test_training_epoch_native_backward; the math is pinned on
// the CPU (oracle/kge_fold.py against autograd and against gradients of the live reference,
// tests/test_fold_algebra.py), the kernels below transcribe it.
//
//   z  = Q T^T                       recomputed with the validated scorer (plain-store epilogue)
//   G  = sigmoid(z + off) - y        grad_planes_kernel: written ONCE as fp16 hi/lo planes in both layouts,
//                                    G [nq, Ep] and G^T [E, Np] (scale 2^14; 1/n rides in the row scale)
//   dT = G^T Q   [E, K]              pre-split fp16 GEMM (pairwise_tc.cu, store epilogue) on G^T and Q^T planes
//   dQ = G  T    [nq, K]             same on G and T^T planes
//   (da, dp) = unfold(a, p, dQ)      unfold_kernel: row-wise vector-Jacobian products of the relation fold,
//                                    atomically added into the entity / relation gradient tables
// This version trades HBM traffic for simplicity (scores and both G layouts are materialised, operands are
// transposed through HBM).  Both GEMMs run split-K (512-element segments added in fp32, pairwise_tc.cu): the
// tensor core's fp32 accumulator error grows with the reduction length, and dQ = G T reduces over all E entities.
#include <cuda_fp16.h>
#include "dropmask.cuh"
#include "fold.cuh"
#include "tc_common.cuh"

namespace b200kge {

namespace {

// ---------------------------------------------------------------------------------------------
// dst[c, r] = src[r, c]   (fp32, 32x32 tiles through shared memory); dst columns [R, ldd) are zeroed
__global__ void __launch_bounds__(256)
transpose_kernel(const float* __restrict__ src, int64_t lds, int64_t R, int64_t C, float* __restrict__ dst,
                 int64_t ldd) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;       // 32 x 8
  const int64_t r0 = (int64_t)blockIdx.x * 32, c0 = (int64_t)blockIdx.y * 32;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int64_t r = r0 + ty + 8 * k, c = c0 + tx;
    tile[ty + 8 * k][tx] = (r < R && c < C) ? __ldg(src + r * lds + c) : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int64_t c = c0 + ty + 8 * k, r = r0 + tx;
    if (c < C && r < ldd) dst[c * ldd + r] = tile[tx][ty + 8 * k];   // r >= R carries the zeros loaded above
  }
}

__device__ __forceinline__ void split_store(__half* __restrict__ hi, __half* __restrict__ lo, int64_t pos, float g) {
  const float s = g * 16384.f;
  const __half h = __float2half_rn(s);
  hi[pos] = h;
  lo[pos] = __float2half_rn(s - __half2float(h));
}

// KL needs the row's log-sum-exp and label mass first: row_stat[2i] = logsumexp_j z_ij, row_stat[2i+1] = sum_j y_ij
// (loss.py:198-213).  One block per row.
__global__ void __launch_bounds__(256)
row_lse_kernel(const float* __restrict__ z, int64_t ldz, int64_t E, const int64_t* __restrict__ label_idx,
               const float* __restrict__ label_dense, int64_t ldl, float* __restrict__ row_stat) {
  __shared__ float red[3][8];
  const int64_t i = blockIdx.x;
  const float* __restrict__ zr = z + i * ldz;
  float mx = -INFINITY, ys = 0.f;
  for (int64_t e = threadIdx.x; e < E; e += blockDim.x) {
    mx = fmaxf(mx, zr[e]);
    if (label_dense) ys += label_dense[i * ldl + e];
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    ys += __shfl_xor_sync(0xffffffffu, ys, o);
  }
  if (lane == 0) { red[0][warp] = mx; red[1][warp] = ys; }
  __syncthreads();
  mx = red[0][0]; ys = red[1][0];
#pragma unroll
  for (int w = 1; w < 8; ++w) { mx = fmaxf(mx, red[0][w]); ys += red[1][w]; }
  float se = 0.f;
  for (int64_t e = threadIdx.x; e < E; e += blockDim.x) se += expf(zr[e] - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
  if (lane == 0) red[2][warp] = se;
  __syncthreads();
  if (threadIdx.x == 0) {
    se = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) se += red[2][w];
    row_stat[2 * i] = mx + logf(se);
    row_stat[2 * i + 1] = label_idx ? ((label_idx[i] >= 0 && label_idx[i] < E) ? 1.f : 0.f) : ys;
  }
}

// G = dL/dz * n as fp16 hi/lo planes, row-major [nq, Ep] and transposed [E, Np]; pads zeroed.
//   BCE (row_stat == nullptr): G = sigmoid(z + off) - y          KL: G = w * exp(z - lse) - y / yc,  yc = max(sum y, 1e-12), w = sum y / yc
// grid = (Ep/64, Np/64), block = 32 x 8: 64 x 64 tiles, every thread two neighbouring elements per step so both layouts
// are written with 4-byte half2 stores (the 32 x 32 / 2-byte version: 125 us at [2048, 14 541], 2.9 TB/s).
__device__ __forceinline__ void split_store2(__half* __restrict__ hi, __half* __restrict__ lo, int64_t pos, float g0, float g1) {
  const float s0 = g0 * 16384.f, s1 = g1 * 16384.f;
  const __half h0 = __float2half_rn(s0), h1 = __float2half_rn(s1);
  *reinterpret_cast<__half2*>(hi + pos) = __halves2half2(h0, h1);                       // pos even, planes 256-byte aligned
  *reinterpret_cast<__half2*>(lo + pos) = __halves2half2(__float2half_rn(s0 - __half2float(h0)),
                                                         __float2half_rn(s1 - __half2float(h1)));
}

__global__ void __launch_bounds__(256)
grad_planes_kernel(const float* __restrict__ z, int64_t ldz, int64_t nq, int64_t E,
                   const int64_t* __restrict__ label_idx, const float* __restrict__ label_dense, int64_t ldl,
                   const float* __restrict__ row_stat, float y_base,
                   float offset, float inv_n, __half* __restrict__ g_hi, __half* __restrict__ g_lo, int64_t Ep,
                   __half* __restrict__ gt_hi, __half* __restrict__ gt_lo, int64_t Np,
                   float* __restrict__ g_scale, float* __restrict__ gt_scale) {
  __shared__ float tile[64][65];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int64_t e0 = (int64_t)blockIdx.x * 64, i0 = (int64_t)blockIdx.y * 64;
  const float inv = inv_n * (1.0f / 16384.f);
  // The first version spent ~110 instructions per element (ncu: 71 % issue utilisation, DRAM at 2.4 TB/s): 64-bit index
  // arithmetic and label compares per element, IEEE division and expf.  Row bases and the label's position inside the
  // tile are now per-row values, sigmoid / softmax use the fast exponential and reciprocal (2 ulp: far below the fp16
  // hi+lo representation error of G).
  const int ecols = (int)min((int64_t)64, E - e0);                     // valid columns of this tile
  const bool vec2 = ((ldz & 1) == 0) && ((reinterpret_cast<uintptr_t>(z) & 7) == 0);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int64_t i = i0 + ty + 8 * k;
    float g[2] = {0.f, 0.f};
    if (i < nq) {
      float lse = 0.f, w = 1.f, inv_yc = 1.f;
      if (row_stat) {
        const float ys = row_stat[2 * i + 1], yc = fmaxf(ys, 1e-12f);      // labels are normalised by their row sum first (loss.py:209-213)
        lse = row_stat[2 * i]; inv_yc = 1.0f / yc; w = ys * inv_yc;
      }
      int lab = -1;                                                          // label column relative to the tile
      if (label_idx) { const int64_t l = label_idx[i] - e0; lab = (l >= 0 && l < 64) ? (int)l : -1; }
      const float* __restrict__ zr = z + i * ldz + e0;
      const float* __restrict__ yr = label_dense ? label_dense + i * ldl + e0 : nullptr;
      const int c = 2 * tx;
      float x[2] = {0.f, 0.f};
      if (vec2 && c + 1 < ecols) { const float2 v = __ldg(reinterpret_cast<const float2*>(zr + c)); x[0] = v.x; x[1] = v.y; }
      else { if (c < ecols) x[0] = __ldg(zr + c); if (c + 1 < ecols) x[1] = __ldg(zr + c + 1); }
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        if (c + j < ecols) {
          const float xv = x[j] + offset;
          const float y = label_idx ? ((lab == c + j) ? 1.f : 0.f) : (yr ? __ldg(yr + c + j) : y_base);   // CSR labels: fixed up below
          g[j] = row_stat ? w * __expf(xv - lse) - y * inv_yc : __fdividef(1.0f, 1.0f + __expf(-xv)) - y;
        }
      }
      split_store2(g_hi, g_lo, i * Ep + e0 + c, g[0], g[1]);          // e < Ep by construction of the grid
      if (blockIdx.x == 0 && tx == 0) g_scale[i] = inv;
    }
    tile[ty + 8 * k][2 * tx] = g[0];
    tile[ty + 8 * k][2 * tx + 1] = g[1];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int el = ty + 8 * k;
    const int64_t e = e0 + el;
    if (e < E) {
      split_store2(gt_hi, gt_lo, e * Np + i0 + 2 * tx, tile[2 * tx][el], tile[2 * tx + 1][el]);   // i < Np by construction
      if (blockIdx.y == 0 && tx == 0) gt_scale[e] = inv;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// CSR multi-hot labels (train_KvsAll.py:242-266): y_ij = a * count_ij + b.  The planes are first written with y = b
// everywhere (grad_planes_kernel, y_base), then the nnz listed entries are recomputed with their labels and patched
// into both layouts — no [n, E] label matrix.  KL needs the row label mass a * nnz_i + b * E in row_stat first.
__global__ void __launch_bounds__(256)
csr_row_mass_kernel(const int64_t* __restrict__ off, int64_t n, float a, float b, float E, float* __restrict__ row_stat) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) row_stat[2 * i + 1] = a * (float)(off[i + 1] - off[i]) + b * E;
}

__global__ void __launch_bounds__(256)
csr_grad_fix_kernel(const float* __restrict__ z, int64_t ldz, int64_t n, const int64_t* __restrict__ off,
                    const int64_t* __restrict__ col, const float* __restrict__ row_stat, float a, float b, float offset,
                    __half* __restrict__ g_hi, __half* __restrict__ g_lo, int64_t Ep, __half* __restrict__ gt_hi,
                    __half* __restrict__ gt_lo, int64_t Np) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);      // one warp per row
  if (i >= n) return;
  const int64_t t0 = off[i], t1 = off[i + 1];
  for (int64_t t = t0 + lane; t < t1; t += 32) {
    if (t > t0 && col[t] == col[t - 1]) continue;             // a run of equal columns is handled by its first entry
    int64_t c = 1;
    while (t + c < t1 && col[t + c] == col[t]) ++c;
    const int64_t e = col[t];
    const float y = a * (float)c + b;
    const float x = z[i * ldz + e] + offset;
    float g;
    if (row_stat) {
      const float ys = row_stat[2 * i + 1], yc = fmaxf(ys, 1e-12f);
      g = (ys / yc) * expf(x - row_stat[2 * i]) - y / yc;
    } else {
      g = 1.0f / (1.0f + expf(-x)) - y;
    }
    split_store(g_hi, g_lo, i * Ep + e, g);
    split_store(gt_hi, gt_lo, e * Np + i, g);
  }
}

// ---------------------------------------------------------------------------------------------
// Row-wise unfold: block b handles query row b.  dir < 0: rows [0,n) are sp_ (a = subject), rows [n,2n) are
// _po (a = object) — the stacked layout of prep_1vsall_kernel; dir = 0 / 1: all rows sp_ / _po.  RECIP (dir < 0): the
// reciprocal layout, rows [n,2n) are sp_ with a = object and relation row p + num_rel.
// MAP (unfold_rows_kernel): the gradient rows are row-mapped, da = d_ent + pe[a] * lde and dp = d_rel + pr[p] * ldr
template <int MODEL, bool RECIP, bool MAP>
__device__ __forceinline__ void unfold_body(const Rows& ent, const Rows& rel, const int64_t* __restrict__ tri, int64_t n,
                                            int dir, const float* __restrict__ dQ, int64_t ldq, float* __restrict__ d_ent,
                                            int64_t lde, float* __restrict__ d_rel, int64_t ldr, int64_t num_rel,
                                            const int32_t* __restrict__ pe, const int32_t* __restrict__ pr) {
  const int64_t b = blockIdx.x;
  const bool second = dir < 0 && b >= n;
  const bool sp = RECIP || (dir < 0 ? (b < n) : (dir == 0));
  const int64_t i = second ? b - n : b;
  const int64_t si = tri[3 * i], oi = tri[3 * i + 2];
  const int64_t pi = RECIP && second ? tri[3 * i + 1] + num_rel : tri[3 * i + 1];
  const int64_t ai = RECIP ? (second ? oi : si) : (sp ? si : oi);
  const float* __restrict__ a = ent.base + ai * ent.ld;
  const float* __restrict__ p = rel.base + pi * rel.ld;
  const float* __restrict__ g = dQ + b * ldq;
  float* __restrict__ da = d_ent + (MAP ? (int64_t)pe[ai] : ai) * lde;
  float* __restrict__ dp = d_rel + (MAP ? (int64_t)pr[pi] : pi) * ldr;
  const int D = ent.dim, h = D >> 1;

  if constexpr (MODEL == B200KGE_RESCAL) {
    // sp_: q = a^T M  => da_i = sum_j M[i,j] g_j,  dM[i,j] = a_i g_j
    // _po: q = M a    => da_j = sum_i g_i M[i,j],  dM[i,j] = g_i a_j
    extern __shared__ float sh[];
    float* sa = sh;
    float* sg = sh + D;
    for (int k = threadIdx.x; k < D; k += blockDim.x) { sa[k] = a[k]; sg[k] = g[k]; }
    __syncthreads();
    if (sp) {
      const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
      for (int r = warp; r < D; r += nw) {
        float acc = 0.f;
        for (int j = lane; j < D; j += 32) acc = fmaf(p[(int64_t)r * D + j], sg[j], acc);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
        if (lane == 0) atomicAdd(da + r, acc);
      }
    } else {
      for (int j = threadIdx.x; j < D; j += blockDim.x) {
        float acc = 0.f;
        for (int r = 0; r < D; ++r) acc = fmaf(sg[r], p[(int64_t)r * D + j], acc);
        atomicAdd(da + j, acc);
      }
    }
    for (int idx = threadIdx.x; idx < D * D; idx += blockDim.x) {
      const int r = idx / D, j = idx - r * D;
      atomicAdd(dp + idx, sp ? sa[r] * sg[j] : sg[r] * sa[j]);
    }
  } else if constexpr (MODEL == B200KGE_COMPLEX) {
    for (int k = threadIdx.x; k < h; k += blockDim.x) {
      const float a_re = a[k], a_im = a[k + h], p_re = p[k], p_im = p[k + h], g_re = g[k], g_im = g[k + h];
      if (sp) {   // Q_re = a_re p_re - a_im p_im ; Q_im = a_im p_re + a_re p_im
        atomicAdd(da + k, g_re * p_re + g_im * p_im);
        atomicAdd(da + k + h, -g_re * p_im + g_im * p_re);
        atomicAdd(dp + k, g_re * a_re + g_im * a_im);
        atomicAdd(dp + k + h, -g_re * a_im + g_im * a_re);
      } else {    // Q_re = p_re a_re + p_im a_im ; Q_im = p_re a_im - p_im a_re
        atomicAdd(da + k, g_re * p_re - g_im * p_im);
        atomicAdd(da + k + h, g_re * p_im + g_im * p_re);
        atomicAdd(dp + k, g_re * a_re + g_im * a_im);
        atomicAdd(dp + k + h, g_re * a_im - g_im * a_re);
      }
    }
  } else if constexpr (MODEL == B200KGE_DISTMULT) {
    for (int k = threadIdx.x; k < D; k += blockDim.x) {
      atomicAdd(da + k, g[k] * p[k]);
      atomicAdd(dp + k, g[k] * a[k]);
    }
  } else if constexpr (MODEL == B200KGE_SIMPLE) {
    for (int k = threadIdx.x; k < h; k += blockDim.x) {
      const float a_h = a[k], a_t = a[k + h], p_f = p[k], p_b = p[k + h];
      const float g0 = 0.5f * g[k], g1 = 0.5f * g[k + h];
      if (sp) {   // Q = 1/2 [a_t p_b | a_h p_f]
        atomicAdd(da + k, g1 * p_f);
        atomicAdd(da + k + h, g0 * p_b);
        atomicAdd(dp + k, g1 * a_h);
        atomicAdd(dp + k + h, g0 * a_t);
      } else {    // Q = 1/2 [a_t p_f | a_h p_b]
        atomicAdd(da + k, g1 * p_b);
        atomicAdd(da + k + h, g0 * p_f);
        atomicAdd(dp + k, g0 * a_t);
        atomicAdd(dp + k + h, g1 * a_h);
      }
    }
  } else {  // CP: sp_ Q = a[:h] p (vs cand[:, h:]);  _po Q = a[h:] p (vs cand[:, :h])
    const int ao = sp ? 0 : h;
    for (int k = threadIdx.x; k < h; k += blockDim.x) {
      atomicAdd(da + ao + k, g[k] * p[k]);
      atomicAdd(dp + k, g[k] * a[ao + k]);
    }
  }
}

template <int MODEL, bool RECIP>
__global__ void __launch_bounds__(128)
unfold_kernel(Rows ent, Rows rel, const int64_t* __restrict__ tri, int64_t n, int dir,
              const float* __restrict__ dQ, int64_t ldq, float* __restrict__ d_ent, int64_t lde,
              float* __restrict__ d_rel, int64_t ldr, int64_t num_rel) {
  unfold_body<MODEL, RECIP, false>(ent, rel, tri, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, num_rel, nullptr, nullptr);
}

template <int MODEL>
__global__ void __launch_bounds__(128)
unfold_rows_kernel(Rows ent, Rows rel, const int64_t* __restrict__ tri, int64_t n, int dir,
                   const float* __restrict__ dQ, int64_t ldq, float* __restrict__ d_ent, int64_t lde,
                   float* __restrict__ d_rel, int64_t ldr, const int32_t* __restrict__ pe,
                   const int32_t* __restrict__ pr) {
  unfold_body<MODEL, false, true>(ent, rel, tri, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, 0, pe, pr);
}

// ---------------------------------------------------------------------------------------------
// Lp / N3 penalty of embedding rows (lookup_embedder.py:123-177): sum over the selected rows of
// count_r * sum_k |x_rk|^p  (N3 in complex space: x -> sqrt(re^2 + im^2 + 1e-14), p = 3), times scale.
// One block per PEN_ROWS rows, per-block partial sums, last block (ticket) adds them in block order.
constexpr int PEN_ROWS = 8;

__device__ __forceinline__ float pow_p(float a, float p, int ip) {
  if (ip == 1) return a;
  if (ip == 2) return a * a;
  if (ip == 3) return a * a * a;
  return powf(a, p);
}

__global__ void __launch_bounds__(256)
penalty_kernel(Rows tab, const float* __restrict__ counts, float p, int complex_abs, float scale,
               float* __restrict__ partial, unsigned int* __restrict__ ticket, float* __restrict__ out) {
  __shared__ float red[8];
  __shared__ bool last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * PEN_ROWS + warp;
  const int ip = (p == 1.f) ? 1 : (p == 2.f) ? 2 : (p == 3.f) ? 3 : 0;
  float acc = 0.f;
  if (r < tab.rows) {
    const float* __restrict__ x = tab.row(r);
    if (complex_abs) {
      const int h = tab.dim >> 1;
      for (int k = lane; k < h; k += 32) {
        const float re = x[k], im = x[k + h];
        acc += pow_p(sqrtf(re * re + im * im + 1e-14f), p, ip);
      }
    } else {
      for (int k = lane; k < tab.dim; k += 32) acc += pow_p(fabsf(x[k]), p, ip);
    }
    if (counts) acc *= counts[r];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < PEN_ROWS; ++w) t += red[w];
    partial[blockIdx.x] = t;
    __threadfence();
    last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (last) {
    float t = 0.f;
    for (unsigned b = threadIdx.x; b < gridDim.x; b += blockDim.x) t += __ldcg(partial + b);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    __syncthreads();
    if (lane == 0) red[warp] = t;
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) tot += red[w];
      *out = tot * scale;
      *ticket = 0u;
    }
  }
}

// rows scaled to unit Lp norm in place (F.normalize, eps = 1e-12; lookup_embedder.py:64-69). One warp per row.
__global__ void __launch_bounds__(256)
normalize_rows_kernel(float* __restrict__ w, int64_t ld, int64_t rows, int dim, float p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * 8 + warp;
  if (r >= rows) return;
  float* __restrict__ x = w + r * ld;
  const int ip = (p == 1.f) ? 1 : (p == 2.f) ? 2 : (p == 3.f) ? 3 : 0;
  float acc = 0.f;
  for (int k = lane; k < dim; k += 32) acc += pow_p(fabsf(x[k]), p, ip);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  const float nrm = (ip == 1) ? acc : (ip == 2) ? sqrtf(acc) : powf(acc, 1.0f / p);
  const float inv = 1.0f / fmaxf(nrm, 1e-12f);
  for (int k = lane; k < dim; k += 32) x[k] *= inv;
}

// ---------------------------------------------------------------------------------------------
// Backward of one negative-sampling slot with BCE (train_negative_sampling.py:113-164), S and O slots: block
// (i, y) folds the positive triple's (other entity, relation) into q once — as ns_kernel does — and walks 64
// of the row's 1 + K columns (column 0 = the positive, label 1; columns 1..K = sampled ids, label 0): per
// column it recomputes z = pair(q, t), g = (sigmoid(z + off) - y) / batch, adds g * dpair/dt into the sampled
// row of d_ent (atomics: the scatter is inherent) and accumulates g * dpair/dq per lane; the block's dq is
// added into dQ[i, :], which unfold_kernel then pushes through the relation fold.  With G given (any other loss:
// G = dL/dz * scale from ns_loss_kernel) g = G[i, c] replaces the BCE formula; the rest is unchanged.
constexpr int NSB_WARPS = 4, NSB_PER_BLOCK = 64, NSB_MAXK = 1024;   // lane-local dq: K / 32 <= 32 registers

// MASK (ns_backward_kernel_masked, the `batch` negatives with dropout): `fa` / `rel` hold masked copies of the fixed rows
// under identity triples, column 0 (the positive, drawn on other streams) is skipped, and every sampled row is masked
// by its entity id (draw tm) where it is loaded and where its gradient is scattered.
// MAP (ns_backward_rows_kernel, ns_backward_rows_kernel_masked): entity e's gradient row is d_ent + pe[e] * lde.
template <int MODEL, bool MASK, bool MAP>
__device__ __forceinline__ void ns_backward_body(const Rows& fa, const Rows& ent, const Rows& rel, const int64_t* __restrict__ tri,
                                                 int sp, const int64_t* __restrict__ neg, int64_t Kneg, const Folded& f,
                                                 float l_norm, float offset, float inv_batch, const float* __restrict__ G,
                                                 int64_t ldg, float* __restrict__ d_ent, int64_t lde, float* __restrict__ dQ,
                                                 int64_t ldq, const DropMask& tm, const int32_t* __restrict__ pe) {
  extern __shared__ __align__(16) float sh[];  // q[K] | dq[K] (+ entity row for RESCAL)
  const int64_t i = blockIdx.x;
  const int64_t si = tri[3 * i], pi = tri[3 * i + 1], oi = tri[3 * i + 2];
  const int D = ent.dim, h = D >> 1, K = f.K;
  const float* __restrict__ a = fa.base + (sp ? si : oi) * fa.ld;
  const float* __restrict__ p = rel.base + pi * rel.ld;
  float* q = sh;
  float* sdq = sh + K;
  if constexpr (MODEL == B200KGE_RESCAL) {
    float* sa = sh + 2 * K;
    for (int k = threadIdx.x; k < D; k += blockDim.x) sa[k] = a[k];
    __syncthreads();
    fold_rescal_block(sp != 0, sa, p, D, [&](int k, float v) { q[k] = v; });
  } else {
    for (int k = threadIdx.x; k < K; k += blockDim.x) q[k] = fold_element<MODEL>(sp != 0, a, p, k, h);
  }
  for (int k = threadIdx.x; k < K; k += blockDim.x) sdq[k] = 0.f;
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t c0 = (int64_t)blockIdx.y * NSB_PER_BLOCK;
  const int hk = K >> 1;
  float dq[NSB_MAXK / 32];
#pragma unroll
  for (int j = 0; j < NSB_MAXK / 32; ++j) dq[j] = 0.f;
  for (int64_t c = c0 + warp; c < c0 + NSB_PER_BLOCK && c <= Kneg; c += NSB_WARPS) {
    if constexpr (MASK) { if (c == 0) continue; }
    // column 0 is the positive triple (its open slot holds the true entity), columns 1..K the samples
    const int64_t e = (c == 0) ? (sp ? oi : si) : neg[i * Kneg + (c - 1)];
    const float y = (c == 0) ? 1.f : 0.f;
    const float* __restrict__ t = ent.base + e * ent.ld + f.col_off;
    float* __restrict__ dt = d_ent + (MAP ? (int64_t)pe[e] : e) * lde + f.col_off;
    // T(k): element k of the sampled row, DT_ADD(k, v): its gradient — through the entity's mask under MASK
#define T(k) (MASK ? t[k] * drop_mask1(tm, (uint64_t)e, D, f.col_off + (k)) : t[k])
#define DT_ADD(k, v)                                                                   \
    do {                                                                               \
      if constexpr (MASK) {                                                            \
        const float m_ = drop_mask1(tm, (uint64_t)e, D, f.col_off + (k));              \
        if (m_ != 0.f) atomicAdd(dt + (k), (v) * m_);                                  \
      } else {                                                                         \
        atomicAdd(dt + (k), (v));                                                      \
      }                                                                                \
    } while (0)
    float acc = 0.f;
    if (f.pair_op == PAIR_DOT) {
      for (int k = lane; k < K; k += 32) acc = fmaf(q[k], T(k), acc);
    } else if (f.pair_op == PAIR_L1) {
      for (int k = lane; k < K; k += 32) acc += fabsf(q[k] - T(k));
    } else if (f.pair_op == PAIR_L2) {
      for (int k = lane; k < K; k += 32) { const float d = q[k] - T(k); acc = fmaf(d, d, acc); }
    } else {   // PAIR_CMOD_L1
      for (int k = lane; k < hk; k += 32) {
        const float d_re = q[k] - T(k), d_im = q[k + hk] - T(k + hk);
        acc += sqrtf(fmaf(d_im, d_im, d_re * d_re));
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    float z = acc, nrm = 1.f;
    if (f.pair_op == PAIR_L1 || f.pair_op == PAIR_CMOD_L1) z = -acc;
    else if (f.pair_op == PAIR_L2) { nrm = sqrtf(acc); z = -nrm; }
    const float g = G ? G[i * ldg + c] : (1.0f / (1.0f + expf(-(z + offset))) - y) * inv_batch;
    if (f.pair_op == PAIR_DOT) {
      for (int k = lane, j = 0; k < K; k += 32, ++j) {
        dq[j] = fmaf(g, T(k), dq[j]);
        DT_ADD(k, g * q[k]);
      }
    } else if (f.pair_op == PAIR_L1) {          // z = -sum |q - t|
      for (int k = lane, j = 0; k < K; k += 32, ++j) {
        const float d = q[k] - T(k);
        const float w = (d > 0.f) ? -g : (d < 0.f ? g : 0.f);
        dq[j] += w;
        DT_ADD(k, -w);
      }
    } else if (f.pair_op == PAIR_L2) {          // z = -||q - t||_2
      const float inv = (nrm > 0.f) ? g / nrm : 0.f;
      for (int k = lane, j = 0; k < K; k += 32, ++j) {
        const float w = -(q[k] - T(k)) * inv;
        dq[j] += w;
        DT_ADD(k, -w);
      }
    } else {                                     // z = -sum_k |q_k - t_k| (complex modulus)
      for (int k = lane, j = 0; k < hk; k += 32, j += 2) {
        const float d_re = q[k] - T(k), d_im = q[k + hk] - T(k + hk);
        const float m = sqrtf(fmaf(d_im, d_im, d_re * d_re));
        const float inv = (m > 0.f) ? g / m : 0.f;
        const float w_re = -d_re * inv, w_im = -d_im * inv;
        dq[j] += w_re;
        dq[j + 1] += w_im;
        DT_ADD(k, -w_re);
        DT_ADD(k + hk, -w_im);
      }
    }
  }
#undef T
#undef DT_ADD
  // block-level dq: lanes own disjoint columns, warps add up through shared memory
  if (f.pair_op == PAIR_CMOD_L1) {
    for (int k = lane, j = 0; k < hk; k += 32, j += 2) { atomicAdd(sdq + k, dq[j]); atomicAdd(sdq + k + hk, dq[j + 1]); }
  } else {
    for (int k = lane, j = 0; k < K; k += 32, ++j) atomicAdd(sdq + k, dq[j]);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x) atomicAdd(dQ + i * ldq + k, sdq[k]);
}

template <int MODEL>
__global__ void __launch_bounds__(NSB_WARPS * 32)
ns_backward_kernel(Rows ent, Rows rel, const int64_t* __restrict__ tri, int sp, const int64_t* __restrict__ neg,
                   int64_t Kneg, Folded f, float l_norm, float offset, float inv_batch, const float* __restrict__ G,
                   int64_t ldg, float* __restrict__ d_ent, int64_t lde, float* __restrict__ dQ, int64_t ldq) {
  ns_backward_body<MODEL, false, false>(ent, ent, rel, tri, sp, neg, Kneg, f, l_norm, offset, inv_batch, G, ldg, d_ent, lde,
                                        dQ, ldq, DropMask{}, nullptr);
}

template <int MODEL>
__global__ void __launch_bounds__(NSB_WARPS * 32)
ns_backward_rows_kernel(Rows ent, Rows rel, const int64_t* __restrict__ tri, int sp, const int64_t* __restrict__ neg,
                        int64_t Kneg, Folded f, float l_norm, float offset, float inv_batch, const float* __restrict__ G,
                        int64_t ldg, float* __restrict__ d_ent, int64_t lde, float* __restrict__ dQ, int64_t ldq,
                        const int32_t* __restrict__ pe) {
  ns_backward_body<MODEL, false, true>(ent, ent, rel, tri, sp, neg, Kneg, f, l_norm, offset, inv_batch, G, ldg, d_ent, lde,
                                       dQ, ldq, DropMask{}, pe);
}

template <int MODEL>
__global__ void __launch_bounds__(NSB_WARPS * 32)
ns_backward_kernel_masked(Rows fa, Rows ent, Rows rel, const int64_t* __restrict__ tri, int sp,
                          const int64_t* __restrict__ neg, int64_t Kneg, Folded f, float l_norm,
                          const float* __restrict__ G, int64_t ldg, float* __restrict__ d_ent, int64_t lde,
                          float* __restrict__ dQ, int64_t ldq, DropMask tm) {
  ns_backward_body<MODEL, true, false>(fa, ent, rel, tri, sp, neg, Kneg, f, l_norm, 0.f, 1.f, G, ldg, d_ent, lde, dQ, ldq,
                                       tm, nullptr);
}

template <int MODEL>
__global__ void __launch_bounds__(NSB_WARPS * 32)
ns_backward_rows_kernel_masked(Rows fa, Rows ent, Rows rel, const int64_t* __restrict__ tri, int sp,
                               const int64_t* __restrict__ neg, int64_t Kneg, Folded f, float l_norm,
                               const float* __restrict__ G, int64_t ldg, float* __restrict__ d_ent, int64_t lde,
                               float* __restrict__ dQ, int64_t ldq, DropMask tm, const int32_t* __restrict__ pe) {
  ns_backward_body<MODEL, true, true>(fa, ent, rel, tri, sp, neg, Kneg, f, l_norm, 0.f, 1.f, G, ldg, d_ent, lde, dQ, ldq,
                                      tm, pe);
}

// unfold for the distance family (TransE: Q = a +- p; RotatE: rotation) — appended to the dot-family unfold
// (RECIP: the reciprocal layout of unfold_kernel)
// (MAP: row-mapped gradient rows, as unfold_body)
template <int MODEL, bool RECIP, bool MAP>
__device__ __forceinline__ void unfold_distance_body(const Rows& ent, const Rows& rel, const int64_t* __restrict__ tri,
                                                     int64_t n, int dir, const float* __restrict__ dQ, int64_t ldq,
                                                     float* __restrict__ d_ent, int64_t lde, float* __restrict__ d_rel,
                                                     int64_t ldr, int64_t num_rel, const int32_t* __restrict__ pe,
                                                     const int32_t* __restrict__ pr) {
  const int64_t b = blockIdx.x;
  const bool second = dir < 0 && b >= n;
  const bool sp = RECIP || (dir < 0 ? (b < n) : (dir == 0));
  const int64_t i = second ? b - n : b;
  const int64_t si = tri[3 * i], oi = tri[3 * i + 2];
  const int64_t pi = RECIP && second ? tri[3 * i + 1] + num_rel : tri[3 * i + 1];
  const int64_t ai = RECIP ? (second ? oi : si) : (sp ? si : oi);
  const float* __restrict__ a = ent.base + ai * ent.ld;
  const float* __restrict__ p = rel.base + pi * rel.ld;
  const float* __restrict__ g = dQ + b * ldq;
  float* __restrict__ da = d_ent + (MAP ? (int64_t)pe[ai] : ai) * lde;
  float* __restrict__ dp = d_rel + (MAP ? (int64_t)pr[pi] : pi) * ldr;
  const int D = ent.dim, h = D >> 1;
  if constexpr (MODEL == B200KGE_TRANSE) {      // Q = a + p | Q = a - p
    for (int k = threadIdx.x; k < D; k += blockDim.x) {
      atomicAdd(da + k, g[k]);
      atomicAdd(dp + k, sp ? g[k] : -g[k]);
    }
  } else {                                        // RotatE, p = phases [h]
    for (int k = threadIdx.x; k < h; k += blockDim.x) {
      float sn, c;
      sincosf(p[k], &sn, &c);
      const float a_re = a[k], a_im = a[k + h], g_re = g[k], g_im = g[k + h];
      if (sp) {   // Q_re = a_re c - a_im s ; Q_im = a_re s + a_im c
        atomicAdd(da + k, g_re * c + g_im * sn);
        atomicAdd(da + k + h, -g_re * sn + g_im * c);
        atomicAdd(dp + k, g_re * (-a_re * sn - a_im * c) + g_im * (a_re * c - a_im * sn));
      } else {    // Q_re = c a_re + s a_im ; Q_im = c a_im - s a_re
        atomicAdd(da + k, g_re * c - g_im * sn);
        atomicAdd(da + k + h, g_re * sn + g_im * c);
        atomicAdd(dp + k, g_re * (-sn * a_re + c * a_im) + g_im * (-sn * a_im - c * a_re));
      }
    }
  }
}

template <int MODEL, bool RECIP>
__global__ void __launch_bounds__(128)
unfold_distance_kernel(Rows ent, Rows rel, const int64_t* __restrict__ tri, int64_t n, int dir,
                       const float* __restrict__ dQ, int64_t ldq, float* __restrict__ d_ent, int64_t lde,
                       float* __restrict__ d_rel, int64_t ldr, int64_t num_rel) {
  unfold_distance_body<MODEL, RECIP, false>(ent, rel, tri, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, num_rel, nullptr,
                                            nullptr);
}

template <int MODEL>
__global__ void __launch_bounds__(128)
unfold_distance_rows_kernel(Rows ent, Rows rel, const int64_t* __restrict__ tri, int64_t n, int dir,
                            const float* __restrict__ dQ, int64_t ldq, float* __restrict__ d_ent, int64_t lde,
                            float* __restrict__ d_rel, int64_t ldr, const int32_t* __restrict__ pe,
                            const int32_t* __restrict__ pr) {
  unfold_distance_body<MODEL, false, true>(ent, rel, tri, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, 0, pe, pr);
}

}  // namespace

int launch_ns_backward(int model, float l_norm, const Rows& ent, const Rows& rel, const int64_t* triples, int slot,
                       const int64_t* neg, int64_t n, int64_t K, float offset, float inv_batch, const float* G,
                       int64_t ldg, float* d_ent, int64_t lde, float* d_rel, int64_t ldr, float* dQ, int64_t ldq,
                       cudaStream_t st, const int32_t* pe, const int32_t* pr) {
  if (n == 0) return 0;
  if (slot != 0 && slot != 2) { set_error("the fused negative-sampling backward covers the S and O slots"); return B200KGE_ERR_UNSUPPORTED; }
  const int sp = (slot == 2) ? 1 : 0;      // O slot: fold (s,p), candidates are objects
  Folded f = folded_problem(model, sp ? B200KGE_SP_ : B200KGE__PO, ent.dim, l_norm);
  if (f.pair_op == PAIR_LP || f.pair_op == PAIR_CMOD_LP) { set_error("the negative-sampling backward covers l_norm 1 and 2 (TransE) / 1 (RotatE)"); return B200KGE_ERR_UNSUPPORTED; }
  if (f.K > NSB_MAXK) { set_error("embedding width %d exceeds the backward kernel's limit of %d", f.K, NSB_MAXK); return B200KGE_ERR_UNSUPPORTED; }
  if (ldq < f.K) { set_error("dQ is narrower than the folded width"); return B200KGE_ERR_INVALID; }
  cudaError_t e = cudaMemsetAsync(dQ, 0, (size_t)n * ldq * 4, st);
  if (e != cudaSuccess) return check_cuda(e, "cudaMemsetAsync(dQ)");
  size_t smem = (size_t)2 * f.K * sizeof(float) + (model == B200KGE_RESCAL ? (size_t)ent.dim * sizeof(float) : 0);
  const int64_t by = (K + 1 + NSB_PER_BLOCK - 1) / NSB_PER_BLOCK;
  if (by > 65535) { set_error("too many negatives per row (%lld)", (long long)K); return B200KGE_ERR_UNSUPPORTED; }
  dim3 grid((unsigned)n, (unsigned)by), block(NSB_WARPS * 32);
#define B2K_NSB(M)                                                                                                             \
  case M:                                                                                                                      \
    if (pe) ns_backward_rows_kernel<M><<<grid, block, smem, st>>>(ent, rel, triples, sp, neg, K, f, l_norm, offset, inv_batch, \
                                                                  G, ldg, d_ent, lde, dQ, ldq, pe);                            \
    else ns_backward_kernel<M><<<grid, block, smem, st>>>(ent, rel, triples, sp, neg, K, f, l_norm, offset, inv_batch, G, ldg, \
                                                          d_ent, lde, dQ, ldq);                                                \
    break;
  switch (model) {
    B2K_NSB(B200KGE_COMPLEX) B2K_NSB(B200KGE_DISTMULT) B2K_NSB(B200KGE_SIMPLE) B2K_NSB(B200KGE_CP)
    B2K_NSB(B200KGE_RESCAL) B2K_NSB(B200KGE_TRANSE) B2K_NSB(B200KGE_ROTATE)
    default: set_error("unknown model %d", model); return B200KGE_ERR_INVALID;
  }
#undef B2K_NSB
  B2K_LAUNCH_CHECK("ns_backward_kernel");
  const int dir = sp ? 0 : 1;
  if (pe) {
    if (model == B200KGE_TRANSE || model == B200KGE_ROTATE)
      return launch_unfold_distance(model, ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, st, 0, pe, pr);
    return launch_unfold(model, ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, st, 0, pe, pr);
  }
  if (model == B200KGE_TRANSE || model == B200KGE_ROTATE) {
    dim3 g2((unsigned)n), b2(128);
    if (model == B200KGE_TRANSE)
      unfold_distance_kernel<B200KGE_TRANSE, false><<<g2, b2, 0, st>>>(ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, 0);
    else
      unfold_distance_kernel<B200KGE_ROTATE, false><<<g2, b2, 0, st>>>(ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, 0);
    B2K_LAUNCH_CHECK("unfold_distance_kernel");
    return 0;
  }
  return launch_unfold(model, ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, st);
}

int launch_ns_backward_masked(int model, float l_norm, const Rows& a, const Rows& p, const Rows& table, int slot,
                              const int64_t* neg, int64_t n, int64_t K, const DropMask& mt, const float* G, int64_t ldg,
                              float* d_ent, int64_t lde, float* dQ, int64_t ldq, int64_t* tri_ws, float* dA, float* dP,
                              cudaStream_t st, const int32_t* pe) {
  if (n == 0) return 0;
  if (slot != 0 && slot != 2) { set_error("the masked negative-sampling backward covers the S and O slots"); return B200KGE_ERR_UNSUPPORTED; }
  const int sp = (slot == 2) ? 1 : 0;
  Folded f = folded_problem(model, sp ? B200KGE_SP_ : B200KGE__PO, table.dim, l_norm);
  if (model == B200KGE_RESCAL || f.pair_op == PAIR_LP || f.pair_op == PAIR_CMOD_LP || f.K > NSB_MAXK) {
    set_error("the masked negative-sampling backward covers the non-RESCAL models with l_norm 1 / 2 and K <= %d", NSB_MAXK);
    return B200KGE_ERR_UNSUPPORTED;
  }
  int rc;
  if ((rc = launch_identity_triples(n, tri_ws, st))) return rc;
  B2K_CUDA(cudaMemsetAsync(dQ, 0, (size_t)n * ldq * 4, st));
  B2K_CUDA(cudaMemsetAsync(dA, 0, (size_t)n * a.dim * 4, st));
  B2K_CUDA(cudaMemsetAsync(dP, 0, (size_t)n * p.dim * 4, st));
  if (K > 0) {
    const size_t smem = (size_t)2 * f.K * sizeof(float);
    const int64_t by = (K + 1 + NSB_PER_BLOCK - 1) / NSB_PER_BLOCK;
    if (by > 65535) { set_error("too many negatives per row (%lld)", (long long)K); return B200KGE_ERR_UNSUPPORTED; }
    dim3 grid((unsigned)n, (unsigned)by), block(NSB_WARPS * 32);
#define B2K_NSBM(M)                                                                                                    \
  case M:                                                                                                              \
    if (pe) ns_backward_rows_kernel_masked<M><<<grid, block, smem, st>>>(a, table, p, tri_ws, sp, neg, K, f, l_norm, G, \
                                                                         ldg, d_ent, lde, dQ, ldq, mt, pe);             \
    else ns_backward_kernel_masked<M><<<grid, block, smem, st>>>(a, table, p, tri_ws, sp, neg, K, f, l_norm, G, ldg,    \
                                                                 d_ent, lde, dQ, ldq, mt);                              \
    break;
    switch (model) {
      B2K_NSBM(B200KGE_COMPLEX) B2K_NSBM(B200KGE_DISTMULT) B2K_NSBM(B200KGE_SIMPLE) B2K_NSBM(B200KGE_CP)
      B2K_NSBM(B200KGE_TRANSE) B2K_NSBM(B200KGE_ROTATE)
      default: set_error("unknown model %d", model); return B200KGE_ERR_INVALID;
    }
#undef B2K_NSBM
    B2K_LAUNCH_CHECK("ns_backward_kernel_masked");
  }
  // the row gradients of the masked copies: the unfold on identity triples writes row i's into row i of dA / dP
  const int dir = sp ? 0 : 1;
  if (model == B200KGE_TRANSE || model == B200KGE_ROTATE)
    return launch_unfold_distance(model, a, p, tri_ws, n, dir, dQ, ldq, dA, a.dim, dP, p.dim, st);
  return launch_unfold(model, a, p, tri_ws, n, dir, dQ, ldq, dA, a.dim, dP, p.dim, st);
}

int launch_unfold_distance(int model, const Rows& ent, const Rows& rel, const int64_t* triples, int64_t n, int dir,
                           const float* dQ, int64_t ldq, float* d_ent, int64_t lde, float* d_rel, int64_t ldr,
                           cudaStream_t st, int64_t num_rel, const int32_t* pe, const int32_t* pr) {
  if (n == 0) return 0;
  if (num_rel > 0 && dir >= 0) { set_error("the reciprocal unfold needs the stacked layout"); return B200KGE_ERR_INVALID; }
  if (pe && (num_rel > 0 || dir < 0)) { set_error("the row-mapped unfold covers one direction"); return B200KGE_ERR_INVALID; }
  dim3 g2((unsigned)(dir < 0 ? 2 * n : n)), b2(128);
  if (pe && model == B200KGE_TRANSE)
    unfold_distance_rows_kernel<B200KGE_TRANSE><<<g2, b2, 0, st>>>(ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, pe, pr);
  else if (pe && model == B200KGE_ROTATE)
    unfold_distance_rows_kernel<B200KGE_ROTATE><<<g2, b2, 0, st>>>(ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, pe, pr);
  else if (model == B200KGE_TRANSE && num_rel > 0)
    unfold_distance_kernel<B200KGE_TRANSE, true><<<g2, b2, 0, st>>>(ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, num_rel);
  else if (model == B200KGE_ROTATE && num_rel > 0)
    unfold_distance_kernel<B200KGE_ROTATE, true><<<g2, b2, 0, st>>>(ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, num_rel);
  else if (model == B200KGE_TRANSE)
    unfold_distance_kernel<B200KGE_TRANSE, false><<<g2, b2, 0, st>>>(ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, 0);
  else if (model == B200KGE_ROTATE)
    unfold_distance_kernel<B200KGE_ROTATE, false><<<g2, b2, 0, st>>>(ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, 0);
  else { set_error("not a distance-family model (%d)", model); return B200KGE_ERR_INVALID; }
  B2K_LAUNCH_CHECK("unfold_distance_kernel");
  return 0;
}

int launch_row_lse(const float* z, int64_t ldz, int64_t nq, int64_t E, const int64_t* label_idx, float* row_stat,
                   cudaStream_t st) {
  if (nq == 0) return 0;
  row_lse_kernel<<<(unsigned)nq, 256, 0, st>>>(z, ldz, E, label_idx, nullptr, 0, row_stat);
  B2K_LAUNCH_CHECK("row_lse_kernel");
  return 0;
}

int launch_penalty(const Rows& tab, const float* counts, float p, int complex_abs, float scale, float* scratch,
                   size_t scratch_floats, float* out, cudaStream_t st) {
  const int64_t blocks = (tab.rows + PEN_ROWS - 1) / PEN_ROWS;
  if (blocks == 0) { return check_cuda(cudaMemsetAsync(out, 0, 4, st), "cudaMemsetAsync(penalty)"); }
  if ((size_t)blocks + 1 > scratch_floats || blocks >= (1ll << 31)) { set_error("workspace too small for the penalty partials"); return B200KGE_ERR_WORKSPACE; }
  unsigned int* ticket = reinterpret_cast<unsigned int*>(scratch + blocks);
  cudaError_t e = cudaMemsetAsync(ticket, 0, 4, st);
  if (e != cudaSuccess) return check_cuda(e, "cudaMemsetAsync(ticket)");
  penalty_kernel<<<(unsigned)blocks, 256, 0, st>>>(tab, counts, p, complex_abs, scale, scratch, ticket, out);
  B2K_LAUNCH_CHECK("penalty_kernel");
  return 0;
}

int launch_normalize_rows(float* w, int64_t ld, int64_t rows, int dim, float p, cudaStream_t st) {
  if (rows == 0 || !(p > 0.f)) return 0;
  normalize_rows_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(w, ld, rows, dim, p);
  B2K_LAUNCH_CHECK("normalize_rows_kernel");
  return 0;
}

int launch_transpose(const float* src, int64_t lds, int64_t R, int64_t C, float* dst, int64_t ldd, cudaStream_t st) {
  if (R == 0 || C == 0) return 0;
  dim3 grid((unsigned)((ldd + 31) / 32), (unsigned)((C + 31) / 32));
  transpose_kernel<<<grid, 256, 0, st>>>(src, lds, R, C, dst, ldd);
  B2K_LAUNCH_CHECK("transpose_kernel");
  return 0;
}

int launch_grad_planes(const float* z, int64_t ldz, int64_t nq, int64_t E, const int64_t* label_idx,
                       const float* label_dense, int64_t ldl, float* row_stat /* [2*nq] scratch: KL; null: BCE */,
                       float offset, float inv_n, void* g_hi, void* g_lo,
                       int64_t Ep, void* gt_hi, void* gt_lo, int64_t Np, float* g_scale, float* gt_scale,
                       cudaStream_t st) {
  if (nq == 0 || E == 0) return 0;
  if (row_stat) {
    row_lse_kernel<<<(unsigned)nq, 256, 0, st>>>(z, ldz, E, label_idx, label_dense, ldl, row_stat);
    B2K_LAUNCH_CHECK("row_lse_kernel");
  }
  dim3 grid((unsigned)(Ep / 64), (unsigned)(Np / 64));
  grad_planes_kernel<<<grid, 256, 0, st>>>(z, ldz, nq, E, label_idx, label_dense, ldl, row_stat, 0.f, offset, inv_n,
                                            (__half*)g_hi, (__half*)g_lo, Ep, (__half*)gt_hi, (__half*)gt_lo, Np,
                                            g_scale, gt_scale);
  B2K_LAUNCH_CHECK("grad_planes_kernel");
  return 0;
}

int launch_grad_planes_csr(const float* z, int64_t ldz, int64_t nq, int64_t E, const int64_t* csr_off,
                           const int64_t* csr_col, float a, float b, float* row_stat /* KL scratch [2nq] or null */,
                           float offset, float inv_n, void* g_hi, void* g_lo, int64_t Ep, void* gt_hi, void* gt_lo,
                           int64_t Np, float* g_scale, float* gt_scale, cudaStream_t st) {
  if (nq == 0 || E == 0) return 0;
  if (row_stat) {
    row_lse_kernel<<<(unsigned)nq, 256, 0, st>>>(z, ldz, E, nullptr, nullptr, 0, row_stat);
    B2K_LAUNCH_CHECK("row_lse_kernel");
    csr_row_mass_kernel<<<(unsigned)((nq + 255) / 256), 256, 0, st>>>(csr_off, nq, a, b, (float)E, row_stat);
    B2K_LAUNCH_CHECK("csr_row_mass_kernel");
  }
  dim3 grid((unsigned)(Ep / 64), (unsigned)(Np / 64));
  grad_planes_kernel<<<grid, 256, 0, st>>>(z, ldz, nq, E, nullptr, nullptr, 0, row_stat, b, offset, inv_n, (__half*)g_hi,
                                            (__half*)g_lo, Ep, (__half*)gt_hi, (__half*)gt_lo, Np, g_scale, gt_scale);
  B2K_LAUNCH_CHECK("grad_planes_kernel");
  csr_grad_fix_kernel<<<(unsigned)((nq + 7) / 8), 256, 0, st>>>(z, ldz, nq, csr_off, csr_col, row_stat, a, b, offset,
                                                               (__half*)g_hi, (__half*)g_lo, Ep, (__half*)gt_hi,
                                                               (__half*)gt_lo, Np);
  B2K_LAUNCH_CHECK("csr_grad_fix_kernel");
  return 0;
}

int launch_unfold(int model, const Rows& ent, const Rows& rel, const int64_t* triples, int64_t n, int dir,
                  const float* dQ, int64_t ldq, float* d_ent, int64_t lde, float* d_rel, int64_t ldr, cudaStream_t st,
                  int64_t num_rel, const int32_t* pe, const int32_t* pr) {
  if (n == 0) return 0;
  if (num_rel > 0 && dir >= 0) { set_error("the reciprocal unfold needs the stacked layout"); return B200KGE_ERR_INVALID; }
  if (pe && (num_rel > 0 || dir < 0)) { set_error("the row-mapped unfold covers one direction"); return B200KGE_ERR_INVALID; }
  const int64_t nq = dir < 0 ? 2 * n : n;
  dim3 grid((unsigned)nq), block(128);
  const int D = ent.dim;
#define B2K_UNFOLD(M, SM) case M: unfold_kernel<M, false><<<grid, block, SM, st>>>(ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, 0); break;
#define B2K_UNFOLD_R(M, SM) case M: unfold_kernel<M, true><<<grid, block, SM, st>>>(ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, num_rel); break;
#define B2K_UNFOLD_M(M, SM) case M: unfold_rows_kernel<M><<<grid, block, SM, st>>>(ent, rel, triples, n, dir, dQ, ldq, d_ent, lde, d_rel, ldr, pe, pr); break;
  if (pe) {
    switch (model) {
      B2K_UNFOLD_M(B200KGE_COMPLEX, 0) B2K_UNFOLD_M(B200KGE_DISTMULT, 0) B2K_UNFOLD_M(B200KGE_SIMPLE, 0)
      B2K_UNFOLD_M(B200KGE_CP, 0) B2K_UNFOLD_M(B200KGE_RESCAL, 2 * D * sizeof(float))
      default: set_error("the analytic backward covers the dot family only (model %d)", model); return B200KGE_ERR_UNSUPPORTED;
    }
  } else if (num_rel > 0) {
    switch (model) {
      B2K_UNFOLD_R(B200KGE_COMPLEX, 0) B2K_UNFOLD_R(B200KGE_DISTMULT, 0) B2K_UNFOLD_R(B200KGE_SIMPLE, 0)
      B2K_UNFOLD_R(B200KGE_CP, 0) B2K_UNFOLD_R(B200KGE_RESCAL, 2 * D * sizeof(float))
      default: set_error("the analytic backward covers the dot family only (model %d)", model); return B200KGE_ERR_UNSUPPORTED;
    }
  } else {
    switch (model) {
      B2K_UNFOLD(B200KGE_COMPLEX, 0) B2K_UNFOLD(B200KGE_DISTMULT, 0) B2K_UNFOLD(B200KGE_SIMPLE, 0)
      B2K_UNFOLD(B200KGE_CP, 0) B2K_UNFOLD(B200KGE_RESCAL, 2 * D * sizeof(float))
      default: set_error("the analytic backward covers the dot family only (model %d)", model); return B200KGE_ERR_UNSUPPORTED;
    }
  }
#undef B2K_UNFOLD
#undef B2K_UNFOLD_R
#undef B2K_UNFOLD_M
  B2K_LAUNCH_CHECK("unfold_kernel");
  return 0;
}

}  // namespace b200kge
