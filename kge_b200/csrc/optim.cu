// optim.cu — the optimizer step of torch.optim.Adagrad (dense and row-sparse gradients) and torch.optim.SparseAdam in
// one pass over the elements they update.  Every operation is an explicit round-to-nearest intrinsic written in the
// order of torch 2.11's kernels (adagrad.py, _functional.sparse_adam), with an FMA exactly where torch's compiled
// kernels have one, so the compiler cannot contract or split anything differently.
//   dense    adagrad_dense_kernel: grid-stride over p / sum / g, float4 body and scalar tail (20 B per element)
//   sparse   a coalesced gradient (sorted unique rows + [nnz, D] values) is read in place; an uncoalesced one is
//            coalesced first: launch_row_set (rowset.cu) over the COO row ids gives the sorted unique rows, their
//            number u (device) and pos[id], then rows_accumulate_kernel adds every value row into vals[pos[id]]
//   update   adagrad_rows_kernel / sparse_adam_rows_kernel: one pass over the u rows, reading u on the device
#include "common.cuh"

namespace b200kge {

namespace {

inline size_t op_up(size_t b) { return (b + 255) / 256 * 256; }

// one wave of 8 blocks of 256 threads per SM: the grid of the loops whose trip count is only known on the device
int one_wave(unsigned* grid) {
  int dev = 0, sms = 0;
  B2K_CUDA(cudaGetDevice(&dev));
  B2K_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  *grid = (unsigned)sms * 8;
  return 0;
}

inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// Adagrad on one element with clr' = -clr, rounded as torch 2.11's CUDA kernels round it.  Their addcmul / addcdiv /
// add-with-alpha are compiled to FMAs (a + alpha * b): the gradient with weight decay is fma(wd, p, g) and the dense sum
// fma(g, g, s).  The orders:
//   AG_FOREACH  _multi_tensor_adagrad (dense):     p + (g * clr') / (sqrt(s) + eps)      (addcdiv with value 1)
//   AG_SINGLE   _single_tensor_adagrad (dense):    fma(g / (sqrt(s) + eps), clr', p)     (addcdiv with value clr')
//   AG_SPARSE   _single_tensor_adagrad (sparse):   s + round(v v), then p + round(clr' (v / (sqrt(s) + eps)))
//               (pow, index_add and a separate mul: nothing fused)
enum { AG_FOREACH = 0, AG_SINGLE = 1, AG_SPARSE = 2 };

template <int ORDER>
__device__ __forceinline__ void adagrad_elem(float& p, float& s, float g, float neg_clr, float eps, float wd) {
  if (ORDER != AG_SPARSE && wd != 0.f) g = __fmaf_rn(wd, p, g);
  s = ORDER == AG_SPARSE ? __fadd_rn(s, __fmul_rn(g, g)) : __fmaf_rn(g, g, s);
  const float den = __fadd_rn(__fsqrt_rn(s), eps);
  if (ORDER == AG_FOREACH) p = __fadd_rn(p, __fdiv_rn(__fmul_rn(g, neg_clr), den));
  else if (ORDER == AG_SINGLE) p = __fmaf_rn(__fdiv_rn(g, den), neg_clr, p);
  else p = __fadd_rn(p, __fmul_rn(neg_clr, __fdiv_rn(g, den)));
}

// SparseAdam on one element: omb1 = 1 - beta1, omb2 = 1 - beta2 (rounded from double on the host, as torch's scalar
// arguments are), neg_step = -step_size
__device__ __forceinline__ void sparse_adam_elem(float& p, float& m, float& q, float v, float omb1, float omb2,
                                                 float eps, float neg_step) {
  const float m_old = m, q_old = q;
  const float mu = __fmul_rn(__fsub_rn(v, m_old), omb1);
  const float qu = __fmul_rn(__fsub_rn(__fmul_rn(v, v), q_old), omb2);
  m = __fadd_rn(m_old, mu);
  q = __fadd_rn(q_old, qu);
  const float den = __fadd_rn(__fsqrt_rn(__fadd_rn(qu, q_old)), eps);
  p = __fadd_rn(p, __fmul_rn(neg_step, __fdiv_rn(__fadd_rn(mu, m_old), den)));
}

// n elements; vec: p, s and g 16-byte aligned, so the first n / 4 * 4 go as float4
template <int ORDER>
__global__ void __launch_bounds__(256)
adagrad_dense_kernel(float* __restrict__ p, float* __restrict__ s, const float* __restrict__ g, int64_t n, int vec,
                     float neg_clr, float eps, float wd) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x, t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t head = 0;
  if (vec) {
    head = n / 4 * 4;
    float4* p4 = reinterpret_cast<float4*>(p);
    float4* s4 = reinterpret_cast<float4*>(s);
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (int64_t i = t; i < n / 4; i += stride) {
      float4 pv = p4[i], sv = s4[i];
      const float4 gv = __ldcs(g4 + i);
      adagrad_elem<ORDER>(pv.x, sv.x, gv.x, neg_clr, eps, wd);
      adagrad_elem<ORDER>(pv.y, sv.y, gv.y, neg_clr, eps, wd);
      adagrad_elem<ORDER>(pv.z, sv.z, gv.z, neg_clr, eps, wd);
      adagrad_elem<ORDER>(pv.w, sv.w, gv.w, neg_clr, eps, wd);
      p4[i] = pv;
      s4[i] = sv;
    }
  }
  for (int64_t i = head + t; i < n; i += stride) adagrad_elem<ORDER>(p[i], s[i], __ldcs(g + i), neg_clr, eps, wd);
}

// vals[pos[idx[j]]] += g[j] for the nnz value rows of an uncoalesced gradient; VEC: dim % 4 == 0, both blocks 16-byte
// aligned (one float4 atomic per four columns)
template <bool VEC>
__global__ void __launch_bounds__(256)
rows_accumulate_kernel(const float* __restrict__ g, const int64_t* __restrict__ idx, int64_t nnz, int64_t dim,
                       const int32_t* __restrict__ pos, float* __restrict__ vals) {
  const int64_t w = VEC ? dim / 4 : dim, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz * w; i += stride) {
    const int64_t r = i / w, dst = (int64_t)pos[idx[r]] * w + (i - r * w);
    if constexpr (VEC) atomicAdd(reinterpret_cast<float4*>(vals) + dst, __ldcs(reinterpret_cast<const float4*>(g) + i));
    else atomicAdd(vals + dst, __ldcs(g + i));
  }
}

// Row r < u (u = *count, or n when count is NULL) of the gradient updates row rows[r] of p and the state.  VEC as above,
// for p, the state and vals.
template <bool VEC>
__global__ void __launch_bounds__(256)
adagrad_rows_kernel(float* __restrict__ p, float* __restrict__ s, const float* __restrict__ vals,
                    const int64_t* __restrict__ rows, const int64_t* __restrict__ count, int64_t n, int64_t dim,
                    float neg_clr, float eps) {
  const int64_t u = count ? *count : n, w = VEC ? dim / 4 : dim, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < u * w; i += stride) {
    const int64_t r = i / w, dst = rows[r] * w + (i - r * w);
    if constexpr (VEC) {
      float4 pv = reinterpret_cast<float4*>(p)[dst], sv = reinterpret_cast<float4*>(s)[dst];
      const float4 v = reinterpret_cast<const float4*>(vals)[i];
      adagrad_elem<AG_SPARSE>(pv.x, sv.x, v.x, neg_clr, eps, 0.f);
      adagrad_elem<AG_SPARSE>(pv.y, sv.y, v.y, neg_clr, eps, 0.f);
      adagrad_elem<AG_SPARSE>(pv.z, sv.z, v.z, neg_clr, eps, 0.f);
      adagrad_elem<AG_SPARSE>(pv.w, sv.w, v.w, neg_clr, eps, 0.f);
      reinterpret_cast<float4*>(p)[dst] = pv;
      reinterpret_cast<float4*>(s)[dst] = sv;
    } else {
      adagrad_elem<AG_SPARSE>(p[dst], s[dst], vals[i], neg_clr, eps, 0.f);
    }
  }
}

template <bool VEC>
__global__ void __launch_bounds__(256)
sparse_adam_rows_kernel(float* __restrict__ p, float* __restrict__ m, float* __restrict__ q,
                        const float* __restrict__ vals, const int64_t* __restrict__ rows,
                        const int64_t* __restrict__ count, int64_t n, int64_t dim, float omb1, float omb2, float eps,
                        float neg_step) {
  const int64_t u = count ? *count : n, w = VEC ? dim / 4 : dim, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < u * w; i += stride) {
    const int64_t r = i / w, dst = rows[r] * w + (i - r * w);
    if constexpr (VEC) {
      float4 pv = reinterpret_cast<float4*>(p)[dst], mv = reinterpret_cast<float4*>(m)[dst],
             qv = reinterpret_cast<float4*>(q)[dst];
      const float4 v = reinterpret_cast<const float4*>(vals)[i];
      sparse_adam_elem(pv.x, mv.x, qv.x, v.x, omb1, omb2, eps, neg_step);
      sparse_adam_elem(pv.y, mv.y, qv.y, v.y, omb1, omb2, eps, neg_step);
      sparse_adam_elem(pv.z, mv.z, qv.z, v.z, omb1, omb2, eps, neg_step);
      sparse_adam_elem(pv.w, mv.w, qv.w, v.w, omb1, omb2, eps, neg_step);
      reinterpret_cast<float4*>(p)[dst] = pv;
      reinterpret_cast<float4*>(m)[dst] = mv;
      reinterpret_cast<float4*>(q)[dst] = qv;
    } else {
      sparse_adam_elem(p[dst], m[dst], q[dst], vals[i], omb1, omb2, eps, neg_step);
    }
  }
}

// The row-sparse gradient as the update kernels read it: rows[r], r < u, with u = *count or n when count is NULL
struct RowGrad {
  const int64_t* rows;
  const int64_t* count;
  const float* vals;
  int64_t n;
};

// coalesced: the caller's rows and values; otherwise their sum per unique row, built in the workspace
int stage_rows(int64_t rows, int64_t dim, const float* grad, const int64_t* grad_rows, int64_t nnz, int coalesced,
               void* workspace, cudaStream_t st, RowGrad* out) {
  if (coalesced) { *out = RowGrad{grad_rows, nullptr, grad, nnz}; return 0; }
  const int64_t cap = nnz < rows ? nnz : rows;
  uint8_t* at = (uint8_t*)workspace + row_set_workspace_bytes(rows);
  int64_t* u_rows = (int64_t*)at;
  at += op_up((size_t)cap * 8);
  int64_t* count = (int64_t*)at;
  at += op_up(8);
  float* vals = (float*)at;
  const IdList list{grad_rows, nnz, 1};
  int rc = launch_row_set(rows, &list, 1, workspace, u_rows, count, vals, dim, st);
  if (rc) return rc;
  unsigned grid;
  if ((rc = one_wave(&grid))) return rc;
  const int32_t* pos = (const int32_t*)workspace;
  if (dim % 4 == 0 && aligned16(grad) && aligned16(vals))
    rows_accumulate_kernel<true><<<grid, 256, 0, st>>>(grad, grad_rows, nnz, dim, pos, vals);
  else
    rows_accumulate_kernel<false><<<grid, 256, 0, st>>>(grad, grad_rows, nnz, dim, pos, vals);
  B2K_LAUNCH_CHECK("rows_accumulate_kernel");
  *out = RowGrad{u_rows, count, vals, cap};
  return 0;
}

}  // namespace

size_t optim_step_workspace_bytes(int64_t rows, int64_t dim, int64_t nnz, int coalesced) {
  if (coalesced || rows <= 0 || dim <= 0 || nnz <= 0) return 0;
  const int64_t cap = nnz < rows ? nnz : rows;
  return row_set_workspace_bytes(rows) + op_up((size_t)cap * 8) + op_up(8) + op_up((size_t)cap * dim * 4);
}

int launch_adagrad_step(float* param, float* state_sum, int64_t rows, int64_t dim, const float* grad,
                        const int64_t* grad_rows, int64_t nnz, int coalesced, int foreach_order, float clr, float eps,
                        float weight_decay, void* workspace, cudaStream_t st) {
  unsigned grid;
  int rc = one_wave(&grid);
  if (rc) return rc;
  if (!grad_rows) {
    const int64_t n = rows * dim;
    if (n == 0) return 0;
    const int vec = aligned16(param) && aligned16(state_sum) && aligned16(grad);
    const int64_t work = vec ? n / 4 + 1 : n;
    const unsigned blocks = (unsigned)(work / 256 + 1 < (int64_t)grid ? work / 256 + 1 : grid);
    if (foreach_order)
      adagrad_dense_kernel<AG_FOREACH><<<blocks, 256, 0, st>>>(param, state_sum, grad, n, vec, -clr, eps, weight_decay);
    else
      adagrad_dense_kernel<AG_SINGLE><<<blocks, 256, 0, st>>>(param, state_sum, grad, n, vec, -clr, eps, weight_decay);
    B2K_LAUNCH_CHECK("adagrad_dense_kernel");
    return 0;
  }
  if (nnz == 0 || rows == 0) return 0;
  RowGrad g;
  if ((rc = stage_rows(rows, dim, grad, grad_rows, nnz, coalesced, workspace, st, &g))) return rc;
  if (dim % 4 == 0 && aligned16(param) && aligned16(state_sum) && aligned16(g.vals))
    adagrad_rows_kernel<true><<<grid, 256, 0, st>>>(param, state_sum, g.vals, g.rows, g.count, g.n, dim, -clr, eps);
  else
    adagrad_rows_kernel<false><<<grid, 256, 0, st>>>(param, state_sum, g.vals, g.rows, g.count, g.n, dim, -clr, eps);
  B2K_LAUNCH_CHECK("adagrad_rows_kernel");
  return 0;
}

int launch_sparse_adam_step(float* param, float* exp_avg, float* exp_avg_sq, int64_t rows, int64_t dim,
                            const float* grad, const int64_t* grad_rows, int64_t nnz, int coalesced,
                            float one_minus_beta1, float one_minus_beta2, float eps, float step_size, void* workspace,
                            cudaStream_t st) {
  if (nnz == 0 || rows == 0) return 0;
  unsigned grid;
  int rc = one_wave(&grid);
  if (rc) return rc;
  RowGrad g;
  if ((rc = stage_rows(rows, dim, grad, grad_rows, nnz, coalesced, workspace, st, &g))) return rc;
  if (dim % 4 == 0 && aligned16(param) && aligned16(exp_avg) && aligned16(exp_avg_sq) && aligned16(g.vals))
    sparse_adam_rows_kernel<true><<<grid, 256, 0, st>>>(param, exp_avg, exp_avg_sq, g.vals, g.rows, g.count, g.n, dim,
                                                        one_minus_beta1, one_minus_beta2, eps, -step_size);
  else
    sparse_adam_rows_kernel<false><<<grid, 256, 0, st>>>(param, exp_avg, exp_avg_sq, g.vals, g.rows, g.count, g.n,
                                                         dim, one_minus_beta1, one_minus_beta2, eps, -step_size);
  B2K_LAUNCH_CHECK("sparse_adam_rows_kernel");
  return 0;
}

}  // namespace b200kge
