// ns_shared.cu — shared negative sampling (b200kge_ns_shared_score / b200kge_ns_shared_backward).
//
// With `negative_sampling.shared: True` every row of a batch draws its negatives from the same U' shared ids
// (`unique`, sampler.py:597-698): column 1 + c of row i holds the sample j = c < U ? c : repeat[c - U], and under the
// `default` type the row's dropped sample drop[i] is replaced by the extra id unique[U]:
//   u(i, c) = (j == drop[i]) ? U : j                     (naive: u = j, no drop)
// (DefaultSharedNegativeSample.score / NaiveSharedNegativeSample.score, sampler.py:428-463,537-578).  So the slot is the
// small dense problem Z = score(fixed pair of row i, unique[u]) [n, U'] plus these kernels:
//   assemble   out[i, 1 + c] = Z[i, u(i, c)]: one block per row
//   collapse   C[i, u] = sum over the columns c with u(i, c) = u of G[i, 1 + c]: one block per row, one thread per u,
//              the repeats staged through shared memory; sums in column order, no atomics (as ns_p_collapse_kernel)
//   used ids   the ids the rows of a sub-batch actually use (the `triple` row set of a sparse gradient): unique[u] is
//              unused exactly when every row has drop[i] == u
//   eps        pairwise_distance's eps folded into TransE's queries (the reference's `triple` scoring, transe.py:18)
//   row add    dT [U', K] ADDED into the rows unique[u] (or their row-set positions): distinct rows, no contention
#include "common.cuh"

namespace b200kge {

namespace {

constexpr int NSS_THREADS = 256;
constexpr int NSS_CHUNK = 1024;          // repeats staged per pass of the collapse

__global__ void __launch_bounds__(NSS_THREADS)
ns_shared_assemble_kernel(const float* __restrict__ Z, int64_t ldz, int64_t K, int64_t U,
                          const int64_t* __restrict__ repeat, const int64_t* __restrict__ drop, float* __restrict__ out,
                          int64_t ldo) {
  const int64_t i = blockIdx.x;
  const int64_t d = drop ? drop[i] : -1;
  const float* __restrict__ z = Z + i * ldz;
  float* __restrict__ o = out + i * ldo + 1;
  for (int64_t c = threadIdx.x; c < K; c += NSS_THREADS) {
    const int64_t j = c < U ? c : repeat[c - U];
    o[c] = z[j == d ? U : j];
  }
}

__global__ void __launch_bounds__(NSS_THREADS)
ns_shared_collapse_kernel(const float* __restrict__ G, int64_t ldg, int64_t K, int64_t U, int64_t nu,
                          const int64_t* __restrict__ repeat, const int64_t* __restrict__ drop, float* __restrict__ C,
                          int64_t ldc) {
  __shared__ int64_t srep[NSS_CHUNK];
  __shared__ float sg[NSS_CHUNK];
  const int64_t i = blockIdx.x, nrep = K - U;
  const int64_t d = drop ? drop[i] : -1;
  const float* __restrict__ g = G + i * ldg + 1;
  for (int64_t u0 = 0; u0 < nu; u0 += NSS_THREADS) {
    const int64_t u = u0 + threadIdx.x;
    // the sample whose columns feed u: u itself, or for the extra id the row's dropped sample (none if d == U)
    const int64_t j = u == U ? d : u;
    const bool live = u < nu && (u == U ? d < U : u != d);
    float acc = live ? g[j] : 0.f;
    for (int64_t r0 = 0; r0 < nrep; r0 += NSS_CHUNK) {
      const int len = (int)(nrep - r0 < NSS_CHUNK ? nrep - r0 : NSS_CHUNK);
      __syncthreads();
      for (int r = threadIdx.x; r < len; r += NSS_THREADS) {
        srep[r] = repeat[r0 + r];
        sg[r] = g[U + r0 + r];
      }
      __syncthreads();
      if (live)
        for (int r = 0; r < len; ++r)
          if (srep[r] == j) acc += sg[r];
    }
    if (u < nu) C[i * ldc + u] = acc;
  }
}

__global__ void __launch_bounds__(NSS_THREADS)
ns_shared_drop_count_kernel(const int64_t* __restrict__ drop, int64_t n, int* __restrict__ cnt) {
  const int64_t i = (int64_t)blockIdx.x * NSS_THREADS + threadIdx.x;
  if (i < n) atomicAdd(cnt + drop[i], 1);
}

// used[u] = unique[u] if some row uses it, else `fill` (an id already in the row set)
__global__ void __launch_bounds__(NSS_THREADS)
ns_shared_used_kernel(const int64_t* __restrict__ unique, int64_t nu, const int* __restrict__ cnt, int64_t n,
                      const int64_t* __restrict__ fill, int64_t* __restrict__ used) {
  const int64_t u = (int64_t)blockIdx.x * NSS_THREADS + threadIdx.x;
  if (u < nu) used[u] = cnt[u] == n ? *fill : unique[u];
}

__global__ void __launch_bounds__(NSS_THREADS)
ns_shared_eps_kernel(float* __restrict__ Q, int64_t ldq, int D, float eps) {
  float* __restrict__ q = Q + (int64_t)blockIdx.x * ldq;
  for (int k = threadIdx.x; k < D; k += NSS_THREADS) q[k] += eps;
}

__global__ void __launch_bounds__(128)
ns_shared_row_add_kernel(const float* __restrict__ dT, int64_t ldt, int K, const int64_t* __restrict__ unique,
                         const int32_t* __restrict__ pe, float* __restrict__ d_ent, int64_t lde, int col_off) {
  const int64_t u = blockIdx.x, e = unique[u];
  float* __restrict__ dst = d_ent + (pe ? (int64_t)pe[e] : e) * lde + col_off;
  const float* __restrict__ src = dT + u * ldt;
  for (int k = threadIdx.x; k < K; k += 128) dst[k] += src[k];
}

}  // namespace

int launch_ns_shared_assemble(const float* Z, int64_t ldz, int64_t n, int64_t K, int64_t U, const int64_t* repeat,
                              const int64_t* drop, float* out, int64_t ldo, cudaStream_t st) {
  if (n == 0 || K == 0) return 0;
  ns_shared_assemble_kernel<<<(unsigned)n, NSS_THREADS, 0, st>>>(Z, ldz, K, U, repeat, drop, out, ldo);
  B2K_LAUNCH_CHECK("ns_shared_assemble_kernel");
  return 0;
}

int launch_ns_shared_collapse(const float* G, int64_t ldg, int64_t n, int64_t K, int64_t U, int64_t nu,
                              const int64_t* repeat, const int64_t* drop, float* C, int64_t ldc, cudaStream_t st) {
  if (n == 0 || nu == 0) return 0;
  ns_shared_collapse_kernel<<<(unsigned)n, NSS_THREADS, 0, st>>>(G, ldg, K, U, nu, repeat, drop, C, ldc);
  B2K_LAUNCH_CHECK("ns_shared_collapse_kernel");
  return 0;
}

int launch_ns_shared_used(const int64_t* unique, int64_t nu, const int64_t* drop, int64_t n, const int64_t* fill,
                          int* cnt, int64_t* used, cudaStream_t st) {
  if (nu == 0 || n == 0) return 0;
  B2K_CUDA(cudaMemsetAsync(cnt, 0, (size_t)nu * 4, st));
  ns_shared_drop_count_kernel<<<(unsigned)((n + NSS_THREADS - 1) / NSS_THREADS), NSS_THREADS, 0, st>>>(drop, n, cnt);
  B2K_LAUNCH_CHECK("ns_shared_drop_count_kernel");
  ns_shared_used_kernel<<<(unsigned)((nu + NSS_THREADS - 1) / NSS_THREADS), NSS_THREADS, 0, st>>>(unique, nu, cnt, n,
                                                                                                 fill, used);
  B2K_LAUNCH_CHECK("ns_shared_used_kernel");
  return 0;
}

int launch_ns_shared_eps(float* Q, int64_t ldq, int64_t n, int D, float eps, cudaStream_t st) {
  if (n == 0 || eps == 0.f) return 0;
  ns_shared_eps_kernel<<<(unsigned)n, NSS_THREADS, 0, st>>>(Q, ldq, D, eps);
  B2K_LAUNCH_CHECK("ns_shared_eps_kernel");
  return 0;
}

int launch_ns_shared_row_add(const float* dT, int64_t ldt, int64_t nu, int K, const int64_t* unique, const int32_t* pe,
                             float* d_ent, int64_t lde, int col_off, cudaStream_t st) {
  if (nu == 0) return 0;
  ns_shared_row_add_kernel<<<(unsigned)nu, 128, 0, st>>>(dT, ldt, K, unique, pe, d_ent, lde, col_off);
  B2K_LAUNCH_CHECK("ns_shared_row_add_kernel");
  return 0;
}

}  // namespace b200kge
