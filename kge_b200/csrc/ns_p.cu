// ns_p.cu — the backward of the negative-sampling P slot (b200kge_ns_p_backward).
//
// Row i of a P-slot block scores (s_i, r, o_i) for r = p_i (column 0) and for its K sampled relation ids, so the
// score depends on (i, r) only and the block's gradient G [n, 1+K] sums exactly into one coefficient per (row,
// relation): C[i, r] = sum over the columns c of row i with id r of G[i, c].  The backward is then an all-relations
// backward with weights C, and no contribution is ever scattered per sample into the R hot relation rows.
//   collapse      C from G, the positives' p and the sampled ids: one block per row, one thread per relation, the
//                 row's ids and G staged through shared memory; sums in column order (deterministic)
//   unpack        s, o of the triples as index vectors, and their destination rows (the row-set map of a sparse
//                 entity gradient, else the ids themselves)
//   distance      TransE (L1, L2) and RotatE (L1): the VJP of -|| x(s_i, r, o_i) || over the nonzero C[i, r]:
//                   l2 norms  (TransE L2) C[i, r] /= || x ||, one warp per (i, r)
//                   entities  one block per row i over the row's nonzero C[i, :] (staged in shared memory): d s_i,
//                             d o_i, added into the destination rows
//                   relations one block per (relation, chunk of rows) walking C transposed: a partial d rel[r] per
//                             chunk, no atomics
//   rel add       the relation gradient (the chunk partials of the distance family, dT of the dot family's GEMM)
//                 summed per row and ADDED into the dense gradient or into the row-sparse value block
#include "common.cuh"

namespace b200kge {

namespace {

constexpr int NSP_THREADS = 256;         // collapse, l2 norms
constexpr int NSP_CHUNK = 1024;          // columns of G staged per pass of the collapse
constexpr int NSP_ROW_THREADS = 128;     // entity / relation / add passes
constexpr int NSP_ROWS_PER_PART = 8;     // least rows per relation-pass chunk

__global__ void __launch_bounds__(NSP_THREADS)
ns_p_collapse_kernel(const int64_t* __restrict__ triples, const int64_t* __restrict__ neg, int64_t K,
                     const float* __restrict__ G, int64_t ldg, int R, float* __restrict__ C, int64_t ldc) {
  __shared__ int sid[NSP_CHUNK];
  __shared__ float sg[NSP_CHUNK];
  const int64_t i = blockIdx.x, m = K + 1;
  const float* __restrict__ g = G + i * ldg;
  const int64_t* __restrict__ ng = neg + i * K;
  for (int r0 = 0; r0 < R; r0 += NSP_THREADS) {
    const int r = r0 + threadIdx.x;
    float acc = 0.f;
    for (int64_t c0 = 0; c0 < m; c0 += NSP_CHUNK) {
      const int len = (int)(m - c0 < NSP_CHUNK ? m - c0 : NSP_CHUNK);
      __syncthreads();
      for (int c = threadIdx.x; c < len; c += NSP_THREADS) {
        const int64_t col = c0 + c;
        sid[c] = (int)(col == 0 ? triples[i * 3 + 1] : ng[col - 1]);
        sg[c] = g[col];
      }
      __syncthreads();
      for (int c = 0; c < len; ++c)
        if (sid[c] == r) acc += sg[c];
    }
    if (r < R) C[i * ldc + r] = acc;
  }
}

__global__ void __launch_bounds__(256)
ns_p_unpack_kernel(const int64_t* __restrict__ triples, int64_t n, const int32_t* __restrict__ pe,
                   int64_t* __restrict__ s_idx, int64_t* __restrict__ o_idx, int64_t* __restrict__ s_dst,
                   int64_t* __restrict__ o_dst) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t s = triples[i * 3], o = triples[i * 3 + 2];
  s_idx[i] = s;
  o_idx[i] = o;
  s_dst[i] = pe ? (int64_t)pe[s] : s;
  o_dst[i] = pe ? (int64_t)pe[o] : o;
}

// TransE: x_k = (s_k + p_k) - o_k + eps, spo_kernel's order (rowwise.cu)
__device__ __forceinline__ float transe_x(float s, float p, float o) { return ((s + p) - o) + 1e-6f; }

// TransE L2: C[i, r] /= || x(s_i, r, o_i) ||_2 (0 where the norm is 0: torch's norm backward there)
__global__ void __launch_bounds__(NSP_THREADS)
ns_p_l2_scale_kernel(Rows E, Rows Rl, const int64_t* __restrict__ s_idx, const int64_t* __restrict__ o_idx, int R,
                     float* __restrict__ C, int64_t ldc) {
  const int64_t i = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = NSP_THREADS >> 5, D = E.dim;
  const float* __restrict__ s = E.base + s_idx[i] * E.ld;
  const float* __restrict__ o = E.base + o_idx[i] * E.ld;
  for (int r = warp; r < R; r += nw) {
    const float w = C[i * ldc + r];
    if (w == 0.f) continue;
    const float* __restrict__ p = Rl.base + (int64_t)r * Rl.ld;
    float acc = 0.f;
    for (int k = lane; k < D; k += 32) {
      const float x = transe_x(s[k], p[k], o[k]);
      acc = fmaf(x, x, acc);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) {
      const float z = sqrtf(acc);
      C[i * ldc + r] = z > 0.f ? w / z : 0.f;
    }
  }
}

// dscore/dx_k times the weight w of TransE: L1 -w sign(x), L2 -w x (w already divided by the norm)
template <bool L2>
__device__ __forceinline__ float transe_g(float w, float x) {
  if constexpr (L2) return -w * x;
  return x > 0.f ? -w : (x < 0.f ? w : 0.f);
}

// RotatE L1 element k of (s_i, theta, o_i): the rotated subject q, and the weighted gradient (g_re, g_im) of
// -|q - o| with respect to the difference (0 where |q - o| = 0, torch's norm backward there)
struct RotElem { float c, sn, q_re, q_im, g_re, g_im; };
__device__ __forceinline__ RotElem rotate_elem(float w, float s_re, float s_im, float th, float o_re, float o_im) {
  RotElem e;
  sincosf(th, &e.sn, &e.c);
  e.q_re = s_re * e.c - s_im * e.sn;
  e.q_im = s_re * e.sn + s_im * e.c;
  const float d_re = e.q_re - o_re, d_im = e.q_im - o_im;
  const float m = sqrtf(fmaf(d_im, d_im, d_re * d_re));
  const float f = m > 0.f ? -w / m : 0.f;
  e.g_re = f * d_re;
  e.g_im = f * d_im;
  return e;
}

// d s_i and d o_i over the nonzero C[i, :], ADDED into rows s_dst[i] / o_dst[i] of d_ent
template <int MODEL, bool L2>
__global__ void __launch_bounds__(NSP_ROW_THREADS)
ns_p_ent_kernel(Rows E, Rows Rl, const int64_t* __restrict__ s_idx, const int64_t* __restrict__ o_idx, int R,
                const float* __restrict__ C, int64_t ldc, float* __restrict__ d_ent, int64_t lde,
                const int64_t* __restrict__ s_dst, const int64_t* __restrict__ o_dst) {
  __shared__ float sc[B200KGE_NS_P_MAX_RELATIONS];
  const int64_t i = blockIdx.x;
  for (int r = threadIdx.x; r < R; r += NSP_ROW_THREADS) sc[r] = C[i * ldc + r];
  __syncthreads();
  const float* __restrict__ s = E.base + s_idx[i] * E.ld;
  const float* __restrict__ o = E.base + o_idx[i] * E.ld;
  float* __restrict__ ds = d_ent + s_dst[i] * lde;
  float* __restrict__ dO = d_ent + o_dst[i] * lde;
  const int D = E.dim, h = D >> 1;
  if constexpr (MODEL == B200KGE_TRANSE) {
    for (int k = threadIdx.x; k < D; k += NSP_ROW_THREADS) {
      const float sk = s[k], ok = o[k];
      float acc = 0.f;
      for (int r = 0; r < R; ++r) {
        const float w = sc[r];
        if (w == 0.f) continue;
        acc += transe_g<L2>(w, transe_x(sk, Rl.base[(int64_t)r * Rl.ld + k], ok));
      }
      atomicAdd(ds + k, acc);          // dx/ds = 1, dx/do = -1
      atomicAdd(dO + k, -acc);
    }
  } else {  // ROTATE, l_norm 1
    for (int k = threadIdx.x; k < h; k += NSP_ROW_THREADS) {
      const float s_re = s[k], s_im = s[k + h], o_re = o[k], o_im = o[k + h];
      float as_re = 0.f, as_im = 0.f, ao_re = 0.f, ao_im = 0.f;
      for (int r = 0; r < R; ++r) {
        const float w = sc[r];
        if (w == 0.f) continue;
        const RotElem e = rotate_elem(w, s_re, s_im, Rl.base[(int64_t)r * Rl.ld + k], o_re, o_im);
        as_re += e.g_re * e.c + e.g_im * e.sn;
        as_im += e.g_im * e.c - e.g_re * e.sn;
        ao_re -= e.g_re;
        ao_im -= e.g_im;
      }
      atomicAdd(ds + k, as_re);
      atomicAdd(ds + k + h, as_im);
      atomicAdd(dO + k, ao_re);
      atomicAdd(dO + k + h, ao_im);
    }
  }
}

// block (r, chunk): sum over the chunk's rows i with C[i, r] != 0 of the relation row's gradient, STORED into
// parts[chunk][r] (every element written)
template <int MODEL, bool L2>
__global__ void __launch_bounds__(NSP_ROW_THREADS)
ns_p_rel_kernel(Rows E, Rows Rl, const int64_t* __restrict__ s_idx, const int64_t* __restrict__ o_idx, int64_t n,
                int64_t rows_per_part, const float* __restrict__ C, int64_t ldc, float* __restrict__ parts) {
  const int r = blockIdx.x, R = (int)Rl.rows, Dr = Rl.dim, h = E.dim >> 1;
  const int64_t i0 = (int64_t)blockIdx.y * rows_per_part;
  const int64_t i1 = i0 + rows_per_part < n ? i0 + rows_per_part : n;
  const float* __restrict__ p = Rl.base + (int64_t)r * Rl.ld;
  float* __restrict__ out = parts + ((int64_t)blockIdx.y * R + r) * Dr;
  for (int k = threadIdx.x; k < Dr; k += NSP_ROW_THREADS) {
    const float pk = p[k];
    float acc = 0.f;
    for (int64_t i = i0; i < i1; ++i) {
      const float w = C[i * ldc + r];
      if (w == 0.f) continue;
      const float* __restrict__ s = E.base + s_idx[i] * E.ld;
      const float* __restrict__ o = E.base + o_idx[i] * E.ld;
      if constexpr (MODEL == B200KGE_TRANSE) {
        acc += transe_g<L2>(w, transe_x(s[k], pk, o[k]));      // dx/dp = 1
      } else {
        const RotElem e = rotate_elem(w, s[k], s[k + h], pk, o[k], o[k + h]);
        acc += e.g_im * e.q_re - e.g_re * e.q_im;            // d(q - o)/dtheta = (-q_im, q_re)
      }
    }
    out[k] = acc;
  }
}

// out[dst(j)] += sum_c parts[c][rel(j)] for j < u: (rel, dst) = (rows[j], j) over a row set of u = *count rows, or
// (j, j) over all R rows
__global__ void __launch_bounds__(NSP_ROW_THREADS)
ns_p_rel_add_kernel(const float* __restrict__ parts, int64_t ldp, int64_t part_stride, int nparts, int Dr,
                    const int64_t* __restrict__ rows, const int64_t* __restrict__ count, float* __restrict__ out,
                    int64_t ldo) {
  const int64_t j = blockIdx.x;
  if (count && j >= *count) return;
  const int64_t r = rows ? rows[j] : j;
  float* __restrict__ dst = out + j * ldo;
  for (int k = threadIdx.x; k < Dr; k += NSP_ROW_THREADS) {
    float acc = 0.f;
    for (int c = 0; c < nparts; ++c) acc += parts[c * part_stride + r * ldp + k];
    dst[k] += acc;
  }
}

}  // namespace

int ns_p_parts(int64_t n, int64_t R) {
  // about 4096 (relation, chunk) blocks at most: their partials stay below 4096 relation rows
  const int64_t by_rows = (n + NSP_ROWS_PER_PART - 1) / NSP_ROWS_PER_PART;
  const int64_t by_rel = R > 0 ? (B200KGE_NS_P_MAX_RELATIONS + R - 1) / R : 1;
  const int64_t p = by_rows < by_rel ? by_rows : by_rel;
  return (int)(p > 0 ? p : 1);
}

int launch_ns_p_unpack(const int64_t* triples, int64_t n, const int32_t* pe, int64_t* s_idx, int64_t* o_idx,
                       int64_t* s_dst, int64_t* o_dst, cudaStream_t st) {
  if (n == 0) return 0;
  ns_p_unpack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(triples, n, pe, s_idx, o_idx, s_dst, o_dst);
  B2K_LAUNCH_CHECK("ns_p_unpack_kernel");
  return 0;
}

int launch_ns_p_collapse(const int64_t* triples, const int64_t* neg, int64_t n, int64_t K, const float* G, int64_t ldg,
                         int64_t R, float* C, int64_t ldc, cudaStream_t st) {
  if (n == 0 || R == 0) return 0;
  ns_p_collapse_kernel<<<(unsigned)n, NSP_THREADS, 0, st>>>(triples, neg, K, G, ldg, (int)R, C, ldc);
  B2K_LAUNCH_CHECK("ns_p_collapse_kernel");
  return 0;
}

int launch_ns_p_distance(int model, float l_norm, const Rows& E, const Rows& Rl, const int64_t* s_idx,
                         const int64_t* o_idx, int64_t n, float* C, int64_t ldc, float* d_ent, int64_t lde,
                         const int64_t* s_dst, const int64_t* o_dst, float* parts, cudaStream_t st) {
  if (n == 0 || Rl.rows == 0) return 0;
  const int R = (int)Rl.rows, P = ns_p_parts(n, R);
  const int64_t rows_per_part = (n + P - 1) / P;
  const bool l2 = model == B200KGE_TRANSE && l_norm == 2.0f;
  if (l2) {
    ns_p_l2_scale_kernel<<<(unsigned)n, NSP_THREADS, 0, st>>>(E, Rl, s_idx, o_idx, R, C, ldc);
    B2K_LAUNCH_CHECK("ns_p_l2_scale_kernel");
  }
  const dim3 rel_grid((unsigned)R, (unsigned)P);
#define B2K_NSP(M, L)                                                                                               \
  ns_p_ent_kernel<M, L><<<(unsigned)n, NSP_ROW_THREADS, 0, st>>>(E, Rl, s_idx, o_idx, R, C, ldc, d_ent, lde, s_dst,  \
                                                                 o_dst);                                            \
  B2K_LAUNCH_CHECK("ns_p_ent_kernel");                                                                              \
  ns_p_rel_kernel<M, L><<<rel_grid, NSP_ROW_THREADS, 0, st>>>(E, Rl, s_idx, o_idx, n, rows_per_part, C, ldc, parts);  \
  B2K_LAUNCH_CHECK("ns_p_rel_kernel");
  if (model == B200KGE_TRANSE && l2) { B2K_NSP(B200KGE_TRANSE, true) }
  else if (model == B200KGE_TRANSE && l_norm == 1.0f) { B2K_NSP(B200KGE_TRANSE, false) }
  else if (model == B200KGE_ROTATE && l_norm == 1.0f) { B2K_NSP(B200KGE_ROTATE, false) }
  else { set_error("the P-slot distance backward covers TransE l_norm 1 and 2 and RotatE l_norm 1"); return B200KGE_ERR_UNSUPPORTED; }
#undef B2K_NSP
  return 0;
}

int launch_ns_p_rel_add(const float* parts, int64_t ldp, int64_t part_stride, int nparts, int64_t R, int Dr,
                        const int64_t* rows, const int64_t* count, float* out, int64_t ldo, cudaStream_t st) {
  if (R == 0) return 0;
  ns_p_rel_add_kernel<<<(unsigned)R, NSP_ROW_THREADS, 0, st>>>(parts, ldp, part_stride, nparts, Dr, rows, count, out,
                                                               ldo);
  B2K_LAUNCH_CHECK("ns_p_rel_add_kernel");
  return 0;
}

}  // namespace b200kge
