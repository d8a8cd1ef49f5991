// ns_dropout.cu — embedding dropout of the negative-sampling training step (train_negative_sampling.py:139-148 with
// LookupEmbedder._postprocess, lookup_embedder.py:96-105), S and O slots, without storing a mask.
//
// Columns of a slot's [n, 1+K] block and the kernels that serve them (mask layout: include/b200kge.h):
//   positive            t = i          mask row row_base + i                      (streams 6+6 slot + 0, 1, 2)
//   `triple` negatives  t = i K + j    mask row (row_base + i) K + j, all three    (streams 6+6 slot + 3, 4, 5)
//   `batch` negatives   fixed slots masked at row_base + i, the open slot at its entity id
// The positive and `triple` (and RESCAL's `batch`) run here as row-wise score_spo of logical triples, one warp each, whose
// operands name a table row and a mask row; the backward forms g * dscore/d(s~, p~, o~) per element and scatters
// mask * scale * that into d_ent / d_rel with atomics.  The other `batch` negatives run ns_kernel / ns_backward_kernel
// with a mask policy (rowwise.cu, grad.cu): q folded once per row from the masked fixed rows, sampled rows masked by id,
// the fixed rows' gradients reduced per row by the unfold and scattered once per row through their masks (below).
// Masks are regenerated where operands are loaded: a group of four elements k..k+3 (k % 4 == 0) is one Philox block.
#include "dropmask.cuh"
#include "fold.cuh"

namespace b200kge {

namespace {

// One operand of the logical triples: table row id(t) = idx[(t / div) * istride] (idx == NULL: t / div); mask row
// by_id ? id(t) : m.row_base + t / mdiv.
struct NsOp {
  const float* base;
  int64_t ld;
  int width;
  const int64_t* idx;
  int64_t istride, div, mdiv;
  int by_id;
  DropMask m;
  __device__ __forceinline__ int64_t id(int64_t t) const {
    const int64_t j = div > 1 ? t / div : t;
    return idx ? idx[j * istride] : j;
  }
  __device__ __forceinline__ uint64_t mrow(int64_t t, int64_t rid) const {
    return by_id ? (uint64_t)rid : (uint64_t)(m.row_base + (mdiv > 1 ? t / mdiv : t));
  }
};

// masked operand group: v[j] = x[k + j] * mk[j]  (the kept value x * (1 / (1 - p)), as dropout_gather_kernel)
struct G4 {
  float v[4], mk[4];
  __device__ __forceinline__ void load(const NsOp& op, const float* x, uint64_t mrow, int k) {
    drop_mask4(op.m, mrow, op.width, k, mk);
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = x[k + j] * mk[j];
  }
  // d[k + j] += mk[j] * dv[j]: the gradient of a masked element reaches the table through the same mask
  __device__ __forceinline__ void scatter(float* d, int k, const float (&dv)[4]) const {
#pragma unroll
    for (int j = 0; j < 4; ++j) if (mk[j] != 0.f) atomicAdd(d + k + j, dv[j] * mk[j]);
  }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// The lane's share of score_spo of logical triple t (BWD = false: returns the partial reduction, spo_kernel's
// arithmetic), or of its vector-Jacobian product (BWD = true: g = dL/dscore, nrm = the L2 distance of TransE L2;
// scatters into d_ent / d_rel and returns 0).  MAP: row-mapped gradient rows, d_ent + pe[id] * lde, d_rel + pr[id] * ldr.
template <int MODEL, bool BWD, bool MAP = false>
__device__ __forceinline__ float ns_drop_triple(const NsOp& S, const NsOp& P, const NsOp& O, int64_t t, int lane,
                                                float l_norm, float teps, float g, float nrm, float* __restrict__ d_ent,
                                                int64_t lde, float* __restrict__ d_rel, int64_t ldr,
                                                const int32_t* __restrict__ pe = nullptr,
                                                const int32_t* __restrict__ pr = nullptr) {
  const int64_t si = S.id(t), pi = P.id(t), oi = O.id(t);
  const uint64_t ms = S.mrow(t, si), mp = P.mrow(t, pi), mo = O.mrow(t, oi);
  const float* __restrict__ s = S.base + si * S.ld;
  const float* __restrict__ p = P.base + pi * P.ld;
  const float* __restrict__ o = O.base + oi * O.ld;
  float* ds = BWD ? d_ent + (MAP ? (int64_t)pe[si] : si) * lde : nullptr;
  float* dp = BWD ? d_rel + (MAP ? (int64_t)pr[pi] : pi) * ldr : nullptr;
  float* dO = BWD ? d_ent + (MAP ? (int64_t)pe[oi] : oi) * lde : nullptr;
  const int D = S.width, h = D >> 1;
  float acc = 0.f;
  if constexpr (MODEL == B200KGE_DISTMULT) {
    for (int k = 4 * lane; k < D; k += 128) {
      G4 a, b, c;
      a.load(S, s, ms, k); b.load(P, p, mp, k); c.load(O, o, mo, k);
      if constexpr (!BWD) {
#pragma unroll
        for (int j = 0; j < 4; ++j) acc = fmaf(a.v[j] * b.v[j], c.v[j], acc);
      } else {
        float da[4], db[4], dc[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) { da[j] = g * b.v[j] * c.v[j]; db[j] = g * a.v[j] * c.v[j]; dc[j] = g * a.v[j] * b.v[j]; }
        a.scatter(ds, k, da); b.scatter(dp, k, db); c.scatter(dO, k, dc);
      }
    }
  } else if constexpr (MODEL == B200KGE_COMPLEX) {
    for (int k = 4 * lane; k < h; k += 128) {
      G4 sr, si_, pr, pim, orr, oim;
      sr.load(S, s, ms, k); si_.load(S, s, ms, k + h); pr.load(P, p, mp, k); pim.load(P, p, mp, k + h);
      orr.load(O, o, mo, k); oim.load(O, o, mo, k + h);
      if constexpr (!BWD) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          acc += sr.v[j] * pr.v[j] * orr.v[j] + si_.v[j] * pr.v[j] * oim.v[j] + sr.v[j] * pim.v[j] * oim.v[j] -
                 si_.v[j] * pim.v[j] * orr.v[j];
      } else {
        float a0[4], a1[4], b0[4], b1[4], c0[4], c1[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float s_re = sr.v[j], s_im = si_.v[j], p_re = pr.v[j], p_im = pim.v[j], o_re = orr.v[j], o_im = oim.v[j];
          a0[j] = g * (p_re * o_re + p_im * o_im); a1[j] = g * (p_re * o_im - p_im * o_re);
          b0[j] = g * (s_re * o_re + s_im * o_im); b1[j] = g * (s_re * o_im - s_im * o_re);
          c0[j] = g * (s_re * p_re - s_im * p_im); c1[j] = g * (s_im * p_re + s_re * p_im);
        }
        sr.scatter(ds, k, a0); si_.scatter(ds, k + h, a1); pr.scatter(dp, k, b0); pim.scatter(dp, k + h, b1);
        orr.scatter(dO, k, c0); oim.scatter(dO, k + h, c1);
      }
    }
  } else if constexpr (MODEL == B200KGE_SIMPLE) {
    for (int k = 4 * lane; k < h; k += 128) {
      G4 s0, s1, p0, p1, o0, o1;
      s0.load(S, s, ms, k); s1.load(S, s, ms, k + h); p0.load(P, p, mp, k); p1.load(P, p, mp, k + h);
      o0.load(O, o, mo, k); o1.load(O, o, mo, k + h);
      if constexpr (!BWD) {
#pragma unroll
        for (int j = 0; j < 4; ++j) acc += 0.5f * (s0.v[j] * p0.v[j] * o1.v[j] + s1.v[j] * p1.v[j] * o0.v[j]);
      } else {
        float a0[4], a1[4], b0[4], b1[4], c0[4], c1[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float gh = 0.5f * g;
          a0[j] = gh * p0.v[j] * o1.v[j]; a1[j] = gh * p1.v[j] * o0.v[j];
          b0[j] = gh * s0.v[j] * o1.v[j]; b1[j] = gh * s1.v[j] * o0.v[j];
          c1[j] = gh * s0.v[j] * p0.v[j]; c0[j] = gh * s1.v[j] * p1.v[j];
        }
        s0.scatter(ds, k, a0); s1.scatter(ds, k + h, a1); p0.scatter(dp, k, b0); p1.scatter(dp, k + h, b1);
        o0.scatter(dO, k, c0); o1.scatter(dO, k + h, c1);
      }
    }
  } else if constexpr (MODEL == B200KGE_CP) {
    for (int k = 4 * lane; k < h; k += 128) {
      G4 a, b, c;
      a.load(S, s, ms, k); b.load(P, p, mp, k); c.load(O, o, mo, k + h);
      if constexpr (!BWD) {
#pragma unroll
        for (int j = 0; j < 4; ++j) acc = fmaf(a.v[j] * b.v[j], c.v[j], acc);
      } else {
        float da[4], db[4], dc[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) { da[j] = g * b.v[j] * c.v[j]; db[j] = g * a.v[j] * c.v[j]; dc[j] = g * a.v[j] * b.v[j]; }
        a.scatter(ds, k, da); b.scatter(dp, k, db); c.scatter(dO, k + h, dc);
      }
    }
  } else if constexpr (MODEL == B200KGE_RESCAL) {
    // score = sum_{r,c} s~_r M~_rc o~_c over float4 groups of the D x D relation row (rescal.py:27-35); correctness
    // over speed: the scalar masks of s~_r and o~_c are regenerated per group
    const int dd = D * D;
    for (int e = 4 * lane; e < dd; e += 128) {
      const int r = e / D, c = e - r * D;
      G4 M, oc;
      M.load(P, p, mp, e); oc.load(O, o, mo, c);
      const float msr = drop_mask1(S.m, ms, D, r), sr = s[r] * msr;
      if constexpr (!BWD) {
#pragma unroll
        for (int j = 0; j < 4; ++j) acc = fmaf(sr * M.v[j], oc.v[j], acc);
      } else {
        float dM[4], dc[4], dsr = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          dM[j] = g * sr * oc.v[j]; dc[j] = g * sr * M.v[j];
          dsr = fmaf(M.v[j], oc.v[j], dsr);
        }
        M.scatter(dp, e, dM); oc.scatter(dO, c, dc);
        if (msr != 0.f) atomicAdd(ds + r, g * dsr * msr);
      }
    }
  } else if constexpr (MODEL == B200KGE_TRANSE) {
    for (int k = 4 * lane; k < D; k += 128) {
      G4 a, b, c;
      a.load(S, s, ms, k); b.load(P, p, mp, k); c.load(O, o, mo, k);
      float d[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) d[j] = ((a.v[j] + b.v[j]) - c.v[j]) + teps;   // F.pairwise_distance eps, transe.py:18
      if constexpr (!BWD) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (l_norm == 1.0f) acc += fabsf(d[j]);
          else acc = fmaf(d[j], d[j], acc);
        }
      } else {        // z = -||d||: dz/ds = dz/dp = -dz/do = -sign(d) (L1) | -d / ||d|| (L2)
        float w[4], nw[4];
        const float inv = (nrm > 0.f) ? g / nrm : 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          w[j] = (l_norm == 1.0f) ? ((d[j] > 0.f) ? -g : (d[j] < 0.f ? g : 0.f)) : -d[j] * inv;
          nw[j] = -w[j];
        }
        a.scatter(ds, k, w); b.scatter(dp, k, w); c.scatter(dO, k, nw);
      }
    }
  } else {  // ROTATE, l_norm 1: z = -sum_k |s_k e^{i p_k} - o_k|
    for (int k = 4 * lane; k < h; k += 128) {
      G4 sr, sim, ph, orr, oim;
      sr.load(S, s, ms, k); sim.load(S, s, ms, k + h); ph.load(P, p, mp, k); orr.load(O, o, mo, k);
      oim.load(O, o, mo, k + h);
      float a0[4], a1[4], b0[4], c0[4], c1[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float sn, cs;
        sincosf(ph.v[j], &sn, &cs);
        const float s_re = sr.v[j], s_im = sim.v[j];
        const float q_re = s_re * cs - s_im * sn, q_im = s_re * sn + s_im * cs;
        const float d_re = q_re - orr.v[j], d_im = q_im - oim.v[j];
        const float m = sqrtf(fmaf(d_im, d_im, d_re * d_re));
        if constexpr (!BWD) {
          acc += m;
        } else {
          const float inv = (m > 0.f) ? g / m : 0.f;
          const float w_re = -d_re * inv, w_im = -d_im * inv;        // dL/dq
          a0[j] = w_re * cs + w_im * sn; a1[j] = -w_re * sn + w_im * cs;
          b0[j] = w_re * (-s_re * sn - s_im * cs) + w_im * (s_re * cs - s_im * sn);
          c0[j] = -w_re; c1[j] = -w_im;
        }
      }
      if constexpr (BWD) {
        sr.scatter(ds, k, a0); sim.scatter(ds, k + h, a1); ph.scatter(dp, k, b0);
        orr.scatter(dO, k, c0); oim.scatter(dO, k + h, c1);
      }
    }
  }
  return acc;
}

template <int MODEL>
__device__ __forceinline__ float ns_drop_finish(float acc, float l_norm) {
  if constexpr (MODEL == B200KGE_TRANSE || MODEL == B200KGE_ROTATE) return (l_norm == 1.0f) ? -acc : -sqrtf(acc);
  return acc;
}

// forward: out[(t / out_div) * ldo + col0 + t % out_div] = score of logical triple t; one warp per triple
template <int MODEL>
__global__ void __launch_bounds__(256)
ns_drop_score_kernel(NsOp S, NsOp P, NsOp O, int64_t N, float l_norm, float teps, float* __restrict__ out, int64_t ldo,
                     int64_t out_div, int64_t col0) {
  const int lane = threadIdx.x & 31;
  const int64_t t = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= N) return;
  float acc = warp_sum(ns_drop_triple<MODEL, false>(S, P, O, t, lane, l_norm, teps, 0.f, 0.f, nullptr, 0, nullptr, 0));
  if (lane == 0) {
    const int64_t r = t / out_div, c = t - r * out_div;
    out[r * ldo + col0 + c] = ns_drop_finish<MODEL>(acc, l_norm);
  }
}

// backward: g = G[(t / out_div) * ldg + col0 + t % out_div]; TransE L2 first recomputes the distance
template <int MODEL, bool MAP>
__device__ __forceinline__ void ns_drop_backward_body(const NsOp& S, const NsOp& P, const NsOp& O, int64_t N, float l_norm,
                                                      float teps, const float* __restrict__ G, int64_t ldg,
                                                      int64_t out_div, int64_t col0, float* __restrict__ d_ent,
                                                      int64_t lde, float* __restrict__ d_rel, int64_t ldr,
                                                      const int32_t* __restrict__ pe, const int32_t* __restrict__ pr) {
  const int lane = threadIdx.x & 31;
  const int64_t t = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= N) return;
  const int64_t r = t / out_div, c = t - r * out_div;
  const float g = G[r * ldg + col0 + c];
  if (g == 0.f) return;
  float nrm = 0.f;
  if (MODEL == B200KGE_TRANSE && l_norm == 2.0f)
    nrm = sqrtf(warp_sum(ns_drop_triple<MODEL, false>(S, P, O, t, lane, l_norm, teps, 0.f, 0.f, nullptr, 0, nullptr, 0)));
  ns_drop_triple<MODEL, true, MAP>(S, P, O, t, lane, l_norm, teps, g, nrm, d_ent, lde, d_rel, ldr, pe, pr);
}

template <int MODEL>
__global__ void __launch_bounds__(256)
ns_drop_backward_kernel(NsOp S, NsOp P, NsOp O, int64_t N, float l_norm, float teps, const float* __restrict__ G,
                        int64_t ldg, int64_t out_div, int64_t col0, float* __restrict__ d_ent, int64_t lde,
                        float* __restrict__ d_rel, int64_t ldr) {
  ns_drop_backward_body<MODEL, false>(S, P, O, N, l_norm, teps, G, ldg, out_div, col0, d_ent, lde, d_rel, ldr, nullptr,
                                      nullptr);
}

template <int MODEL>
__global__ void __launch_bounds__(256)
ns_drop_backward_rows_kernel(NsOp S, NsOp P, NsOp O, int64_t N, float l_norm, float teps, const float* __restrict__ G,
                             int64_t ldg, int64_t out_div, int64_t col0, float* __restrict__ d_ent, int64_t lde,
                             float* __restrict__ d_rel, int64_t ldr, const int32_t* __restrict__ pe,
                             const int32_t* __restrict__ pr) {
  ns_drop_backward_body<MODEL, true>(S, P, O, N, l_norm, teps, G, ldg, out_div, col0, d_ent, lde, d_rel, ldr, pe, pr);
}

// dst[i, :] = mask(row_base + i, :) * tab[tri[3 i + c], :]  (width % 4 == 0; one thread per four-element group)
__global__ void __launch_bounds__(256)
ns_drop_gather_kernel(DropMask m, const float* __restrict__ base, int64_t ld, int width, const int64_t* __restrict__ tri,
                      int c, int64_t n, float* __restrict__ dst) {
  const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, w4 = width >> 2;
  if (g >= n * w4) return;
  const int64_t i = g / w4;
  const int k = (int)(g - i * w4) * 4;
  float mk[4];
  drop_mask4(m, (uint64_t)(m.row_base + i), width, k, mk);
  const float* src = base + tri[3 * i + c] * ld;
#pragma unroll
  for (int j = 0; j < 4; ++j) dst[i * width + k + j] = src[k + j] * mk[j];
}

// d[tri[3 i + c], :] += mask(row_base + i, :) * src[i, :]  (atomic: rows repeat; MAP: row pos[tri[3 i + c]] of d)
template <bool MAP>
__device__ __forceinline__ void ns_drop_scatter_body(const DropMask& m, const float* __restrict__ src, int width,
                                                     const int64_t* __restrict__ tri, int c, int64_t n,
                                                     float* __restrict__ d, int64_t ldd, const int32_t* __restrict__ pos) {
  const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, w4 = width >> 2;
  if (g >= n * w4) return;
  const int64_t i = g / w4;
  const int k = (int)(g - i * w4) * 4;
  float mk[4];
  drop_mask4(m, (uint64_t)(m.row_base + i), width, k, mk);
  const int64_t id = tri[3 * i + c];
  float* dst = d + (MAP ? (int64_t)pos[id] : id) * ldd;
#pragma unroll
  for (int j = 0; j < 4; ++j) if (mk[j] != 0.f) atomicAdd(dst + k + j, src[i * width + k + j] * mk[j]);
}

__global__ void __launch_bounds__(256)
ns_drop_scatter_kernel(DropMask m, const float* __restrict__ src, int width, const int64_t* __restrict__ tri, int c,
                       int64_t n, float* __restrict__ d, int64_t ldd) {
  ns_drop_scatter_body<false>(m, src, width, tri, c, n, d, ldd, nullptr);
}

__global__ void __launch_bounds__(256)
ns_drop_scatter_rows_kernel(DropMask m, const float* __restrict__ src, int width, const int64_t* __restrict__ tri, int c,
                            int64_t n, float* __restrict__ d, int64_t ldd, const int32_t* __restrict__ pos) {
  ns_drop_scatter_body<true>(m, src, width, tri, c, n, d, ldd, pos);
}

inline unsigned groups_grid(int64_t n, int width) { return (unsigned)((n * (width / 4) + 255) / 256); }

NsOp ns_op(const Rows& tab, const int64_t* idx, int64_t istride, int64_t div, const DropMask& m, int64_t mdiv,
           int by_id) {
  NsOp op;
  op.base = tab.base; op.ld = tab.ld; op.width = tab.dim; op.idx = idx; op.istride = istride; op.div = div;
  op.mdiv = mdiv; op.by_id = by_id; op.m = m;
  return op;
}

int launch_drop_triples(int model, bool bwd, const NsOp& S, const NsOp& P, const NsOp& O, int64_t N, float l_norm,
                        float teps, const float* G, int64_t ldg, float* out, int64_t ldo, int64_t out_div,
                        int64_t col0, float* d_ent, int64_t lde, float* d_rel, int64_t ldr, cudaStream_t st,
                        const int32_t* pe, const int32_t* pr) {
  if (N == 0) return 0;
  const int64_t blocks = (N + 7) / 8;
  if (blocks > 2147483647LL) { set_error("too many triples"); return B200KGE_ERR_UNSUPPORTED; }
  dim3 grid((unsigned)blocks), block(256);
#define B2K_NSD(M)                                                                                                  \
  case M:                                                                                                           \
    if (bwd && pe) ns_drop_backward_rows_kernel<M><<<grid, block, 0, st>>>(S, P, O, N, l_norm, teps, G, ldg,        \
                                                                           out_div, col0, d_ent, lde, d_rel, ldr,   \
                                                                           pe, pr);                                 \
    else if (bwd) ns_drop_backward_kernel<M><<<grid, block, 0, st>>>(S, P, O, N, l_norm, teps, G, ldg, out_div,     \
                                                                     col0, d_ent, lde, d_rel, ldr);                 \
    else ns_drop_score_kernel<M><<<grid, block, 0, st>>>(S, P, O, N, l_norm, teps, out, ldo, out_div, col0);        \
    break;
  switch (model) {
    B2K_NSD(B200KGE_COMPLEX) B2K_NSD(B200KGE_DISTMULT) B2K_NSD(B200KGE_SIMPLE) B2K_NSD(B200KGE_CP)
    B2K_NSD(B200KGE_RESCAL) B2K_NSD(B200KGE_TRANSE) B2K_NSD(B200KGE_ROTATE)
    default: set_error("unknown model %d", model); return B200KGE_ERR_INVALID;
  }
#undef B2K_NSD
  B2K_LAUNCH_CHECK(bwd ? "ns_drop_backward_kernel" : "ns_drop_score_kernel");
  return 0;
}

}  // namespace

size_t ns_dropout_workspace_bytes(int model, int64_t n, int32_t D) {
  const int64_t Dr = relation_dim(model, D), ldq = (D + 31) / 32 * 32;
  const auto up = [](int64_t b) { return (size_t)((b + 255) / 256 * 256); };
  return up(n * D * 4) * 2 + up(n * Dr * 4) * 2 + up(n * ldq * 4) + up(n * 3 * 8);
}

int launch_ns_dropout(int model, float l_norm, const Rows& ent, const Rows& rel, const int64_t* triples, int slot,
                      const int64_t* neg, int64_t n, int64_t K, int impl, const NsDropKeys& keys, const float* G,
                      int64_t ldg, float* out, int64_t ldo, float* d_ent, int64_t lde, float* d_rel, int64_t ldr,
                      void* workspace, size_t workspace_bytes, cudaStream_t st, const int32_t* pe,
                      const int32_t* pr) {
  const bool bwd = G != nullptr;
  const int64_t rb = keys.row_base;
  const int sb = 6 + 6 * slot;                         // first stream of the slot
  auto mk = [&](bool is_rel, int j, int64_t row_base) {
    DropMask m = is_rel ? keys.rel : keys.ent;
    m.stream = sb + j; m.row_base = row_base;
    return m;
  };
  const float eps = (model == B200KGE_TRANSE) ? 1e-6f : 0.f;
  // positive column: score_spo(s, p, o) over the n rows, draws 0-2
  NsOp S = ns_op(ent, triples + 0, 3, 1, mk(false, 0, rb), 1, 0);
  NsOp P = ns_op(rel, triples + 1, 3, 1, mk(true, 1, rb), 1, 0);
  NsOp O = ns_op(ent, triples + 2, 3, 1, mk(false, 2, rb), 1, 0);
  int rc = launch_drop_triples(model, bwd, S, P, O, n, l_norm, eps, G, ldg, out, ldo, 1, 0, d_ent, lde, d_rel, ldr, st,
                               pe, pr);
  if (rc || K == 0) return rc;
  const bool triple = impl == B200KGE_NS_TRIPLE;
  if (!triple && model != B200KGE_RESCAL) {
    // `batch`: ns_kernel / ns_backward_kernel with the mask policy — q folded once per row from the masked fixed rows,
    // every sampled row masked by its id (draw 3 + slot), the fixed rows' gradient reduced per row by the unfold
    const int ca = (slot == 2) ? 0 : 2;                // the fixed entity column
    const DropMask ma = mk(false, 3 + ca, rb), mp = mk(true, 4, rb), mt = mk(false, 3 + slot, 0);
    if (!bwd) return launch_ns_masked(model, l_norm, ent, rel, triples, slot, neg, n, K, ma, mp, mt, out, ldo, 1, st);
    const int D = ent.dim, Dr = rel.dim;
    const int64_t ldq = (D + 31) / 32 * 32;
    if (workspace_bytes < ns_dropout_workspace_bytes(model, n, D) || !workspace) {
      set_error("workspace too small (see b200kge_ns_backward_workspace_bytes)");
      return B200KGE_ERR_WORKSPACE;
    }
    uint8_t* w = (uint8_t*)workspace;
    const auto take = [&](int64_t bytes) { uint8_t* r = w; w += (bytes + 255) / 256 * 256; return r; };
    float* Am = (float*)take(n * D * 4);
    float* Pm = (float*)take(n * Dr * 4);
    float* dA = (float*)take(n * D * 4);
    float* dP = (float*)take(n * Dr * 4);
    float* dQ = (float*)take(n * ldq * 4);
    int64_t* tri = (int64_t*)take(n * 3 * 8);
    ns_drop_gather_kernel<<<groups_grid(n, D), 256, 0, st>>>(ma, ent.base, ent.ld, D, triples, ca, n, Am);
    B2K_LAUNCH_CHECK("ns_drop_gather_kernel");
    ns_drop_gather_kernel<<<groups_grid(n, Dr), 256, 0, st>>>(mp, rel.base, rel.ld, Dr, triples, 1, n, Pm);
    B2K_LAUNCH_CHECK("ns_drop_gather_kernel");
    Rows a{Am, nullptr, n, D, D}, p{Pm, nullptr, n, Dr, Dr};
    if ((rc = launch_ns_backward_masked(model, l_norm, a, p, ent, slot, neg, n, K, mt, G, ldg, d_ent, lde, dQ, ldq, tri,
                                        dA, dP, st, pe))) return rc;
    if (pe) {
      ns_drop_scatter_rows_kernel<<<groups_grid(n, D), 256, 0, st>>>(ma, dA, D, triples, ca, n, d_ent, lde, pe);
      B2K_LAUNCH_CHECK("ns_drop_scatter_rows_kernel");
      ns_drop_scatter_rows_kernel<<<groups_grid(n, Dr), 256, 0, st>>>(mp, dP, Dr, triples, 1, n, d_rel, ldr, pr);
      B2K_LAUNCH_CHECK("ns_drop_scatter_rows_kernel");
      return 0;
    }
    ns_drop_scatter_kernel<<<groups_grid(n, D), 256, 0, st>>>(ma, dA, D, triples, ca, n, d_ent, lde);
    B2K_LAUNCH_CHECK("ns_drop_scatter_kernel");
    ns_drop_scatter_kernel<<<groups_grid(n, Dr), 256, 0, st>>>(mp, dP, Dr, triples, 1, n, d_rel, ldr);
    B2K_LAUNCH_CHECK("ns_drop_scatter_kernel");
    return 0;
  }
  // `triple` (and RESCAL's `batch`, whose D x D relation row is not copied per row): logical triple t = i K + j, the
  // open slot reads neg[t]; draws 3-5
  NsOp ops[3];
  for (int c = 0; c < 3; ++c) {
    const Rows& tab = (c == 1) ? rel : ent;
    if (c == slot)                                      // the sampled entity: its own row per triple | its id
      ops[c] = ns_op(tab, neg, 1, 1, mk(false, 3 + c, triple ? rb * K : 0), 1, triple ? 0 : 1);
    else                                                // a fixed operand of row i = t / K
      ops[c] = ns_op(tab, triples + c, 3, K, mk(c == 1, 3 + c, triple ? rb * K : rb), triple ? 1 : K, 0);
  }
  return launch_drop_triples(model, bwd, ops[0], ops[1], ops[2], n * K, l_norm, triple ? eps : 0.f, G, ldg, out, ldo,
                             K, 1, d_ent, lde, d_rel, ldr, st, pe, pr);
}

}  // namespace b200kge
