// rowwise.cu — row-wise triple scoring (combine="spo") and fused negative-sample scoring.
//
//  * spo_kernel: one warp per triple; gathers the three rows by index and reduces the model's
//    trilinear form / distance in registers.  Replaces KgeModel.score_spo (kge_model.py:663-680) +
//    score_emb(combine="spo") of complex.py:34-35, distmult.py:16-17, simple.py:21-23,
//    cp.py:21-22, rescal.py:27-35, transe.py:17-18, rotate.py:30-41.
//  * ns_kernel: BatchNegativeSample.score (sampler.py:263-344) for the S and O slots: the CTA folds
//    (other entity, relation) of its positive triple into q once, then each warp gathers sampled
//    rows and reduces pair(q, row) — the gather of the sampled indexes is fused with the
//    per-negative dot/distance; nothing of size [n*K, D] is materialised (the reference's `triple`
//    implementation gathers 3 x [n*K, D]).  The P slot goes through spo_kernel with row divisors.
#include "dropmask.cuh"
#include "fold.cuh"

namespace b200kge {

namespace {

struct RowsDiv {
  Rows r;
  int64_t div;  // logical row t reads operand row t / div
  __device__ __forceinline__ const float* row(int64_t t) const { return r.row(div > 1 ? t / div : t); }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

template <int MODEL>
__global__ void __launch_bounds__(256)
spo_kernel(RowsDiv S, RowsDiv Pr, RowsDiv O, int64_t n, float l_norm, float* __restrict__ out,
           int64_t out_ld, int64_t out_div, int64_t col0) {
  const int lane = threadIdx.x & 31;
  const int64_t t = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= n) return;
  const float* __restrict__ s = S.row(t);
  const float* __restrict__ p = Pr.row(t);
  const float* __restrict__ o = O.row(t);
  const int D = S.r.dim, h = D >> 1;
  float acc = 0.f;
  if constexpr (MODEL == B200KGE_COMPLEX) {
    for (int k = lane; k < h; k += 32) {
      const float s_re = s[k], s_im = s[k + h], p_re = p[k], p_im = p[k + h], o_re = o[k], o_im = o[k + h];
      acc += s_re * p_re * o_re + s_im * p_re * o_im + s_re * p_im * o_im - s_im * p_im * o_re;
    }
  } else if constexpr (MODEL == B200KGE_DISTMULT) {
    for (int k = lane; k < D; k += 32) acc = fmaf(s[k] * p[k], o[k], acc);
  } else if constexpr (MODEL == B200KGE_SIMPLE) {
    for (int k = lane; k < h; k += 32)
      acc += 0.5f * (s[k] * p[k] * o[k + h] + s[k + h] * p[k + h] * o[k]);
  } else if constexpr (MODEL == B200KGE_CP) {
    for (int k = lane; k < h; k += 32) acc = fmaf(s[k] * p[k], o[k + h], acc);
  } else if constexpr (MODEL == B200KGE_RESCAL) {
    const int64_t dd = (int64_t)D * D;
    for (int64_t e = lane; e < dd; e += 32) {
      const int r = (int)(e / D), c = (int)(e - (int64_t)r * D);
      acc = fmaf(s[r] * p[e], o[c], acc);
    }
  } else if constexpr (MODEL == B200KGE_TRANSE) {
    for (int k = lane; k < D; k += 32) {
      const float d = fabsf(((s[k] + p[k]) - o[k]) + 1e-6f);  // F.pairwise_distance eps, transe.py:18
      if (l_norm == 1.0f) acc += d;
      else if (l_norm == 2.0f) acc = fmaf(d, d, acc);
      else acc += __powf(d, l_norm);
    }
  } else {  // ROTATE
    for (int k = lane; k < h; k += 32) {
      float sn, c;
      sincosf(p[k], &sn, &c);
      const float q_re = s[k] * c - s[k + h] * sn, q_im = s[k] * sn + s[k + h] * c;
      const float d_re = q_re - o[k], d_im = q_im - o[k + h];
      const float m2 = fmaf(d_im, d_im, d_re * d_re);
      if (l_norm == 1.0f) acc += sqrtf(m2);
      else acc += __powf(m2, 0.5f * l_norm);
    }
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    if constexpr (MODEL == B200KGE_TRANSE || MODEL == B200KGE_ROTATE) {
      if (l_norm == 1.0f) acc = -acc;
      else if (l_norm == 2.0f) acc = -sqrtf(acc);
      else acc = -powf(acc, 1.0f / l_norm);
    }
    // logical triple t lands at out[(t / out_div) * out_ld + col0 + t % out_div]
    int64_t r = t, c = 0;
    if (out_div > 1) { r = t / out_div; c = t - r * out_div; }
    out[r * out_ld + col0 + c] = acc;
  }
}

int launch_spo_div(int model, float l_norm, const RowsDiv& s, const RowsDiv& p, const RowsDiv& o,
                   int64_t n, float* out, int64_t out_ld, int64_t out_div, int64_t col0,
                   cudaStream_t st) {
  if (n == 0) return 0;
  const int wpb = 8;
  const int64_t blocks = (n + wpb - 1) / wpb;
  if (blocks > 2147483647LL) { set_error("too many triples"); return B200KGE_ERR_UNSUPPORTED; }
  dim3 grid((unsigned)blocks), block(wpb * 32);
#define B2K_SPO(M) case M: spo_kernel<M><<<grid, block, 0, st>>>(s, p, o, n, l_norm, out, out_ld, out_div, col0); break;
  switch (model) {
    B2K_SPO(B200KGE_COMPLEX) B2K_SPO(B200KGE_DISTMULT) B2K_SPO(B200KGE_SIMPLE) B2K_SPO(B200KGE_CP)
    B2K_SPO(B200KGE_RESCAL) B2K_SPO(B200KGE_TRANSE) B2K_SPO(B200KGE_ROTATE)
    default: set_error("unknown model %d", model); return B200KGE_ERR_INVALID;
  }
#undef B2K_SPO
  B2K_LAUNCH_CHECK("spo_kernel");
  return 0;
}

// ---------------------------------------------------------------------------------------------
constexpr int NS_WARPS = 8, NS_PER_BLOCK = 256;

__device__ __forceinline__ float sqrt_approx(float x) {
  float y;
  asm("sqrt.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// pair(q, t) partial sum of one lane over a row, 16-byte loads: lane handles float4 groups lane, lane + 32, ...
// (complex pair ops: the re group at k4 pairs with the im group at k4 + hk/4)
// MASK: the sampled row is entity `e` of a dropout draw `tm` over rows of width `tw`, its group k starting at column
// col_off + 4 k (the `batch` negatives of b200kge_ns_score_dropout: one mask per entity id)
__device__ __forceinline__ float4 ns_masked(float4 t, const DropMask& tm, int64_t e, int tw, int col) {
  float mk[4];
  drop_mask4(tm, (uint64_t)e, tw, col, mk);
  t.x *= mk[0]; t.y *= mk[1]; t.z *= mk[2]; t.w *= mk[3];
  return t;
}

template <int PAIR, bool MASK = false>
__device__ __forceinline__ float ns_row_partial(const float4* __restrict__ q4, const float4* __restrict__ t4, int n4, int lane,
                                                const DropMask& tm = DropMask{}, int64_t e = 0, int tw = 0, int col_off = 0) {
  float acc = 0.f;
  if constexpr (PAIR == PAIR_CMOD_L1) {
    const int h4 = n4 >> 1;
    for (int k = lane; k < h4; k += 32) {
      float4 tr = __ldg(t4 + k), ti = __ldg(t4 + k + h4);
      if constexpr (MASK) { tr = ns_masked(tr, tm, e, tw, col_off + 4 * k); ti = ns_masked(ti, tm, e, tw, col_off + 4 * (k + h4)); }
      const float4 qr = q4[k], qi = q4[k + h4];
      float dr, di;
      dr = qr.x - tr.x; di = qi.x - ti.x; acc += sqrt_approx(fmaf(di, di, dr * dr));
      dr = qr.y - tr.y; di = qi.y - ti.y; acc += sqrt_approx(fmaf(di, di, dr * dr));
      dr = qr.z - tr.z; di = qi.z - ti.z; acc += sqrt_approx(fmaf(di, di, dr * dr));
      dr = qr.w - tr.w; di = qi.w - ti.w; acc += sqrt_approx(fmaf(di, di, dr * dr));
    }
  } else {
    for (int k = lane; k < n4; k += 32) {
      float4 t = __ldg(t4 + k);
      if constexpr (MASK) t = ns_masked(t, tm, e, tw, col_off + 4 * k);
      const float4 q = q4[k];
      if constexpr (PAIR == PAIR_DOT) {
        acc = fmaf(q.x, t.x, acc); acc = fmaf(q.y, t.y, acc); acc = fmaf(q.z, t.z, acc); acc = fmaf(q.w, t.w, acc);
      } else if constexpr (PAIR == PAIR_L1) {
        acc += fabsf(q.x - t.x); acc += fabsf(q.y - t.y); acc += fabsf(q.z - t.z); acc += fabsf(q.w - t.w);
      } else {  // PAIR_L2
        float d;
        d = q.x - t.x; acc = fmaf(d, d, acc); d = q.y - t.y; acc = fmaf(d, d, acc);
        d = q.z - t.z; acc = fmaf(d, d, acc); d = q.w - t.w; acc = fmaf(d, d, acc);
      }
    }
  }
  return acc;
}

// the warp's rows kk, kk + NS_WARPS, ... of this CTA's range, TWO at a time (both rows' loads are in flight together)
template <int PAIR, bool MASK = false>
__device__ __forceinline__ void ns_rows_vec(const float* q, const Rows& table, int col_off, int K, const int64_t* __restrict__ neg_row,
                                            int64_t k0, int64_t kend, int warp, int lane, float* __restrict__ out_row,
                                            const DropMask& tm = DropMask{}) {
  const float4* q4 = reinterpret_cast<const float4*>(q);
  const int n4 = K >> 2;
  for (int64_t kk = k0 + warp; kk < kend; kk += 2 * NS_WARPS) {
    const int64_t kb = kk + NS_WARPS;
    const bool two = kb < kend;
    const int64_t e0 = __ldg(neg_row + kk), e1 = two ? __ldg(neg_row + kb) : e0;
    const float4* t0 = reinterpret_cast<const float4*>(table.base + e0 * table.ld + col_off);
    const float4* t1 = reinterpret_cast<const float4*>(table.base + e1 * table.ld + col_off);
    float a0 = ns_row_partial<PAIR, MASK>(q4, t0, n4, lane, tm, e0, table.dim, col_off);
    float a1 = two ? ns_row_partial<PAIR, MASK>(q4, t1, n4, lane, tm, e1, table.dim, col_off) : 0.f;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      a0 += __shfl_xor_sync(0xffffffffu, a0, off);
      a1 += __shfl_xor_sync(0xffffffffu, a1, off);
    }
    if (lane == 0) {
      if constexpr (PAIR == PAIR_L1 || PAIR == PAIR_CMOD_L1) { a0 = -a0; a1 = -a1; }
      else if constexpr (PAIR == PAIR_L2) { a0 = -sqrtf(a0); a1 = -sqrtf(a1); }
      out_row[kk] = a0;
      if (two) out_row[kb] = a1;
    }
  }
}

// Dropout of the `batch` negatives (ns_kernel_masked): the fixed entity row (draw `a`, mask row a.row_base + i) and the
// relation row (draw `p`) are masked once per row before the fold, every sampled row by its entity id (draw `t`).
struct NsRowMasks {
  DropMask a, p, t;
};

template <int MODEL, bool MASK>
__device__ __forceinline__ void ns_body(const Rows& A, const Rows& Pr, const Rows& table, int sp, const int64_t* __restrict__ neg,
                                        int64_t Kneg, const Folded& f, float l_norm, float* __restrict__ out, int64_t ldo,
                                        int col0, int vec_ok, const NsRowMasks& mk, const int64_t* __restrict__ tri = nullptr,
                                        int ca = 0) {
  extern __shared__ __align__(16) float sh[];  // q[K] (+ entity row for RESCAL) (MASK: + masked entity and relation rows)
  const int64_t i = blockIdx.x;
  const int D = A.dim, h = D >> 1, K = f.K;
  const float* __restrict__ a = A.row(i);
  const float* __restrict__ p = Pr.row(i);
  float* q = sh;
  if constexpr (MASK) {       // the fold reads masked copies in shared memory (D, Dr multiples of 4)
    a = A.base + tri[3 * i + ca] * A.ld;      // the fixed rows of triple i: entity column ca, relation column 1
    p = Pr.base + tri[3 * i + 1] * Pr.ld;
    float* sa = sh + ((K + 3) & ~3);
    float* spr = sa + D;
    for (int g = 4 * threadIdx.x; g < D + Pr.dim; g += 4 * blockDim.x) {
      const bool ent = g < D;
      const int k = ent ? g : g - D;
      float m4[4];
      drop_mask4(ent ? mk.a : mk.p, (uint64_t)((ent ? mk.a.row_base : mk.p.row_base) + i), ent ? D : Pr.dim, k, m4);
      const float* src = ent ? a : p;
      float* dst = ent ? sa : spr;
#pragma unroll
      for (int j = 0; j < 4; ++j) dst[k + j] = src[k + j] * m4[j];
    }
    __syncthreads();
    a = sa; p = spr;
  }
  if constexpr (MODEL == B200KGE_RESCAL) {
    float* sa = sh + ((K + 3) & ~3);
    for (int k = threadIdx.x; k < D; k += blockDim.x) sa[k] = a[k];
    __syncthreads();
    fold_rescal_block(sp != 0, sa, p, D, [&](int k, float v) { q[k] = v; });
  } else {
    for (int k = threadIdx.x; k < K; k += blockDim.x) q[k] = fold_element<MODEL>(sp != 0, a, p, k, h);
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t k0 = (int64_t)blockIdx.y * NS_PER_BLOCK;
  const int64_t kend = (k0 + NS_PER_BLOCK < Kneg) ? k0 + NS_PER_BLOCK : Kneg;
  const int64_t* __restrict__ neg_row = neg + i * Kneg;
  float* __restrict__ out_row = out + i * ldo + col0;
  if (vec_ok) {
    // 16-byte loads, two rows in flight per warp (the scalar form below gathered at 3.4 TB/s from an L2-resident table)
    switch (f.pair_op) {
      case PAIR_DOT:     ns_rows_vec<PAIR_DOT, MASK>(q, table, f.col_off, K, neg_row, k0, kend, warp, lane, out_row, mk.t); return;
      case PAIR_L1:      ns_rows_vec<PAIR_L1, MASK>(q, table, f.col_off, K, neg_row, k0, kend, warp, lane, out_row, mk.t); return;
      case PAIR_L2:      ns_rows_vec<PAIR_L2, MASK>(q, table, f.col_off, K, neg_row, k0, kend, warp, lane, out_row, mk.t); return;
      case PAIR_CMOD_L1: ns_rows_vec<PAIR_CMOD_L1, MASK>(q, table, f.col_off, K, neg_row, k0, kend, warp, lane, out_row, mk.t); return;
      default: break;
    }
  }
  if constexpr (MASK) return;          // the masked launch requires the vector path (checked by launch_ns_masked)
  const int hk = K >> 1;
  for (int64_t kk = k0 + warp; kk < kend; kk += NS_WARPS) {
    const int64_t e = neg_row[kk];
    const float* __restrict__ t = table.base + e * table.ld + f.col_off;
    float acc = 0.f;
    if (f.pair_op == PAIR_DOT) {
      for (int k = lane; k < K; k += 32) acc = fmaf(q[k], t[k], acc);
    } else if (f.pair_op == PAIR_L1) {
      for (int k = lane; k < K; k += 32) acc += fabsf(q[k] - t[k]);
    } else if (f.pair_op == PAIR_L2) {
      for (int k = lane; k < K; k += 32) { const float d = q[k] - t[k]; acc = fmaf(d, d, acc); }
    } else if (f.pair_op == PAIR_LP) {
      for (int k = lane; k < K; k += 32) acc += __powf(fabsf(q[k] - t[k]), l_norm);
    } else {
      for (int k = lane; k < hk; k += 32) {
        const float d_re = q[k] - t[k], d_im = q[k + hk] - t[k + hk];
        const float m2 = fmaf(d_im, d_im, d_re * d_re);
        acc += (f.pair_op == PAIR_CMOD_L1) ? sqrtf(m2) : __powf(m2, 0.5f * l_norm);
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) {
      if (f.pair_op == PAIR_L1 || f.pair_op == PAIR_CMOD_L1) acc = -acc;
      else if (f.pair_op == PAIR_L2) acc = -sqrtf(acc);
      else if (f.pair_op != PAIR_DOT) acc = -powf(acc, 1.0f / l_norm);
      out_row[kk] = acc;
    }
  }
}

template <int MODEL>
__global__ void __launch_bounds__(NS_WARPS * 32)
ns_kernel(Rows A, Rows Pr, Rows table, int sp, const int64_t* __restrict__ neg, int64_t Kneg,
          Folded f, float l_norm, float* __restrict__ out, int64_t ldo, int col0, int vec_ok) {
  ns_body<MODEL, false>(A, Pr, table, sp, neg, Kneg, f, l_norm, out, ldo, col0, vec_ok, NsRowMasks{});
}

template <int MODEL>
__global__ void __launch_bounds__(NS_WARPS * 32)
ns_kernel_masked(Rows A, Rows Pr, Rows table, const int64_t* __restrict__ tri, int sp, const int64_t* __restrict__ neg,
                 int64_t Kneg, Folded f, float l_norm, float* __restrict__ out, int64_t ldo, int col0, NsRowMasks mk) {
  ns_body<MODEL, true>(A, Pr, table, sp, neg, Kneg, f, l_norm, out, ldo, col0, 1, mk, tri, sp ? 0 : 2);
}

}  // namespace

int launch_spo(int model, float l_norm, const Rows& s, const Rows& p, const Rows& o, int64_t n,
               float* out, int64_t out_stride, cudaStream_t st) {
  RowsDiv S{s, 1}, P{p, 1}, O{o, 1};
  return launch_spo_div(model, l_norm, S, P, O, n, out, out_stride, 1, 0, st);
}

int launch_ns(int model, float l_norm, const Rows& s, const Rows& p, const Rows& o,
              const Rows& table, int slot, const int64_t* neg, int64_t n, int64_t K, float* out,
              int64_t ldo, int col0, cudaStream_t st) {
  if (n == 0 || K == 0) return 0;
  if (slot == 1) {
    // P slot: score(s_i, neg[i,k], o_i) for every (i,k) through the row-wise kernel: logical triple
    // t = i*K + k reads s/o row t/K and relation row neg[t]  (num_samples.p defaults to 0, so this
    // path is rare; config-default.yaml:346-349).
    Rows pneg = table; pneg.idx = neg; pneg.rows = n * K;
    RowsDiv S{s, K}, P{pneg, 1}, O{o, K};
    return launch_spo_div(model, l_norm, S, P, O, n * K, out, ldo, K, col0, st);
  }
  const int sp = (slot == 2) ? 1 : 0;  // O slot: fold (s,p) and score against sampled objects
  const Rows& a = sp ? s : o;
  Folded f = folded_problem(model, sp ? B200KGE_SP_ : B200KGE__PO, a.dim, l_norm);
  size_t smem = (size_t)((f.K + 3) & ~3) * sizeof(float) + (model == B200KGE_RESCAL ? (size_t)a.dim * sizeof(float) : 0);
  // 16-byte loads: rows of the sampled table start 16-byte aligned and the reduction splits into float4 groups
  const bool cm = (f.pair_op == PAIR_CMOD_L1 || f.pair_op == PAIR_CMOD_LP);
  const int vec_ok = (table.ld % 4 == 0 && f.col_off % 4 == 0 && f.K % (cm ? 8 : 4) == 0 &&
                      (reinterpret_cast<uintptr_t>(table.base) & 15) == 0) ? 1 : 0;
  const int64_t by = (K + NS_PER_BLOCK - 1) / NS_PER_BLOCK;
  if (by > 65535) { set_error("too many negatives per row (%lld)", (long long)K); return B200KGE_ERR_UNSUPPORTED; }
  dim3 grid((unsigned)n, (unsigned)by), block(NS_WARPS * 32);
#define B2K_NS(M) case M: ns_kernel<M><<<grid, block, smem, st>>>(a, p, table, sp, neg, K, f, l_norm, out, ldo, col0, vec_ok); break;
  switch (model) {
    B2K_NS(B200KGE_COMPLEX) B2K_NS(B200KGE_DISTMULT) B2K_NS(B200KGE_SIMPLE) B2K_NS(B200KGE_CP)
    B2K_NS(B200KGE_RESCAL) B2K_NS(B200KGE_TRANSE) B2K_NS(B200KGE_ROTATE)
    default: set_error("unknown model %d", model); return B200KGE_ERR_INVALID;
  }
#undef B2K_NS
  B2K_LAUNCH_CHECK("ns_kernel");
  return 0;
}

// The `batch` negatives of one slot with dropout (b200kge_ns_score_dropout): ns_kernel's gather + pair reduction with the
// fixed rows of triple i (the slot's other entity and the relation) masked once per row and each sampled row masked by
// its id.  Not for
// RESCAL, whose D x D relation row does not fit the shared-memory copy.
int launch_ns_masked(int model, float l_norm, const Rows& ent, const Rows& rel, const int64_t* triples, int slot,
                     const int64_t* neg, int64_t n, int64_t K, const DropMask& ma, const DropMask& mp, const DropMask& mt,
                     float* out, int64_t ldo, int col0, cudaStream_t st) {
  const Rows& a = ent; const Rows& p = rel; const Rows& table = ent;
  if (n == 0 || K == 0) return 0;
  const int sp = (slot == 2) ? 1 : 0;
  Folded f = folded_problem(model, sp ? B200KGE_SP_ : B200KGE__PO, a.dim, l_norm);
  const bool cm = (f.pair_op == PAIR_CMOD_L1 || f.pair_op == PAIR_CMOD_LP);
  if (model == B200KGE_RESCAL || f.pair_op == PAIR_LP || f.pair_op == PAIR_CMOD_LP || a.dim % 4 || p.dim % 4 ||
      table.ld % 4 || f.col_off % 4 || f.K % (cm ? 8 : 4) || (reinterpret_cast<uintptr_t>(table.base) & 15)) {
    set_error("the masked negative-sample kernel needs a 16-byte aligned table, widths that are multiples of 4 and a "
              "non-RESCAL model with l_norm 1 / 2");
    return B200KGE_ERR_UNSUPPORTED;
  }
  const size_t smem = (size_t)(((f.K + 3) & ~3) + a.dim + p.dim) * sizeof(float);
  const int64_t by = (K + NS_PER_BLOCK - 1) / NS_PER_BLOCK;
  if (by > 65535) { set_error("too many negatives per row (%lld)", (long long)K); return B200KGE_ERR_UNSUPPORTED; }
  dim3 grid((unsigned)n, (unsigned)by), block(NS_WARPS * 32);
  NsRowMasks mk{ma, mp, mt};
#define B2K_NSM(M) case M: ns_kernel_masked<M><<<grid, block, smem, st>>>(a, p, table, triples, sp, neg, K, f, l_norm, out, ldo, col0, mk); break;
  switch (model) {
    B2K_NSM(B200KGE_COMPLEX) B2K_NSM(B200KGE_DISTMULT) B2K_NSM(B200KGE_SIMPLE) B2K_NSM(B200KGE_CP)
    B2K_NSM(B200KGE_TRANSE) B2K_NSM(B200KGE_ROTATE)
    default: set_error("unknown model %d", model); return B200KGE_ERR_INVALID;
  }
#undef B2K_NSM
  B2K_LAUNCH_CHECK("ns_kernel_masked");
  return 0;
}

// ---------------------------------------------------------------------------------------------
// On-device uniform negative sampling (SURVEY 8f-4): KgeUniformSampler._sample (sampler.py:588-596) is
// torch.randint(vocabulary_size, (n, num_samples)) on the CPU inside DataLoader workers, followed by a host->device copy
// of n*K int64 per slot; here the ids are drawn where they are consumed.  Counter-based Philox4x32-10 (Salmon et al.,
// SC'11): element e of the call uses counter (e / 2, offset) under key (seed), so results depend on (seed, offset, e)
// only — reproducible, no generator state.  Each 64-bit draw r maps to floor(r * vocab / 2^64) (bias <= vocab / 2^64).
namespace {

__global__ void __launch_bounds__(256)
sample_uniform_kernel(uint64_t seed, uint64_t offset, uint64_t vocab, int64_t total, int64_t* __restrict__ out) {
  const int64_t pair = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;      // two ids per Philox block
  if (2 * pair >= total) return;
  uint32_t c[4] = {(uint32_t)pair, (uint32_t)((uint64_t)pair >> 32), (uint32_t)offset, (uint32_t)(offset >> 32)};
  philox4x32_10(c, seed);
  const uint64_t r0 = ((uint64_t)c[1] << 32) | c[0], r1 = ((uint64_t)c[3] << 32) | c[2];
  out[2 * pair] = (int64_t)__umul64hi(r0, vocab);
  if (2 * pair + 1 < total) out[2 * pair + 1] = (int64_t)__umul64hi(r1, vocab);
}

// Filtered uniform sampling (KgeSampler with filtering.<slot>, sampler.py:108-128,163-196,700-752).  Element
// e = i*K + k first takes sample_uniform_kernel's draw x (block (e/2, offset) under key seed, words (0,1) | (2,3) by the
// parity of e).  If x is not one of the m sorted, distinct positives of row i's key, the output is x.  Otherwise one
// second draw u = floor(r' * (vocab - m) / 2^64) picks the u-th non-positive id, where r' is word pair (e & 1) of block
// (e/2 | 2^63, offset) under the same key: a counter the first draw never reaches (its block index is below 2^62).
// P(y) = 1/V + (m/V) * 1/(V-m) = 1/(V-m) for every non-positive y: the distribution of the reference's redraw loop, with
// no loop whose length depends on chance.  The u-th non-positive is u + c, c = #{j : values[j] - j <= u} (values[j] - j
// counts the non-positives below values[j] and does not decrease in j).  A row whose key is absent has m = 0; a row
// with m >= vocab has no non-positive and gets -1.
constexpr uint64_t FILTER_DOMAIN = 1ull << 63;

__device__ __forceinline__ uint64_t philox_u64(uint64_t seed, uint64_t offset, uint64_t block, bool odd) {
  uint32_t c[4] = {(uint32_t)block, (uint32_t)(block >> 32), (uint32_t)offset, (uint32_t)(offset >> 32)};
  philox4x32_10(c, seed);
  return odd ? ((uint64_t)c[3] << 32) | c[2] : ((uint64_t)c[1] << 32) | c[0];
}

// thread 0's lookup of row i's key (tri[3i + c0], tri[3i + c1]) among the sorted keys of a filter index: the start and
// count of its values, (0, 0) for an absent key
__device__ __forceinline__ void key_values(const int64_t* __restrict__ tri, int64_t i, int c0, int c1,
                                           const int64_t* __restrict__ keys, const int64_t* __restrict__ offsets,
                                           int64_t num_keys, int64_t& begin, int64_t& m) {
  const int64_t a = tri[3 * i + c0], b = tri[3 * i + c1];
  int64_t lo = 0, hi = num_keys;
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    const int64_t ka = keys[2 * mid], kb = keys[2 * mid + 1];
    if (ka < a || (ka == a && kb < b)) lo = mid + 1;
    else hi = mid;
  }
  begin = 0;
  m = 0;
  if (lo < num_keys && keys[2 * lo] == a && keys[2 * lo + 1] == b) {
    begin = offsets[lo];
    m = offsets[lo + 1] - begin;
  }
}

// lower bound of x among the m sorted positives v
__device__ __forceinline__ int64_t positive_lower_bound(const int64_t* __restrict__ v, int64_t m, int64_t x) {
  int64_t lo = 0, hi = m;
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(v + mid) < x) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// one CTA per row: thread 0 looks the row's key up once, every thread then takes elements k, k + blockDim.x, ...
__global__ void __launch_bounds__(256)
sample_uniform_filtered_kernel(uint64_t seed, uint64_t offset, uint64_t vocab, int64_t K, const int64_t* __restrict__ tri,
                               int c0, int c1, const int64_t* __restrict__ keys, const int64_t* __restrict__ offsets,
                               const int64_t* __restrict__ values, int64_t num_keys, int64_t* __restrict__ out) {
  __shared__ int64_t s_begin, s_m;
  const int64_t i = blockIdx.x;
  if (threadIdx.x == 0) {
    int64_t begin, m;
    key_values(tri, i, c0, c1, keys, offsets, num_keys, begin, m);
    s_begin = begin;
    s_m = m;
  }
  __syncthreads();
  const int64_t* __restrict__ v = values + s_begin;
  const int64_t m = s_m;
  int64_t* __restrict__ orow = out + i * K;
  if ((uint64_t)m >= vocab) {
    for (int64_t k = threadIdx.x; k < K; k += blockDim.x) orow[k] = -1;
    return;
  }
  for (int64_t k = threadIdx.x; k < K; k += blockDim.x) {
    const uint64_t e = (uint64_t)(i * K + k);
    const int64_t x = (int64_t)__umul64hi(philox_u64(seed, offset, e >> 1, e & 1), vocab);
    int64_t lo = positive_lower_bound(v, m, x), hi;
    if (lo == m || __ldg(v + lo) != x) { orow[k] = x; continue; }
    const int64_t u = (int64_t)__umul64hi(philox_u64(seed, offset, (e >> 1) | FILTER_DOMAIN, e & 1), vocab - (uint64_t)m);
    lo = 0; hi = m;                          // c = #{j : v[j] - j <= u}
    while (lo < hi) {
      const int64_t mid = lo + ((hi - lo) >> 1);
      if (__ldg(v + mid) - mid <= u) lo = mid + 1;
      else hi = mid;
    }
    orow[k] = u + lo;
  }
}

// Frequency sampling (KgeFrequencySampler, sampler.py:755-793): P(x) = q_x / Q over the integer weights q of
// b200kge_frequency_cdf_build, given as the exclusive prefix cdf[0..V] (cdf[0] = 0, cdf[V] = Q).  A 64-bit draw r maps
// to t = floor(r * Q / 2^64) and then to the largest x with cdf[x] <= t: the preimage of x is an interval of q_x / Q of
// the r range (to within 2^-64), and an id of zero weight is never drawn.
//
// The largest x in [0, len - 1) with cdf[x] <= t[j], for N targets at once: a branchless lower bound whose trip count,
// ceil(log2(len)), depends on len only, so the lanes of a warp never diverge.  Needs cdf[0] <= t[j] < cdf[len - 1].
template <int N>
__device__ __forceinline__ void cdf_search(const uint64_t* __restrict__ cdf, int64_t len, const uint64_t (&t)[N],
                                           int64_t (&x)[N]) {
#pragma unroll
  for (int j = 0; j < N; ++j) x[j] = 0;
  for (int64_t w = len; w > 1;) {
    const int64_t half = w >> 1;
#pragma unroll
    for (int j = 0; j < N; ++j) x[j] += __ldg(cdf + x[j] + half) <= t[j] ? half : 0;
    w -= half;
  }
}

// two elements per Philox block, exactly the words sample_uniform_kernel takes; the two searches run interleaved
__global__ void __launch_bounds__(256)
sample_frequency_kernel(uint64_t seed, uint64_t offset, const uint64_t* __restrict__ cdf, int64_t len, int64_t total,
                        int64_t* __restrict__ out) {
  const int64_t pair = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (2 * pair >= total) return;
  uint32_t c[4] = {(uint32_t)pair, (uint32_t)((uint64_t)pair >> 32), (uint32_t)offset, (uint32_t)(offset >> 32)};
  philox4x32_10(c, seed);
  const uint64_t Q = __ldg(cdf + len - 1);
  const uint64_t t[2] = {__umul64hi(((uint64_t)c[1] << 32) | c[0], Q), __umul64hi(((uint64_t)c[3] << 32) | c[2], Q)};
  int64_t x[2];
  cdf_search(cdf, len, t, x);
  out[2 * pair] = x[0];
  if (2 * pair + 1 < total) out[2 * pair + 1] = x[1];
}

// Filtered frequency sampling: i.i.d. from q restricted to the non-positives of row i's key, P(y) = q_y / (Q - M_i) with
// M_i the mass of the key's m positives v_0 < ... < v_{m-1} (the law of the reference's redraw loop).  Element e first
// takes sample_frequency_kernel's draw x; if x is not a positive it is the output.  Otherwise u = floor(r' * (Q - M_i) /
// 2^64), r' word pair (e & 1) of block (e/2 | 2^63, offset), picks the u-th unit of non-positive mass.  below[j] =
// G_j = cdf[v_j] - sum_{l<j} q_{v_l} is the non-positive mass below v_j (non-decreasing in j); with g = #{j : G_j <= u}
// and PW_g = sum_{l<g} q_{v_l} = cdf[v_{g-1} + 1] - G_{g-1}, the target u + PW_g lies in [cdf[v_{g-1} + 1], cdf[v_g]),
// so the CDF search lands strictly between two positives on an id of nonzero weight.  No loop's length depends on
// chance.  Absent keys are unfiltered; a row whose positives carry all the mass (Q - M_i = 0) gets -1.
__global__ void __launch_bounds__(256)
sample_frequency_filtered_kernel(uint64_t seed, uint64_t offset, const uint64_t* __restrict__ cdf, int64_t len,
                                 int64_t K, const int64_t* __restrict__ tri, int c0, int c1,
                                 const int64_t* __restrict__ keys, const int64_t* __restrict__ offsets,
                                 const int64_t* __restrict__ values, const uint64_t* __restrict__ below,
                                 int64_t num_keys, int64_t* __restrict__ out) {
  __shared__ int64_t s_begin, s_m;
  __shared__ uint64_t s_q, s_rest;
  const int64_t i = blockIdx.x;
  if (threadIdx.x == 0) {
    int64_t begin, m;
    key_values(tri, i, c0, c1, keys, offsets, num_keys, begin, m);
    const uint64_t Q = cdf[len - 1];
    s_begin = begin;
    s_m = m;
    s_q = Q;
    s_rest = m > 0 ? Q - (cdf[values[begin + m - 1] + 1] - below[begin + m - 1]) : Q;
  }
  __syncthreads();
  const int64_t* __restrict__ v = values + s_begin;
  const uint64_t* __restrict__ G = below + s_begin;
  const int64_t m = s_m;
  const uint64_t Q = s_q, rest = s_rest;
  int64_t* __restrict__ orow = out + i * K;
  if (rest == 0) {
    for (int64_t k = threadIdx.x; k < K; k += blockDim.x) orow[k] = -1;
    return;
  }
  for (int64_t k = threadIdx.x; k < K; k += blockDim.x) {
    const uint64_t e = (uint64_t)(i * K + k);
    uint64_t t[1] = {__umul64hi(philox_u64(seed, offset, e >> 1, e & 1), Q)};
    int64_t x[1];
    cdf_search(cdf, len, t, x);
    int64_t lo = positive_lower_bound(v, m, x[0]), hi;
    if (lo == m || __ldg(v + lo) != x[0]) { orow[k] = x[0]; continue; }
    const uint64_t u = __umul64hi(philox_u64(seed, offset, (e >> 1) | FILTER_DOMAIN, e & 1), rest);
    lo = 0; hi = m;                          // g = #{j : G_j <= u}
    while (lo < hi) {
      const int64_t mid = lo + ((hi - lo) >> 1);
      if (__ldg(G + mid) <= u) lo = mid + 1;
      else hi = mid;
    }
    t[0] = u + (lo == 0 ? 0 : __ldg(cdf + __ldg(v + lo - 1) + 1) - __ldg(G + lo - 1));
    cdf_search(cdf, len, t, x);
    orow[k] = x[0];
  }
}

}  // namespace

int launch_sample_frequency(uint64_t seed, uint64_t offset, int64_t vocab, const uint64_t* cdf, int64_t total,
                            int64_t* out, cudaStream_t st) {
  if (total <= 0) return 0;
  const int64_t pairs = (total + 1) / 2;
  sample_frequency_kernel<<<(unsigned)((pairs + 255) / 256), 256, 0, st>>>(seed, offset, cdf, vocab + 1, total, out);
  B2K_LAUNCH_CHECK("sample_frequency_kernel");
  return 0;
}

int launch_sample_frequency_filtered(uint64_t seed, uint64_t offset, int64_t vocab, int64_t n, int64_t K,
                                     const int64_t* triples, int slot, const int64_t* keys, const int64_t* offsets,
                                     const int64_t* values, int64_t num_keys, const uint64_t* cdf,
                                     const uint64_t* below, int64_t* out, cudaStream_t st) {
  if (n <= 0 || K <= 0) return 0;
  if (n > 2147483647LL) { set_error("too many rows (%lld)", (long long)n); return B200KGE_ERR_UNSUPPORTED; }
  const int c0 = slot == 0 ? 1 : 0, c1 = slot == 2 ? 1 : 2;   // the key pair of the slot, as launch_sample_uniform_filtered
  const int threads = K >= 256 ? 256 : (int)((K + 31) / 32) * 32;
  sample_frequency_filtered_kernel<<<(unsigned)n, threads, 0, st>>>(seed, offset, cdf, vocab + 1, K, triples, c0, c1,
                                                                     keys, offsets, values, below, num_keys, out);
  B2K_LAUNCH_CHECK("sample_frequency_filtered_kernel");
  return 0;
}

int launch_sample_uniform_filtered(uint64_t seed, uint64_t offset, int64_t vocab, int64_t n, int64_t K,
                                   const int64_t* triples, int slot, const int64_t* keys, const int64_t* offsets,
                                   const int64_t* values, int64_t num_keys, int64_t* out, cudaStream_t st) {
  if (n <= 0 || K <= 0) return 0;
  if (n > 2147483647LL) { set_error("too many rows (%lld)", (long long)n); return B200KGE_ERR_UNSUPPORTED; }
  // the key pair of each slot: (p, o) for S, (s, o) for P, (s, p) for O (sampler.py:167-173)
  const int c0 = slot == 0 ? 1 : 0, c1 = slot == 2 ? 1 : 2;
  const int threads = K >= 256 ? 256 : (int)((K + 31) / 32) * 32;
  sample_uniform_filtered_kernel<<<(unsigned)n, threads, 0, st>>>(seed, offset, (uint64_t)vocab, K, triples, c0, c1,
                                                                   keys, offsets, values, num_keys, out);
  B2K_LAUNCH_CHECK("sample_uniform_filtered_kernel");
  return 0;
}

int launch_sample_uniform(uint64_t seed, uint64_t offset, int64_t vocab, int64_t total, int64_t* out, cudaStream_t st) {
  if (total <= 0) return 0;
  const int64_t pairs = (total + 1) / 2;
  sample_uniform_kernel<<<(unsigned)((pairs + 255) / 256), 256, 0, st>>>(seed, offset, (uint64_t)vocab, total, out);
  B2K_LAUNCH_CHECK("sample_uniform_kernel");
  return 0;
}

}  // namespace b200kge
