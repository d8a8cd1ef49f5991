// tc_common.cuh — pieces shared by the tensor-core scorer (pairwise_tc.cu) and its callers.
#pragma once
#include <cuda.h>
#include <cstdlib>
#include "common.cuh"
#include "ptx.cuh"

namespace b200kge {
namespace tc {

__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}

__device__ __forceinline__ float4 trunc_tf32_4(const float4 v) {
  return make_float4(__uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u), __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u),
                     __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u), __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u));
}
// lo = rn_tf32(x - trunc_tf32(x)) for 4 packed floats
__device__ __forceinline__ float4 split_lo4(const float4 v) {
  float4 l;
  l.x = tf32_rna(v.x - __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u));
  l.y = tf32_rna(v.y - __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u));
  l.z = tf32_rna(v.z - __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u));
  l.w = tf32_rna(v.w - __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u));
  return l;
}

// ---------------------------------------------------------------------------------------------
// explicit shared-space vector accesses (the compiler otherwise emits generic LD.E/ST.E for pointers
// carved out of the dynamic smem buffer by integer arithmetic)
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const float4 v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// lo tile = split_lo(raw tile) for NBYTES bytes, by `nthreads` threads (thread index t); the raw tile is
// rewritten as trunc_tf32(raw), so the tf32 MMA's hi operand is exact whether the tensor core truncates or rounds
// the low mantissa bits.  All loads of a thread are issued before its stores so the smem latency is paid once.
template <int NBYTES, int NTHR>
__device__ __forceinline__ void split_tile(uint32_t src, uint32_t dst, int t) {
  constexpr int PER = NBYTES / 16 / NTHR;   // float4s per thread
  static_assert(PER * NTHR * 16 == NBYTES, "tile must divide evenly");
  float4 v[PER];
#pragma unroll
  for (int i = 0; i < PER; ++i) v[i] = lds128(src + (uint32_t)(t + i * NTHR) * 16u);
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    sts128(dst + (uint32_t)(t + i * NTHR) * 16u, split_lo4(v[i]));
    sts128(src + (uint32_t)(t + i * NTHR) * 16u, trunc_tf32_4(v[i]));
  }
}

// Mixed mode (tf32 hi*hi + bf16 cross terms): from a raw fp32 K-major tile [ROWS][32] in the 128-B
// swizzled layout, derive two bf16 K-major tiles [ROWS][32] in the 64-B swizzled layout:
//   hi16 = bf16_rn(x)            (hi operand of the cross terms)
//   lo16 = bf16_rn(x - trunc_tf32(x))   (remainder w.r.t. the tf32 MMA's hi operand)
// and rewrite the raw tile as trunc_tf32(x) (the tf32 MMA's hi operand, exact in tf32).
// One item = (row r, group c of 8 consecutive k): reads fp32 16-B chunks 2c, 2c+1 of row r (physical
// chunk = logical ^ (r & 7)), writes bf16 16-B chunk c of row r (physical = c ^ ((r >> 1) & 3)).
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));   // low half <- a, high half <- b
  return r;
}
template <int ROWS, int NTHR>
__device__ __forceinline__ void split_tile_bf16(uint32_t src, uint32_t dst_hi, uint32_t dst_lo, int t) {
  constexpr int ITEMS = ROWS * 4, PER = ITEMS / NTHR, RSTEP = NTHR / 4;
  static_assert(PER * NTHR == ITEMS && RSTEP % 8 == 0, "tile must divide evenly; row step keeps the swizzle phase");
  // item i of thread t: row r = (t >> 2) + i * RSTEP, k-group c = t & 3.  RSTEP is a multiple of 8, so
  // the swizzle terms (r & 7) and ((r >> 1) & 3) are per-thread constants and all addresses are
  // base + i * constant.
  const int r0 = t >> 2, c = t & 3;
  const uint32_t s0 = src + (uint32_t)r0 * 128u + (uint32_t)(((2 * c) ^ (r0 & 7)) * 16);
  const uint32_t s1 = src + (uint32_t)r0 * 128u + (uint32_t)(((2 * c + 1) ^ (r0 & 7)) * 16);
  const uint32_t doff = (uint32_t)r0 * 64u + (uint32_t)((c ^ ((r0 >> 1) & 3)) * 16);
  float4 v0[PER], v1[PER];
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    v0[i] = lds128(s0 + (uint32_t)(i * RSTEP * 128));
    v1[i] = lds128(s1 + (uint32_t)(i * RSTEP * 128));
  }
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const float x[8] = {v0[i].x, v0[i].y, v0[i].z, v0[i].w, v1[i].x, v1[i].y, v1[i].z, v1[i].w};
    float lo[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) lo[k] = x[k] - __uint_as_float(__float_as_uint(x[k]) & 0xFFFFE000u);
    const uint32_t roff = (uint32_t)(i * RSTEP * 128);
    sts128(s0 + roff, trunc_tf32_4(v0[i]));
    sts128(s1 + roff, trunc_tf32_4(v1[i]));
    const uint32_t off = doff + (uint32_t)(i * RSTEP * 64);
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst_hi + off), "r"(pack_bf16x2(x[0], x[1])),
                 "r"(pack_bf16x2(x[2], x[3])), "r"(pack_bf16x2(x[4], x[5])), "r"(pack_bf16x2(x[6], x[7])) : "memory");
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst_lo + off), "r"(pack_bf16x2(lo[0], lo[1])),
                 "r"(pack_bf16x2(lo[2], lo[3])), "r"(pack_bf16x2(lo[4], lo[5])), "r"(pack_bf16x2(lo[6], lo[7])) : "memory");
  }
}

// Epilogue, straight from the wgmma accumulator fragment (layout in ptx.cuh).  The calling thread holds 32 scores of
// one query row of a 128-column tile: v[2j + p] is column c0 + 8j + p (j < 16, p < 2) with c0 = tile start +
// 2 * (lane % 4), so the four lanes of a quad together hold the row's 128 columns.  Per-row state stays lane-local
// until the flush, which combines the quad's states (epi_lane_reduce) in a fixed order.  Columns >= m are skipped.

constexpr float LOG2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;

__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// offset of fragment element k from the lane's first column
__device__ __forceinline__ constexpr int frag_col(int k) { return 8 * (k >> 1) + (k & 1); }

// fragment element holding tile column `tc` (0..127) if lane q of the quad holds it, else -1
__device__ __forceinline__ int frag_elem(int tc, int q) {
  return ((tc >> 1) & 3) == q ? 2 * (tc >> 3) + (tc & 1) : -1;
}

__device__ __forceinline__ float frag_get(const float (&v)[32], int k) {
  float x = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i)
    if (i == k) x = v[i];
  return x;
}

// FULL: all 128 columns of the tile are < m (then nvalid is not read)
template <int EPI, bool FULL>
__device__ __forceinline__ void epi_row_body(const EpiParams& P, RowState<EPI>& st, const float (&v)[32], int64_t row,
                                             int64_t e0, int64_t c0, int nvalid, int q, int64_t lab) {
  if constexpr (EPI == EPI_BCE) {
    // sum softplus(z) - sum y*z,  softplus(z) = max(z,0) + log(1 + exp(-|z|))   (loss.py:150-157;
    // torch's kernel also evaluates log(1+e) with a plain log, so tiny e drop out identically)
    // The lane's 32 logarithms are taken as one: log(prod(1 + e)).  Each factor 1 + e lies in [1, 2], so the product
    // of 32 stays within [1, 2^32] (no overflow, no denormal), a NaN score still propagates and z = +-inf still adds
    // a factor of exactly 1.
    const float off = P.offset;
    float amax = 0.f, prod = 1.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) {
      if (FULL || frag_col(k) < nvalid) {
        const float z = v[k] + off;
        const float e = fast_ex2(-fabsf(z) * LOG2E);
        prod *= 1.0f + e;
        amax += fmaxf(z, 0.f);
      }
    }
    st.a += fmaf(__log2f(prod), LN2, amax);
    if (P.label_dense) {
      const float* __restrict__ y = P.label_dense + row * P.ldl + c0;
      float b = 0.f;
#pragma unroll
      for (int k = 0; k < 32; ++k)
        if (FULL || frag_col(k) < nvalid) b = fmaf(__ldg(y + frag_col(k)), v[k] + off, b);
      st.b += b;
    } else if (P.label_idx) {
      const int k = (lab >= e0 && lab < e0 + 128 && (FULL || lab - c0 < nvalid)) ? frag_elem((int)(lab - e0), q) : -1;
      if (k >= 0) st.b += frag_get(v, k) + off;
    }
  } else if constexpr (EPI == EPI_KL) {
    // online logsumexp: the lane's max first, then ONE exp per element   (loss.py:198-213)
    float cm = B2K_NEG_HUGE;
#pragma unroll
    for (int k = 0; k < 32; ++k)
      if (FULL || frag_col(k) < nvalid) cm = fmaxf(cm, v[k]);
    const float mn = fmaxf(st.m, cm);
    const float mn2 = mn * LOG2E;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k)
      if (FULL || frag_col(k) < nvalid) acc += fast_ex2(fmaf(v[k], LOG2E, -mn2));
    st.s = fmaf(st.s, fast_ex2((st.m - mn) * LOG2E), acc);
    st.m = mn;
    if (P.label_dense) {
      const float* __restrict__ y = P.label_dense + row * P.ldl + c0;
#pragma unroll
      for (int k = 0; k < 32; ++k) {
        if (FULL || frag_col(k) < nvalid) {
          const float yy = __ldg(y + frag_col(k));
          if (yy != 0.f) {
            st.y_sum += yy;
            st.yx = fmaf(yy, v[k], st.yx);
            st.ylogy = fmaf(yy, __logf(yy), st.ylogy);
          }
        }
      }
    } else if (P.label_idx) {
      const int k = (lab >= e0 && lab < e0 + 128 && (FULL || lab - c0 < nvalid)) ? frag_elem((int)(lab - e0), q) : -1;
      if (k >= 0) { st.y_sum += 1.0f; st.yx += frag_get(v, k); }
    }
  } else if constexpr (EPI == EPI_RANK || EPI == EPI_RANK_EVAL) {
    // eval_entity_ranking.py:561-596; `allowed` depends on the row only -> hoisted
    const float t = epi_row_aux<EPI_RANK>(P, row);
    const float allowed = __fadd_rn(P.atol, fabsf(__fmul_rn(P.rtol, t)));
    const float* __restrict__ f = (EPI == EPI_RANK && P.filter) ? P.filter + row * P.ldf + c0 : nullptr;
    unsigned int gt = 0, cl = 0;
#pragma unroll
    for (int k = 0; k < 32; ++k) {
      if (FULL || frag_col(k) < nvalid) {
        float x = v[k];
        if (f) x = __fsub_rn(x, __ldg(f + frag_col(k)));
        if (isnan(x)) x = -INFINITY;
        const float actual = fabsf(__fsub_rn(x, t));
        const bool close = (x == t) || (isfinite(actual) && actual <= allowed);
        cl += close ? 1u : 0u;
        gt += (!close && x > t) ? 1u : 0u;
      }
    }
    st.greater += gt;
    st.close += cl;
  } else if constexpr (EPI == EPI_STORE) {
    int64_t r = row, cb = 0;
    if (P.n_rows_out > 0 && r >= P.n_rows_out) { r -= P.n_rows_out; cb = P.col_block; }   // sp|po seam
    const int64_t at = r * P.ldo + cb + c0;
    // a quad writes 32 contiguous bytes of the row per j: full sectors whatever the row stride is
    auto put = [&](float* __restrict__ p) {
      const bool vec = (reinterpret_cast<uintptr_t>(p) & 7) == 0;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        if (vec && (FULL || 8 * j + 1 < nvalid)) {
          *reinterpret_cast<float2*>(p + 8 * j) = make_float2(v[2 * j], v[2 * j + 1]);
        } else {
          if (FULL || 8 * j < nvalid) p[8 * j] = v[2 * j];
          if (FULL || 8 * j + 1 < nvalid) p[8 * j + 1] = v[2 * j + 1];
        }
      }
    };
    if (P.accumulate_out) {
      float* __restrict__ p = P.out + at;
#pragma unroll
      for (int k = 0; k < 32; ++k)
        if (FULL || frag_col(k) < nvalid) atomicAdd(p + frag_col(k), v[k]);
    } else {
      put(P.out + at);
      for (int g = 0; g < P.n_peers; ++g) put(P.out_peer[g] + at);   // same offsets in the peers' symmetric buffers
    }
  }
}

// EPI_RANK_EVAL after the raw counts of a tile: the row's listed columns inside the tile (F, then the test answers not
// in F) swap their raw contribution for that of -inf (RankFix), except the own answer, whose score goes to own_score.
// Every lane of the quad walks the lists and acts on the columns it holds.
__device__ __forceinline__ void rank_eval_row(const EpiParams& P, const float (&v)[32], int64_t row, int64_t e0, int64_t m,
                                              int q) {
  const float t = epi_row_aux<EPI_RANK_EVAL>(P, row);
  const int64_t lim = e0 + 128 < m ? e0 + 128 : m;
  const int64_t own = __ldg(P.csr_skip + row);
  if (own >= e0 && own < lim) {
    const int k = frag_elem((int)(own - e0), q);
    if (k >= 0) P.own_score[row] = frag_get(v, k);
  }
  RankFix fix;
#pragma unroll
  for (int list = 0; list < 2; ++list) {
    const int64_t* __restrict__ off = list ? P.csr2_off : P.csr_off;
    const int64_t* __restrict__ col = list ? P.csr2_col : P.csr_col;
    if (!off) continue;
    const int64_t end = __ldg(off + row + 1);
    for (int64_t cur = csr_lower_bound(col, __ldg(off + row), end, e0); cur < end; ++cur) {
      const int64_t cj = __ldg(col + cur);
      if (cj >= lim) break;
      const int k = frag_elem((int)(cj - e0), q);
      if (k >= 0 && cj != own) fix.add(list == 1, frag_get(v, k), t, P.rtol, P.atol);
    }
  }
  fix.commit(P, row);
}

// One row's share of a tile: e0 = first column of the tile, q = lane % 4, c0 = e0 + 2q.  lab = P.label_idx[row], loaded
// by the caller ahead of the accumulators (read by BCE / KL with label_idx only).  v is clobbered (rank: CSR filtered
// columns become -inf).
template <int EPI>
__device__ __forceinline__ void epi_row(const EpiParams& P, RowState<EPI>& st, float (&v)[32], int64_t row,
                                        int64_t e0, int64_t m, int q, int64_t lab) {
  const int64_t c0 = e0 + 2 * q;
  if constexpr (EPI == EPI_RANK_EVAL) {
    if (e0 + 128 <= m) epi_row_body<EPI, true>(P, st, v, row, e0, c0, 128, q, lab);
    else               epi_row_body<EPI, false>(P, st, v, row, e0, c0, (int)(m - c0), q, lab);
    rank_eval_row(P, v, row, e0, m, q);
    return;
  }
  if constexpr (EPI != EPI_STORE) {
    if (P.csr_off) {
      // listed columns of this row inside the tile: emit their scores (losses) or filter them (rank).  Every lane of
      // the quad walks the list and acts on the columns it holds.
      const int64_t end = __ldg(P.csr_off + row + 1);
      const int64_t lim = e0 + 128 < m ? e0 + 128 : m;
      const int64_t skip = (EPI == EPI_RANK && P.csr_skip) ? __ldg(P.csr_skip + row) : -1;
      for (int64_t cur = csr_lower_bound(P.csr_col, __ldg(P.csr_off + row), end, e0); cur < end; ++cur) {
        const int64_t cj = __ldg(P.csr_col + cur);
        if (cj >= lim) break;
        const int k = frag_elem((int)(cj - e0), q);
        if (k < 0) continue;
        if constexpr (EPI == EPI_RANK) {
          if (cj != skip) {
#pragma unroll
            for (int i = 0; i < 32; ++i)
              if (i == k) v[i] = -INFINITY;               // neither greater nor close (for a finite true score)
          }
        } else {
          P.csr_out[cur] = frag_get(v, k);
        }
      }
    }
    if constexpr (EPI == EPI_BCE || EPI == EPI_KL) {
      if (P.csr_extra && e0 == 0 && q == 0) P.csr_out[P.csr_nnz + row] = v[0];
    }
  }
  if (e0 + 128 <= m) epi_row_body<EPI, true>(P, st, v, row, e0, c0, 128, q, lab);
  else               epi_row_body<EPI, false>(P, st, v, row, e0, c0, (int)(m - c0), q, lab);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D fp32 tensor map over [rows, cols] with row stride ld floats; box = box_cols x box_rows,
// swizzle = box_cols*4 bytes (64 or 128).
inline int make_map(CUtensorMap* map, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_cols,
                    int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled not available from the driver"); return B200KGE_ERR_CUDA; }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMapSwizzle sw = (box_cols * 4 == 128) ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld", (int)r, (long long)rows,
              (long long)cols, (long long)ld);
    return B200KGE_ERR_CUDA;
  }
  return 0;
}

// 2-D fp16 tensor map over [rows, cols] halfs with row stride ld halfs; box = box_cols x box_rows with
// box_cols = 64 (128-byte rows, 128-byte swizzle) or 32 (64-byte rows, 64-byte swizzle).
inline int make_map_f16(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows,
                        int box_cols = 64) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled not available from the driver"); return B200KGE_ERR_CUDA; }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, box_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(f16) failed (%d) rows=%lld cols=%lld ld=%lld", (int)r, (long long)rows,
              (long long)cols, (long long)ld);
    return B200KGE_ERR_CUDA;
  }
  return 0;
}

inline int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

}  // namespace tc

// Pre-split fp16 path (presplit.cu + pairwise_tc.cu).  One row set of the operand split: rows of `src` (optionally gathered through idx, starting at column
// col_off, K columns) -> hi/lo fp16 planes [rows, Kp] (Kp = round_up(K, 64), zero padded) and the
// per-row power-of-two factor inv_scale[rows_pad] that undoes the row scaling (0 beyond `rows`).
struct SplitSet {
  const float* src; int64_t ld; const int64_t* idx; int col_off;
  int64_t rows, rows_pad;
  int K, Kp;
  void* hi; void* lo; float* inv_scale;
};
int launch_presplit(const SplitSet& A, const SplitSet& B, cudaStream_t st);   // B.rows may be 0
// fold + split of the 2n stacked query rows of a 1vsAll batch AND the split of the table, labels, ticket: one launch
// (num_rel > 0: the reciprocal layout of launch_prep_1vsall)
int launch_prep_split_1vsall(int model, const Rows& ent, const Rows& rel, const int64_t* triples, int64_t n,
                             const SplitSet& Qs, const SplitSet& Ts, int64_t* labels2n, unsigned int* ticket,
                             cudaStream_t st, int64_t num_rel = 0);
int launch_pairwise_tc3(int epi_kind, const SplitSet& Q, const SplitSet& T, const EpiParams& P, cudaStream_t st);

// Backward pieces (grad.cu), experimental.
int launch_transpose(const float* src, int64_t lds, int64_t R, int64_t C, float* dst, int64_t ldd, cudaStream_t st);
int launch_grad_planes(const float* z, int64_t ldz, int64_t nq, int64_t E, const int64_t* label_idx,
                       const float* label_dense, int64_t ldl, float* row_stat, float offset, float inv_n, void* g_hi, void* g_lo,
                       int64_t Ep, void* gt_hi, void* gt_lo, int64_t Np, float* g_scale, float* gt_scale,
                       cudaStream_t st);
// distance-family backward (grad_distance.cu, grad.cu)
int launch_pair_rowgrad(int pair_op, const float* A, int64_t lda, int64_t ra, const float* B, int64_t ldb, int64_t rb, int K,
                        const float* Wt, int64_t ldwt, float* dA, int64_t ldda, cudaStream_t st);   // Wt: [rb, >= ra]
int launch_grad_dense(const float* z, int64_t ldz, int64_t nq, int64_t E, const int64_t* label_idx, const float* row_stat,
                      float offset, float inv_n, int div_z, float* G, int64_t ldg, cudaStream_t st);
// G for CSR labels y = a * count + b (KvsAll); row_stat: KL row log-sum-exp in row_stat[2 i] (else null)
int launch_grad_csr(const float* z, int64_t ldz, int64_t nq, int64_t E, const int64_t* csr_off, const int64_t* csr_col,
                    float a, float b, const float* row_stat, float offset, float inv_n, int div_z, float* G, int64_t ldg,
                    cudaStream_t st);
int launch_div_scores(const float* g, int64_t ldg, const float* z, int64_t ldz, int64_t n, int64_t E, float* W, int64_t ldw,
                      cudaStream_t st);
int launch_row_lse(const float* z, int64_t ldz, int64_t nq, int64_t E, const int64_t* label_idx, float* row_stat,
                   cudaStream_t st);
// num_rel > 0 (dir < 0 only): the reciprocal layout, rows [n,2n) unfold as sp_ into d_ent[o], d_rel[p + num_rel]
int launch_unfold_distance(int model, const Rows& ent, const Rows& rel, const int64_t* triples, int64_t n, int dir,
                           const float* dQ, int64_t ldq, float* d_ent, int64_t lde, float* d_rel, int64_t ldr,
                           cudaStream_t st, int64_t num_rel = 0, const int32_t* pe = nullptr,
                           const int32_t* pr = nullptr);
int launch_grad_planes_csr(const float* z, int64_t ldz, int64_t nq, int64_t E, const int64_t* csr_off,
                           const int64_t* csr_col, float a, float b, float* row_stat, float offset, float inv_n,
                           void* g_hi, void* g_lo, int64_t Ep, void* gt_hi, void* gt_lo, int64_t Np, float* g_scale,
                           float* gt_scale, cudaStream_t st);
// CSR-label losses (csr_loss.cu).
int launch_csr_expand(const int64_t* off, const int64_t* col, int64_t n, int64_t nnz, int extra, const int64_t* q_idx,
                      const int64_t* p_idx, int64_t* qsel, int64_t* psel, int64_t* esel, cudaStream_t st);
// zsum (label smoothing, else null): zsum_chunks partial score sums per row, [n, zsum_chunks]
int launch_csr_rows(int loss_kind, const int64_t* off, const int64_t* col, const float* zpos, int64_t n, int64_t nnz,
                    const float* fused, const float* zsum, int zsum_chunks, float a, float b, float E, float offset,
                    float* row_loss, cudaStream_t st);
int launch_rows_sum(const float* rows, int64_t n, float scale, float* out, cudaStream_t st);
int launch_row_score_sums(const float* Q, int64_t ldq, int64_t n, const float* T, int64_t ldt, int64_t E, int K,
                          float* scratch, float* zsum, cudaStream_t st);
// G (optional, [n, 1+K], row stride ldg): dL/dz already scaled, read instead of the BCE gradient.  pe / pr (both or
// neither): row maps, entity e's gradient row is d_ent + pe[e] * lde, relation r's d_rel + pr[r] * ldr.
int launch_ns_backward(int model, float l_norm, const Rows& ent, const Rows& rel, const int64_t* triples, int slot,
                       const int64_t* neg, int64_t n, int64_t K, float offset, float inv_batch, const float* G,
                       int64_t ldg, float* d_ent, int64_t lde, float* d_rel, int64_t ldr, float* dQ, int64_t ldq,
                       cudaStream_t st, const int32_t* pe = nullptr, const int32_t* pr = nullptr);
// row-wise KgeLoss of a negative-sampling block (ns_loss.cu): part[2 i] = row loss (BCE finaliser layout), G optional
int launch_ns_loss(int loss_kind, const float* scores, int64_t lds, int64_t n, int64_t m, const int64_t* label_idx,
                   float arg, float temperature, float scale, float* part, float* G, int64_t ldg, cudaStream_t st);
int launch_penalty(const Rows& tab, const float* counts, float p, int complex_abs, float scale, float* scratch,
                   size_t scratch_floats, float* out, cudaStream_t st);
int launch_normalize_rows(float* w, int64_t ld, int64_t rows, int dim, float p, cudaStream_t st);
int launch_unfold(int model, const Rows& ent, const Rows& rel, const int64_t* triples, int64_t n, int dir,
                  const float* dQ, int64_t ldq, float* d_ent, int64_t lde, float* d_rel, int64_t ldr, cudaStream_t st,
                  int64_t num_rel = 0, const int32_t* pe = nullptr, const int32_t* pr = nullptr);

}  // namespace b200kge
