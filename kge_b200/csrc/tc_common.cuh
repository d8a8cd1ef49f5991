// tc_common.cuh — pieces shared by the tensor-core scorer (pairwise_tc.cu) and its callers.
#pragma once
#include <cuda.h>
#include <cstdlib>
#include "common.cuh"
#include "ptx.cuh"

namespace b200kge {
namespace tc {

constexpr int STG_LD = 33;   // padded row of the per-warp transpose staging buffer

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

// Epilogue.  The accumulator tile is staged in shared memory with one row per thread, so one thread owns
// one query row and walks 32-column chunks; every per-row reduction is thread-local.  Warp-uniform fast
// paths for full chunks, optional operands resolved once per chunk, the one-hot label handled outside the
// element loop, and two threads per row (each takes half of the tile's columns).

constexpr float LOG2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;

__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// 32 columns [c0, c0+32) of row `row`; v = raw accumulator bits.  FULL: all 32 columns < m.
// `side`: this row's 32 entries of the dense label matrix (BCE/KL) or of the filter matrix (rank),
// already staged in shared memory by the warp (coalesced loads), or nullptr.
template <int EPI, bool FULL>
__device__ __forceinline__ void epi_chunk32(const EpiParams& P, RowState<EPI>& st, int64_t row, float aux,
                                            const uint32_t (&v)[32], int64_t c0, int64_t m,
                                            const float* __restrict__ side) {
  const int nvalid = FULL ? 32 : (int)(m - c0);   // > 0 by construction
  if constexpr (EPI == EPI_BCE) {
    // sum softplus(z) - sum y*z,  softplus(z) = max(z,0) + log(1 + exp(-|z|))   (loss.py:150-157;
    // torch's kernel also evaluates log(1+e) with a plain log, so tiny e drop out identically)
    const float off = P.offset;
    float amax = 0.f, alg = 0.f;
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      if (FULL || c < nvalid) {
        const float z = __uint_as_float(v[c]) + off;
        const float e = fast_ex2(-fabsf(z) * LOG2E);
        alg += __log2f(1.0f + e);
        amax += fmaxf(z, 0.f);
      }
    }
    st.a += fmaf(alg, LN2, amax);
    if (side) {
      float b = 0.f;
#pragma unroll
      for (int c = 0; c < 32; ++c)
        if (FULL || c < nvalid) b = fmaf(side[c], __uint_as_float(v[c]) + off, b);
      st.b += b;
    } else {
      const int rel = __float_as_int(aux) - (int)c0;      // one-hot label relative to this chunk
      if ((unsigned)rel < (unsigned)nvalid) {
#pragma unroll
        for (int c = 0; c < 32; ++c)
          if (c == rel) st.b += __uint_as_float(v[c]) + off;
      }
    }
  } else if constexpr (EPI == EPI_KL) {
    // online logsumexp: chunk max first, then ONE exp per element   (loss.py:198-213)
    float cm = B2K_NEG_HUGE;
#pragma unroll
    for (int c = 0; c < 32; ++c)
      if (FULL || c < nvalid) cm = fmaxf(cm, __uint_as_float(v[c]));
    const float mn = fmaxf(st.m, cm);
    const float mn2 = mn * LOG2E;
    float acc = 0.f;
#pragma unroll
    for (int c = 0; c < 32; ++c)
      if (FULL || c < nvalid) acc += fast_ex2(fmaf(__uint_as_float(v[c]), LOG2E, -mn2));
    st.s = fmaf(st.s, fast_ex2((st.m - mn) * LOG2E), acc);
    st.m = mn;
    if (side) {
#pragma unroll
      for (int c = 0; c < 32; ++c) {
        if (FULL || c < nvalid) {
          const float yy = side[c];
          if (yy != 0.f) {
            st.y_sum += yy;
            st.yx = fmaf(yy, __uint_as_float(v[c]), st.yx);
            st.ylogy = fmaf(yy, __logf(yy), st.ylogy);
          }
        }
      }
    } else {
      const int rel = __float_as_int(aux) - (int)c0;
      if ((unsigned)rel < (unsigned)nvalid) {
#pragma unroll
        for (int c = 0; c < 32; ++c)
          if (c == rel) { st.y_sum += 1.0f; st.yx += __uint_as_float(v[c]); }
      }
    }
  } else if constexpr (EPI == EPI_RANK) {
    // eval_entity_ranking.py:561-596; `allowed` depends on the row only -> hoisted
    const float t = aux;
    const float allowed = __fadd_rn(P.atol, fabsf(__fmul_rn(P.rtol, t)));
    const float* __restrict__ f = side;
    unsigned int gt = 0, cl = 0;
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      if (FULL || c < nvalid) {
        float x = __uint_as_float(v[c]);
        if (f) x = __fsub_rn(x, f[c]);
        if (isnan(x)) x = -INFINITY;
        const float actual = fabsf(__fsub_rn(x, t));
        const bool close = (x == t) || (isfinite(actual) && actual <= allowed);
        cl += close ? 1u : 0u;
        gt += (!close && x > t) ? 1u : 0u;
      }
    }
    st.greater += gt;
    st.close += cl;
  }
}

// Epilogue of NCH 32-column chunks of one accumulator tile for the warp owning 32 of its rows and columns
// [col_first, col_first + 32*NCH); `acc` points at this thread's row, first column of the span.
// SCALED (pre-split fp16 planes): the accumulator holds the product of row-scaled
// operands; score = acc * row_scale * col_scale[column] (both exact powers of two).  col_scale must be
// readable (and 16-byte aligned) for 32 floats from any chunk start < m.
template <int EPI, int NCH, bool SCALED = false>
__device__ __forceinline__ void epilogue_tile(const EpiParams& P, RowState<EPI>& st, float aux,
                                              const float* acc,
                                              int64_t tile_row0 /* first row of this warp's 32 */,
                                              int64_t e0 /* global column of the first chunk */, int64_t nq,
                                              int64_t m, float* my_stg, int lane, float row_scale = 1.f,
                                              const float* __restrict__ col_scale = nullptr,
                                              int64_t csr_end = 0 /* end of this row's CSR segment (0: none) */) {
  const int64_t row = tile_row0 + lane;
  const bool row_ok = row < nq;
  // CSR side input: position of the first listed column >= e0 in this row's segment (one binary search per span)
  int64_t csr_cur = 0;
  if (csr_end > 0) csr_cur = csr_lower_bound(P.csr_col, __ldg(P.csr_off + row), csr_end, e0);
#pragma unroll 1
  for (int j = 0; j < NCH; ++j) {
    const int64_t c0 = e0 + j * 32;
    if (c0 >= m) break;                                   // warp-uniform: chunk entirely out of range
    uint32_t v[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) v[c] = __float_as_uint(acc[j * 32 + c]);
    if constexpr (SCALED) {
      float4 cs[8];
#pragma unroll
      for (int g = 0; g < 8; ++g) cs[g] = __ldg(reinterpret_cast<const float4*>(col_scale + c0) + g);
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        v[4 * g + 0] = __float_as_uint(__uint_as_float(v[4 * g + 0]) * (row_scale * cs[g].x));
        v[4 * g + 1] = __float_as_uint(__uint_as_float(v[4 * g + 1]) * (row_scale * cs[g].y));
        v[4 * g + 2] = __float_as_uint(__uint_as_float(v[4 * g + 2]) * (row_scale * cs[g].z));
        v[4 * g + 3] = __float_as_uint(__uint_as_float(v[4 * g + 3]) * (row_scale * cs[g].w));
      }
    }
    if (csr_cur < csr_end) {
      // listed columns of this row inside [c0, c0 + 32): emit their scores (losses) or filter them (rank)
      int64_t cj = __ldg(P.csr_col + csr_cur);
      while (cj < c0 + 32) {
        const int rel = (int)(cj - c0);
        if constexpr (EPI == EPI_RANK) {
          if (!P.csr_skip || __ldg(P.csr_skip + row) != cj) {
#pragma unroll
            for (int c = 0; c < 32; ++c)
              if (c == rel) v[c] = 0xff800000u;            // -inf: neither greater nor close (for a finite true score)
          }
        } else {
          uint32_t x = 0;
#pragma unroll
          for (int c = 0; c < 32; ++c)
            if (c == rel) x = v[c];
          if (cj < m) P.csr_out[csr_cur] = __uint_as_float(x);
        }
        if (++csr_cur >= csr_end) break;
        cj = __ldg(P.csr_col + csr_cur);
      }
    }
    if constexpr (EPI == EPI_BCE || EPI == EPI_KL) {
      if (P.csr_extra && c0 == 0 && row_ok) P.csr_out[P.csr_nnz + row] = __uint_as_float(v[0]);
    }
    if constexpr (EPI == EPI_STORE) {
      // transpose a 32x32 block through smem: each store instruction then writes 32 consecutive
      // entities of ONE query row (coalesced 128 B) whatever the row stride is
#pragma unroll
      for (int c = 0; c < 32; ++c) my_stg[lane * STG_LD + c] = __uint_as_float(v[c]);
      __syncwarp();
      const int64_t col = c0 + lane;
      // rows of this warp map to consecutive output rows unless the block straddles the sp|po seam
      const bool seam = P.n_rows_out > 0 && tile_row0 < P.n_rows_out && tile_row0 + 32 > P.n_rows_out;
      if (!seam) {
        int64_t r0 = tile_row0, cb = 0;
        if (P.n_rows_out > 0 && r0 >= P.n_rows_out) { r0 -= P.n_rows_out; cb = P.col_block; }
        float* __restrict__ p = P.out + r0 * P.ldo + cb + col;
        const int nrows = (int)((nq - tile_row0) < 32 ? (nq - tile_row0) : 32);
        float t[32];
#pragma unroll
        for (int rr = 0; rr < 32; ++rr) t[rr] = my_stg[rr * STG_LD + lane];
        if (col < m && P.accumulate_out) {
#pragma unroll
          for (int rr = 0; rr < 32; ++rr)
            if (rr < nrows) atomicAdd(p + rr * P.ldo, t[rr]);
        } else if (col < m) {
          if (nrows == 32) {
#pragma unroll
            for (int rr = 0; rr < 32; ++rr) p[rr * P.ldo] = t[rr];
          } else {
#pragma unroll
            for (int rr = 0; rr < 32; ++rr)
              if (rr < nrows) p[rr * P.ldo] = t[rr];
          }
          for (int g = 0; g < P.n_peers; ++g) {        // same offsets in the peers' symmetric buffers
            float* __restrict__ pp = P.out_peer[g] + (p - P.out);
#pragma unroll
            for (int rr = 0; rr < 32; ++rr)
              if (rr < nrows) pp[rr * P.ldo] = t[rr];
          }
        }
      } else if (col < m) {
        for (int rr = 0; rr < 32; ++rr) {
          int64_t r = tile_row0 + rr;
          if (r < nq) {
            int64_t cb = 0;
            if (r >= P.n_rows_out) { r -= P.n_rows_out; cb = P.col_block; }
            const int64_t at = r * P.ldo + cb + col;
            const float xv = my_stg[rr * STG_LD + lane];
            P.out[at] = xv;
            for (int g = 0; g < P.n_peers; ++g) P.out_peer[g][at] = xv;
          }
        }
      }
      __syncwarp();
    } else {
      // dense side matrix (labels / filter): the warp stages its 32x32 block through shared memory
      // with coalesced 128-B row reads; each thread then reads its own row from smem (reading the
      // matrix directly would touch 32 different rows per load instruction)
      const float* gside = nullptr;
      int64_t gld = 0;
      if constexpr (EPI == EPI_RANK) { gside = P.filter; gld = P.ldf; }
      else { gside = P.label_dense; gld = P.ldl; }
      const float* side = nullptr;
      if (gside) {
        const int64_t col = c0 + lane;
        const bool col_ok = col < m;
#pragma unroll 8
        for (int rr = 0; rr < 32; ++rr) {
          const int64_t r = tile_row0 + rr;
          my_stg[rr * STG_LD + lane] = (col_ok && r < nq) ? __ldg(gside + r * gld + col) : 0.f;
        }
        __syncwarp();
        side = my_stg + lane * STG_LD;
      }
      if (row_ok) {
        if (c0 + 32 <= m) epi_chunk32<EPI, true>(P, st, row, aux, v, c0, m, side);
        else              epi_chunk32<EPI, false>(P, st, row, aux, v, c0, m, side);
      }
      if (gside) __syncwarp();
    }
  }
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
int launch_div_scores(const float* g, int64_t ldg, const float* z, int64_t ldz, int64_t n, int64_t E, float* W, int64_t ldw,
                      cudaStream_t st);
int launch_row_lse(const float* z, int64_t ldz, int64_t nq, int64_t E, const int64_t* label_idx, float* row_stat,
                   cudaStream_t st);
// num_rel > 0 (dir < 0 only): the reciprocal layout, rows [n,2n) unfold as sp_ into d_ent[o], d_rel[p + num_rel]
int launch_unfold_distance(int model, const Rows& ent, const Rows& rel, const int64_t* triples, int64_t n, int dir,
                           const float* dQ, int64_t ldq, float* d_ent, int64_t lde, float* d_rel, int64_t ldr,
                           cudaStream_t st, int64_t num_rel = 0);
int launch_grad_planes_csr(const float* z, int64_t ldz, int64_t nq, int64_t E, const int64_t* csr_off,
                           const int64_t* csr_col, float a, float b, float* row_stat, float offset, float inv_n,
                           void* g_hi, void* g_lo, int64_t Ep, void* gt_hi, void* gt_lo, int64_t Np, float* g_scale,
                           float* gt_scale, cudaStream_t st);
// CSR-label losses (csr_loss.cu).
int launch_csr_expand(const int64_t* off, const int64_t* col, int64_t n, int64_t nnz, int extra, const int64_t* q_idx,
                      const int64_t* p_idx, int64_t* qsel, int64_t* psel, int64_t* esel, cudaStream_t st);
int launch_csr_rows(int loss_kind, const int64_t* off, const int64_t* col, const float* zpos, int64_t n, int64_t nnz,
                    const float* fused, const float* zsum, float a, float b, float E, float offset, float* row_loss,
                    cudaStream_t st);
int launch_rows_sum(const float* rows, int64_t n, float scale, float* out, cudaStream_t st);
int launch_row_score_sums(const float* Q, int64_t ldq, int64_t n, const float* T, int64_t ldt, int64_t E, int K,
                          float* scratch, float* zsum, cudaStream_t st);
// G (optional, [n, 1+K], row stride ldg): dL/dz already scaled, read instead of the BCE gradient
int launch_ns_backward(int model, float l_norm, const Rows& ent, const Rows& rel, const int64_t* triples, int slot,
                       const int64_t* neg, int64_t n, int64_t K, float offset, float inv_batch, const float* G,
                       int64_t ldg, float* d_ent, int64_t lde, float* d_rel, int64_t ldr, float* dQ, int64_t ldq,
                       cudaStream_t st);
// row-wise KgeLoss of a negative-sampling block (ns_loss.cu): part[2 i] = row loss (BCE finaliser layout), G optional
int launch_ns_loss(int loss_kind, const float* scores, int64_t lds, int64_t n, int64_t m, const int64_t* label_idx,
                   float arg, float temperature, float scale, float* part, float* G, int64_t ldg, cudaStream_t st);
int launch_penalty(const Rows& tab, const float* counts, float p, int complex_abs, float scale, float* scratch,
                   size_t scratch_floats, float* out, cudaStream_t st);
int launch_normalize_rows(float* w, int64_t ld, int64_t rows, int dim, float p, cudaStream_t st);
int launch_unfold(int model, const Rows& ent, const Rows& rel, const int64_t* triples, int64_t n, int dir,
                  const float* dQ, int64_t ldq, float* d_ent, int64_t lde, float* d_rel, int64_t ldr, cudaStream_t st,
                  int64_t num_rel = 0);

}  // namespace b200kge
