// presplit.cu — operand split for the pre-split fp16 tensor-core kernel (pairwise_tc.cu, F16X3 mode): the
// default path of the dot family (B200KGE_PREC_AUTO / F16X3).
//
// A fp32 value x of row r is represented as  x = inv_scale[r] * (hi + lo),  hi = fp16_rn(x * 2^s),
// lo = fp16_rn(x * 2^s - hi),  2^s chosen per row so that max|x * 2^s| lies in [2^13, 2^14): 22 significant
// bits, no fp16 overflow, lo in the normal range for every element within 2^-13 of the row maximum.  The
// three products hi*hi + hi*lo + lo*hi on the f16 tensor pipe (fp32 accumulate) then reproduce the fp32 GEMM
// of the reference (torch.mm in complex.py:37,39 etc.) to ~5e-7 of the score rms before accumulation
// round-off — the same accuracy class as the in-kernel tf32+bf16 split, at 6 instead of 8 MMA slots per 32
// reduction elements and without any shared-memory round trip in the main loop.
//
// One warp per row, two passes over the row (|max|, then convert; the second read hits L1).  HBM-bound:
// 4 B read + 4 B written per element.
#include <cuda_fp16.h>
#include "fold.cuh"
#include "tc_common.cuh"

namespace b200kge {

namespace {

constexpr int PS_WARPS = 8;

__device__ __forceinline__ void presplit_row(const SplitSet& S, int64_t r, int lane) {
  if (r >= S.rows) {
    if (r < S.rows_pad && lane == 0) S.inv_scale[r] = 0.f;
    return;
  }
  const int64_t src_row = S.idx ? S.idx[r] : r;
  const float* __restrict__ x = S.src + src_row * S.ld + S.col_off;
  const int K = S.K, Kp = S.Kp;
  const bool vec = (K % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
  float amax = 0.f;
  bool bad = false;
  if (vec) {
    for (int k = lane * 4; k < K; k += 128) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(x + k));
      amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
      bad |= !(isfinite(v.x) && isfinite(v.y) && isfinite(v.z) && isfinite(v.w));
    }
  } else {
    for (int k = lane; k < K; k += 32) {
      const float v = __ldg(x + k);
      amax = fmaxf(amax, fabsf(v));
      bad |= !isfinite(v);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  bad = __any_sync(0xffffffffu, bad);
  int e = 13;                                    // => scale 1 for all-zero or non-finite rows
  if (amax > 0.f && !bad) {
    e = ilogbf(amax);
    e = e < -60 ? -60 : (e > 60 ? 60 : e);
  }
  const float mul = scalbnf(1.f, 13 - e), inv = scalbnf(1.f, e - 13);
  __half* __restrict__ hi = reinterpret_cast<__half*>(S.hi) + r * Kp;
  __half* __restrict__ lo = reinterpret_cast<__half*>(S.lo) + r * Kp;
  if (vec) {
    for (int k = lane * 4; k < Kp; k += 128) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k < K) v = __ldg(reinterpret_cast<const float4*>(x + k));
      const float s[4] = {v.x * mul, v.y * mul, v.z * mul, v.w * mul};
      __half h[4], l[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        h[i] = __float2half_rn(s[i]);
        l[i] = __float2half_rn(s[i] - __half2float(h[i]));
      }
      uint2 ph, pl;
      ph.x = (uint32_t)__half_as_ushort(h[0]) | ((uint32_t)__half_as_ushort(h[1]) << 16);
      ph.y = (uint32_t)__half_as_ushort(h[2]) | ((uint32_t)__half_as_ushort(h[3]) << 16);
      pl.x = (uint32_t)__half_as_ushort(l[0]) | ((uint32_t)__half_as_ushort(l[1]) << 16);
      pl.y = (uint32_t)__half_as_ushort(l[2]) | ((uint32_t)__half_as_ushort(l[3]) << 16);
      *reinterpret_cast<uint2*>(hi + k) = ph;     // Kp % 64 == 0 and 256-byte aligned planes: 8-byte aligned
      *reinterpret_cast<uint2*>(lo + k) = pl;
    }
  } else {
    for (int k = lane; k < Kp; k += 32) {
      const float s = (k < K) ? __ldg(x + k) * mul : 0.f;
      const __half h = __float2half_rn(s);
      hi[k] = h;
      lo[k] = __float2half_rn(s - __half2float(h));
    }
  }
  if (lane == 0) S.inv_scale[r] = inv;
}

__global__ void __launch_bounds__(PS_WARPS * 32)
presplit_kernel(const SplitSet A, const SplitSet B, const int blocks_a) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if ((int)blockIdx.x < blocks_a) presplit_row(A, (int64_t)blockIdx.x * PS_WARPS + warp, lane);
  else presplit_row(B, (int64_t)(blockIdx.x - blocks_a) * PS_WARPS + warp, lane);
}

// Long rows (the transposed operands of the backward GEMMs: K = E or 2n elements per row, only ~1000 rows): one warp per
// row leaves most SMs idle and walks 114 strides per pass (83.6 us for 2 x 30 MB at E = 14 541).  One CTA per row instead.
__global__ void __launch_bounds__(PS_WARPS * 32)
presplit_longrow_kernel(const SplitSet A, const SplitSet B, const int rows_a) {
  __shared__ float red[PS_WARPS];
  __shared__ int bad_any;
  const bool first = (int)blockIdx.x < rows_a;
  const SplitSet& S = first ? A : B;
  const int64_t r = first ? blockIdx.x : blockIdx.x - rows_a;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (r >= S.rows) {
    if (threadIdx.x == 0) S.inv_scale[r] = 0.f;
    return;
  }
  const int64_t src_row = S.idx ? S.idx[r] : r;
  const float* __restrict__ x = S.src + src_row * S.ld + S.col_off;
  const int K = S.K, Kp = S.Kp;
  if (threadIdx.x == 0) bad_any = 0;
  float amax = 0.f;
  bool bad = false;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float v = __ldg(x + k);
    amax = fmaxf(amax, fabsf(v));
    bad |= !isfinite(v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  __syncthreads();
  if (__any_sync(0xffffffffu, bad) && lane == 0) bad_any = 1;
  if (lane == 0) red[warp] = amax;
  __syncthreads();
  amax = red[0];
#pragma unroll
  for (int w = 1; w < PS_WARPS; ++w) amax = fmaxf(amax, red[w]);
  int e = 13;                                    // same scaling rule as presplit_row
  if (amax > 0.f && !bad_any) {
    e = ilogbf(amax);
    e = e < -60 ? -60 : (e > 60 ? 60 : e);
  }
  const float mul = scalbnf(1.f, 13 - e);
  __half2* __restrict__ hi = reinterpret_cast<__half2*>(reinterpret_cast<__half*>(S.hi) + r * Kp);
  __half2* __restrict__ lo = reinterpret_cast<__half2*>(reinterpret_cast<__half*>(S.lo) + r * Kp);
  for (int k = threadIdx.x * 2; k < Kp; k += blockDim.x * 2) {        // Kp is even; second read hits L1 / L2
    const float s0 = (k < K) ? __ldg(x + k) * mul : 0.f, s1 = (k + 1 < K) ? __ldg(x + k + 1) * mul : 0.f;
    const __half h0 = __float2half_rn(s0), h1 = __float2half_rn(s1);
    hi[k >> 1] = __halves2half2(h0, h1);
    lo[k >> 1] = __halves2half2(__float2half_rn(s0 - __half2float(h0)), __float2half_rn(s1 - __half2float(h1)));
  }
  if (threadIdx.x == 0) S.inv_scale[r] = scalbnf(1.f, e - 13);
}

// ---------------------------------------------------------------------------------------------
// The whole prologue of a fused 1vsAll step in ONE launch (train_1vsAll.py:59-65,75-76 up to the scorer):
//   blocks [0, 2n)   : query row b — gather + relation fold of (s_b, p_b) for the sp_ direction (b < n) or of
//                      (o_b, p_b) for _po (b >= n) into shared memory, row scale, hi/lo planes, inverse scale, and
//                      the row's label (o_b | s_b); block 0 also zeroes the finalisation ticket
//   blocks [2n, ...) : table rows, one warp per row (presplit_row)
// replaces prep_1vsall_kernel + presplit_kernel (one launch and one launch gap less per step; the folded fp32 query
// matrix never reaches HBM).
constexpr int PQ_THREADS = PS_WARPS * 32;

// RECIP: the reciprocal layout of prep_1vsall_kernel (fold.cu) — block n+b folds (o_b, p_b + num_rel) with the sp_ fold.
template <int MODEL, bool RECIP>
__global__ void __launch_bounds__(PQ_THREADS)
prep_split_1vsall_kernel(Rows ent, Rows rel, const int64_t* __restrict__ tri, int64_t n, const SplitSet Qs,
                         const SplitSet Ts, int64_t* __restrict__ labels2n, unsigned int* ticket, int K,
                         int64_t num_rel) {
  extern __shared__ float sh[];      // [Kp] folded row (+ [D] entity row for RESCAL)
  const int64_t b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (b >= 2 * n) {
    presplit_row(Ts, (b - 2 * n) * PS_WARPS + warp, lane);
    return;
  }
  __shared__ float red[PS_WARPS];
  __shared__ int bad_any;
  const bool first = b < n;
  const bool sp = RECIP || first;
  const int64_t i = first ? b : b - n;
  const int64_t si = tri[3 * i], pi = tri[3 * i + 1], oi = tri[3 * i + 2];
  const float* __restrict__ a = ent.base + (first ? si : oi) * ent.ld;
  const float* __restrict__ p = rel.base + (RECIP && !first ? pi + num_rel : pi) * rel.ld;
  const int D = ent.dim, h = D >> 1, Kp = Qs.Kp;
  if (threadIdx.x == 0) {
    labels2n[b] = first ? oi : si;
    bad_any = 0;
  }
  if (b == 0 && ticket && threadIdx.x == 0) *ticket = 0u;                   // the finaliser's last-block counter
  float* q = sh;
  if constexpr (MODEL == B200KGE_RESCAL) {
    float* sh_a = sh + Kp;
    for (int k = threadIdx.x; k < D; k += blockDim.x) sh_a[k] = a[k];
    __syncthreads();
    fold_rescal_block(sp, sh_a, p, D, [&](int k, float v) { q[k] = v; });
  } else {
    for (int k = threadIdx.x; k < K; k += blockDim.x) q[k] = fold_element<MODEL>(sp, a, p, k, h);
  }
  for (int k = K + threadIdx.x; k < Kp; k += blockDim.x) q[k] = 0.f;
  __syncthreads();
  float amax = 0.f;
  bool bad = false;
  for (int k = threadIdx.x; k < K; k += blockDim.x) { const float v = q[k]; amax = fmaxf(amax, fabsf(v)); bad |= !isfinite(v); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if (__any_sync(0xffffffffu, bad) && lane == 0) bad_any = 1;
  if (lane == 0) red[warp] = amax;
  __syncthreads();
  amax = red[0];
#pragma unroll
  for (int w = 1; w < PS_WARPS; ++w) amax = fmaxf(amax, red[w]);
  int e = 13;                                    // same scaling rule as presplit_row
  if (amax > 0.f && !bad_any) {
    e = ilogbf(amax);
    e = e < -60 ? -60 : (e > 60 ? 60 : e);
  }
  const float mul = scalbnf(1.f, 13 - e);
  __half* __restrict__ hi = reinterpret_cast<__half*>(Qs.hi) + b * Kp;
  __half* __restrict__ lo = reinterpret_cast<__half*>(Qs.lo) + b * Kp;
  for (int k = threadIdx.x * 4; k < Kp; k += blockDim.x * 4) {
    __half hh[4], ll[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float sv = q[k + j] * mul;
      hh[j] = __float2half_rn(sv);
      ll[j] = __float2half_rn(sv - __half2float(hh[j]));
    }
    uint2 ph, pl;
    ph.x = (uint32_t)__half_as_ushort(hh[0]) | ((uint32_t)__half_as_ushort(hh[1]) << 16);
    ph.y = (uint32_t)__half_as_ushort(hh[2]) | ((uint32_t)__half_as_ushort(hh[3]) << 16);
    pl.x = (uint32_t)__half_as_ushort(ll[0]) | ((uint32_t)__half_as_ushort(ll[1]) << 16);
    pl.y = (uint32_t)__half_as_ushort(ll[2]) | ((uint32_t)__half_as_ushort(ll[3]) << 16);
    *reinterpret_cast<uint2*>(hi + k) = ph;
    *reinterpret_cast<uint2*>(lo + k) = pl;
  }
  if (threadIdx.x == 0) Qs.inv_scale[b] = scalbnf(1.f, e - 13);
}

}  // namespace

int launch_prep_split_1vsall(int model, const Rows& ent, const Rows& rel, const int64_t* triples, int64_t n,
                             const SplitSet& Qs, const SplitSet& Ts, int64_t* labels2n, unsigned int* ticket,
                             cudaStream_t st, int64_t num_rel) {
  if (n == 0) return 0;
  const int D = ent.dim;
  const int K = (model == B200KGE_CP) ? D / 2 : D;
  const int64_t tb = (Ts.rows_pad + PS_WARPS - 1) / PS_WARPS;
  if (2 * n + tb >= (1ll << 31)) { set_error("too many rows for the fused prologue"); return B200KGE_ERR_INVALID; }
  const size_t smem = ((size_t)Qs.Kp + (model == B200KGE_RESCAL ? D : 0)) * sizeof(float);
  if (smem > 48 * 1024) { set_error("embedding too wide for the fused prologue"); return B200KGE_ERR_UNSUPPORTED; }
  dim3 grid((unsigned)(2 * n + tb)), block(PQ_THREADS);
#define B2K_PS(M) case M: prep_split_1vsall_kernel<M, false><<<grid, block, smem, st>>>(ent, rel, triples, n, Qs, Ts, labels2n, ticket, K, 0); break;
#define B2K_PS_R(M) case M: prep_split_1vsall_kernel<M, true><<<grid, block, smem, st>>>(ent, rel, triples, n, Qs, Ts, labels2n, ticket, K, num_rel); break;
  if (num_rel > 0) {
    // reciprocal: both halves are sp_ queries, so CP (table columns [h, D)) stacks too
    switch (model) {
      B2K_PS_R(B200KGE_COMPLEX) B2K_PS_R(B200KGE_DISTMULT) B2K_PS_R(B200KGE_SIMPLE) B2K_PS_R(B200KGE_CP)
      B2K_PS_R(B200KGE_RESCAL)
      default: set_error("model %d has no fused pre-split prologue", model); return B200KGE_ERR_UNSUPPORTED;
    }
  } else {
    switch (model) {
      B2K_PS(B200KGE_COMPLEX) B2K_PS(B200KGE_DISTMULT) B2K_PS(B200KGE_SIMPLE) B2K_PS(B200KGE_RESCAL)
      default: set_error("model %d has no fused pre-split prologue", model); return B200KGE_ERR_UNSUPPORTED;
    }
  }
#undef B2K_PS
#undef B2K_PS_R
  B2K_LAUNCH_CHECK("prep_split_1vsall_kernel");
  return 0;
}

int launch_presplit(const SplitSet& A, const SplitSet& B, cudaStream_t st) {
  const int64_t ba = (A.rows_pad + PS_WARPS - 1) / PS_WARPS, bb = (B.rows_pad + PS_WARPS - 1) / PS_WARPS;
  if (ba + bb == 0) return 0;
  if (ba + bb >= (1ll << 31)) { set_error("too many rows for the operand split"); return B200KGE_ERR_INVALID; }
  if ((A.K >= 4096 || (B.rows_pad > 0 && B.K >= 4096)) && A.rows_pad + B.rows_pad < (1ll << 31)) {
    presplit_longrow_kernel<<<(unsigned)(A.rows_pad + B.rows_pad), PS_WARPS * 32, 0, st>>>(A, B, (int)A.rows_pad);
    B2K_LAUNCH_CHECK("presplit_longrow_kernel");
    return 0;
  }
  presplit_kernel<<<(unsigned)(ba + bb), PS_WARPS * 32, 0, st>>>(A, B, (int)ba);
  B2K_LAUNCH_CHECK("presplit_kernel");
  return 0;
}

}  // namespace b200kge
