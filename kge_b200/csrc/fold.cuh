// fold.cuh — per-element relation folding shared by fold.cu (prologue) and rowwise.cu (NS).
#pragma once
#include "common.cuh"

namespace b200kge {

// q[k] for the non-RESCAL scorers; `sp` selects the sp_ fold (a = subject row) or the _po fold
// (a = object row).  h = D/2.  See fold.cu for the algebra and reference citations.
template <int MODEL>
__device__ __forceinline__ float fold_element(bool sp, const float* __restrict__ a,
                                              const float* __restrict__ p, int k, int h) {
  float v;
  if constexpr (MODEL == B200KGE_COMPLEX) {
    const int kk = (k < h) ? k : k - h;
    const float a_re = a[kk], a_im = a[kk + h], p_re = p[kk], p_im = p[kk + h];
    if (sp) v = (k < h) ? (a_re * p_re - a_im * p_im) : (a_im * p_re + a_re * p_im);
    else    v = (k < h) ? (p_re * a_re + p_im * a_im) : (p_re * a_im - p_im * a_re);
  } else if constexpr (MODEL == B200KGE_DISTMULT) {
    v = a[k] * p[k];
  } else if constexpr (MODEL == B200KGE_SIMPLE) {
    const int kk = (k < h) ? k : k - h;
    if (sp) v = (k < h) ? 0.5f * a[h + kk] * p[h + kk] : 0.5f * a[kk] * p[kk];
    else    v = (k < h) ? 0.5f * a[h + kk] * p[kk] : 0.5f * a[kk] * p[h + kk];
  } else if constexpr (MODEL == B200KGE_CP) {
    v = sp ? a[k] * p[k] : a[h + k] * p[k];
  } else if constexpr (MODEL == B200KGE_TRANSE) {
    v = sp ? a[k] + p[k] : a[k] - p[k];
  } else {  // ROTATE
    const int kk = (k < h) ? k : k - h;
    float sn, c;
    sincosf(p[kk], &sn, &c);
    const float a_re = a[kk], a_im = a[kk + h];
    if (sp) v = (k < h) ? (a_re * c - a_im * sn) : (a_re * sn + a_im * c);
    else    v = (k < h) ? (c * a_re + sn * a_im) : (c * a_im - sn * a_re);
  }
  return v;
}

// q[k] of the s_o fold (relation prediction, kge_model.py:727-747): score(s, r, o) = q . rel[r][0:K] with the
// spo_kernel formulas (rowwise.cu) regrouped around the relation row.  Not RESCAL (fold_so_kernel).  h = D/2.
template <int MODEL>
__device__ __forceinline__ float fold_so_element(const float* __restrict__ s, const float* __restrict__ o, int k, int h) {
  if constexpr (MODEL == B200KGE_COMPLEX) {
    const int kk = (k < h) ? k : k - h;
    const float s_re = s[kk], s_im = s[kk + h], o_re = o[kk], o_im = o[kk + h];
    return (k < h) ? (s_re * o_re + s_im * o_im) : (s_re * o_im - s_im * o_re);
  } else if constexpr (MODEL == B200KGE_DISTMULT) {
    return s[k] * o[k];
  } else if constexpr (MODEL == B200KGE_SIMPLE) {
    return 0.5f * s[k] * o[k < h ? k + h : k - h];
  } else {  // CP: K = h
    return s[k] * o[k + h];
  }
}

// RESCAL fold for one row by a whole CTA: sh_a holds the entity row (length D) in shared memory,
// emit(k, value) receives q[k].
template <class Emit>
__device__ __forceinline__ void fold_rescal_block(bool sp, const float* sh_a,
                                                  const float* __restrict__ p, int D, Emit emit) {
  if (sp) {  // q_j = sum_i s_i M[i,j]      rescal.py:37-40
    for (int j = threadIdx.x; j < D; j += blockDim.x) {
      float acc = 0.f;
      for (int r = 0; r < D; ++r) acc = fmaf(sh_a[r], p[(int64_t)r * D + j], acc);
      emit(j, acc);
    }
  } else {   // q_i = sum_j M[i,j] o_j      rescal.py:43-46
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    for (int r = warp; r < D; r += nw) {
      float acc = 0.f;
      for (int j = lane; j < D; j += 32) acc = fmaf(p[(int64_t)r * D + j], sh_a[j], acc);
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
      if (lane == 0) emit(r, acc);
    }
  }
}

// Folded-problem descriptor of a model: pair op, reduction length, candidate column offset.
__host__ __device__ inline Folded folded_problem(int model, int combine, int D, float l_norm) {
  Folded f;
  f.K = D; f.col_off = 0; f.pair_op = PAIR_DOT;
  if (model == B200KGE_CP) { f.K = D / 2; f.col_off = (combine == B200KGE_SP_) ? D / 2 : 0; }
  else if (model == B200KGE_TRANSE) f.pair_op = (l_norm == 1.0f) ? PAIR_L1 : (l_norm == 2.0f ? PAIR_L2 : PAIR_LP);
  else if (model == B200KGE_ROTATE) f.pair_op = (l_norm == 1.0f) ? PAIR_CMOD_L1 : PAIR_CMOD_LP;
  return f;
}

}  // namespace b200kge
