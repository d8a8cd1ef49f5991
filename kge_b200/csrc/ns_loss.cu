// ns_loss.cu — the row-wise KgeLoss of a negative-sampling block and its gradient.
//
//  * ns_loss_kernel: one block per row of an [n, m] score block (column l_i = the row's positive, label 1; every
//    other column label 0).  Up to three sweeps over the row — a max (log-sum-exp / softmax stabiliser), the sums,
//    and the gradient G = dL/dz * scale when asked — so any m works, from K = 1 to rows far wider than a block.
//    Per row, with z_l the positive, z_c the negatives (K = m - 1), o = offset and sp(x) = log(1 + e^x):
//      bce                   sum_c bce(z_c + o, y_c)                                           loss.py:153-159
//      kl                    lse(z) - z_l                                                      loss.py:198-213
//      bce_mean              (bce(z_l + o, 1) + sum_c bce(z_c + o, 0) / K) / 2                 loss.py:160-168
//      bce_self_adversarial  (bce(z_l + o, 1) + sum_c w_c bce(z_c + o, 0)) / 2,
//                            w = softmax(T (z_c + o)) over the negatives, detached             loss.py:169-187
//      margin_ranking        sum_c max(0, margin - z_l + z_c)  (a tie counts as active)        loss.py:240-252
//      soft_margin           sp(-z_l) + sum_c sp(z_c)                                          loss.py:216-224
//      se                    (z_l - 1)^2 + sum_c z_c^2                                         loss.py:267-274
//    The row loss goes to part[2 i] (part[2 i + 1] = 0), the layout of the BCE finaliser, so the scalar is reduced
//    by loss_finalize_kernel in its fixed order.
#include "common.cuh"

namespace b200kge {

namespace {

constexpr int NL_THREADS = 256, NL_WARPS = NL_THREADS / 32;

// softplus(x) = log(1 + e^x), stable for any |x| (the form of the BCE epilogue with y = 0)
__device__ __forceinline__ float softplus_f(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }

// fixed-order block reductions: shuffle tree per warp, warp results added in warp order by every thread
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < NL_WARPS; ++w) t += red[w];
  __syncthreads();
  return t;
}

__device__ __forceinline__ float block_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = -INFINITY;
#pragma unroll
  for (int w = 0; w < NL_WARPS; ++w) t = fmaxf(t, red[w]);
  __syncthreads();
  return t;
}

template <int KIND>
__global__ void __launch_bounds__(NL_THREADS)
ns_loss_kernel(const float* __restrict__ z, int64_t lds, int64_t m, const int64_t* __restrict__ label_idx,
               float arg, float temperature, float scale, float* __restrict__ part, float* __restrict__ G,
               int64_t ldg) {
  __shared__ float red[NL_WARPS];
  const int64_t i = blockIdx.x;
  const float* __restrict__ x = z + i * lds;
  const int64_t l = label_idx ? label_idx[i] : 0;
  const float zl = x[l];
  const float o = arg;                                   // offset (BCE family) or margin (margin ranking)
  const float inv_k = 1.0f / (float)(m - 1);

  // sweep 1: the stabiliser of the softmax (kl: over the row; self-adversarial: over the negatives' T (z + o))
  float mx = 0.f;
  if constexpr (KIND == B200KGE_LOSS_KL || KIND == B200KGE_LOSS_BCE_SELF_ADV) {
    float v = -INFINITY;
    for (int64_t c = threadIdx.x; c < m; c += NL_THREADS) {
      if (KIND == B200KGE_LOSS_KL) v = fmaxf(v, x[c]);
      else if (c != l) v = fmaxf(v, temperature * (x[c] + o));
    }
    mx = block_max(v, red);
  }

  // sweep 2: the row sums.  a: the loss terms of the negatives (or the exp sum); b: the softmax denominator of the
  // self-adversarial weights / the number of active margin terms
  float a = 0.f, b = 0.f;
  for (int64_t c = threadIdx.x; c < m; c += NL_THREADS) {
    const float v = x[c];
    if constexpr (KIND == B200KGE_LOSS_KL) {
      const float e = expf(v - mx);
      a += e;
      if (c != l) b += e;                                // 1 - softmax_l without the cancellation
    } else if (c != l) {
      if constexpr (KIND == B200KGE_LOSS_BCE || KIND == B200KGE_LOSS_BCE_MEAN) {
        a += softplus_f(v + o);
      } else if constexpr (KIND == B200KGE_LOSS_BCE_SELF_ADV) {
        const float e = expf(temperature * (v + o) - mx);
        a += e * softplus_f(v + o);
        b += e;
      } else if constexpr (KIND == B200KGE_LOSS_MARGIN_RANKING) {
        const float h = -(zl - v) + o;                   // torch: clamp_min(-y (x1 - x2) + margin, 0), y = 1
        if (h >= 0.f) { a += h; b += 1.f; }
      } else if constexpr (KIND == B200KGE_LOSS_SOFT_MARGIN) {
        a += softplus_f(v);
      } else {                                           // SE
        a = fmaf(v, v, a);
      }
    }
  }
  a = block_sum(a, red);
  if constexpr (KIND != B200KGE_LOSS_BCE && KIND != B200KGE_LOSS_BCE_MEAN && KIND != B200KGE_LOSS_SOFT_MARGIN &&
                KIND != B200KGE_LOSS_SE)
    b = block_sum(b, red);

  const float pos_bce = softplus_f(-(zl + o));           // bce(z_l + o, 1)
  if (threadIdx.x == 0) {
    float rl;
    if constexpr (KIND == B200KGE_LOSS_BCE) rl = pos_bce + a;
    else if constexpr (KIND == B200KGE_LOSS_KL) rl = (mx - zl) + logf(a);
    else if constexpr (KIND == B200KGE_LOSS_BCE_MEAN) rl = 0.5f * (pos_bce + a * inv_k);
    else if constexpr (KIND == B200KGE_LOSS_BCE_SELF_ADV) rl = 0.5f * (pos_bce + a / b);
    else if constexpr (KIND == B200KGE_LOSS_MARGIN_RANKING) rl = a;
    else if constexpr (KIND == B200KGE_LOSS_SOFT_MARGIN) rl = softplus_f(-zl) + a;
    else { const float d = zl - 1.f; rl = fmaf(d, d, a); }
    part[2 * i] = rl;
    part[2 * i + 1] = 0.f;
  }
  if (G == nullptr) return;

  // sweep 3: G[i, c] = dL/dz_ic * scale; the positive's sigma(x) - 1 is taken as -sigma(-x) and 1 - softmax_l as
  // the negatives' share, which keeps full relative precision when the positive already wins
  float* __restrict__ g = G + i * ldg;
  const float inv_a = 1.0f / a, inv_b = 1.0f / b;
  for (int64_t c = threadIdx.x; c < m; c += NL_THREADS) {
    const float v = x[c];
    const bool pos = (c == l);
    float d;
    if constexpr (KIND == B200KGE_LOSS_BCE) {
      d = pos ? -sigmoid_f(-(v + o)) : sigmoid_f(v + o);
    } else if constexpr (KIND == B200KGE_LOSS_KL) {
      d = pos ? -(b * inv_a) : expf(v - mx) * inv_a;
    } else if constexpr (KIND == B200KGE_LOSS_BCE_MEAN) {
      d = pos ? -0.5f * sigmoid_f(-(v + o)) : 0.5f * sigmoid_f(v + o) * inv_k;
    } else if constexpr (KIND == B200KGE_LOSS_BCE_SELF_ADV) {
      d = pos ? -0.5f * sigmoid_f(-(v + o))
              : 0.5f * (expf(temperature * (v + o) - mx) * inv_b) * sigmoid_f(v + o);
    } else if constexpr (KIND == B200KGE_LOSS_MARGIN_RANKING) {
      d = pos ? -b : ((-(zl - v) + o >= 0.f) ? 1.f : 0.f);
    } else if constexpr (KIND == B200KGE_LOSS_SOFT_MARGIN) {
      d = pos ? -sigmoid_f(-v) : sigmoid_f(v);
    } else {
      d = 2.f * (v - (pos ? 1.f : 0.f));
    }
    g[c] = d * scale;
  }
}

}  // namespace

int launch_ns_loss(int loss_kind, const float* scores, int64_t lds, int64_t n, int64_t m, const int64_t* label_idx,
                   float arg, float temperature, float scale, float* part, float* G, int64_t ldg, cudaStream_t st) {
  if (n == 0) return 0;
  if (n > 0x7fffffffll) { set_error("too many rows for one launch (%lld)", (long long)n); return B200KGE_ERR_UNSUPPORTED; }
#define B2K_NSL(L) case L: ns_loss_kernel<L><<<(unsigned)n, NL_THREADS, 0, st>>>(scores, lds, m, label_idx, arg, temperature, scale, part, G, ldg); break;
  switch (loss_kind) {
    B2K_NSL(B200KGE_LOSS_BCE) B2K_NSL(B200KGE_LOSS_KL) B2K_NSL(B200KGE_LOSS_BCE_MEAN) B2K_NSL(B200KGE_LOSS_BCE_SELF_ADV)
    B2K_NSL(B200KGE_LOSS_MARGIN_RANKING) B2K_NSL(B200KGE_LOSS_SOFT_MARGIN) B2K_NSL(B200KGE_LOSS_SE)
    default: set_error("unknown loss kind %d", loss_kind); return B200KGE_ERR_INVALID;
  }
#undef B2K_NSL
  B2K_LAUNCH_CHECK("ns_loss_kernel");
  return 0;
}

}  // namespace b200kge
