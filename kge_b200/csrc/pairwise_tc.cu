// pairwise_tc.cu — Hopper (sm_90a) tensor-core 1-vs-N scorer for the dot-product family (ComplEx / DistMult /
// SimplE / CP / RESCAL after folding), fp32-equivalent through an operand split, with the consumer of the scores
// (the plain [n,E] store, BCE / KL loss, rank counting) fused into the epilogue.
//
//   S[q, e] = sum_k Q[q,k] * T[e,k]          Q: folded queries [nq, K]     T: entity table [m, K]
//
// replaces the reference's torch.mm over concatenated operands (complex.py:37,39, distmult.py:19,21,
// simple.py:25-29, cp.py:24,26, rescal.py:41,47) AND whatever consumes the scores next in ONE kernel.
//
// Operand forms (MODE), one kernel:
//   F16X3   pre-split fp16 planes (presplit.cu / grad.cu, THE default): S = qs*ts*(Qh*Th + Qh*Tl + Ql*Th), qs / ts
//           per-row powers of two.  Per 64-wide K chunk TMA lands four 16 KB boxes; nothing else touches smem.
//   TF32    raw fp32 tiles, one tf32 product (experiments).
//   TF32X3  raw fp32 tiles, splitter warps derive lo = rn_tf32(x - trunc_tf32(x)) in smem: Q*T + Ql*T + Q*Tl (tf32).
//   MIXED   raw fp32 tiles, splitter warps derive bf16 hi / lo tiles: Q*T [tf32] + Ql16*Th16 + Qh16*Tl16 [bf16].
// The reference is a true fp32 GEMM; single-pass TF32 misses the 1e-4 bar, the three split forms meet it.
//
// CTA = 3 (4 with splitters) warpgroups, one CTA per SM, persistent over a contiguous range of the flattened work
// items (query tile, entity tile[, K segment]): every CTA runs floor or ceil of items / SMs, so a range may straddle
// query tiles.
//   warpgroup 0   warp 0 lane 0: TMA producer (the warpgroup hands its registers to the consumers)
//   warpgroups 1-2 consumers, wgmma m64n128 with the fp32 accumulator in registers; the epilogue runs on the
//                 accumulator fragment itself (no shared-memory staging).
//                 F16X3 / TF32, "ping-pong": warpgroup g owns whole 128x128 tiles (two accumulators), the CTA's tiles
//                 g, g+2, g+4, ... of its range, so one warpgroup's epilogue runs under the other's wgmmas.
//                 TF32X3 / MIXED (four warpgroups, 128 registers per thread): warpgroup g owns query rows [64g, +64)
//                 of every tile.
//   warpgroup 3   (TF32X3 / MIXED) splitters
// Ring of NSTAGE stages of 64 KB; a stage is one K chunk of both operands in every plane the mode uses.  Chunks are
// consumed in ring order, which is also what hands the tensor cores from one ping-pong warpgroup to the other.
//   full[s]    TMA bytes landed                              -> splitters, consumers
//   split[s]   splitter warps wrote + fenced derived tiles    -> consumers
//   empty[s]   every consuming warp's wgmmas on s retired     -> producer
// Loss rows: the per-row state is flushed once per (query tile, CTA) into slot 2j + h of the row: j = the CTA's place
// among the CTAs covering the query tile, h = the consumer warpgroup (ping-pong) or the half of the lane quad (row
// split).  The CTA that ends a query tile writes neutral states into the slots no CTA reached, so the finaliser sums
// the same slots in the same order whatever the schedule.
#include "tc_common.cuh"

namespace b200kge {

namespace {

enum Mode : int { MODE_F16X3 = 0, MODE_TF32 = 1, MODE_TF32X3 = 2, MODE_MIXED = 3 };

constexpr int TM = 128;             // queries per tile
constexpr int TN = 128;             // entities per tile (wgmma N)
constexpr int NSTAGE = 3;
constexpr int STAGE_BYTES = 64 * 1024;
constexpr int BOX_BYTES = 16 * 1024;        // one 128-row box of 128-byte rows
// per-row loss / rank state of the consumers between tiles: 256 consumer threads x 4 rows x the largest RowState
constexpr int STATE_BYTES = 256 * 4 * (int)sizeof(RowState<EPI_KL>);
static_assert(sizeof(RowState<EPI_RANK_EVAL>) <= sizeof(RowState<EPI_KL>), "row state slots are sized for KL");
constexpr int SMEM_BYTES = 1024 /*align slack*/ + NSTAGE * STAGE_BYTES + 256 /*barriers*/ + STATE_BYTES;
static_assert(SMEM_BYTES <= 227 * 1024, "exceeds the H100's 227 KB of shared memory per block");

template <int MODE> struct ModeCfg {
  static constexpr bool SPLIT = MODE == MODE_TF32X3 || MODE == MODE_MIXED;
  static constexpr bool PP = !SPLIT;                                              // ping-pong consumers
  static constexpr int MH = PP ? 2 : 1;                                           // m64 accumulators per consumer
  static constexpr int NTHREADS = (SPLIT ? 4 : 3) * 128;
  static constexpr int TK = MODE == MODE_F16X3 ? 64 : 32;                        // K elements per chunk
  static constexpr uint32_t TX = MODE == MODE_F16X3 ? 4 * BOX_BYTES : 2 * BOX_BYTES;   // TMA bytes per stage
  static constexpr uint32_t STAGE_CONSUMERS = PP ? 4 : 8;                        // warps releasing each stage
};

struct TcParams {
  int64_t nq, m;
  int nk;           // K chunks
  int q_tiles, e_tiles;
  int ksplit;       // > 1: split-K GEMM mode (EPI_STORE only): the reduction is cut into `ksplit` segments of `kseg`
  int kseg;         //      K chunks; every (tile, segment) is its own work item and ADDS into the zeroed output
  int64_t items;    // q_tiles * e_tiles * ksplit; CTA b runs items [b * items / grid, (b + 1) * items / grid)
  int grid;
  int nsl;          // slot pairs per row (EpiParams::nchunks = 2 * nsl)
  const float* q_scale;   // F16X3: [nq]
  const float* t_scale;   // F16X3: [m + 32], zero beyond m
  EpiParams epi;
};

struct Item { int qt, et, k0, k1; };
__device__ __forceinline__ Item item_at(const TcParams& p, int64_t i) {
  Item it;
  int ks = 0;
  if (p.ksplit > 1) { ks = (int)(i % p.ksplit); i /= p.ksplit; }
  it.qt = (int)(i / p.e_tiles);
  it.et = (int)(i - (int64_t)it.qt * p.e_tiles);
  it.k0 = ks * p.kseg;
  it.k1 = it.k0 + p.kseg < p.nk ? it.k0 + p.kseg : p.nk;
  return it;
}

// Stage layout (byte offsets).  F16X3: Qh | Th | Ql | Tl.  Raw modes: Q | T | derived tiles:
//   TF32X3: Ql (16 KB) | Tl (16 KB)      MIXED: Qh16 | Ql16 | Th16 | Tl16 (8 KB each, 64-byte rows)
// h: which 64 query rows of the stage's 128
template <int MODE>
__device__ __forceinline__ void mma_chunk(float (&d)[64], uint32_t st, int h) {
  const uint32_t a = st + (uint32_t)h * (BOX_BYTES / 2), b = st + BOX_BYTES;
  if constexpr (MODE == MODE_F16X3) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t o = k * 32;
      ptx::wgmma_f16(d, ptx::wg_desc_sw128(a + o), ptx::wg_desc_sw128(b + o));
      ptx::wgmma_f16(d, ptx::wg_desc_sw128(a + o), ptx::wg_desc_sw128(b + 2 * BOX_BYTES + o));
      ptx::wgmma_f16(d, ptx::wg_desc_sw128(a + 2 * BOX_BYTES + o), ptx::wg_desc_sw128(b + o));
    }
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k)
      ptx::wgmma_tf32(d, ptx::wg_desc_sw128(a + k * 32), ptx::wg_desc_sw128(b + k * 32));
    if constexpr (MODE == MODE_TF32X3) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        ptx::wgmma_tf32(d, ptx::wg_desc_sw128(a + 2 * BOX_BYTES + k * 32), ptx::wg_desc_sw128(b + k * 32));
        ptx::wgmma_tf32(d, ptx::wg_desc_sw128(a + k * 32), ptx::wg_desc_sw128(b + 2 * BOX_BYTES + k * 32));
      }
    } else if constexpr (MODE == MODE_MIXED) {
      const uint32_t hq = st + 2 * BOX_BYTES + (uint32_t)h * (BOX_BYTES / 4);   // Qh16 rows of these 64 queries
      const uint32_t lq = hq + BOX_BYTES / 2;                                    // Ql16
      const uint32_t th = st + 3 * BOX_BYTES, tl = th + BOX_BYTES / 2;           // Th16, Tl16
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        ptx::wgmma_bf16(d, ptx::wg_desc_sw64(lq + k * 32), ptx::wg_desc_sw64(th + k * 32));
        ptx::wgmma_bf16(d, ptx::wg_desc_sw64(hq + k * 32), ptx::wg_desc_sw64(tl + k * 32));
      }
    }
  }
}

template <int EPI, int MODE>
__global__ void __launch_bounds__(ModeCfg<MODE>::NTHREADS, 1)
pairwise_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmT,
                   const __grid_constant__ CUtensorMap tmQl, const __grid_constant__ CUtensorMap tmTl,
                   const TcParams prm) {
  using C = ModeCfg<MODE>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + NSTAGE * STAGE_BYTES);
  uint64_t* full = bars;                  // [NSTAGE]
  uint64_t* split = bars + NSTAGE;        // [NSTAGE]
  uint64_t* empty = bars + 2 * NSTAGE;    // [NSTAGE]
  uint64_t* turn = bars + 3 * NSTAGE;     // [2] ping-pong: warpgroup g may start waiting on its next tile's chunks

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t i0 = (int64_t)blockIdx.x * prm.items / prm.grid, i1 = (int64_t)(blockIdx.x + 1) * prm.items / prm.grid;

  if (threadIdx.x == 0) {
    ptx::prefetch_tensormap(&tmQ);
    ptx::prefetch_tensormap(&tmT);
    if constexpr (MODE == MODE_F16X3) {
      ptx::prefetch_tensormap(&tmQl);
      ptx::prefetch_tensormap(&tmTl);
    }
    for (int s = 0; s < NSTAGE; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&split[s], 4);
      ptx::mbar_init(&empty[s], C::STAGE_CONSUMERS);
    }
    ptx::mbar_init(&turn[0], 1);
    ptx::mbar_init(&turn[1], 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ================================ TMA producer =========================================
    if constexpr (C::PP) ptx::setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      uint32_t c = 0;
      for (int64_t i = i0; i < i1; ++i) {
        const Item it = item_at(prm, i);
        for (int kc = it.k0; kc < it.k1; ++kc, ++c) {
          const int s = (int)(c % NSTAGE);
          ptx::mbar_wait_bounded(&empty[s], ((c / NSTAGE) & 1) ^ 1);
          uint8_t* sp = smem + s * STAGE_BYTES;
          ptx::mbar_arrive_expect_tx(&full[s], C::TX);
          ptx::tma_load_2d(sp, &tmQ, &full[s], kc * C::TK, it.qt * TM);
          ptx::tma_load_2d(sp + BOX_BYTES, &tmT, &full[s], kc * C::TK, it.et * TN);
          if constexpr (MODE == MODE_F16X3) {
            ptx::tma_load_2d(sp + 2 * BOX_BYTES, &tmQl, &full[s], kc * C::TK, it.qt * TM);
            ptx::tma_load_2d(sp + 3 * BOX_BYTES, &tmTl, &full[s], kc * C::TK, it.et * TN);
          }
        }
      }
    }
  } else if (warp >= 12) {
    // ================================ splitters (TF32X3 / MIXED) ============================
    if constexpr (C::SPLIT) {
      const int t = threadIdx.x - 12 * 32;
      uint32_t c = 0;
      for (int64_t i = i0; i < i1; ++i) {
        const Item it = item_at(prm, i);
        for (int kc = it.k0; kc < it.k1; ++kc, ++c) {
          const int s = (int)(c % NSTAGE);
          ptx::mbar_wait_bounded(&full[s], (c / NSTAGE) & 1);
          const uint32_t sp = ptx::smem_u32(smem + s * STAGE_BYTES);
          if constexpr (MODE == MODE_TF32X3) {
            tc::split_tile<BOX_BYTES, 128>(sp, sp + 2 * BOX_BYTES, t);
            tc::split_tile<BOX_BYTES, 128>(sp + BOX_BYTES, sp + 3 * BOX_BYTES, t);
          } else {
            tc::split_tile_bf16<TM, 128>(sp, sp + 2 * BOX_BYTES, sp + 2 * BOX_BYTES + BOX_BYTES / 2, t);
            tc::split_tile_bf16<TN, 128>(sp + BOX_BYTES, sp + 3 * BOX_BYTES, sp + 3 * BOX_BYTES + BOX_BYTES / 2, t);
          }
          ptx::fence_proxy_async_smem();
          __syncwarp();
          if (lane == 0) ptx::mbar_arrive(&split[s]);
        }
      }
    }
  } else {
    // ================================ consumers: wgmma + epilogue ===========================
    if constexpr (C::PP) ptx::setmaxnreg_inc<232>();
    const int g = (warp - 4) >> 2;            // consumer warpgroup
    const int tg = threadIdx.x & 127, q = tg & 3;
    // tile row of this thread's accumulator row rr: accumulator rr / 2, +8 for odd rr (fragment layout in ptx.cuh)
    const int row_in_tile = (C::PP ? 0 : 64 * g) + 16 * (tg >> 5) + ((tg & 31) >> 2);
    const EpiParams& P = prm.epi;
    // Row state lives in shared memory between tiles (thread-private slots, stride 256 states), so it does not hold
    // registers next to the accumulators during the main loop.
    RowState<EPI>* st = reinterpret_cast<RowState<EPI>*>(smem + NSTAGE * STAGE_BYTES + 256) + (threadIdx.x - 128);
#pragma unroll
    for (int rr = 0; rr < 2 * C::MH; ++rr) st[256 * rr].init();
    uint32_t c = 0;
    for (int64_t i = i0; i < i1; ++i) {
      const Item it = item_at(prm, i);
      const int nkc = it.k1 - it.k0;
      if (!C::PP || (int)((i - i0) & 1) == g) {
        // Ping-pong: the k-th tile of warpgroup g waits until the other warpgroup has waited on every chunk of the
        // tile before it.  Without this a warpgroup would wait on a full[] phase two ring passes ahead, and the
        // parity wait would return on an earlier chunk.
        const uint32_t k = (uint32_t)((i - i0) >> 1);
        if (C::PP && (g == 1 || k > 0)) ptx::mbar_wait_bounded(&turn[g], (g == 1 ? k : k - 1) & 1);
        float d[C::MH][64];
#pragma unroll
        for (int h = 0; h < C::MH; ++h)
#pragma unroll
          for (int e = 0; e < 64; ++e) d[h][e] = 0.f;
        for (int kk = 0; kk < nkc; ++kk) {
          const uint32_t cc = c + kk;
          const int s = (int)(cc % NSTAGE);
          ptx::mbar_wait_bounded(&full[s], (cc / NSTAGE) & 1);
          if constexpr (C::SPLIT) ptx::mbar_wait_bounded(&split[s], (cc / NSTAGE) & 1);
          // Hand the ring to the other warpgroup as soon as this tile's last chunk has landed, before its wgmmas are
          // issued, so the other warpgroup's first chunk queues behind this one's last.  Safe: this thread has waited
          // on every chunk of the tile in order, and before the tile (through turn[g]) the other warpgroup's thread 0
          // had waited on every earlier chunk, so every full[] phase up to this one has completed.  The other
          // warpgroup's next waits are on phases at most one ring pass ahead; the stages it waits on cannot be
          // refilled beyond that before every warp of this warpgroup releases them through empty[].
          if (C::PP && kk == nkc - 1 && tg == 0) ptx::mbar_arrive(&turn[g ^ 1]);
          ptx::wg_fence();
#pragma unroll
          for (int h = 0; h < C::MH; ++h) mma_chunk<MODE>(d[h], ptx::smem_u32(smem + s * STAGE_BYTES), C::PP ? h : g);
          ptx::wg_commit();
          if (kk > 0) {
            ptx::wg_wait<1>();                 // the previous chunk's wgmmas retired: release its stage
            __syncwarp();
            if (lane == 0) ptx::mbar_arrive(&empty[(cc - 1) % NSTAGE]);
          }
        }
        // The epilogue's operands do not depend on the accumulators: load them before the wait, so their latency runs
        // under this tile's last wgmmas instead of after them.
        const int64_t e0 = (int64_t)it.et * TN;
        float qs[2 * C::MH];      // F16X3 row factors
        float2 ts[16];            // F16X3 column factors of columns e0 + 2q + 8j (+1)
        int64_t lab[2 * C::MH];   // BCE / KL with label_idx: the row's label
#pragma unroll
        for (int rr = 0; rr < 2 * C::MH; ++rr) {
          const int64_t row = (int64_t)it.qt * TM + row_in_tile + 64 * (rr >> 1) + 8 * (rr & 1);
          if constexpr (MODE == MODE_F16X3) qs[rr] = row < prm.nq ? __ldg(prm.q_scale + row) : 0.f;
          lab[rr] = -1;
          if constexpr (EPI == EPI_BCE || EPI == EPI_KL)
            if (P.label_idx && row < prm.nq) lab[rr] = P.label_idx[row];
        }
        if constexpr (MODE == MODE_F16X3) {
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int64_t col = e0 + 2 * q + 8 * j;
            ts[j] = col < prm.m ? __ldg(reinterpret_cast<const float2*>(prm.t_scale + col)) : make_float2(0.f, 0.f);
          }
        }
        ptx::wg_wait<0>();
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty[(c + nkc - 1) % NSTAGE]);

        if constexpr (MODE == MODE_F16X3) {
          // score = acc * (row factor * column factor), both exact powers of two
#pragma unroll
          for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int rr = 0; rr < 2 * C::MH; ++rr) {
              float* a = &d[rr >> 1][4 * j + 2 * (rr & 1)];
              a[0] = a[0] * (qs[rr] * ts[j].x);
              a[1] = a[1] * (qs[rr] * ts[j].y);
            }
          }
        }
#pragma unroll
        for (int rr = 0; rr < 2 * C::MH; ++rr) {
          const int64_t row = (int64_t)it.qt * TM + row_in_tile + 64 * (rr >> 1) + 8 * (rr & 1);
          if (row < prm.nq) {
            float v[32];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              v[2 * j] = d[rr >> 1][4 * j + 2 * (rr & 1)];
              v[2 * j + 1] = d[rr >> 1][4 * j + 2 * (rr & 1) + 1];
            }
            RowState<EPI> rs = st[256 * rr];
            tc::epi_row<EPI>(P, rs, v, row, e0, prm.m, q, lab[rr]);
            st[256 * rr] = rs;
          }
        }
      }
      c += nkc;
      if constexpr (EPI != EPI_STORE) {
        // losses and ranks never split K: item i is tile (i / e_tiles, i % e_tiles)
        const bool ends_qt = (i + 1) % prm.e_tiles == 0;
        if (ends_qt || i + 1 == i1) {
          const int qt = (int)(i / prm.e_tiles);
          const int64_t first = (((int64_t)qt * prm.e_tiles + 1) * prm.grid - 1) / prm.items;   // CTA of its 1st item
          const int j = (int)(blockIdx.x - first);
          const int h = C::PP ? g : (q >> 1);
          const bool writer = C::PP ? q == 0 : (q & 1) == 0;
#pragma unroll
          for (int rr = 0; rr < 2 * C::MH; ++rr) {
            RowState<EPI> rs = st[256 * rr];
            epi_lane_reduce<EPI>(rs, C::PP ? 4 : 2);
            const int64_t row = (int64_t)qt * TM + row_in_tile + 64 * (rr >> 1) + 8 * (rr & 1);
            if (writer && row < prm.nq) {
              epi_flush<EPI>(P, rs, row, 2 * j + h);
              if constexpr (EPI != EPI_RANK && EPI != EPI_RANK_EVAL) {
                if (ends_qt) {
                  RowState<EPI> z;
                  z.init();
                  for (int jj = j + 1; jj < prm.nsl; ++jj) epi_flush<EPI>(P, z, row, 2 * jj + h);
                }
              }
            }
            st[256 * rr].init();
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
using tc::num_sms;

// Flattened work items split into contiguous ranges over min(#SMs, items) CTAs.
void schedule(int64_t nq, int64_t m, int ksplit, TcParams& prm) {
  prm.q_tiles = (int)((nq + TM - 1) / TM);
  if (prm.q_tiles < 1) prm.q_tiles = 1;
  prm.e_tiles = (int)((m + TN - 1) / TN);
  prm.ksplit = ksplit;
  prm.items = (int64_t)prm.q_tiles * prm.e_tiles * ksplit;
  prm.grid = prm.items < num_sms() ? (int)prm.items : num_sms();
  // every range holds >= per items, so a query tile's e_tiles items meet at most ceil(e_tiles / per) + 1 ranges, and
  // never more than there are CTAs: nsl <= #SMs keeps the partials within 2 * #SMs slots per row (the workspace size)
  const int64_t per = prm.items / prm.grid;
  const int64_t nsl = (prm.e_tiles + per - 1) / per + 1;
  prm.nsl = nsl < prm.grid ? (int)nsl : prm.grid;
}

template <int EPI, int MODE>
int launch_k(const CUtensorMap (&maps)[4], const TcParams& prm, cudaStream_t st) {
  auto kern = pairwise_tc_kernel<EPI, MODE>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute(pairwise_tc_kernel)");
  profile_begin(st);
  kern<<<prm.grid, ModeCfg<MODE>::NTHREADS, SMEM_BYTES, st>>>(maps[0], maps[1], maps[2], maps[3], prm);
  profile_end(st);
  B2K_LAUNCH_CHECK("pairwise_tc_kernel");
  return 0;
}

template <int MODE>
int launch_mode(int epi_kind, const CUtensorMap (&maps)[4], const TcParams& prm, cudaStream_t st) {
  switch (epi_kind) {
    case EPI_STORE: return launch_k<EPI_STORE, MODE>(maps, prm, st);
    case EPI_BCE:   return launch_k<EPI_BCE, MODE>(maps, prm, st);
    case EPI_KL:    return launch_k<EPI_KL, MODE>(maps, prm, st);
    case EPI_RANK:  return launch_k<EPI_RANK, MODE>(maps, prm, st);
    case EPI_RANK_EVAL:   // pre-split planes only; run_block refuses the in-kernel split modes before any launch
      if constexpr (MODE == MODE_F16X3) return launch_k<EPI_RANK_EVAL, MODE>(maps, prm, st);
      break;
  }
  set_error("bad epilogue kind %d", epi_kind);
  return B200KGE_ERR_INVALID;
}

}  // namespace

bool tc_supported(int pair_op, int K, const Rows& cand, int col_off) {
  if (pair_op != PAIR_DOT) return false;
  if (K < 32) return false;
  if (cand.ld % 4 != 0 || col_off % 4 != 0) return false;
  if ((reinterpret_cast<uintptr_t>(cand.base) & 15) != 0) return false;
  if (cand.rows >= (1ll << 31)) return false;
  return true;
}

int tc_nchunks(int64_t nq, int64_t m) {
  TcParams prm;
  schedule(nq, m, 1, prm);
  return 2 * prm.nsl;
}

// in-kernel split of raw fp32 operands: passes 1 = TF32, 2 = MIXED, 3 = TF32X3
int launch_pairwise_tc(int epi_kind, int passes, const float* Q, int64_t ldq,
                       int64_t nq, const float* T, int64_t ldt, int64_t m, int K,
                       const EpiParams& P, cudaStream_t st) {
  if (nq == 0 || m == 0) return 0;
  CUtensorMap maps[4];
  int rc;
  if ((rc = tc::make_map(&maps[0], Q, nq, K, ldq, 32, TM))) return rc;
  if ((rc = tc::make_map(&maps[1], T, m, K, ldt, 32, TN))) return rc;
  maps[2] = maps[0]; maps[3] = maps[1];
  TcParams prm;
  prm.nq = nq; prm.m = m; prm.nk = (K + 31) / 32;
  schedule(nq, m, 1, prm);
  prm.kseg = prm.nk;
  prm.q_scale = nullptr; prm.t_scale = nullptr;
  prm.epi = P;
  prm.epi.nchunks = 2 * prm.nsl;
  if (passes == 3) return launch_mode<MODE_TF32X3>(epi_kind, maps, prm, st);
  if (passes == 2) return launch_mode<MODE_MIXED>(epi_kind, maps, prm, st);
  return launch_mode<MODE_TF32>(epi_kind, maps, prm, st);
}

// pre-split fp16 planes (F16X3)
int launch_pairwise_tc3(int epi_kind, const SplitSet& Q, const SplitSet& T, const EpiParams& P, cudaStream_t st) {
  const int64_t nq = Q.rows, m = T.rows;
  if (nq == 0 || m == 0) return 0;
  if (Q.Kp != T.Kp || Q.Kp % 64 != 0) { set_error("operand planes disagree on the padded reduction length"); return B200KGE_ERR_INVALID; }
  TcParams prm;
  prm.nq = nq; prm.m = m; prm.nk = Q.Kp / 64;
  prm.kseg = prm.nk;
  if (P.accumulate_out) {
    // split-K GEMM: segments of 8 chunks (512 reduction elements) bound the tensor core's accumulator error, which
    // grows with the reduction length; segment results are added in fp32 by the epilogue (red.global.add).
    if (epi_kind != EPI_STORE) { set_error("split-K accumulation is a GEMM (store) mode"); return B200KGE_ERR_INVALID; }
    prm.kseg = 8;
  }
  schedule(nq, m, (prm.nk + prm.kseg - 1) / prm.kseg, prm);
  prm.q_scale = Q.inv_scale; prm.t_scale = T.inv_scale;
  CUtensorMap maps[4];
  int rc;
  if ((rc = tc::make_map_f16(&maps[0], Q.hi, nq, Q.Kp, Q.Kp, TM))) return rc;
  if ((rc = tc::make_map_f16(&maps[1], T.hi, m, T.Kp, T.Kp, TN))) return rc;
  if ((rc = tc::make_map_f16(&maps[2], Q.lo, nq, Q.Kp, Q.Kp, TM))) return rc;
  if ((rc = tc::make_map_f16(&maps[3], T.lo, m, T.Kp, T.Kp, TN))) return rc;
  prm.epi = P;
  prm.epi.nchunks = 2 * prm.nsl;
  return launch_mode<MODE_F16X3>(epi_kind, maps, prm, st);
}

}  // namespace b200kge
