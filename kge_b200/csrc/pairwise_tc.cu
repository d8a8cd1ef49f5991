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
// CTA = 3 (4 with splitters) warpgroups, one CTA per SM, persistent over (query tile, range of entity tiles):
//   warpgroup 0   warp 0 lane 0: TMA producer
//   warpgroups 1-2 consumers: warpgroup g owns query rows [64g, 64g+64) of the 128-row tile; wgmma m64n128 with the
//                 fp32 accumulator in registers, then the accumulator goes to a shared-memory tile (one row per
//                 thread) and the same warps run the epilogue: warp w of the group takes rows 32*(w&1) and
//                 columns 64*(w>>1) of the 128-entity tile
//   warpgroup 3   (TF32X3 / MIXED) splitters
// Ring of NSTAGE stages of 64 KB; a stage is one K chunk of both operands in every plane the mode uses.
//   full[s]    TMA bytes landed                              -> splitters, consumers
//   split[s]   splitter warps wrote + fenced derived tiles    -> consumers
//   empty[s]   every consumer warp's wgmmas on s retired      -> producer
// While the consumers run the epilogue of tile i the producer already fills the ring for tile i+1.
#include "tc_common.cuh"

namespace b200kge {

namespace {

enum Mode : int { MODE_F16X3 = 0, MODE_TF32 = 1, MODE_TF32X3 = 2, MODE_MIXED = 3 };

constexpr int TM = 128;             // queries per tile (two consumer warpgroups x 64)
constexpr int TN = 128;             // entities per tile (wgmma N)
constexpr int NSTAGE = 2;
constexpr int STAGE_BYTES = 64 * 1024;
constexpr int BOX_BYTES = 16 * 1024;        // one 128-row box of 128-byte rows
constexpr int ACC_LD = TN + 1;              // padded row of the staged accumulator (conflict-free row-per-thread reads)
constexpr int ACC_BYTES = TM * ACC_LD * 4;
constexpr int EPI_WARPS = 8;
using tc::STG_LD;
constexpr int STG_BYTES = EPI_WARPS * 32 * STG_LD * 4;
constexpr int SMEM_BYTES = 1024 /*align slack*/ + NSTAGE * STAGE_BYTES + ACC_BYTES + STG_BYTES + 256 /*barriers*/;
static_assert(SMEM_BYTES <= 227 * 1024, "exceeds the H100's 227 KB of shared memory per block");

template <int MODE> struct ModeCfg {
  static constexpr bool SPLIT = MODE == MODE_TF32X3 || MODE == MODE_MIXED;
  static constexpr int NTHREADS = (SPLIT ? 4 : 3) * 128;
  static constexpr int TK = MODE == MODE_F16X3 ? 64 : 32;                        // K elements per chunk
  static constexpr uint32_t TX = MODE == MODE_F16X3 ? 4 * BOX_BYTES : 2 * BOX_BYTES;   // TMA bytes per stage
};

struct TcParams {
  int64_t nq, m;
  int nk;           // K chunks
  int q_tiles, e_tiles, echunks;
  int ksplit;       // > 1: split-K GEMM mode (EPI_STORE only): the reduction is cut into `ksplit` segments of `kseg`
  int kseg;         //      K chunks; every (tile, segment) is its own work item and ADDS into the zeroed output
  const float* q_scale;   // F16X3: [nq]
  const float* t_scale;   // F16X3: [m + 32], zero beyond m
  EpiParams epi;
};

// Stage layout (byte offsets).  F16X3: Qh | Th | Ql | Tl.  Raw modes: Q | T | derived tiles:
//   TF32X3: Ql (16 KB) | Tl (16 KB)      MIXED: Qh16 | Ql16 | Th16 | Tl16 (8 KB each, 64-byte rows)
template <int MODE>
__device__ __forceinline__ void mma_chunk(float (&d)[64], uint32_t st, int g) {
  const uint32_t a = st + (uint32_t)g * (BOX_BYTES / 2), b = st + BOX_BYTES;   // this warpgroup's 64 query rows
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
      const uint32_t h = st + 2 * BOX_BYTES + (uint32_t)g * (BOX_BYTES / 4);    // Qh16 rows of this warpgroup
      const uint32_t l = h + BOX_BYTES / 2;                                      // Ql16
      const uint32_t th = st + 3 * BOX_BYTES, tl = th + BOX_BYTES / 2;           // Th16, Tl16
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        ptx::wgmma_bf16(d, ptx::wg_desc_sw64(l + k * 32), ptx::wg_desc_sw64(th + k * 32));
        ptx::wgmma_bf16(d, ptx::wg_desc_sw64(h + k * 32), ptx::wg_desc_sw64(tl + k * 32));
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
  float* accs = reinterpret_cast<float*>(smem + NSTAGE * STAGE_BYTES);
  float* stg = reinterpret_cast<float*>(smem + NSTAGE * STAGE_BYTES + ACC_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + NSTAGE * STAGE_BYTES + ACC_BYTES + STG_BYTES);
  uint64_t* full = bars;                  // [NSTAGE]
  uint64_t* split = bars + NSTAGE;        // [NSTAGE]
  uint64_t* empty = bars + 2 * NSTAGE;    // [NSTAGE]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_work = prm.q_tiles * prm.echunks * prm.ksplit;

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
      ptx::mbar_init(&empty[s], EPI_WARPS);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  int k0 = 0, k1 = prm.nk;      // K-chunk range of the current work item (split-K mode: one segment)
  auto work_range = [&](int w, int& qt, int& et0, int& et1, int& ec) {
    if (prm.ksplit > 1) {
      const int ks = w % prm.ksplit;
      w /= prm.ksplit;
      k0 = ks * prm.kseg;
      k1 = (k0 + prm.kseg < prm.nk) ? k0 + prm.kseg : prm.nk;
    }
    qt = w / prm.echunks;
    ec = w - qt * prm.echunks;
    const int base = prm.e_tiles / prm.echunks, rem = prm.e_tiles % prm.echunks;
    et0 = ec * base + (ec < rem ? ec : rem);
    et1 = et0 + base + (ec < rem ? 1 : 0);
  };

  if (warp == 0) {
    // ================================ TMA producer =========================================
    if (lane == 0) {
      uint32_t c = 0;
      for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
        int qt, et0, et1, ec;
        work_range(w, qt, et0, et1, ec);
        for (int et = et0; et < et1; ++et) {
          for (int kc = k0; kc < k1; ++kc, ++c) {
            const int s = (int)(c % NSTAGE);
            ptx::mbar_wait_bounded(&empty[s], ((c / NSTAGE) & 1) ^ 1);
            uint8_t* sp = smem + s * STAGE_BYTES;
            ptx::mbar_arrive_expect_tx(&full[s], C::TX);
            ptx::tma_load_2d(sp, &tmQ, &full[s], kc * C::TK, qt * TM);
            ptx::tma_load_2d(sp + BOX_BYTES, &tmT, &full[s], kc * C::TK, et * TN);
            if constexpr (MODE == MODE_F16X3) {
              ptx::tma_load_2d(sp + 2 * BOX_BYTES, &tmQl, &full[s], kc * C::TK, qt * TM);
              ptx::tma_load_2d(sp + 3 * BOX_BYTES, &tmTl, &full[s], kc * C::TK, et * TN);
            }
          }
        }
      }
    }
  } else if (warp >= 12) {
    // ================================ splitters (TF32X3 / MIXED) ============================
    if constexpr (C::SPLIT) {
      const int t = threadIdx.x - 12 * 32;
      uint32_t c = 0;
      for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
        int qt, et0, et1, ec;
        work_range(w, qt, et0, et1, ec);
        for (int et = et0; et < et1; ++et) {
          for (int kc = k0; kc < k1; ++kc, ++c) {
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
    }
  } else if (warp >= 4) {
    // ================================ consumers: wgmma + epilogue ===========================
    const int g = (warp - 4) >> 2;            // consumer warpgroup: query rows [64g, +64) of the tile
    const int wl = warp & 3;                  // warp within the group
    const int quad = wl & 1, half = wl >> 1;  // epilogue: rows [32*quad, +32) of the group, columns [64*half, +64)
    const int tg = threadIdx.x & 127;
    float* acc_g = accs + g * 64 * ACC_LD;
    float* my_stg = stg + (warp - 4) * 32 * STG_LD;
    const EpiParams& P = prm.epi;
    uint32_t c = 0;
    for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
      int qt, et0, et1, ec;
      work_range(w, qt, et0, et1, ec);
      const int64_t tile_row0 = (int64_t)qt * TM + g * 64 + quad * 32;
      const int64_t row = tile_row0 + lane;   // this thread's query row in the epilogue
      const bool row_ok = row < prm.nq;
      RowState<EPI> st;
      st.init();
      const float aux = row_ok ? epi_row_aux<EPI>(P, row) : 0.f;
      const float qs = (MODE == MODE_F16X3 && row_ok) ? __ldg(prm.q_scale + row) : 0.f;
      const int64_t csr_end = (P.csr_off && row_ok) ? __ldg(P.csr_off + row + 1) : 0;
      for (int et = et0; et < et1; ++et) {
        float d[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) d[i] = 0.f;
        for (int kc = k0; kc < k1; ++kc, ++c) {
          const int s = (int)(c % NSTAGE);
          ptx::mbar_wait_bounded(&full[s], (c / NSTAGE) & 1);
          if constexpr (C::SPLIT) ptx::mbar_wait_bounded(&split[s], (c / NSTAGE) & 1);
          ptx::wg_fence();
          mma_chunk<MODE>(d, ptx::smem_u32(smem + s * STAGE_BYTES), g);
          ptx::wg_commit();
          if (kc > k0) {
            ptx::wg_wait<1>();                 // the previous chunk's wgmmas retired: release its stage
            __syncwarp();
            if (lane == 0) ptx::mbar_arrive(&empty[(c - 1) % NSTAGE]);
          }
        }
        ptx::wg_wait<0>();
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty[(c - 1) % NSTAGE]);
        // accumulator -> shared tile (one row per thread afterwards)
        ptx::bar_sync(1 + g, 128);             // the previous tile's epilogue is done reading acc_g
        {
          const int r = 16 * (tg >> 5) + ((tg & 31) >> 2), cc = 2 * (tg & 3);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            acc_g[r * ACC_LD + 8 * j + cc] = d[4 * j];
            acc_g[r * ACC_LD + 8 * j + cc + 1] = d[4 * j + 1];
            acc_g[(r + 8) * ACC_LD + 8 * j + cc] = d[4 * j + 2];
            acc_g[(r + 8) * ACC_LD + 8 * j + cc + 1] = d[4 * j + 3];
          }
        }
        ptx::bar_sync(1 + g, 128);
        const int64_t tile_end = (int64_t)(et + 1) * TN;
        tc::epilogue_tile<EPI, 2, MODE == MODE_F16X3>(P, st, aux, acc_g + (quad * 32 + lane) * ACC_LD + half * 64,
                                                      tile_row0, (int64_t)et * TN + half * 64, prm.nq,
                                                      tile_end < prm.m ? tile_end : prm.m, my_stg, lane, qs,
                                                      prm.t_scale, csr_end);
      }
      if constexpr (EPI != EPI_STORE) {
        if (row_ok) epi_flush<EPI>(P, st, row, ec * 2 + half);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
using tc::num_sms;

// entity tiles split into `echunks` ranges so that q_tiles * echunks ~ #SMs
void plan(int64_t nq, int64_t m, int& q_tiles, int& e_tiles, int& echunks) {
  q_tiles = (int)((nq + TM - 1) / TM);
  if (q_tiles < 1) q_tiles = 1;
  e_tiles = (int)((m + TN - 1) / TN);
  int per = num_sms() / q_tiles;
  if (per < 1) per = 1;
  if (per > e_tiles) per = e_tiles;
  echunks = per;
}

template <int EPI, int MODE>
int launch_k(const CUtensorMap (&maps)[4], const TcParams& prm, cudaStream_t st) {
  auto kern = pairwise_tc_kernel<EPI, MODE>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute(pairwise_tc_kernel)");
  const int total = prm.q_tiles * prm.echunks * prm.ksplit;
  const int grid = total < num_sms() ? total : num_sms();
  profile_begin(st);
  kern<<<grid, ModeCfg<MODE>::NTHREADS, SMEM_BYTES, st>>>(maps[0], maps[1], maps[2], maps[3], prm);
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
  int qt, et, ec;
  plan(nq, m, qt, et, ec);
  return 2 * ec;
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
  plan(nq, m, prm.q_tiles, prm.e_tiles, prm.echunks);
  prm.ksplit = 1; prm.kseg = prm.nk;
  prm.q_scale = nullptr; prm.t_scale = nullptr;
  prm.epi = P;
  prm.epi.nchunks = 2 * prm.echunks;   // two epilogue threads (column halves) per row
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
  plan(nq, m, prm.q_tiles, prm.e_tiles, prm.echunks);
  prm.ksplit = 1; prm.kseg = prm.nk;
  if (P.accumulate_out) {
    // split-K GEMM: segments of 8 chunks (512 reduction elements) bound the tensor core's accumulator error, which
    // grows with the reduction length; segment results are added in fp32 by the epilogue (red.global.add).  One
    // entity tile per work item.
    if (epi_kind != EPI_STORE) { set_error("split-K accumulation is a GEMM (store) mode"); return B200KGE_ERR_INVALID; }
    prm.kseg = 8;
    prm.ksplit = (prm.nk + prm.kseg - 1) / prm.kseg;
    prm.echunks = prm.e_tiles;
  }
  prm.q_scale = Q.inv_scale; prm.t_scale = T.inv_scale;
  CUtensorMap maps[4];
  int rc;
  if ((rc = tc::make_map_f16(&maps[0], Q.hi, nq, Q.Kp, Q.Kp, TM))) return rc;
  if ((rc = tc::make_map_f16(&maps[1], T.hi, m, T.Kp, T.Kp, TN))) return rc;
  if ((rc = tc::make_map_f16(&maps[2], Q.lo, nq, Q.Kp, Q.Kp, TM))) return rc;
  if ((rc = tc::make_map_f16(&maps[3], T.lo, m, T.Kp, T.Kp, TN))) return rc;
  prm.epi = P;
  prm.epi.nchunks = 2 * prm.echunks;
  return launch_mode<MODE_F16X3>(epi_kind, maps, prm, st);
}

}  // namespace b200kge
