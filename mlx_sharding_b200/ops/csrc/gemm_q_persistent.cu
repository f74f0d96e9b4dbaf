// Persistent quantised-weight GEMM (MLX affine int4 / int8, in-kernel dequant) — the production path for 4-bit /
// 8-bit checkpoints (BASELINE config 2).  Structure = gemm_persistent.cu (static round-robin tile list, the TMA ring
// keeps streaming the next tile during the epilogue) plus a *decoupled* dequant stage:
//
//   TMA ring (deep, cheap stages)     : packed codes [128 x 32|64 B] + scales/biases rows + bf16 token tile
//   dequant warps (4, one per row)    : ring stage -> bf16 A tile in a small 128B-swizzled ring (DQ buffers)
//   MMA warpgroup                     : A tile ring + token tile of the ring stage -> register accumulator, then the
//                                       epilogue: registers -> shared -> global (shared epilogue semantics)
//
// HBM sees 4.5 / 8.5 bits per weight; the deep ring hides HBM latency with ~13-17 KB stages while the expensive
// 16 KB bf16 tiles only exist DQ (2-3) at a time.
#include <type_traits>

#include "gemm_q_common.cuh"
#include "launch.h"

namespace b200 {

using namespace gemm;

namespace {

constexpr int kQPThreads = kNumThreads + 128;  // warps 0..3 MMA + epilogue, 4 TMA, 5..8 dequant

__host__ __device__ constexpr int qp_packed_bytes(int bits) { return kTileM * (kBlockK * bits / 8); }
__host__ __device__ constexpr int qp_stage_bytes(int BN, bool dual, int bits) {
  const int d = dual ? 2 : 1;
  return (BN * kBlockK * 2 + (qp_packed_bytes(bits) + 512) * d + 1023) / 1024 * 1024;
}
__host__ __device__ constexpr int qp_dq(int BN, bool dual) { return BN <= 64 && !dual ? 3 : 2; }  // bf16 A-tile buffers
__host__ __device__ constexpr int qp_staging_bytes(int BN, int out_bytes) { return staging_bytes(BN, kTileM, out_bytes); }
__host__ __device__ constexpr int qp_num_stages(int BN, bool dual, int bits, int out_bytes) {
  const int fixed = qp_dq(BN, dual) * kATileBytes * (dual ? 2 : 1) + acc_bytes(BN, dual) + qp_staging_bytes(BN, out_bytes) + 1024;
  int s = (225 * 1024 - fixed) / qp_stage_bytes(BN, dual, bits);
  return s > 10 ? 10 : s;
}

}  // namespace

// Kernel body; LORA adds the adapter term (LoraParams) in the epilogue.
template <int BN, bool DUAL, typename OutT, int BITS, bool LORA>
__device__ __forceinline__ void q_persistent_body(const CUtensorMap& tmap_wq, const CUtensorMap& tmap_wq2, const CUtensorMap& tmap_s,
                                                  const CUtensorMap& tmap_b, const CUtensorMap& tmap_s2, const CUtensorMap& tmap_b2,
                                                  const CUtensorMap& tmap_x, const GemmParams& p, const int group_kblocks,
                                                  const int tiles_n, const int tiles_m, const int num_tiles, const LoraParams* lora) {
  constexpr int D = DUAL ? 2 : 1;
  constexpr int STAGES = qp_num_stages(BN, DUAL, BITS, sizeof(OutT));
  constexpr int STAGE_BYTES = qp_stage_bytes(BN, DUAL, BITS);
  constexpr int PACKED_BYTES = qp_packed_bytes(BITS);
  constexpr int OFF_PACKED = BN * kBlockK * 2;             // stage layout: [B tile | packed x D | (scales, biases) x D]
  constexpr int OFF_SCALE = OFF_PACKED + PACKED_BYTES * D;
  constexpr uint32_t TX_BYTES = BN * kBlockK * 2 + (PACKED_BYTES + 512) * D;
  constexpr int DQ = qp_dq(BN, DUAL);
  static_assert(STAGES >= 2, "ring too small");

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024 B alignment by *pointer arithmetic* on the __shared__ array: an integer round-trip loses the address space and
  // turns every LDS/STS below into a generic LD.E/ST.E (checked with cuobjdump -sass)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* a_ring = smem;                                        // [DQ][D][16 KB]   (1024-aligned)
  uint8_t* ring = a_ring + DQ * D * kATileBytes;                 // [STAGES][STAGE_BYTES]
  float* acc_smem = reinterpret_cast<float*>(ring + STAGES * STAGE_BYTES);   // [BN * D][128] fp32
  OutT* stg = reinterpret_cast<OutT*>(ring + STAGES * STAGE_BYTES + acc_bytes(BN, DUAL));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(stg) + qp_staging_bytes(BN, sizeof(OutT)));
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* dq_full = empty_bar + STAGES;    // [DQ]
  uint64_t* dq_empty = dq_full + DQ;         // [DQ]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const bool pdl_early = p.expert_offsets != nullptr;
  if (pdl_early) pdl_wait();

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&tmap_wq);
    tma_prefetch_desc(&tmap_s);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_x);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);  // one arrival per MMA warp
    }
    for (int j = 0; j < DQ; ++j) {
      mbar_init(&dq_full[j], 4);   // one arrival per dequant warp
      mbar_init(&dq_empty[j], 4);  // one arrival per MMA warp
    }
    mbar_fence_init();
  }
  __syncthreads();
  if (!pdl_early) pdl_wait();
  pdl_launch_dependents();

  const int kb_total = p.k / kBlockK;

  if (warp == kProducerWarp) {
    // ============================================================== TMA producer
    if (elect_one()) {  // one elected lane: uniform-datapath issue, no per-instruction ELECT loop (ptx.cuh)
      uint32_t it = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const TileInfo ti = decode_tile(p, t, tiles_n, tiles_m, BN);
        if (ti.rows_valid <= 0) continue;
        for (int kb = 0; kb < kb_total; ++kb, ++it) {
          const uint32_t s = it % STAGES, ph = (it / STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* st = ring + s * STAGE_BYTES;
          const int gi = kb / group_kblocks;
          mbar_arrive_expect_tx(&full_bar[s], TX_BYTES);
          tma_load_2d(st + OFF_PACKED, &tmap_wq, &full_bar[s], kb * (kBlockK * BITS / 32), ti.w_row, kEvictFirst);
          tma_load_2d(st + OFF_SCALE, &tmap_s, &full_bar[s], ti.w_row, gi, kEvictFirst);
          tma_load_2d(st + OFF_SCALE + 256, &tmap_b, &full_bar[s], ti.w_row, gi, kEvictFirst);
          if (DUAL) {
            tma_load_2d(st + OFF_PACKED + PACKED_BYTES, &tmap_wq2, &full_bar[s], kb * (kBlockK * BITS / 32), ti.w_row, kEvictFirst);
            tma_load_2d(st + OFF_SCALE + 512, &tmap_s2, &full_bar[s], ti.w_row, gi, kEvictFirst);
            tma_load_2d(st + OFF_SCALE + 768, &tmap_b2, &full_bar[s], ti.w_row, gi, kEvictFirst);
          }
          tma_load_2d(st, &tmap_x, &full_bar[s], kb * kBlockK, ti.row_base, kEvictLast);
        }
      }
    }
  } else if (warp < 4) {
    // ============================================================== MMA warpgroup, then epilogue (128 threads)
    const bool leader = lane == 0;
    uint32_t it = 0, tc = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const TileInfo ti = decode_tile(p, t, tiles_n, tiles_m, BN);
      if (ti.rows_valid <= 0) continue;
      float acc[2][BN / 2], acc2[2][BN / 2];
      acc_zero<BN>(acc);
      if (DUAL) acc_zero<BN>(acc2);
      for (int kb = 0; kb < kb_total; ++kb, ++it) {
        const uint32_t s = it % STAGES, ph = (it / STAGES) & 1;
        const uint32_t j = it % DQ, jph = (it / DQ) & 1;
        mbar_wait(&full_bar[s], ph);   // token tile landed
        mbar_wait(&dq_full[j], jph);   // weight tile dequantised + fenced
        const uint32_t a_addr = smem_u32(a_ring + j * D * kATileBytes);
        const uint32_t b_addr = smem_u32(ring + s * STAGE_BYTES);
        wgmma_fence();
        mma_kblock<BN>(acc, a_addr, b_addr);
        if (DUAL) mma_kblock<BN>(acc2, a_addr + kATileBytes, b_addr);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs are done: release its ring stage and A buffer
        if (kb > 0 && leader) {
          mbar_arrive(&empty_bar[(it - 1) % STAGES]);
          mbar_arrive(&dq_empty[(it - 1) % DQ]);
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        wgmma_fence_acc(acc[h]);
        if (DUAL) wgmma_fence_acc(acc2[h]);
      }
      if (kb_total > 0 && leader) {
        mbar_arrive(&empty_bar[(it - 1) % STAGES]);
        mbar_arrive(&dq_empty[(it - 1) % DQ]);
      }
      acc_store_smem<BN>(acc, acc_smem, 0);
      if (DUAL) acc_store_smem<BN>(acc2, acc_smem, BN);
      named_bar_sync(1, kEpiThreads);
      store_acc_tile<BN, DUAL, OutT, LORA>(p, acc_smem, stg, ti, lora);
      ++tc;
    }
    if (p.signal_flag != nullptr) {
      // fused stage boundary: fence once, then report this CTA's tiles
      __threadfence_system();
      named_bar_sync(1, kEpiThreads);
      if (threadIdx.x == 0) publish_tiles_done(p, tc);
    }
  } else {
    // ============================================================== dequant producers (4 warps, one thread per row)
    const int r = threadIdx.x - kNumThreads;
    uint32_t it = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const TileInfo ti = decode_tile(p, t, tiles_n, tiles_m, BN);
      if (ti.rows_valid <= 0) continue;
      for (int kb = 0; kb < kb_total; ++kb, ++it) {
        const uint32_t s = it % STAGES, ph = (it / STAGES) & 1;
        const uint32_t j = it % DQ, jph = (it / DQ) & 1;
        mbar_wait(&full_bar[s], ph);        // packed codes + scales landed
        mbar_wait(&dq_empty[j], jph ^ 1);   // the MMAs that read this A buffer have completed
        const uint8_t* st = ring + s * STAGE_BYTES;
        uint8_t* a_tile = a_ring + j * D * kATileBytes;
#pragma unroll
        for (int d = 0; d < D; ++d) {
          const __nv_bfloat16* sb = reinterpret_cast<const __nv_bfloat16*>(st + OFF_SCALE + d * 512);
          const float sc = __bfloat162float(sb[r]), bi = __bfloat162float(sb[128 + r]);
          for (int half = 0; half < 2; ++half)
            dequant_half_row<BITS>(st + OFF_PACKED + d * PACKED_BYTES + r * (kBlockK * BITS / 8), sc, bi, a_tile + d * kATileBytes, r,
                                   half);
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(&dq_full[j]);
      }
    }
  }
}

template <int BN, bool DUAL, typename OutT, int BITS>
__global__ void __launch_bounds__(kQPThreads, 1)
gemm_q_persistent_kernel(const __grid_constant__ CUtensorMap tmap_wq, const __grid_constant__ CUtensorMap tmap_wq2,
                         const __grid_constant__ CUtensorMap tmap_s, const __grid_constant__ CUtensorMap tmap_b,
                         const __grid_constant__ CUtensorMap tmap_s2, const __grid_constant__ CUtensorMap tmap_b2,
                         const __grid_constant__ CUtensorMap tmap_x, const GemmParams p, const int group_kblocks, const int tiles_n,
                         const int tiles_m, const int num_tiles) {
  q_persistent_body<BN, DUAL, OutT, BITS, false>(tmap_wq, tmap_wq2, tmap_s, tmap_b, tmap_s2, tmap_b2, tmap_x, p, group_kblocks, tiles_n,
                                                 tiles_m, num_tiles, nullptr);
}

// Adapted weights (bf16 output): the same kernel with the LoRA term in the epilogue.
template <int BN, bool DUAL, int BITS>
__global__ void __launch_bounds__(kQPThreads, 1)
gemm_q_persistent_lora_kernel(const __grid_constant__ CUtensorMap tmap_wq, const __grid_constant__ CUtensorMap tmap_wq2,
                              const __grid_constant__ CUtensorMap tmap_s, const __grid_constant__ CUtensorMap tmap_b,
                              const __grid_constant__ CUtensorMap tmap_s2, const __grid_constant__ CUtensorMap tmap_b2,
                              const __grid_constant__ CUtensorMap tmap_x, const GemmParams p, const int group_kblocks, const int tiles_n,
                              const int tiles_m, const int num_tiles, const LoraParams lora) {
  q_persistent_body<BN, DUAL, __nv_bfloat16, BITS, true>(tmap_wq, tmap_wq2, tmap_s, tmap_b, tmap_s2, tmap_b2, tmap_x, p, group_kblocks,
                                                         tiles_n, tiles_m, num_tiles, &lora);
}

// ================================================================================================ host side
namespace {

template <int BN, bool DUAL, typename OutT, int BITS>
cudaError_t qp_launch_one(const QMaps& t, const GemmParams& p, int gk, const GemmPlan& plan, const LoraParams* lora, cudaStream_t stream) {
  constexpr int STAGES = qp_num_stages(BN, DUAL, BITS, sizeof(OutT));
  constexpr int smem = qp_dq(BN, DUAL) * kATileBytes * (DUAL ? 2 : 1) + STAGES * qp_stage_bytes(BN, DUAL, BITS) + acc_bytes(BN, DUAL) +
                       qp_staging_bytes(BN, sizeof(OutT)) + (2 * STAGES + 2 * qp_dq(BN, DUAL)) * 8 + 1024;
  static_assert(smem <= 227 * 1024, "shared memory budget exceeded");
  if (lora != nullptr) {
    if constexpr (std::is_same_v<OutT, __nv_bfloat16>) {
      constexpr auto kern = gemm_q_persistent_lora_kernel<BN, DUAL, BITS>;
      cudaError_t e = set_max_dynamic_smem_once<kern>(smem);
      if (e != cudaSuccess) return e;
      (void)launch_pdl(kern, plan.grid, dim3(kQPThreads), smem, stream, t.wq, t.wq2, t.s, t.b, t.s2, t.b2, t.x, p, gk, plan.tiles_n,
                       plan.tiles_m, plan.num_tiles, *lora);
      return cudaGetLastError();
    } else {
      return cudaErrorInvalidValue;   // adapters run with bf16 output only
    }
  }
  constexpr auto kern = gemm_q_persistent_kernel<BN, DUAL, OutT, BITS>;
  cudaError_t e = set_max_dynamic_smem_once<kern>(smem);
  if (e != cudaSuccess) return e;
  (void)launch_pdl(kern, plan.grid, dim3(kQPThreads), smem, stream, t.wq, t.wq2, t.s, t.b, t.s2, t.b2, t.x, p, gk, plan.tiles_n,
                   plan.tiles_m, plan.num_tiles);
  return cudaGetLastError();
}

}  // namespace

cudaError_t gemm_q_persistent_launch(const GemmArgs& a, const GemmPlan& plan, cudaStream_t stream) {
  const bool dual = a.w2 != nullptr;
  if (a.expert_offsets != nullptr && (a.n % kTileM) != 0) return cudaErrorInvalidValue;
  if ((a.n % 8) != 0 || (a.k % kBlockK) != 0) return cudaErrorInvalidValue;
  if (dual && a.out_fp32) return cudaErrorInvalidValue;

  QMaps t;
  if (!q_maps(a, plan.bn, &t)) return cudaErrorUnknown;
  const GemmParams p = gemm_params(a, plan);
  const LoraParams lora = lora_params(a);
  const int gk = a.q_group / kBlockK;
  auto dispatch = [&](auto bits) {
    return dispatch_tile<kMaxBN, kMaxBNDual>(plan.bn, dual, a.out_fp32, [&](auto c) {
      using C = decltype(c);
      return qp_launch_one<C::BN, C::DUAL, typename C::OutT, decltype(bits)::value>(t, p, gk, plan, a.lora_r > 0 ? &lora : nullptr,
                                                                                    stream);
    });
  };
  if (a.q_bits == 4) return dispatch(std::integral_constant<int, 4>{});
  return dispatch(std::integral_constant<int, 8>{});
}

}  // namespace b200
