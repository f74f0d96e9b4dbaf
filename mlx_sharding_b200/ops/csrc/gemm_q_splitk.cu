// Quantised-weight variant of the swap-AB wgmma GEMM: MLX affine int4 / int8 checkpoints are dequantised
// *inside* the kernel (SURVEY §2.6 K17, §7.4-2 "Plan A").  The reference gets this from MLX's
// `quantized_matmul` / `gather_qmm` Metal kernels (enabled by `nn.quantize` at shard/utils.py:54-65).
//
// Data path per 64-wide k-block (== one or half a quantisation group):
//   TMA:      packed codes [128 rows x 32|64 B]  + scales[128] + biases[128] (pre-transposed [K/g, rows] at load)
//             + the bf16 token tile (128B swizzle)                                    -> full barrier
//   4 dequant warps (one thread per weight row): unpack LSB-first nibbles/bytes, w = s*q + b in fp32, round to bf16,
//             store into the 128B-swizzled MMA "A" tile, fence.proxy.async            -> dequant barrier
//   MMA warpgroup: wgmma (fp32 accumulators in registers), wait                        -> empty barrier
// so HBM only ever sees 4.5 (or 8.5) bits per weight; everything downstream (epilogue, DUAL gate/up,
// grouped experts, split-K, fused P2P signal) is shared with the dense kernel (gemm_common.cuh).
#include <type_traits>

#include "gemm_q_common.cuh"
#include "gemm_tmap.h"
#include "launch.h"

namespace b200 {

using namespace gemm;

namespace {

constexpr int kQThreads = kNumThreads + 128;  // + warps 5..8: dequant producers (one thread per weight row)

__host__ __device__ constexpr int q_stage_bytes(int BN, bool dual, int bits) {
  const int d = dual ? 2 : 1;
  const int raw = kATileBytes * d + BN * kBlockK * 2 + kTileM * (kBlockK * bits / 8) * d + 512 * d;
  return (raw + 1023) / 1024 * 1024;
}
__host__ __device__ constexpr int q_num_stages(int BN, bool dual, int bits, int out_bytes) {
  int s = (196 * 1024) / q_stage_bytes(BN, dual, bits);
  s = s > 8 ? 8 : s;
  while (s * q_stage_bytes(BN, dual, bits) < acc_bytes(BN, dual) + BN * kTileM * out_bytes) ++s;
  return s;
}

}  // namespace

template <int BN, bool DUAL, typename OutT, int BITS>
__global__ void __launch_bounds__(kQThreads, 1)
gemm_swapab_q_kernel(const __grid_constant__ CUtensorMap tmap_wq, const __grid_constant__ CUtensorMap tmap_wq2,
                     const __grid_constant__ CUtensorMap tmap_s, const __grid_constant__ CUtensorMap tmap_b,
                     const __grid_constant__ CUtensorMap tmap_s2, const __grid_constant__ CUtensorMap tmap_b2,
                     const __grid_constant__ CUtensorMap tmap_x, const GemmParams p, const int group_kblocks) {
  constexpr int D = DUAL ? 2 : 1;
  constexpr int STAGES = q_num_stages(BN, DUAL, BITS, sizeof(OutT));
  constexpr int STAGE_BYTES = q_stage_bytes(BN, DUAL, BITS);
  constexpr int PACKED_BYTES = kTileM * (kBlockK * BITS / 8);
  constexpr int OFF_B = kATileBytes * D;
  constexpr int OFF_PACKED = OFF_B + BN * kBlockK * 2;
  constexpr int OFF_SCALE = OFF_PACKED + PACKED_BYTES * D;  // per weight: scales[128] bf16 then biases[128] bf16
  constexpr uint32_t TX_BYTES = BN * kBlockK * 2 + (PACKED_BYTES + 512) * D;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024 B alignment by *pointer arithmetic* on the __shared__ array: an integer round-trip loses the address space and
  // turns every LDS/STS below into a generic LD.E/ST.E (checked with cuobjdump -sass)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* deq_bar = full_bar + STAGES;
  uint64_t* empty_bar = deq_bar + STAGES;
  uint32_t* flag_smem = reinterpret_cast<uint32_t*>(empty_bar + STAGES);
  // after the main loop the idle ring holds the fp32 accumulator, then the output staging tile
  float* acc_smem = reinterpret_cast<float*>(smem);
  OutT* stg = reinterpret_cast<OutT*>(smem + acc_bytes(BN, DUAL));

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // PDL: grouped launches read expert_offsets (written by the permutation kernel) right away, so they wait first;
  // plain launches overlap their whole prologue (barrier init) with the predecessor's tail.
  const bool pdl_early = p.expert_offsets != nullptr;
  if (pdl_early) pdl_wait();
  const SplitTile sk = splitk_tile(p, BN);
  const TileInfo& ti = sk.ti;
  if (ti.rows_valid <= 0) return;
  const int kb_begin = sk.kb_begin, num_kb = sk.num_kb;

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&tmap_wq);
    tma_prefetch_desc(&tmap_s);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_x);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&deq_bar[s], 4);
      mbar_init(&empty_bar[s], 4);
    }
    mbar_fence_init();
  }
  __syncthreads();
  if (!pdl_early) pdl_wait();
  pdl_launch_dependents();

  if (warp == kProducerWarp) {
    // ============================================================== TMA producer
    if (elect_one()) {  // one elected lane: uniform-datapath issue, no per-instruction ELECT loop (ptx.cuh)
      for (int i = 0; i < num_kb; ++i) {
        const int s = i % STAGES;
        const uint32_t ph = (i / STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* st = smem + s * STAGE_BYTES;
        const int kb = kb_begin + i;
        const int gi = kb / group_kblocks;  // quantisation group row of this k-block
        mbar_arrive_expect_tx(&full_bar[s], TX_BYTES);
        tma_load_2d(st + OFF_PACKED, &tmap_wq, &full_bar[s], kb * (kBlockK * BITS / 32), ti.w_row, kEvictFirst);
        tma_load_2d(st + OFF_SCALE, &tmap_s, &full_bar[s], ti.w_row, gi, kEvictFirst);
        tma_load_2d(st + OFF_SCALE + 256, &tmap_b, &full_bar[s], ti.w_row, gi, kEvictFirst);
        if (DUAL) {
          tma_load_2d(st + OFF_PACKED + PACKED_BYTES, &tmap_wq2, &full_bar[s], kb * (kBlockK * BITS / 32), ti.w_row, kEvictFirst);
          tma_load_2d(st + OFF_SCALE + 512, &tmap_s2, &full_bar[s], ti.w_row, gi, kEvictFirst);
          tma_load_2d(st + OFF_SCALE + 768, &tmap_b2, &full_bar[s], ti.w_row, gi, kEvictFirst);
        }
        tma_load_2d(st + OFF_B, &tmap_x, &full_bar[s], kb * kBlockK, ti.row_base, kEvictLast);
      }
    }
  } else if (warp < 4) {
    // ============================================================== MMA warpgroup, then epilogue (128 threads)
    float acc[2][BN / 2], acc2[2][BN / 2];
    acc_zero<BN>(acc);
    if (DUAL) acc_zero<BN>(acc2);
    mma_mainloop<BN, DUAL, STAGES, STAGE_BYTES, OFF_B>(acc, acc2, smem, empty_bar, 0u, num_kb, [&](uint32_t s, uint32_t ph) {
      mbar_wait(&full_bar[s], ph);  // token tile landed (async proxy)
      mbar_wait(&deq_bar[s], ph);   // weight tile dequantised + fenced by the producer warps
    });
    named_bar_sync(1, kEpiThreads);  // every warp's MMAs are done: the ring is idle
    acc_store_smem<BN>(acc, acc_smem, 0);
    if (DUAL) acc_store_smem<BN>(acc2, acc_smem, BN);
    named_bar_sync(1, kEpiThreads);
    run_epilogue<BN, DUAL, OutT>(p, acc_smem, stg, flag_smem, ti, sk.split);
  } else {
    // ============================================================== dequant producers: one weight row per thread
    const int r = threadIdx.x - kNumThreads;   // weight row of the tile
    for (int i = 0; i < num_kb; ++i) {
      const int s = i % STAGES;
      const uint32_t ph = (i / STAGES) & 1;
      mbar_wait(&full_bar[s], ph);
      uint8_t* st = smem + s * STAGE_BYTES;
#pragma unroll
      for (int d = 0; d < D; ++d) {
        const __nv_bfloat16* sb = reinterpret_cast<const __nv_bfloat16*>(st + OFF_SCALE + d * 512);
        const float sc = __bfloat162float(sb[r]), bi = __bfloat162float(sb[128 + r]);
        for (int half = 0; half < 2; ++half)
          dequant_half_row<BITS>(st + OFF_PACKED + d * PACKED_BYTES + r * (kBlockK * BITS / 8), sc, bi, st + d * kATileBytes, r,
                                 half);
      }
      fence_proxy_async_smem();  // generic-proxy stores -> visible to the tensor core (async proxy)
      __syncwarp();
      if (lane == 0) mbar_arrive(&deq_bar[s]);
    }
  }

}

// ================================================================================================ host side
namespace {

template <int BN, bool DUAL, typename OutT, int BITS>
cudaError_t q_launch_one(const QMaps& t, const GemmParams& p, int group_kblocks, const GemmPlan& plan, cudaStream_t stream) {
  constexpr int STAGES = q_num_stages(BN, DUAL, BITS, sizeof(OutT));
  constexpr int smem = STAGES * q_stage_bytes(BN, DUAL, BITS) + 3 * STAGES * 8 + 16 + 1024;
  static_assert(smem <= 227 * 1024, "shared memory budget exceeded");
  constexpr auto kern = gemm_swapab_q_kernel<BN, DUAL, OutT, BITS>;
  cudaError_t e = set_max_dynamic_smem_once<kern>(smem);
  if (e != cudaSuccess) return e;
  (void)launch_pdl(kern, plan.grid, dim3(kQThreads), smem, stream, t.wq, t.wq2, t.s, t.b, t.s2, t.b2, t.x, p, group_kblocks);
  return cudaGetLastError();
}

}  // namespace

bool q_maps(const GemmArgs& a, int bn, QMaps* t) {
  const uint64_t w_rows = static_cast<uint64_t>(a.n) * (a.expert_offsets != nullptr ? a.num_experts : 1);
  const uint64_t words = static_cast<uint64_t>(a.k) * a.q_bits / 32;
  // packed codes: uint32 [w_rows, words] in unswizzled boxes of 128 rows x one k-block
  auto codes = [&](CUtensorMap* m, const void* ptr) {
    TmapSpec s;
    s.ptr = ptr; s.dtype = CU_TENSOR_MAP_DATA_TYPE_UINT32; s.swizzle = CU_TENSOR_MAP_SWIZZLE_NONE;
    s.dims[0] = words; s.dims[1] = w_rows; s.strides[0] = words * 4;
    s.box[0] = kBlockK * a.q_bits / 32; s.box[1] = kTileM;
    return tmap_cached(m, s);
  };
  // scales / biases: bf16 [k / group, w_rows] in unswizzled boxes of 128 rows of one group
  auto group_rows = [&](CUtensorMap* m, const void* ptr) {
    TmapSpec s;
    s.ptr = ptr; s.swizzle = CU_TENSOR_MAP_SWIZZLE_NONE;
    s.dims[0] = w_rows; s.dims[1] = a.k / a.q_group; s.strides[0] = w_rows * 2;
    s.box[0] = kTileM; s.box[1] = 1;
    return tmap_cached(m, s);
  };
  if (!codes(&t->wq, a.w) || !group_rows(&t->s, a.q_scales_t) || !group_rows(&t->b, a.q_biases_t)) return false;
  if (a.w2 != nullptr) {
    if (!codes(&t->wq2, a.w2) || !group_rows(&t->s2, a.q_scales2_t) || !group_rows(&t->b2, a.q_biases2_t)) return false;
  } else {
    t->wq2 = t->wq; t->s2 = t->s; t->b2 = t->b;
  }
  return gemm_tmap(&t->x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, a.x, a.x_rows, a.k, a.ld_x, bn);
}

bool gemm_q_supported(int bits, int group, int k) {
  return (bits == 4 || bits == 8) && (group == 64 || group == 128) && (k % 64) == 0 && (k % group) == 0;
}

cudaError_t gemm_q_launch(const GemmArgs& a, const GemmPlan& plan, cudaStream_t stream) {
  if (!gemm_q_supported(a.q_bits, a.q_group, a.k)) return cudaErrorNotSupported;
  if (plan.route == kRoutePersistent) return gemm_q_persistent_launch(a, plan, stream);
  const bool dual = a.w2 != nullptr;
  if (a.expert_offsets != nullptr && (a.n % kTileM) != 0) return cudaErrorInvalidValue;
  if ((a.n % 8) != 0) return cudaErrorInvalidValue;
  if (a.workspace == nullptr || a.tile_counters == nullptr) return cudaErrorInvalidValue;
  if (dual && a.out_fp32) return cudaErrorInvalidValue;

  QMaps t;
  if (!q_maps(a, plan.bn, &t)) return cudaErrorUnknown;
  const GemmParams p = gemm_params(a, plan);
  const int gk = a.q_group / kBlockK;  // k-blocks per quantisation group (1 or 2)
  auto dispatch = [&](auto bits) {
    return dispatch_tile<kMaxBN, kMaxBNDual>(plan.bn, dual, a.out_fp32, [&](auto c) {
      using C = decltype(c);
      return q_launch_one<C::BN, C::DUAL, typename C::OutT, decltype(bits)::value>(t, p, gk, plan, stream);
    });
  };
  if (a.q_bits == 4) return dispatch(std::integral_constant<int, 4>{});
  return dispatch(std::integral_constant<int, 8>{});
}

}  // namespace b200
