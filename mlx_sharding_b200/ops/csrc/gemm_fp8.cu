// Block-scaled FP8 (MXFP8) variant of the persistent swap-AB GEMM on wgmma (e4m3 x e4m3, fp32 accumulate).
//
// SURVEY §2.6 K17 / BASELINE north star: "block-scaled fp8 where the checkpoint is 4-bit/8-bit".  MLX-affine int4/int8 weights are
// dequantised in shared memory by gemm_q_*.cu (exact MLX semantics, but the dequant ALU work caps the speed-up); here they are
// converted ONCE at load to OCP MXFP8 — e4m3 elements with one power-of-two (ue8m0) scale per 32 consecutive K values
// (utils/quant.py::to_mxfp8):
//
//   * weights [N, K] e4m3 + scales [N, K/32] ue8m0, activations [T, K] e4m3 + scales [T, K/32] (quantised by
//     elementwise.cu::quant_mxfp8_kernel); 1 byte per element, so a 128 B swizzle row is one 128-element k-block and a stage has
//     the same bytes as in the bf16 kernel;
//   * wgmma K = 32 per instruction = exactly one scale block: each block's product goes to a fresh register tile that the warpgroup
//     scales by (weight scale x token scale) and adds into the fp32 accumulator (sm_90 has no block-scaled MMA).
//
// Everything else — the persistent tile walk, grouped (MoE) mode incl. the fixed-stride scatter layout, the DUAL gate/up act(g)*u
// epilogue, residual / fp32 outputs — is gemm_common.cuh's, as in gemm_persistent.cu.
#include "gemm_common.cuh"
#include "gemm_tmap.h"
#include "launch.h"

namespace b200 {

using namespace gemm;

namespace {

constexpr int kFp8Threads = kNumThreads;
constexpr int kFp8BlockK = 128;             // e4m3 elements per k-block = one 128 B swizzle row

__host__ __device__ constexpr int p_staging_bytes(int BN, int out_bytes) { return staging_bytes(BN, kTileM, out_bytes); }
__host__ __device__ constexpr int p_num_stages(int BN, bool dual, int out_bytes) {
  int s = (225 * 1024 - acc_bytes(BN, dual) - p_staging_bytes(BN, out_bytes) - 512) / stage_bytes(BN, dual);
  return s > 8 ? 8 : s;
}

}  // namespace

// ue8m0 -> fp32: 2^(e - 127)
__device__ __forceinline__ float ue8m0(uint32_t e) { return __uint_as_float(e ? e << 23 : 0x00400000u); }

template <int BN, bool DUAL, typename OutT>
__global__ void __launch_bounds__(kFp8Threads, 1)
gemm_fp8_persistent_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_w2,
                       const __grid_constant__ CUtensorMap tmap_x, const GemmParams p, const int tiles_n, const int tiles_m,
                       const int num_tiles) {
  constexpr int STAGES = p_num_stages(BN, DUAL, sizeof(OutT));
  constexpr int STAGE_BYTES = stage_bytes(BN, DUAL);
  static_assert(STAGES >= 2, "ring too small");

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024 B alignment by *pointer arithmetic* on the __shared__ array: an integer round-trip loses the address space and
  // turns every LDS/STS below into a generic LD.E/ST.E (checked with cuobjdump -sass)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  float* acc_smem = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);   // [BN * (1 + DUAL)][128] fp32
  OutT* stg = reinterpret_cast<OutT*>(smem + STAGES * STAGE_BYTES + acc_bytes(BN, DUAL));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + acc_bytes(BN, DUAL) + p_staging_bytes(BN, sizeof(OutT)));
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const bool pdl_early = p.expert_offsets != nullptr;
  if (pdl_early) pdl_wait();

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&tmap_w);
    tma_prefetch_desc(&tmap_x);
    if (DUAL) tma_prefetch_desc(&tmap_w2);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);  // one arrival per MMA warp
    }
    mbar_fence_init();
  }
  __syncthreads();
  // PDL: let the successor's CTAs become resident now (their pre-wait prologue / weight prefetch overlaps this kernel)
  pdl_launch_dependents();

  const int kb_total = (p.k + kFp8BlockK - 1) / kFp8BlockK;

  if (warp == kProducerWarp) {
    // ============================================================== TMA producer
    if (elect_one()) {  // one elected lane: uniform-datapath issue, no per-instruction ELECT loop (ptx.cuh)
      // Weights never depend on a predecessor kernel: the first ring-full of weight tiles is requested *before*
      // griddepcontrol.wait (HBM latency overlaps the predecessor's tail); the activation tiles follow after it.
      // (un-grouped launches only: iteration i <-> tile blockIdx.x + (i / kb_total) * gridDim.x, k-block i % kb_total)
      uint32_t pre = 0;
      if (!pdl_early) {
        for (; pre < (uint32_t)STAGES; ++pre) {
          const int t = blockIdx.x + (int)(pre / kb_total) * gridDim.x;
          if (t >= num_tiles) break;
          const TileInfo ti = decode_tile(p, t, tiles_n, tiles_m, BN);
          uint8_t* st = smem + pre * STAGE_BYTES;
          const int kc = (int)(pre % kb_total) * kFp8BlockK;
          mbar_arrive_expect_tx(&full_bar[pre], STAGE_BYTES);
          tma_load_2d(st, &tmap_w, &full_bar[pre], kc, ti.w_row, kEvictFirst);
          if (DUAL) tma_load_2d(st + kATileBytes, &tmap_w2, &full_bar[pre], kc, ti.w_row, kEvictFirst);
        }
        pdl_wait();
        for (uint32_t i = 0; i < pre; ++i) {
          const int t = blockIdx.x + (int)(i / kb_total) * gridDim.x;
          const TileInfo ti = decode_tile(p, t, tiles_n, tiles_m, BN);
          tma_load_2d(smem + i * STAGE_BYTES + kATileBytes * (DUAL ? 2 : 1), &tmap_x, &full_bar[i], (int)(i % kb_total) * kFp8BlockK,
                      ti.row_base, kEvictLast);
        }
      }
      uint32_t it = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const TileInfo ti = decode_tile(p, t, tiles_n, tiles_m, BN);
        if (ti.rows_valid <= 0) continue;
        for (int kb = 0; kb < kb_total; ++kb, ++it) {
          if (it < pre) continue;  // issued above
          const uint32_t s = it % STAGES, ph = (it / STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* st = smem + s * STAGE_BYTES;
          const int kc = kb * kFp8BlockK;
          mbar_arrive_expect_tx(&full_bar[s], STAGE_BYTES);
          tma_load_2d(st, &tmap_w, &full_bar[s], kc, ti.w_row, kEvictFirst);
          if (DUAL) tma_load_2d(st + kATileBytes, &tmap_w2, &full_bar[s], kc, ti.w_row, kEvictFirst);
          tma_load_2d(st + kATileBytes * (DUAL ? 2 : 1), &tmap_x, &full_bar[s], kc, ti.row_base, kEvictLast);
        }
      }
    }
  } else {
    // ============================================================== MMA warpgroup, then epilogue (128 threads)
    uint32_t it = 0;
    if (!pdl_early) pdl_wait();  // activation scales, residual and out are ordered after the predecessor
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const TileInfo ti = decode_tile(p, t, tiles_n, tiles_m, BN);
      if (ti.rows_valid <= 0) continue;
      float acc[2][BN / 2], acc2[2][BN / 2];
      acc_zero<BN>(acc);
      if (DUAL) acc_zero<BN>(acc2);
      for (int kb = 0; kb < kb_total; ++kb, ++it) {
        const uint32_t s = it % STAGES, ph = (it / STAGES) & 1;
        // scale words (4 x ue8m0, one per 32-wide K block) of this thread's 4 weight rows and BN / 4 token rows
        uint32_t wa[2][2], wa2[2][2], wb[BN / 4];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const size_t row = static_cast<size_t>(ti.w_row + h * 64 + wg_row(2 * r));
            wa[h][r] = __ldg(p.w_sf + row * p.sf_ld_w + kb);
            wa2[h][r] = DUAL ? __ldg(p.w2_sf + row * p.sf_ld_w + kb) : 0u;
          }
#pragma unroll
        for (int c = 0; c < BN / 4; ++c) {
          const int r = wg_col(4 * (c >> 1) + (c & 1));
          wb[c] = r < ti.rows_valid ? __ldcg(p.x_sf + static_cast<size_t>(ti.row_base + r) * p.sf_ld_x + kb) : 0x7f7f7f7fu;
        }
        mbar_wait(&full_bar[s], ph);
        const uint32_t a_addr = smem_u32(smem + s * STAGE_BYTES);
        const uint64_t bdesc = gmma_desc_sw128(a_addr + kATileBytes * (DUAL ? 2 : 1));
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {   // 4 x (K = 32) per 128-element k-block; scale byte kk of the words
          float part[2][BN / 2], part2[2][BN / 2];
          wgmma_fence();
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            wgmma_e4m3<BN>(part[h], gmma_desc_sw128(a_addr + h * 64 * 128) + 2 * kk, bdesc + 2 * kk);
            if (DUAL) wgmma_e4m3<BN>(part2[h], gmma_desc_sw128(a_addr + kATileBytes + h * 64 * 128) + 2 * kk, bdesc + 2 * kk);
          }
          wgmma_commit();
          wgmma_wait<0>();
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            wgmma_fence_acc(part[h]);
            if (DUAL) wgmma_fence_acc(part2[h]);
#pragma unroll
            for (int j = 0; j < BN / 2; ++j) {
              const float sb = ue8m0((wb[2 * (j >> 2) + (j & 1)] >> (8 * kk)) & 0xFF);
              acc[h][j] += part[h][j] * (ue8m0((wa[h][(j >> 1) & 1] >> (8 * kk)) & 0xFF) * sb);
              if (DUAL) acc2[h][j] += part2[h][j] * (ue8m0((wa2[h][(j >> 1) & 1] >> (8 * kk)) & 0xFF) * sb);
            }
          }
        }
        if (lane == 0) mbar_arrive(&empty_bar[s]);
      }
      acc_store_smem<BN>(acc, acc_smem, 0);
      if (DUAL) acc_store_smem<BN>(acc2, acc_smem, BN);
      named_bar_sync(1, kEpiThreads);
      store_acc_tile<BN, DUAL, OutT>(p, acc_smem, stg, ti);
    }
  }
}

// ================================================================================================ host side
namespace {

template <int BN, bool DUAL, typename OutT>
cudaError_t f_launch_one(const GemmMaps& t, const GemmParams& p, const GemmPlan& plan, cudaStream_t stream) {
  constexpr int STAGES = p_num_stages(BN, DUAL, sizeof(OutT));
  constexpr int smem = STAGES * stage_bytes(BN, DUAL) + acc_bytes(BN, DUAL) + p_staging_bytes(BN, sizeof(OutT)) + 2 * STAGES * 8 + 1024;
  static_assert(smem <= 227 * 1024, "shared memory budget exceeded");
  constexpr auto kern = gemm_fp8_persistent_kernel<BN, DUAL, OutT>;
  cudaError_t e = set_max_dynamic_smem_once<kern>(smem);
  if (e != cudaSuccess) return e;
  (void)launch_pdl(kern, plan.grid, dim3(kFp8Threads), smem, stream, t.w, t.w2, t.x, p, plan.tiles_n, plan.tiles_m, plan.num_tiles);
  return cudaGetLastError();
}

}  // namespace

cudaError_t gemm_fp8_launch(const GemmArgs& a, const GemmPlan& plan, cudaStream_t stream) {
  const bool dual = a.w2 != nullptr;
  if (a.expert_offsets != nullptr && (a.n % kTileM) != 0) return cudaErrorInvalidValue;
  if ((a.k % kFp8BlockK) != 0 || (a.n % kTileM) != 0) return cudaErrorInvalidValue;   // whole k-blocks / weight tiles only
  if (a.w_sf == nullptr || a.x_sf == nullptr || (dual && a.w2_sf == nullptr)) return cudaErrorInvalidValue;
  if (dual && a.out_fp32) return cudaErrorInvalidValue;

  GemmMaps t;
  if (!gemm_maps(a, CU_TENSOR_MAP_DATA_TYPE_UINT8, plan.bn, &t)) return cudaErrorUnknown;
  GemmParams p = gemm_params(a, plan);
  p.w_sf = static_cast<const uint32_t*>(a.w_sf); p.w2_sf = static_cast<const uint32_t*>(a.w2_sf);
  p.x_sf = static_cast<const uint32_t*>(a.x_sf); p.sf_ld_w = a.k / kFp8BlockK; p.sf_ld_x = a.k / kFp8BlockK;
  return dispatch_tile<kFp8MaxBN, kFp8MaxBNDual>(plan.bn, dual, a.out_fp32, [&](auto c) {
    using C = decltype(c);
    return f_launch_one<C::BN, C::DUAL, typename C::OutT>(t, p, plan, stream);
  });
}

}  // namespace b200
