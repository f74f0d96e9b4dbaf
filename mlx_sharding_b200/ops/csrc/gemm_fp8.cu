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
// Everything else — persistent tile walk, grouped (MoE) mode incl. the fixed-stride scatter layout, DUAL gate/up with act(g)*u
// epilogue, residual / fp32 outputs — is shared by construction with gemm_persistent.cu.
#include "gemm_common.cuh"
#include "gemm_tmap.h"
#include "launch.h"

namespace b200 {

using namespace gemm;

namespace {

constexpr int kFp8Threads = kNumThreads;
constexpr int kFp8BlockK = 128;             // e4m3 elements per k-block = one 128 B swizzle row

__host__ __device__ constexpr int p_stg_rows(int BN) { return BN < 64 ? BN : 64; }
__host__ __device__ constexpr int p_staging_bytes(int BN, int out_bytes) { return p_stg_rows(BN) * kTileM * out_bytes; }
__host__ __device__ constexpr int p_num_stages(int BN, bool dual, int out_bytes) {
  int s = (225 * 1024 - acc_bytes(BN, dual) - p_staging_bytes(BN, out_bytes) - 512) / stage_bytes(BN, dual);
  return s > 8 ? 8 : s;
}

struct TileInfo {
  int n0, w_row, row_base, rows_valid, mt;
};

__device__ __forceinline__ TileInfo decode_tile(const GemmParams& p, int t, int tiles_n, int tiles_m, int BN) {
  TileInfo ti;
  const int nt = t % tiles_n;
  const int rest = t / tiles_n;
  ti.mt = rest % tiles_m;
  const int expert = rest / tiles_m;
  ti.n0 = nt * kTileM;
  ti.row_base = 0;
  ti.rows_valid = p.m;
  if (p.expert_offsets != nullptr) {
    if (p.expert_stride > 0) {   // scatter layout: fixed stride per expert, the array holds row counts (written by atomics: no __ldg)
      ti.row_base = expert * p.expert_stride;
      ti.rows_valid = __ldcg(p.expert_offsets + expert);
    } else {
      const int lo = __ldg(p.expert_offsets + expert), hi = __ldg(p.expert_offsets + expert + 1);
      ti.row_base = lo;
      ti.rows_valid = hi - lo;
    }
  }
  ti.rows_valid -= ti.mt * BN;
  ti.row_base += ti.mt * BN;
  if (ti.rows_valid > BN) ti.rows_valid = BN;
  ti.w_row = expert * p.n + ti.n0;
  return ti;
}

}  // namespace

// One thread per CTA, once, after the CTA's last tile (a system fence per *tile* would stall the epilogue on an NVLink round
// trip each time when `out` is peer memory): reports how many tiles of the grid this CTA covered; the arrival that completes
// the grid raises the consumer flag(s) with system scope.  Every CTA fences its own stores before arriving.
__device__ __forceinline__ void fp8_publish_tiles_done(const GemmParams& p, unsigned int n) {
  const unsigned int done = atomicAdd(p.done_counter, n) + n;
  if (done != p.signal_tiles) return;
  *p.done_counter = 0u;
  __threadfence_system();
  if (p.signal_peers != nullptr) {
    for (int i = 0; i < p.num_signal_peers; ++i) atomicAdd_system(reinterpret_cast<unsigned int*>(__ldg(p.signal_peers + i)), 1u);
  } else if (p.signal_value == 0u) {
    atomicAdd_system(p.signal_flag, 1u);
  } else {
    st_release_sys(p.signal_flag, p.signal_value);
  }
}

// ue8m0 -> fp32: 2^(e - 127)
__device__ __forceinline__ float ue8m0(uint32_t e) { return __uint_as_float(e ? e << 23 : 0x00400000u); }

template <int BN, bool DUAL, typename OutT>
__global__ void __launch_bounds__(kFp8Threads, 1)
gemm_fp8_persistent_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_w2,
                       const __grid_constant__ CUtensorMap tmap_x, const GemmParams p, const int tiles_n, const int tiles_m,
                       const int num_tiles) {
  constexpr int STAGES = p_num_stages(BN, DUAL, sizeof(OutT));
  constexpr int STAGE_BYTES = stage_bytes(BN, DUAL);
  constexpr int STG_ROWS = p_stg_rows(BN);
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
    const int f_local = threadIdx.x;
    const int et = threadIdx.x;
    constexpr int kVec = 8, kChunks = kTileM / kVec, kRowsPerIter = kEpiThreads / kChunks;
    uint32_t it = 0, tc = 0, my_tiles = 0;
    if (!pdl_early) pdl_wait();  // activation scales, residual and out are ordered after the predecessor
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const TileInfo ti = decode_tile(p, t, tiles_n, tiles_m, BN);
      if (ti.rows_valid <= 0) {
        ++my_tiles;  // empty tiles are counted too (EP return: signal_tiles = whole grid)
        continue;
      }
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
      const int f_glob = ti.n0 + f_local;
      const float bias = (p.bias != nullptr && f_glob < p.n) ? __bfloat162float(p.bias[f_glob]) : 0.0f;
#pragma unroll 1
      for (int c0 = 0; c0 < BN; c0 += STG_ROWS) {
        if (c0 >= ti.rows_valid) break;
#pragma unroll 1
        for (int c = c0; c < c0 + STG_ROWS; c += 16) {
          if (c >= ti.rows_valid) break;
          float g[16], u[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            g[j] = acc_smem[(c + j) * kTileM + f_local];
            if (DUAL) u[j] = acc_smem[(BN + c + j) * kTileM + f_local];
          }
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            float y = g[j] + bias;
            if (DUAL) y = apply_act(p.act, y) * u[j];
            if (p.softcap > 0.f) y = p.softcap * tanhf(y / p.softcap);
            stage_store<OutT>(&stg[(c - c0 + j) * kTileM + f_local], y);
          }
        }
        named_bar_sync(1, kEpiThreads);
        const int ch = et % kChunks;
        const int f0 = ti.n0 + ch * kVec;
        const int rows_here = min(STG_ROWS, ti.rows_valid - c0);
        if (f0 < p.n) {
          for (int r = et / kChunks; r < rows_here; r += kRowsPerIter) {
            const size_t row = static_cast<size_t>(ti.row_base + c0 + r);
            float vals[kVec];
            if (sizeof(OutT) == 2) {
              const uint4 raw = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(stg) + r * kTileM + ch * kVec);
              const uint32_t w4[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
              for (int j = 0; j < 4; ++j) { vals[2 * j] = bf16_lo(w4[j]); vals[2 * j + 1] = bf16_hi(w4[j]); }
            } else {
              const float4 a = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(stg) + r * kTileM + ch * kVec);
              const float4 b = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(stg) + r * kTileM + ch * kVec + 4);
              vals[0] = a.x; vals[1] = a.y; vals[2] = a.z; vals[3] = a.w;
              vals[4] = b.x; vals[5] = b.y; vals[6] = b.z; vals[7] = b.w;
            }
            if (p.residual != nullptr) {
              const uint4 rr = *reinterpret_cast<const uint4*>(p.residual + row * p.ld_res + f0);
              const uint32_t w4[4] = {rr.x, rr.y, rr.z, rr.w};
#pragma unroll
              for (int j = 0; j < 4; ++j) { vals[2 * j] += bf16_lo(w4[j]); vals[2 * j + 1] += bf16_hi(w4[j]); }
            }
            // destination row: [row] of `out`, or (EP return) wherever the row's owner wants it — possibly peer memory
            OutT* orow = p.row_dst != nullptr ? reinterpret_cast<OutT*>(__ldg(p.row_dst + row))
                                              : reinterpret_cast<OutT*>(p.out) + row * p.ld_out;
            if (sizeof(OutT) == 2) {
              uint4 o;
              o.x = pack_bf16(vals[0], vals[1]); o.y = pack_bf16(vals[2], vals[3]);
              o.z = pack_bf16(vals[4], vals[5]); o.w = pack_bf16(vals[6], vals[7]);
              *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(orow) + f0) = o;
            } else {
              float* o = reinterpret_cast<float*>(orow) + f0;
              *reinterpret_cast<float4*>(o) = make_float4(vals[0], vals[1], vals[2], vals[3]);
              *reinterpret_cast<float4*>(o + 4) = make_float4(vals[4], vals[5], vals[6], vals[7]);
            }
          }
        }
        named_bar_sync(1, kEpiThreads);  // staging buffer (and, after the last chunk, the accumulator) free again
      }
      ++my_tiles;
      ++tc;
    }
    if (p.signal_flag != nullptr || p.signal_peers != nullptr) {
      // fused stage boundary / EP return: `out` rows went to peer memory; fence once, then report this CTA's tiles
      __threadfence_system();
      named_bar_sync(1, kEpiThreads);
      if (et == 0) fp8_publish_tiles_done(p, p.signal_peers != nullptr ? my_tiles : tc);
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
  if (a.signal_peers != nullptr) {
    // EP return: every tile of the grid (empty experts included) is counted, then all peers are signalled
    p.row_dst = a.row_dst; p.signal_peers = a.signal_peers; p.num_signal_peers = a.num_signal_peers;
    p.signal_tiles = static_cast<unsigned int>(plan.num_tiles);
  }
  return dispatch_tile<kFp8MaxBN, kFp8MaxBNDual>(plan.bn, dual, a.out_fp32, [&](auto c) {
    using C = decltype(c);
    return f_launch_one<C::BN, C::DUAL, typename C::OutT>(t, p, plan, stream);
  });
}

}  // namespace b200
