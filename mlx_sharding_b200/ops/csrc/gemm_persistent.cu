// Persistent variant of the swap-AB wgmma GEMM (dense + grouped, no split-K): one CTA per SM walks a static
// round-robin tile list and the TMA ring never drains between tiles, so tile i+1's weight loads stream while tile i's
// epilogue runs.  The fixed prologue cost is paid once per SM and everything else is a continuous weight stream.
//
// Roles (160 threads): warps 0..3 = MMA warpgroup + epilogue, warp 4 = TMA producer.
// Barriers: full/empty per ring stage.
#include <algorithm>

#include "gemm_common.cuh"
#include "gemm_tmap.h"
#include "launch.h"

namespace b200 {

using namespace gemm;

namespace {

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
__device__ __forceinline__ void publish_tiles_done(const GemmParams& p, unsigned int n) {
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

template <int BN, bool DUAL, typename OutT>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_persistent_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_w2,
                       const __grid_constant__ CUtensorMap tmap_x, const GemmParams p_in, const int tiles_n, const int tiles_m,
                       const int num_tiles) {
  GemmParams p = p_in;
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
  if (p.ep_arrive != nullptr) {
    // Expert-parallel receive side: the token rows, their return addresses and the per-expert row counts of this step are written
    // into this rank's buffers by the *other ranks'* dispatch kernels.  Each source publishes the step's sequence number with
    // release.sys after its rows; one thread per CTA acquires all of them (bounded spin), then the whole CTA proceeds.  This wait
    // used to be a separate single-CTA kernel followed by a gather; now the persistent GEMM's CTAs are already resident (PDL).
    if (threadIdx.x == 0) {
      const uint32_t expected = *reinterpret_cast<const volatile uint32_t*>(p.ep_seq);   // == my own dispatch count (lock-step ranks)
      unsigned long long t0;
      asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t0));
      for (int r = 0; r < p.ep_world; ++r) {
        while (static_cast<uint32_t>(ld_acquire_sys_u64(p.ep_arrive + r)) != expected) {
          unsigned long long t1;
          asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t1));
          if (t1 - t0 > 20000000000ull) { if (p.ep_error != nullptr) atomicExch(p.ep_error, 1u); break; }
          __nanosleep(32);
        }
      }
      __threadfence_system();
    }
    __syncthreads();
    const uint32_t par = *reinterpret_cast<const volatile uint32_t*>(p.ep_seq) & 1u;
    const int ne = num_tiles / (tiles_n * tiles_m);      // experts on this rank
    // counts are double-buffered by step parity; the buffer of the *other* parity (last step's) is reset for the next step
    if (p.ep_zero_other && blockIdx.x == 0)
      for (int e = threadIdx.x; e < ne; e += blockDim.x) const_cast<int*>(p.expert_offsets)[(par ^ 1u) * ne + e] = 0;
    p.expert_offsets += par * ne;
  }

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&tmap_w);
    tma_prefetch_desc(&tmap_x);
    if (DUAL) tma_prefetch_desc(&tmap_w2);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);
    }
    mbar_fence_init();
  }
  __syncthreads();
  // PDL: let the successor's CTAs become resident now (their pre-wait prologue / weight prefetch overlaps this kernel)
  pdl_launch_dependents();

  const int kb_total = (p.k + kBlockK - 1) / kBlockK;

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
          const int kc = (int)(pre % kb_total) * kBlockK;
          mbar_arrive_expect_tx(&full_bar[pre], STAGE_BYTES);
          tma_load_2d(st, &tmap_w, &full_bar[pre], kc, ti.w_row, kEvictFirst);
          if (DUAL) tma_load_2d(st + kATileBytes, &tmap_w2, &full_bar[pre], kc, ti.w_row, kEvictFirst);
        }
        pdl_wait();
        for (uint32_t i = 0; i < pre; ++i) {
          const int t = blockIdx.x + (int)(i / kb_total) * gridDim.x;
          const TileInfo ti = decode_tile(p, t, tiles_n, tiles_m, BN);
          tma_load_2d(smem + i * STAGE_BYTES + kATileBytes * (DUAL ? 2 : 1), &tmap_x, &full_bar[i], (int)(i % kb_total) * kBlockK,
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
          const int kc = kb * kBlockK;
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
    bool waited = pdl_early;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const TileInfo ti = decode_tile(p, t, tiles_n, tiles_m, BN);
      if (ti.rows_valid <= 0) {
        ++my_tiles;  // empty tiles are counted too (EP return: signal_tiles = whole grid)
        continue;
      }
      float acc[2][BN / 2], acc2[2][BN / 2];
      acc_zero<BN>(acc);
      if (DUAL) acc_zero<BN>(acc2);
      mma_mainloop<BN, DUAL, STAGES, STAGE_BYTES, kATileBytes * (DUAL ? 2 : 1)>(
          acc, acc2, smem, empty_bar, it, kb_total, [&](uint32_t s, uint32_t ph) { mbar_wait(&full_bar[s], ph); });
      it += kb_total;
      acc_store_smem<BN>(acc, acc_smem, 0);
      if (DUAL) acc_store_smem<BN>(acc2, acc_smem, BN);
      if (!waited) {  // residual / out are ordered after the predecessor
        pdl_wait();
        waited = true;
      }
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
    if (!waited) pdl_wait();
    if (p.signal_flag != nullptr || p.signal_peers != nullptr) {
      // fused stage boundary / EP return: `out` rows went to peer memory; fence once, then report this CTA's tiles
      __threadfence_system();
      named_bar_sync(1, kEpiThreads);
      if (et == 0) publish_tiles_done(p, p.signal_peers != nullptr ? my_tiles : tc);
    }
  }
}

// ================================================================================================ host side
namespace {

int sm_count_cached() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

template <int BN, bool DUAL, typename OutT>
cudaError_t p_launch_one(const CUtensorMap& tw, const CUtensorMap& tw2, const CUtensorMap& tx, const GemmParams& p, int tiles_n,
                         int tiles_m, int num_tiles, cudaStream_t stream) {
  constexpr int STAGES = p_num_stages(BN, DUAL, sizeof(OutT));
  constexpr int smem = STAGES * stage_bytes(BN, DUAL) + acc_bytes(BN, DUAL) + p_staging_bytes(BN, sizeof(OutT)) + 2 * STAGES * 8 + 1024;
  static_assert(smem <= 227 * 1024, "shared memory budget exceeded");
  auto kern = gemm_persistent_kernel<BN, DUAL, OutT>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  const int grid = std::min(num_tiles, sm_count_cached());
  (void)launch_pdl(kern, dim3(grid), dim3(kNumThreads), smem, stream, tw, tw2, tx, p, tiles_n, tiles_m, num_tiles);
  return cudaGetLastError();
}

template <bool DUAL, typename OutT>
cudaError_t p_dispatch_bn(int bn, const CUtensorMap& tw, const CUtensorMap& tw2, const CUtensorMap& tx, const GemmParams& p,
                          int tiles_n, int tiles_m, int num_tiles, cudaStream_t s) {
  switch (bn) {
    case 16: return p_launch_one<16, DUAL, OutT>(tw, tw2, tx, p, tiles_n, tiles_m, num_tiles, s);
    case 32: return p_launch_one<32, DUAL, OutT>(tw, tw2, tx, p, tiles_n, tiles_m, num_tiles, s);
    case 64: return p_launch_one<64, DUAL, OutT>(tw, tw2, tx, p, tiles_n, tiles_m, num_tiles, s);
    case 128:
      if constexpr (!DUAL) return p_launch_one<128, DUAL, OutT>(tw, tw2, tx, p, tiles_n, tiles_m, num_tiles, s);
      return cudaErrorInvalidValue;
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

cudaError_t gemm_persistent_launch(const GemmArgs& a, cudaStream_t stream) {
  const bool dual = a.w2 != nullptr;
  const bool grouped = a.expert_offsets != nullptr;
  const int bn = gemm_clamp_bn(a.bn > 0 ? a.bn : gemm_pick_bn(a.max_rows), dual);
  if (grouped && (a.n % kTileM) != 0) return cudaErrorInvalidValue;
  if ((a.k % 8) != 0 || (a.n % 8) != 0) return cudaErrorInvalidValue;
  if (dual && a.out_fp32) return cudaErrorInvalidValue;

  CUtensorMap tw, tw2, tx;
  const uint64_t w_rows = static_cast<uint64_t>(a.n) * (grouped ? a.num_experts : 1);
  if (!gemm_make_tmap(&tw, a.w, w_rows, a.k, a.ld_w, kTileM)) return cudaErrorUnknown;
  if (dual) {
    if (!gemm_make_tmap(&tw2, a.w2, w_rows, a.k, a.ld_w, kTileM)) return cudaErrorUnknown;
  } else {
    tw2 = tw;
  }
  if (!gemm_make_tmap(&tx, a.x, a.x_rows, a.k, a.ld_x, bn)) return cudaErrorUnknown;

  GemmParams p;
  p.row_dst = nullptr; p.signal_peers = nullptr; p.num_signal_peers = 0; p.w_sf = p.w2_sf = p.x_sf = nullptr; p.sf_ld_w = p.sf_ld_x = 0;
  p.ep_arrive = a.ep_arrive; p.ep_seq = a.ep_seq; p.ep_error = a.ep_error; p.ep_world = a.ep_world; p.ep_zero_other = a.ep_zero_other ? 1 : 0;
  p.m = a.m; p.n = a.n; p.k = a.k; p.splits = 1; p.cluster_splitk = 0;
  p.expert_offsets = a.expert_offsets;
  p.expert_stride = a.expert_stride;
  p.out = a.out; p.ld_out = a.ld_out;
  p.residual = static_cast<const __nv_bfloat16*>(a.residual); p.ld_res = a.ld_res;
  p.bias = static_cast<const __nv_bfloat16*>(a.bias); p.act = a.act; p.softcap = a.softcap;
  p.workspace = nullptr; p.tile_counters = nullptr;
  p.signal_flag = a.signal_flag; p.signal_value = a.signal_value; p.done_counter = a.done_counter;
  const int tiles_n = (a.n + kTileM - 1) / kTileM;
  const int tiles_m = (a.max_rows + bn - 1) / bn;
  const int num_tiles = tiles_n * tiles_m * (grouped ? a.num_experts : 1);
  p.signal_tiles = a.signal_tiles > 0 ? a.signal_tiles : static_cast<unsigned int>(tiles_n * tiles_m);
  if (a.signal_peers != nullptr) {
    // EP return: every tile of the grid (empty experts included) is counted, then all peers are signalled
    p.row_dst = a.row_dst; p.signal_peers = a.signal_peers; p.num_signal_peers = a.num_signal_peers;
    p.signal_tiles = static_cast<unsigned int>(num_tiles);
  }
  if (a.out_fp32) return p_dispatch_bn<false, float>(bn, tw, tw2, tx, p, tiles_n, tiles_m, num_tiles, stream);
  if (dual) return p_dispatch_bn<true, __nv_bfloat16>(bn, tw, tw2, tx, p, tiles_n, tiles_m, num_tiles, stream);
  return p_dispatch_bn<false, __nv_bfloat16>(bn, tw, tw2, tx, p, tiles_n, tiles_m, num_tiles, stream);
}

}  // namespace b200
