// Persistent variant of the swap-AB wgmma GEMM (dense + grouped, no split-K): one CTA per SM walks a static
// round-robin tile list and the TMA ring never drains between tiles, so tile i+1's weight loads stream while tile i's
// epilogue runs.  The fixed prologue cost is paid once per SM and everything else is a continuous weight stream.
//
// Roles (160 threads): warps 0..3 = MMA warpgroup + epilogue, warp 4 = TMA producer.
// Barriers: full/empty per ring stage.
//
// Shared memory is the TMA ring plus one output staging tile; the epilogue works on the wgmma fragments in registers, so no fp32
// accumulator tile competes with the ring (5 stages for the gate/up pair at BN = 64, 8 for a single matrix).  Token tiles are
// loaded in 16-row boxes, only as many as the tile has valid rows: a routed expert of a decode step holds a handful of rows of its
// 64-row segment.
#include "gemm_common.cuh"
#include "gemm_tmap.h"
#include "kernels.h"
#include "launch.h"

namespace b200 {

using namespace gemm;

namespace {

constexpr int kXBoxRows = 16;                             // token rows per TMA box
constexpr int kXBoxBytes = kXBoxRows * kBlockK * 2;       // 2 KB

// Staging row pitch in elements: 16 B of padding per token row.  A fragment store writes 8 consecutive features of 4 token columns
// (2 apart); unpadded, those columns are a multiple of 512 B apart and hit the same banks (4-way conflict), padded they are 32 B apart.
__host__ __device__ constexpr int p_stg_ld(int out_bytes) { return kTileM + 16 / out_bytes; }
__host__ __device__ constexpr int p_staging_bytes(int BN, int out_bytes) { return staging_bytes(BN, p_stg_ld(out_bytes), out_bytes); }
__host__ __device__ constexpr int p_num_stages(int BN, bool dual, int out_bytes) {
  // 227 KB opt-in shared memory less the 1 KB alignment slack, the staging tile and the barriers (at most 8 stages x 2 x 8 B)
  int s = (227 * 1024 - 1024 - p_staging_bytes(BN, out_bytes) - 2 * 8 * 8) / stage_bytes(BN, dual);
  return s > 8 ? 8 : s;
}

}  // namespace

template <int BN, bool DUAL, typename OutT>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_persistent_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_w2,
                       const __grid_constant__ CUtensorMap tmap_x, const GemmParams p_in, const int tiles_n, const int tiles_m,
                       const int num_tiles) {
  GemmParams p = p_in;
  constexpr int STAGES = p_num_stages(BN, DUAL, sizeof(OutT));
  constexpr int STAGE_BYTES = stage_bytes(BN, DUAL);
  constexpr int STG_ROWS = stg_rows(BN);
  constexpr int STG_LD = p_stg_ld(sizeof(OutT));
  constexpr int OFF_X = kATileBytes * (DUAL ? 2 : 1);   // token tile within a stage
  static_assert(STAGES >= 2, "ring too small");
  static_assert(BN % kXBoxRows == 0, "token tile must be whole boxes");

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024 B alignment by *pointer arithmetic* on the __shared__ array: an integer round-trip loses the address space and
  // turns every LDS/STS below into a generic LD.E/ST.E (checked with cuobjdump -sass)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  OutT* stg = reinterpret_cast<OutT*>(smem + STAGES * STAGE_BYTES);   // [STG_ROWS][STG_LD]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + p_staging_bytes(BN, sizeof(OutT)));
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int kb_total = (p.k + kBlockK - 1) / kBlockK;
  const bool pdl_early = p.expert_offsets != nullptr;
  if (pdl_early) {
    // Grouped launches read the router's counts, so they wait for the predecessor before anything else.  The weights do not depend
    // on it: the producer first prefetches the first ring-full of k-blocks of this CTA's first tile into L2, so HBM streams through
    // the router (or the gate/up -> down boundary) instead of idling.  No ring bookkeeping: the loads after the wait hit L2.
    if (warp == kProducerWarp && elect_one()) {
      const int w_row = (blockIdx.x / (tiles_n * tiles_m)) * p.n + (blockIdx.x % tiles_n) * kTileM;
      const int kb_pre = kb_total < STAGES ? kb_total : STAGES;
      for (int kb = 0; kb < kb_pre; ++kb) {
        tma_prefetch_l2_2d(&tmap_w, kb * kBlockK, w_row);
        if (DUAL) tma_prefetch_l2_2d(&tmap_w2, kb * kBlockK, w_row);
      }
    }
    pdl_wait();
  }
  if (p.ep_arrive != nullptr) {
    // Expert-parallel receive side: the token rows, their return addresses and the per-expert row counts of this step are written
    // into this rank's buffers by the *other ranks'* dispatch kernels.  Each source publishes the step's sequence number with
    // release.sys after its rows (ep_dispatch.cuh); one thread per CTA acquires all of them, then the whole CTA proceeds.
    if (threadIdx.x == 0) {
      const uint32_t expected = *reinterpret_cast<const volatile uint32_t*>(p.ep_seq);   // == my own dispatch count (lock-step ranks)
      const unsigned long long t0 = globaltimer_ns();
      for (int r = 0; r < p.ep_world; ++r)
        spin_acquire([&] { return static_cast<uint32_t>(ld_acquire_sys_u64(p.ep_arrive + r)) == expected; }, t0, p.ep_timeout_ns,
                     p.ep_error);
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

  if (warp == kProducerWarp) {
    // ============================================================== TMA producer
    if (elect_one()) {  // one elected lane: uniform-datapath issue, no per-instruction ELECT loop (ptx.cuh)
      // Only the 16-row boxes that hold valid rows are loaded; the token rows of the stage beyond them keep stale data, which only
      // feeds accumulator columns the epilogue never stores.
      auto x_boxes = [](const TileInfo& ti) { return (ti.rows_valid + kXBoxRows - 1) / kXBoxRows; };
      auto stage_tx = [&](const TileInfo& ti) { return (uint32_t)(OFF_X + x_boxes(ti) * kXBoxBytes); };
      auto load_x = [&](uint8_t* st, uint64_t* bar, int kc, const TileInfo& ti) {
        const int nb = x_boxes(ti);
        for (int b = 0; b < nb; ++b) tma_load_2d(st + OFF_X + b * kXBoxBytes, &tmap_x, bar, kc, ti.row_base + b * kXBoxRows, kEvictLast);
      };
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
          mbar_arrive_expect_tx(&full_bar[pre], stage_tx(ti));
          tma_load_2d(st, &tmap_w, &full_bar[pre], kc, ti.w_row, kEvictFirst);
          if (DUAL) tma_load_2d(st + kATileBytes, &tmap_w2, &full_bar[pre], kc, ti.w_row, kEvictFirst);
        }
        pdl_wait();
        for (uint32_t i = 0; i < pre; ++i) {
          const int t = blockIdx.x + (int)(i / kb_total) * gridDim.x;
          const TileInfo ti = decode_tile(p, t, tiles_n, tiles_m, BN);
          load_x(smem + i * STAGE_BYTES, &full_bar[i], (int)(i % kb_total) * kBlockK, ti);
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
          mbar_arrive_expect_tx(&full_bar[s], stage_tx(ti));
          tma_load_2d(st, &tmap_w, &full_bar[s], kc, ti.w_row, kEvictFirst);
          if (DUAL) tma_load_2d(st + kATileBytes, &tmap_w2, &full_bar[s], kc, ti.w_row, kEvictFirst);
          load_x(st, &full_bar[s], kc, ti);
        }
      }
    }
  } else {
    // ============================================================== MMA warpgroup, then epilogue (128 threads)
    const int et = threadIdx.x;
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
      mma_mainloop<BN, DUAL, STAGES, STAGE_BYTES, OFF_X>(
          acc, acc2, smem, empty_bar, it, kb_total, [&](uint32_t s, uint32_t ph) { mbar_wait(&full_bar[s], ph); });
      it += kb_total;
      if (!waited) {  // residual / out are ordered after the predecessor
        pdl_wait();
        waited = true;
      }
      // this thread's fragment rows (features) are h * 64 + wg_row(j), and wg_row(j) only depends on bit 1 of j
      float bias[2][2];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < 2; ++r) bias[h][r] = feature_bias(p, ti.n0 + h * 64 + wg_row(2 * r));
      // Epilogue on the fragments: acc[h][j] and acc2[h][j] are the same (feature, token).  The chunk loop is unrolled so that the
      // fragment index stays a compile-time constant (the accumulators never leave registers); only valid token columns are stored.
#pragma unroll
      for (int c0 = 0; c0 < BN; c0 += STG_ROWS) {
        if (c0 >= ti.rows_valid) break;
#pragma unroll
        for (int j = c0 / 2; j < (c0 + STG_ROWS) / 2; ++j) {
          const int c = wg_col(j);
          if (c >= ti.rows_valid) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h)
            stage_store<OutT>(&stg[(c - c0) * STG_LD + h * 64 + wg_row(j)], epi_value<DUAL>(p, acc[h][j], acc2[h][j], bias[h][(j >> 1) & 1]));
        }
        named_bar_sync(1, kEpiThreads);
        write_rows<OutT>(p, stg, STG_LD, et, ti.n0, ti.row_base + c0, min(STG_ROWS, ti.rows_valid - c0));
        named_bar_sync(1, kEpiThreads);  // staging buffer free again
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

template <int BN, bool DUAL, typename OutT>
cudaError_t p_launch_one(const GemmMaps& t, const GemmParams& p, const GemmPlan& plan, cudaStream_t stream) {
  constexpr int STAGES = p_num_stages(BN, DUAL, sizeof(OutT));
  constexpr int smem = STAGES * stage_bytes(BN, DUAL) + p_staging_bytes(BN, sizeof(OutT)) + 2 * STAGES * 8 + 1024;
  static_assert(smem <= 227 * 1024, "shared memory budget exceeded");
  constexpr auto kern = gemm_persistent_kernel<BN, DUAL, OutT>;
  cudaError_t e = set_max_dynamic_smem_once<kern>(smem);
  if (e != cudaSuccess) return e;
  (void)launch_pdl(kern, plan.grid, dim3(kNumThreads), smem, stream, t.w, t.w2, t.x, p, plan.tiles_n, plan.tiles_m, plan.num_tiles);
  return cudaGetLastError();
}

}  // namespace

cudaError_t gemm_persistent_launch(const GemmArgs& a, const GemmPlan& plan, cudaStream_t stream) {
  const bool dual = a.w2 != nullptr;
  if (a.expert_offsets != nullptr && (a.n % kTileM) != 0) return cudaErrorInvalidValue;
  if ((a.k % 8) != 0 || (a.n % 8) != 0) return cudaErrorInvalidValue;
  if (dual && a.out_fp32) return cudaErrorInvalidValue;

  GemmMaps t;
  if (!gemm_maps(a, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, kXBoxRows, &t)) return cudaErrorUnknown;
  GemmParams p = gemm_params(a, plan);
  if (a.ep_arrive != nullptr) {
    p.ep_arrive = a.ep_arrive; p.ep_seq = a.ep_seq; p.ep_error = a.ep_error; p.ep_timeout_ns = wait_timeout_ns();
    p.ep_world = a.ep_world; p.ep_zero_other = a.ep_zero_other ? 1 : 0;
  }
  if (a.signal_peers != nullptr) {
    // EP return: every tile of the grid (empty experts included) is counted, then all peers are signalled
    p.row_dst = a.row_dst; p.signal_peers = a.signal_peers; p.num_signal_peers = a.num_signal_peers;
    p.signal_tiles = static_cast<unsigned int>(plan.num_tiles);
  }
  return dispatch_tile<kMaxBN, kMaxBNDual>(plan.bn, dual, a.out_fp32, [&](auto c) {
    using C = decltype(c);
    return p_launch_one<C::BN, C::DUAL, typename C::OutT>(t, p, plan, stream);
  });
}

}  // namespace b200
