// Swap-AB wgmma GEMM for LLM inference on sm_90a:  Y[tokens, N] = X[tokens, K] · W[N, K]^T
//
// Implements SURVEY §2.6 K3/K4/K5/K8/K9/K11/K12 (all projection GEMMs, the SwiGLU/GeGLU pair, the MoE
// grouped GEMMs and the LM head) — ops the reference delegates to MLX Metal matmul / gather_qmm
// (shard/server/model/*.py via mlx_lm blocks).
//
// Design:
//  * The *weight* tile is the MMA "A" operand (128 output features = two wgmma M = 64 halves) and the
//    *token* tile is the "B" operand (N = BN in {16..128} tokens).  Decode batches are skinny (1..64
//    tokens) so the tensor-core tile is always full along M and the kernel is a pure HBM weight
//    stream; prefill uses BN = 128 (64 for the gate/up pair: the accumulators live in registers).
//  * TMA (cp.async.bulk.tensor, 128B swizzle) feeds a STAGES-deep shared-memory ring; one warpgroup
//    issues wgmma with fp32 accumulators in registers, then stores them to shared memory, applies the
//    fused epilogue, transposes through shared memory and writes coalesced rows.
//  * DUAL mode streams two weight matrices (gate, up) against the same token tile into two register
//    accumulators and writes act(gate)*up — the SwiGLU intermediate never touches HBM un-fused.
//  * Grouped mode (MoE): blockIdx.y = expert, rows come from a permuted token buffer via per-expert
//    offsets; experts with no tokens exit immediately.
//  * split-K (decode, few output tiles): partial tiles go to an fp32 workspace; the last-arriving CTA of a
//    tile (global atomic ticket) reduces them in split order (deterministic) and runs the epilogue.
//  * Fused stage boundary: `out` may be a peer-mapped pointer (next pipeline stage's inbox over
//    NVLink); when `signal_flag` is set the last CTA of the grid publishes it with st.release.sys
//    after a system-scope fence — GEMM + P2P hand-off in one kernel, no NCCL call, no host hop.
#include "gemm_cluster.cuh"
#include "gemm_tmap.h"
#include "launch.h"

namespace b200 {

using namespace gemm;

template <int BN, bool DUAL, typename OutT>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_swapab_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_w2,
                   const __grid_constant__ CUtensorMap tmap_x, const GemmParams p) {
  constexpr int STAGES = num_stages(BN, DUAL, sizeof(OutT));
  constexpr int STAGE_BYTES = stage_bytes(BN, DUAL);

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024B alignment is required by the 128B swizzle atom (8 rows x 128 B)
  // 1024 B alignment by *pointer arithmetic* on the __shared__ array: an integer round-trip loses the address space and
  // turns every LDS/STS below into a generic LD.E/ST.E (checked with cuobjdump -sass)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint32_t* flag_smem = reinterpret_cast<uint32_t*>(empty_bar + STAGES);
  // after the main loop the idle ring holds the fp32 accumulator [BN * (1 + DUAL)][128], then the output staging tile
  float* acc_smem = reinterpret_cast<float*>(smem);
  OutT* stg = reinterpret_cast<OutT*>(smem + acc_bytes(BN, DUAL));

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // ---------------------------------------------------------------- tile coordinates
  // PDL: grouped launches read expert_offsets (written by the permutation kernel) right away, so they wait first;
  // plain launches overlap their whole prologue (barrier init) with the predecessor's tail.
  const bool pdl_early = p.expert_offsets != nullptr;
  if (pdl_early) pdl_wait();
  const SplitTile sk = splitk_tile(p, BN);
  const TileInfo& ti = sk.ti;
  if (ti.rows_valid <= 0) return;  // uniform across the CTA
  const int kb_begin = sk.kb_begin, num_kb = sk.num_kb;

  // ---------------------------------------------------------------- one-time setup
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
      // Weights never depend on a predecessor kernel: the first ring-full of weight tiles is requested *before*
      // griddepcontrol.wait, so their HBM latency overlaps the predecessor's tail; the activation tiles follow after it.
      const int pre = pdl_early ? 0 : (num_kb < STAGES ? num_kb : STAGES);
      for (int i = 0; i < pre; ++i) {
        uint8_t* st = smem + i * STAGE_BYTES;
        const int kc = (kb_begin + i) * kBlockK;
        mbar_arrive_expect_tx(&full_bar[i], STAGE_BYTES);
        tma_load_2d(st, &tmap_w, &full_bar[i], kc, ti.w_row, kEvictFirst);
        if (DUAL) tma_load_2d(st + kATileBytes, &tmap_w2, &full_bar[i], kc, ti.w_row, kEvictFirst);
      }
      if (!pdl_early) pdl_wait();
      for (int i = 0; i < pre; ++i)
        tma_load_2d(smem + i * STAGE_BYTES + kATileBytes * (DUAL ? 2 : 1), &tmap_x, &full_bar[i], (kb_begin + i) * kBlockK, ti.row_base, kEvictLast);
      for (int i = pre; i < num_kb; ++i) {
        const int s = i % STAGES;
        const uint32_t ph = (i / STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* st = smem + s * STAGE_BYTES;
        const int kc = (kb_begin + i) * kBlockK;
        mbar_arrive_expect_tx(&full_bar[s], STAGE_BYTES);
        // weights are streamed exactly once per launch: evict-first; activations are re-read by every
        // feature tile: evict-last
        tma_load_2d(st, &tmap_w, &full_bar[s], kc, ti.w_row, kEvictFirst);
        if (DUAL) tma_load_2d(st + kATileBytes, &tmap_w2, &full_bar[s], kc, ti.w_row, kEvictFirst);
        tma_load_2d(st + kATileBytes * (DUAL ? 2 : 1), &tmap_x, &full_bar[s], kc, ti.row_base, kEvictLast);
      }
    }
  } else {
    // ============================================================== MMA warpgroup, then epilogue (128 threads)
    float acc[2][BN / 2], acc2[2][BN / 2];
    acc_zero<BN>(acc);
    if (DUAL) acc_zero<BN>(acc2);
    mma_mainloop<BN, DUAL, STAGES, STAGE_BYTES, kATileBytes * (DUAL ? 2 : 1)>(
        acc, acc2, smem, empty_bar, 0u, num_kb, [&](uint32_t s, uint32_t ph) { mbar_wait(&full_bar[s], ph); });
    named_bar_sync(1, kEpiThreads);  // every warp's MMAs are done: the ring is idle
    acc_store_smem<BN>(acc, acc_smem, 0);
    if (DUAL) acc_store_smem<BN>(acc2, acc_smem, BN);
    named_bar_sync(1, kEpiThreads);
    if (!pdl_early) pdl_wait();  // residual / split-K workspace / out are ordered after the predecessor
    if (!p.cluster_splitk)
      gemm::run_epilogue<BN, DUAL, OutT>(p, acc_smem, stg, flag_smem, ti, sk.split);
  }
  if (p.cluster_splitk) {
    // split-K through DSMEM: the `splits` CTAs of this output tile are one cluster (gemm_cluster.cuh); phase A is the
    // accumulator store above
    __syncwarp();
    gemm::cluster_sync_all();
    if (warp < 4) gemm::cluster_epilogue_reduce_store<BN, DUAL, OutT>(p, smem, ti);
    __syncwarp();
    gemm::cluster_sync_all();
    gemm::cluster_signal(p);
  }
}

// ================================================================================================ host side
namespace {

template <int BN, bool DUAL, typename OutT>
cudaError_t launch_one(const GemmMaps& t, const GemmParams& p, const GemmPlan& plan, cudaStream_t stream) {
  constexpr int STAGES = num_stages(BN, DUAL, sizeof(OutT));
  constexpr int smem = STAGES * stage_bytes(BN, DUAL) + 2 * STAGES * 8 + 16 + 1024;
  static_assert(smem <= 227 * 1024, "shared memory budget exceeded");
  constexpr auto kern = gemm_swapab_kernel<BN, DUAL, OutT>;
  cudaError_t e = set_max_dynamic_smem_once<kern>(smem);
  if (e != cudaSuccess) return e;
  (void)launch_pdl_cluster(kern, plan.grid, dim3(kNumThreads), smem, stream, plan.cluster_z, t.w, t.w2, t.x, p);
  return cudaGetLastError();
}

}  // namespace

cudaError_t gemm_launch(const GemmArgs& a, const GemmPlan& plan, cudaStream_t stream) {
  if (plan.route == kRoutePersistent) return gemm_persistent_launch(a, plan, stream);
  const bool dual = a.w2 != nullptr;
  if (a.expert_offsets != nullptr && (a.n % kTileM) != 0) return cudaErrorInvalidValue;
  if ((a.k % 8) != 0 || (a.n % 8) != 0) return cudaErrorInvalidValue;
  if (plan.route == kRouteWorkspaceSplitK && (a.workspace == nullptr || a.tile_counters == nullptr)) return cudaErrorInvalidValue;
  if (dual && a.out_fp32) return cudaErrorInvalidValue;

  GemmMaps t;
  if (!gemm_maps(a, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, plan.bn, &t)) return cudaErrorUnknown;
  const GemmParams p = gemm_params(a, plan);
  return dispatch_tile<kMaxBN, kMaxBNDual>(plan.bn, dual, a.out_fp32, [&](auto c) {
    using C = decltype(c);
    return launch_one<C::BN, C::DUAL, typename C::OutT>(t, p, plan, stream);
  });
}

}  // namespace b200
