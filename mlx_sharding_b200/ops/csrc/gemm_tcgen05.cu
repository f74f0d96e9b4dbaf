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
#include "gemm_tcgen05.h"

#include <algorithm>
#include <mutex>
#include <unordered_map>

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
  const int n0 = blockIdx.x * kTileM;
  const int expert = blockIdx.y;
  const int split = blockIdx.z % p.splits;
  const int mt = blockIdx.z / p.splits;
  int row_base = 0, rows_valid = p.m;
  if (p.expert_offsets != nullptr) {
    if (p.expert_stride > 0) {
      row_base = expert * p.expert_stride;
      rows_valid = __ldcg(p.expert_offsets + expert);
    } else {
      const int lo = p.expert_offsets[expert], hi = p.expert_offsets[expert + 1];
      row_base = lo;
      rows_valid = hi - lo;
    }
  }
  rows_valid -= mt * BN;
  row_base += mt * BN;
  if (rows_valid <= 0) return;  // uniform across the CTA
  if (rows_valid > BN) rows_valid = BN;
  const int w_row = expert * p.n + n0;

  const int kb_total = (p.k + kBlockK - 1) / kBlockK;
  const int kb_per = (kb_total + p.splits - 1) / p.splits;
  const int kb_begin = split * kb_per;
  int kb_end = kb_begin + kb_per;
  if (kb_end > kb_total) kb_end = kb_total;
  const int num_kb = kb_end - kb_begin;  // may be 0 for a trailing split: contributes zeros

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
        tma_load_2d(st, &tmap_w, &full_bar[i], kc, w_row, kEvictFirst);
        if (DUAL) tma_load_2d(st + kATileBytes, &tmap_w2, &full_bar[i], kc, w_row, kEvictFirst);
      }
      if (!pdl_early) pdl_wait();
      for (int i = 0; i < pre; ++i)
        tma_load_2d(smem + i * STAGE_BYTES + kATileBytes * (DUAL ? 2 : 1), &tmap_x, &full_bar[i], (kb_begin + i) * kBlockK, row_base, kEvictLast);
      for (int i = pre; i < num_kb; ++i) {
        const int s = i % STAGES;
        const uint32_t ph = (i / STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* st = smem + s * STAGE_BYTES;
        const int kc = (kb_begin + i) * kBlockK;
        mbar_arrive_expect_tx(&full_bar[s], STAGE_BYTES);
        // weights are streamed exactly once per launch: evict-first; activations are re-read by every
        // feature tile: evict-last
        tma_load_2d(st, &tmap_w, &full_bar[s], kc, w_row, kEvictFirst);
        if (DUAL) tma_load_2d(st + kATileBytes, &tmap_w2, &full_bar[s], kc, w_row, kEvictFirst);
        tma_load_2d(st + kATileBytes * (DUAL ? 2 : 1), &tmap_x, &full_bar[s], kc, row_base, kEvictLast);
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
      gemm::run_epilogue<BN, DUAL, OutT>(p, acc_smem, stg, flag_smem, 0, n0, mt, split, row_base, rows_valid);
  }
  if (p.cluster_splitk) {
    // split-K through DSMEM: the `splits` CTAs of this output tile are one cluster (gemm_cluster.cuh); phase A is the
    // accumulator store above
    __syncwarp();
    gemm::cluster_sync_all();
    if (warp < 4) gemm::cluster_epilogue_reduce_store<BN, DUAL, OutT>(p, smem, 0, n0, row_base, rows_valid);
    __syncwarp();
    gemm::cluster_sync_all();
    gemm::cluster_signal(p, 0);
  }
}

// ================================================================================================ host side
namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || ptr == nullptr) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// Descriptor cache: encoding a tensor map costs a few microseconds of host time; weights (and the static
// activation buffers of graph-captured steps) are encoded once.
struct TmapKey {
  const void* ptr; uint64_t rows, cols, ld; uint32_t box;
  bool operator==(const TmapKey& o) const { return ptr == o.ptr && rows == o.rows && cols == o.cols && ld == o.ld && box == o.box; }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    h ^= std::hash<uint64_t>()(k.rows * 1000003ull + k.cols) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    h ^= std::hash<uint64_t>()(k.ld * 31ull + k.box) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    return h;
  }
};
std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmap_cache;
std::mutex g_tmap_mutex;

bool encode_tmap(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows);

// bf16 row-major [rows, cols] (row stride ld elements) -> tiles of box_rows x 64 with 128B swizzle
bool make_tmap(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  const TmapKey key{ptr, rows, cols, ld, box_rows};
  std::lock_guard<std::mutex> lock(g_tmap_mutex);
  auto it = g_tmap_cache.find(key);
  if (it != g_tmap_cache.end()) { *m = it->second; return true; }
  if (!encode_tmap(m, ptr, rows, cols, ld, box_rows)) return false;
  if (g_tmap_cache.size() > 16384) g_tmap_cache.clear();
  g_tmap_cache.emplace(key, *m);
  return true;
}

bool encode_tmap(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return false;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {kBlockK, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

template <int BN, bool DUAL, typename OutT>
cudaError_t launch_one(const GemmArgs& a, const CUtensorMap& tw, const CUtensorMap& tw2, const CUtensorMap& tx,
                       const GemmParams& p, dim3 grid, cudaStream_t stream) {
  constexpr int STAGES = num_stages(BN, DUAL, sizeof(OutT));
  constexpr int smem = STAGES * stage_bytes(BN, DUAL) + 2 * STAGES * 8 + 16 + 1024;
  static_assert(smem <= 227 * 1024, "shared memory budget exceeded");
  auto kern = gemm_swapab_kernel<BN, DUAL, OutT>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  (void)launch_pdl_cluster(kern, dim3(grid), dim3(kNumThreads), smem, stream, p.cluster_splitk ? (unsigned)p.splits : 1u, tw, tw2, tx, p);
  return cudaGetLastError();
}

template <bool DUAL, typename OutT>
cudaError_t dispatch_bn(int bn, const GemmArgs& a, const CUtensorMap& tw, const CUtensorMap& tw2, const CUtensorMap& tx,
                        const GemmParams& p, dim3 grid, cudaStream_t s) {
  switch (bn) {
    case 16: return launch_one<16, DUAL, OutT>(a, tw, tw2, tx, p, grid, s);
    case 32: return launch_one<32, DUAL, OutT>(a, tw, tw2, tx, p, grid, s);
    case 64: return launch_one<64, DUAL, OutT>(a, tw, tw2, tx, p, grid, s);
    case 128:
      if constexpr (!DUAL) return launch_one<128, DUAL, OutT>(a, tw, tw2, tx, p, grid, s);
      return cudaErrorInvalidValue;
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

bool gemm_make_tmap(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  return make_tmap(m, ptr, rows, cols, ld, box_rows);
}

bool gemm_make_tmap_u8(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  // same cache, keyed with the top bit of the box to keep bf16 and byte maps of one pointer apart
  const TmapKey key{ptr, rows, cols, ld, box_rows | 0x80000000u};
  std::lock_guard<std::mutex> lock(g_tmap_mutex);
  auto it = g_tmap_cache.find(key);
  if (it != g_tmap_cache.end()) { *m = it->second; return true; }
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return false;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld};
  cuuint32_t box[2] = {128, box_rows};
  cuuint32_t estr[2] = {1, 1};
  if (fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return false;
  if (g_tmap_cache.size() > 16384) g_tmap_cache.clear();
  g_tmap_cache.emplace(key, *m);
  return true;
}

int gemm_pick_bn(int max_rows) {
  if (max_rows <= 16) return 16;
  if (max_rows <= 32) return 32;
  if (max_rows <= 64) return 64;
  return kMaxBN;
}

int gemm_clamp_bn(int bn, bool dual) { return std::min(bn, dual ? kMaxBNDual : kMaxBN); }

size_t gemm_workspace_floats(const GemmArgs& a, int bn, int splits) {
  if (splits <= 1) return 0;
  const size_t tiles_n = (a.n + kTileM - 1) / kTileM;
  const size_t tiles_m = (a.max_rows + bn - 1) / bn;
  return tiles_n * (a.num_experts > 0 ? a.num_experts : 1) * tiles_m * splits * (size_t)bn * (a.w2 ? 2 : 1) * kTileM;
}

cudaError_t gemm_launch(const GemmArgs& a, cudaStream_t stream) {
  const bool dual = a.w2 != nullptr;
  const bool grouped = a.expert_offsets != nullptr;
  const int bn = gemm_clamp_bn(a.bn > 0 ? a.bn : gemm_pick_bn(a.max_rows), dual);
  int splits = a.splits > 0 ? a.splits : 1;
  const int kb_total = (a.k + kBlockK - 1) / kBlockK;
  if (splits > kb_total) splits = kb_total;
  if (splits == 1 && a.persistent) return gemm_persistent_launch(a, stream);  // no split-K: persistent tile loop
  if (grouped && (a.n % kTileM) != 0) return cudaErrorInvalidValue;
  if ((a.k % 8) != 0 || (a.n % 8) != 0) return cudaErrorInvalidValue;
  if (splits > 1 && !a.cluster_splitk && (a.workspace == nullptr || a.tile_counters == nullptr)) return cudaErrorInvalidValue;
  if (dual && a.out_fp32) return cudaErrorInvalidValue;

  CUtensorMap tw, tw2, tx;
  const uint64_t w_rows = static_cast<uint64_t>(a.n) * (grouped ? a.num_experts : 1);
  if (!make_tmap(&tw, a.w, w_rows, a.k, a.ld_w, kTileM)) return cudaErrorUnknown;
  if (dual) {
    if (!make_tmap(&tw2, a.w2, w_rows, a.k, a.ld_w, kTileM)) return cudaErrorUnknown;
  } else {
    tw2 = tw;
  }
  if (!make_tmap(&tx, a.x, a.x_rows, a.k, a.ld_x, bn)) return cudaErrorUnknown;

  GemmParams p;
  p.row_dst = nullptr; p.signal_peers = nullptr; p.num_signal_peers = 0; p.w_sf = p.w2_sf = p.x_sf = nullptr; p.sf_ld_w = p.sf_ld_x = 0; p.ep_arrive = nullptr; p.ep_seq = nullptr; p.ep_error = nullptr; p.ep_world = 0; p.ep_zero_other = 0;
  p.m = a.m; p.n = a.n; p.k = a.k; p.splits = splits;
  // DSMEM (cluster) split-K when the fp32 partial tile fits the idle stage ring and the cluster is portable
  p.cluster_splitk = (a.cluster_splitk && splits > 1 && splits <= 8 && bn * (dual ? 2 : 1) <= 128) ? 1 : 0;
  p.expert_offsets = a.expert_offsets;
  p.expert_stride = a.expert_stride;
  p.out = a.out; p.ld_out = a.ld_out;
  p.residual = static_cast<const __nv_bfloat16*>(a.residual); p.ld_res = a.ld_res;
  p.bias = static_cast<const __nv_bfloat16*>(a.bias); p.act = a.act; p.softcap = a.softcap;
  p.workspace = a.workspace; p.tile_counters = a.tile_counters;
  p.signal_flag = a.signal_flag; p.signal_value = a.signal_value; p.done_counter = a.done_counter;

  const int tiles_n = (a.n + kTileM - 1) / kTileM;
  const int tiles_m = (a.max_rows + bn - 1) / bn;
  dim3 grid(tiles_n, grouped ? a.num_experts : 1, tiles_m * splits);
  // tiles that run the epilogue (= tiles that will tick done_counter); for grouped launches the caller
  // passes the exact count (empty experts exit early)
  p.signal_tiles = a.signal_tiles > 0 ? a.signal_tiles : static_cast<unsigned int>(tiles_n * tiles_m);

  if (a.out_fp32) return dispatch_bn<false, float>(bn, a, tw, tw2, tx, p, grid, stream);
  if (dual) return dispatch_bn<true, __nv_bfloat16>(bn, a, tw, tw2, tx, p, grid, stream);
  return dispatch_bn<false, __nv_bfloat16>(bn, a, tw, tw2, tx, p, grid, stream);
}

}  // namespace b200
