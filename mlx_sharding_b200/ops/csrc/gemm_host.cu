// Host code shared by the GEMM launchers: the route planner, the kernel-parameter builder, the SM count and the TMA
// descriptor factory with its cache (also used by mla_decode.cu).  No kernels.
#include <algorithm>
#include <array>
#include <mutex>
#include <unordered_map>

#include "gemm_common.cuh"
#include "gemm_tmap.h"

namespace b200 {

using namespace gemm;

// ================================================================================================ route planner
namespace {

int pick_bn(long long rows) {
  if (rows <= 16) return 16;
  if (rows <= 32) return 32;
  if (rows <= 64) return 64;
  return kMaxBN;
}

// Decode batches: fill ~one wave of SMs with split-K while keeping >= 8 k-blocks per split.
int auto_splits(int tiles_n, int kb, int sms) {
  int s = 1;
  while (tiles_n * (s * 2) <= sms && kb / (s * 2) >= 8 && s < 4) s *= 2;
  return s;
}

}  // namespace

GemmPlan gemm_plan(const GemmArgs& a, GemmKind kind, int sms) {
  const bool dual = a.w2 != nullptr;
  const int experts = a.num_experts > 0 ? a.num_experts : 1;
  GemmPlan pl;
  // Grouped (MoE) token tile: ~2x the average rows per expert but never below 64, so an expert's rows rarely need a second
  // tile; experts with more rows take further tiles of the persistent tile list.
  pl.bn = a.num_experts > 0 && a.expected_rows > 0
              ? pick_bn(std::min<long long>(a.max_rows, std::max<long long>(64, 2 * ((a.expected_rows + experts - 1) / experts))))
              : pick_bn(a.max_rows);
  // the register accumulators bound the token tile
  if (kind == kGemmFp8) pl.bn = std::min(pl.bn, dual ? kFp8MaxBNDual : kFp8MaxBN);
  else pl.bn = std::min(pl.bn, dual ? kMaxBNDual : kMaxBN);
  pl.tiles_n = (a.n + kTileM - 1) / kTileM;
  pl.tiles_m = (a.max_rows + pl.bn - 1) / pl.bn;
  pl.num_tiles = pl.tiles_n * pl.tiles_m * experts;

  // Split-K for small dense batches only.  Quantised weights stream 3.5x fewer bytes per tile, so their batches above 32
  // rows run un-split on the persistent kernel.  MXFP8 has no split-K kernel.
  const int kb = (a.k + kBlockK - 1) / kBlockK;
  if (kind != kGemmFp8) {
    if (a.splits > 0) pl.splits = a.splits;
    else if (a.num_experts == 0 && a.max_rows <= (kind == kGemmQuant ? 32 : 256)) pl.splits = auto_splits(pl.tiles_n, kb, sms);
    pl.splits = std::min(pl.splits, kb);
  }

  if (pl.splits == 1) {
    pl.route = kRoutePersistent;
    pl.grid = dim3(std::min(pl.num_tiles, sms));
    return pl;
  }
  pl.grid = dim3(pl.tiles_n, experts, pl.tiles_m * pl.splits);
  // DSMEM reduction when the fp32 partial tile fits the idle stage ring and the cluster is portable (<= 8 CTAs)
  if (kind == kGemmBf16 && pl.splits <= 8 && pl.bn * (dual ? 2 : 1) <= 128) {
    pl.route = kRouteClusterSplitK;
    pl.cluster_z = pl.splits;
    return pl;
  }
  pl.route = kRouteWorkspaceSplitK;
  pl.workspace_floats = (size_t)pl.tiles_n * experts * pl.tiles_m * pl.splits * pl.bn * (dual ? 2 : 1) * kTileM;
  return pl;
}

GemmParams gemm_params(const GemmArgs& a, const GemmPlan& plan) {
  GemmParams p{};
  p.m = a.m; p.n = a.n; p.k = a.k; p.splits = plan.splits;
  p.cluster_splitk = plan.route == kRouteClusterSplitK ? 1 : 0;
  p.expert_offsets = a.expert_offsets;
  p.expert_stride = a.expert_stride;
  p.out = a.out; p.ld_out = a.ld_out;
  p.residual = static_cast<const __nv_bfloat16*>(a.residual); p.ld_res = a.ld_res;
  p.bias = static_cast<const __nv_bfloat16*>(a.bias); p.act = a.act; p.softcap = a.softcap;
  if (plan.route == kRouteWorkspaceSplitK) { p.workspace = a.workspace; p.tile_counters = a.tile_counters; }
  p.signal_flag = a.signal_flag; p.signal_value = a.signal_value; p.done_counter = a.done_counter;
  // tiles that tick done_counter before signal_flag is raised (fused stage boundary of a dense launch)
  p.signal_tiles = static_cast<unsigned int>(plan.tiles_n * plan.tiles_m);
  return p;
}

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// ================================================================================================ tensor maps
namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
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

using TmapKey = std::array<uint64_t, 13>;
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    size_t h = 0;
    for (uint64_t v : k) h ^= std::hash<uint64_t>()(v) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    return h;
  }
};
std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmap_cache;
std::mutex g_tmap_mutex;

}  // namespace

bool tmap_encode(CUtensorMap* m, const TmapSpec& s) {
  EncodeTiledFn fn = encode_fn();
  if (fn == nullptr) return false;
  const cuuint32_t estr[3] = {1, 1, 1};
  return fn(m, s.dtype, s.rank, const_cast<void*>(s.ptr), s.dims, s.strides, s.box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, s.swizzle,
            s.l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

bool tmap_cached(CUtensorMap* m, const TmapSpec& s) {
  const TmapKey key{reinterpret_cast<uint64_t>(s.ptr), (uint64_t)s.dtype, s.rank, s.dims[0], s.dims[1], s.dims[2],
                    s.strides[0], s.strides[1], s.box[0], s.box[1], s.box[2], (uint64_t)s.swizzle, (uint64_t)s.l2};
  std::lock_guard<std::mutex> lock(g_tmap_mutex);
  auto it = g_tmap_cache.find(key);
  if (it != g_tmap_cache.end()) { *m = it->second; return true; }
  if (!tmap_encode(m, s)) return false;
  if (g_tmap_cache.size() > 16384) g_tmap_cache.clear();
  g_tmap_cache.emplace(key, *m);
  return true;
}

bool gemm_tmap(CUtensorMap* m, CUtensorMapDataType dtype, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld,
               uint32_t box_rows) {
  const uint32_t elem_bytes = dtype == CU_TENSOR_MAP_DATA_TYPE_UINT8 ? 1 : 2;   // e4m3 or bf16
  TmapSpec s;
  s.ptr = ptr;
  s.dtype = dtype;
  s.dims[0] = cols; s.dims[1] = rows;
  s.strides[0] = ld * elem_bytes;
  s.box[0] = 128 / elem_bytes; s.box[1] = box_rows;
  return tmap_cached(m, s);
}

bool gemm_maps(const GemmArgs& a, CUtensorMapDataType dtype, uint32_t x_box_rows, GemmMaps* t) {
  const uint64_t w_rows = static_cast<uint64_t>(a.n) * (a.expert_offsets != nullptr ? a.num_experts : 1);
  if (!gemm_tmap(&t->w, dtype, a.w, w_rows, a.k, a.ld_w, kTileM)) return false;
  if (a.w2 == nullptr) t->w2 = t->w;
  else if (!gemm_tmap(&t->w2, dtype, a.w2, w_rows, a.k, a.ld_w, kTileM)) return false;
  return gemm_tmap(&t->x, dtype, a.x, a.x_rows, a.k, a.ld_x, x_box_rows);
}

}  // namespace b200
