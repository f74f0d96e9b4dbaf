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
#include <mutex>
#include <unordered_map>

#include "gemm_q_common.cuh"
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
  const int n0 = blockIdx.x * kTileM;
  const int expert = blockIdx.y;
  const int split = blockIdx.z % p.splits;
  const int mt = blockIdx.z / p.splits;
  int row_base = 0, rows_valid = p.m;
  if (p.expert_offsets != nullptr) {
    const int lo = p.expert_offsets[expert], hi = p.expert_offsets[expert + 1];
    row_base = lo;
    rows_valid = hi - lo;
  }
  rows_valid -= mt * BN;
  row_base += mt * BN;
  if (rows_valid <= 0) return;
  if (rows_valid > BN) rows_valid = BN;
  const int w_row = expert * p.n + n0;

  const int kb_total = (p.k + kBlockK - 1) / kBlockK;
  const int kb_per = (kb_total + p.splits - 1) / p.splits;
  const int kb_begin = split * kb_per;
  int kb_end = kb_begin + kb_per;
  if (kb_end > kb_total) kb_end = kb_total;
  const int num_kb = kb_end - kb_begin;

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
        tma_load_2d(st + OFF_PACKED, &tmap_wq, &full_bar[s], kb * (kBlockK * BITS / 32), w_row, kEvictFirst);
        tma_load_2d(st + OFF_SCALE, &tmap_s, &full_bar[s], w_row, gi, kEvictFirst);
        tma_load_2d(st + OFF_SCALE + 256, &tmap_b, &full_bar[s], w_row, gi, kEvictFirst);
        if (DUAL) {
          tma_load_2d(st + OFF_PACKED + PACKED_BYTES, &tmap_wq2, &full_bar[s], kb * (kBlockK * BITS / 32), w_row, kEvictFirst);
          tma_load_2d(st + OFF_SCALE + 512, &tmap_s2, &full_bar[s], w_row, gi, kEvictFirst);
          tma_load_2d(st + OFF_SCALE + 768, &tmap_b2, &full_bar[s], w_row, gi, kEvictFirst);
        }
        tma_load_2d(st + OFF_B, &tmap_x, &full_bar[s], kb * kBlockK, row_base, kEvictLast);
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
    run_epilogue<BN, DUAL, OutT>(p, acc_smem, stg, flag_smem, 0, n0, mt, split, row_base, rows_valid);
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

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn q_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

struct QKey {
  const void* ptr; uint64_t d0, d1, ld; uint32_t b0, b1; int kind;
  bool operator==(const QKey& o) const { return ptr == o.ptr && d0 == o.d0 && d1 == o.d1 && ld == o.ld && b0 == o.b0 && b1 == o.b1 && kind == o.kind; }
};
struct QKeyHash {
  size_t operator()(const QKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    h ^= std::hash<uint64_t>()(k.d0 * 1000003ull + k.d1 * 7919ull + k.ld) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    h ^= std::hash<uint64_t>()(((uint64_t)k.b0 << 32) | (k.b1 * 8u + k.kind)) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    return h;
  }
};
std::unordered_map<QKey, CUtensorMap, QKeyHash> g_qcache;
std::mutex g_qmutex;

// kind 0: bf16 128B-swizzled K-major tile (activations); 1: uint32 packed codes, no swizzle; 2: bf16 row vector, no swizzle
bool q_make_tmap(CUtensorMap* m, int kind, const void* ptr, uint64_t d0, uint64_t d1, uint64_t ld_elems, uint32_t b0, uint32_t b1) {
  const QKey key{ptr, d0, d1, ld_elems, b0, b1, kind};
  std::lock_guard<std::mutex> lock(g_qmutex);
  auto it = g_qcache.find(key);
  if (it != g_qcache.end()) { *m = it->second; return true; }
  EncodeTiledFn fn = q_encode_fn();
  if (fn == nullptr) return false;
  const uint32_t esz = kind == 1 ? 4 : 2;
  cuuint64_t dims[2] = {d0, d1};
  cuuint64_t strides[1] = {ld_elems * esz};
  cuuint32_t box[2] = {b0, b1};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, kind == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims,
                  strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, kind == 0 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return false;
  if (g_qcache.size() > 16384) g_qcache.clear();
  g_qcache.emplace(key, *m);
  return true;
}


template <int BN, bool DUAL, typename OutT, int BITS>
cudaError_t q_launch_one(const QMaps& t, const GemmParams& p, int group_kblocks, dim3 grid, cudaStream_t stream) {
  constexpr int STAGES = q_num_stages(BN, DUAL, BITS, sizeof(OutT));
  constexpr int smem = STAGES * q_stage_bytes(BN, DUAL, BITS) + 3 * STAGES * 8 + 16 + 1024;
  static_assert(smem <= 227 * 1024, "shared memory budget exceeded");
  auto kern = gemm_swapab_q_kernel<BN, DUAL, OutT, BITS>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  (void)launch_pdl(kern, dim3(grid), dim3(kQThreads), smem, stream, t.wq, t.wq2, t.s, t.b, t.s2, t.b2, t.x, p, group_kblocks);
  return cudaGetLastError();
}

template <bool DUAL, typename OutT, int BITS>
cudaError_t q_dispatch_bn(int bn, const QMaps& t, const GemmParams& p, int gk, dim3 grid, cudaStream_t s) {
  switch (bn) {
    case 16: return q_launch_one<16, DUAL, OutT, BITS>(t, p, gk, grid, s);
    case 32: return q_launch_one<32, DUAL, OutT, BITS>(t, p, gk, grid, s);
    case 64: return q_launch_one<64, DUAL, OutT, BITS>(t, p, gk, grid, s);
    case 128:
      if constexpr (!DUAL) return q_launch_one<128, DUAL, OutT, BITS>(t, p, gk, grid, s);
      return cudaErrorInvalidValue;
    default: return cudaErrorInvalidValue;
  }
}

template <int BITS>
cudaError_t q_dispatch(bool dual, bool fp32, int bn, const QMaps& t, const GemmParams& p, int gk, dim3 grid, cudaStream_t s) {
  if (fp32) return q_dispatch_bn<false, float, BITS>(bn, t, p, gk, grid, s);
  if (dual) return q_dispatch_bn<true, __nv_bfloat16, BITS>(bn, t, p, gk, grid, s);
  return q_dispatch_bn<false, __nv_bfloat16, BITS>(bn, t, p, gk, grid, s);
}

}  // namespace

bool gemm_q_make_tmap(CUtensorMap* m, int kind, const void* ptr, uint64_t d0, uint64_t d1, uint64_t ld_elems, uint32_t b0, uint32_t b1) {
  return q_make_tmap(m, kind, ptr, d0, d1, ld_elems, b0, b1);
}

bool gemm_q_supported(int bits, int group, int k) {
  return (bits == 4 || bits == 8) && (group == 64 || group == 128) && (k % 64) == 0 && (k % group) == 0;
}

cudaError_t gemm_q_launch(const GemmArgs& a, cudaStream_t stream) {
  if (!gemm_q_supported(a.q_bits, a.q_group, a.k)) return cudaErrorNotSupported;
  const bool dual = a.w2 != nullptr;
  const bool grouped = a.expert_offsets != nullptr;
  const int bn = gemm_clamp_bn(a.bn > 0 ? a.bn : gemm_pick_bn(a.max_rows), dual);
  int splits = a.splits > 0 ? a.splits : 1;
  if (splits == 1 && a.persistent) return gemm_q_persistent_launch(a, stream);
  const int kb_total = a.k / kBlockK;
  if (splits > kb_total) splits = kb_total;
  if (grouped && (a.n % kTileM) != 0) return cudaErrorInvalidValue;
  if ((a.n % 8) != 0) return cudaErrorInvalidValue;
  if (splits > 1 && (a.workspace == nullptr || a.tile_counters == nullptr)) return cudaErrorInvalidValue;
  if (dual && a.out_fp32) return cudaErrorInvalidValue;

  const uint64_t w_rows = static_cast<uint64_t>(a.n) * (grouped ? a.num_experts : 1);
  const uint64_t words = static_cast<uint64_t>(a.k) * a.q_bits / 32;
  const uint64_t ngroups = a.k / a.q_group;
  QMaps t;
  if (!q_make_tmap(&t.wq, 1, a.w, words, w_rows, words, kBlockK * a.q_bits / 32, kTileM)) return cudaErrorUnknown;
  if (!q_make_tmap(&t.s, 2, a.q_scales_t, w_rows, ngroups, w_rows, kTileM, 1)) return cudaErrorUnknown;
  if (!q_make_tmap(&t.b, 2, a.q_biases_t, w_rows, ngroups, w_rows, kTileM, 1)) return cudaErrorUnknown;
  if (dual) {
    if (!q_make_tmap(&t.wq2, 1, a.w2, words, w_rows, words, kBlockK * a.q_bits / 32, kTileM)) return cudaErrorUnknown;
    if (!q_make_tmap(&t.s2, 2, a.q_scales2_t, w_rows, ngroups, w_rows, kTileM, 1)) return cudaErrorUnknown;
    if (!q_make_tmap(&t.b2, 2, a.q_biases2_t, w_rows, ngroups, w_rows, kTileM, 1)) return cudaErrorUnknown;
  } else {
    t.wq2 = t.wq; t.s2 = t.s; t.b2 = t.b;
  }
  if (!q_make_tmap(&t.x, 0, a.x, a.k, a.x_rows, a.ld_x, kBlockK, bn)) return cudaErrorUnknown;

  GemmParams p;
  p.row_dst = nullptr; p.signal_peers = nullptr; p.num_signal_peers = 0; p.w_sf = p.w2_sf = p.x_sf = nullptr; p.sf_ld_w = p.sf_ld_x = 0; p.ep_arrive = nullptr; p.ep_seq = nullptr; p.ep_error = nullptr; p.ep_world = 0; p.ep_zero_other = 0; p.expert_stride = 0;
  p.m = a.m; p.n = a.n; p.k = a.k; p.splits = splits;
  p.cluster_splitk = 0;
  p.expert_offsets = a.expert_offsets;
  p.out = a.out; p.ld_out = a.ld_out;
  p.residual = static_cast<const __nv_bfloat16*>(a.residual); p.ld_res = a.ld_res;
  p.bias = static_cast<const __nv_bfloat16*>(a.bias); p.act = a.act; p.softcap = a.softcap;
  p.workspace = a.workspace; p.tile_counters = a.tile_counters;
  p.signal_flag = a.signal_flag; p.signal_value = a.signal_value; p.done_counter = a.done_counter;
  const int tiles_n = (a.n + kTileM - 1) / kTileM;
  const int tiles_m = (a.max_rows + bn - 1) / bn;
  dim3 grid(tiles_n, grouped ? a.num_experts : 1, tiles_m * splits);
  p.signal_tiles = a.signal_tiles > 0 ? a.signal_tiles : static_cast<unsigned int>(tiles_n * tiles_m);
  const int gk = a.q_group / kBlockK;  // k-blocks per quantisation group (1 or 2)
  if (a.q_bits == 4) return q_dispatch<4>(dual, a.out_fp32, bn, t, p, gk, grid, stream);
  return q_dispatch<8>(dual, a.out_fp32, bn, t, p, gk, grid, stream);
}

}  // namespace b200
