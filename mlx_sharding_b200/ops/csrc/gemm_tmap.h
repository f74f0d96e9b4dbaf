// TMA descriptors (cuTensorMapEncodeTiled, looked up once through the runtime) and the descriptor cache of the GEMMs
// (gemm_host.cu).
#pragma once
#include <cuda.h>
#include <stdint.h>

namespace b200 {

// Every input of one cuTensorMapEncodeTiled call (no interleave, element strides 1, no OOB fill).
struct TmapSpec {
  const void* ptr = nullptr;
  CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  uint32_t rank = 2;
  uint64_t dims[3] = {1, 1, 1};     // elements, innermost first
  uint64_t strides[2] = {0, 0};     // bytes, of dims 1 .. rank - 1
  uint32_t box[3] = {1, 1, 1};      // elements, innermost first
  CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B;
  CUtensorMapL2promotion l2 = CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
};

// Encodes on every call (descriptors of per-call buffers).
bool tmap_encode(CUtensorMap* m, const TmapSpec& s);
// Encodes once per distinct spec: weights and the static activation buffers of graph-captured steps hit the cache, which saves
// a few microseconds of host time per launch.
bool tmap_cached(CUtensorMap* m, const TmapSpec& s);

// GEMM operand: row-major [rows, cols] with a row stride of ld elements, in boxes of box_rows rows x 128 bytes (one 128B
// swizzle row: 64 bf16 or 128 one-byte elements).  Cached.
bool gemm_tmap(CUtensorMap* m, CUtensorMapDataType dtype, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld,
               uint32_t box_rows);

// Weight (w, w2: 128-row boxes; w2 = w without a pair) and token (x_box_rows-row boxes) maps of a bf16 or MXFP8 launch.
struct GemmArgs;
struct GemmMaps { CUtensorMap w, w2, x; };
bool gemm_maps(const GemmArgs& a, CUtensorMapDataType dtype, uint32_t x_box_rows, GemmMaps* t);

}  // namespace b200
