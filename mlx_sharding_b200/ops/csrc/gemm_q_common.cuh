// Shared pieces of the quantised (MLX affine int4/int8) wgmma GEMMs: the in-register dequantiser and the
// TMA descriptors of packed codes / transposed scale rows.
#pragma once
#include "gemm_common.cuh"

namespace b200 {
namespace gemm {

// One thread dequantises half a row of the k-block: 32 weights = 4 chunks of 8 (chunks 4*half .. 4*half+3).
//
// int4 fast path (2 ALU ops / weight instead of ~5.5): nibbles i and i+4 of a (load-time re-packed) word are isolated together with
// (w >> 4i) & 0x000F000F, OR-ed with 0x4300'4300 they are the bf16 pair (128 + q_i, 128 + q_{i+4}) exactly; one HSUB2
// removes the 128 and one HFMA2.BF16 produces bf16(s*q + b) with a *single* rounding.  int8 keeps the fp32 magic-number path (8-bit codes do not fit the bf16 mantissa).
template <int BITS>
__device__ __forceinline__ void dequant_half_row(const uint8_t* packed_row, float s, float b, uint8_t* a_tile, int r, int half) {
  uint8_t* row = a_tile + r * 128;
  if (BITS == 4) {
    const uint4 v = reinterpret_cast<const uint4*>(packed_row)[half];  // 4 words = 32 codes
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    const __nv_bfloat162 s2 = __float2bfloat162_rn(s), b2 = __float2bfloat162_rn(b);
    uint32_t magic, mask4;  // kept in registers (asm volatile-free movs) so the and-or below stays a single LOP3
    asm("mov.b32 %0, 0x43004300;" : "=r"(magic));
    asm("mov.b32 %0, 0x000F000F;" : "=r"(mask4));
    const __nv_bfloat162 c128 = *reinterpret_cast<const __nv_bfloat162*>(&magic);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      uint32_t x[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        uint32_t m;  // (128 + q_i, 128 + q_{i+4}): one LOP3 ((a & b) | c, LUT 0xEA) with both constants in registers
        asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(m) : "r"(w[c] >> (4 * i)), "r"(mask4), "r"(magic));
        __nv_bfloat162 q = __hsub2(*reinterpret_cast<const __nv_bfloat162*>(&m), c128);
        q = __hfma2(s2, q, b2);
        x[i] = *reinterpret_cast<uint32_t*>(&q);
      }
      uint4 o;
      // the loader re-packs every word so that nibble j holds v_{2j} and nibble 4+j holds v_{2j+1} (same bits, TMA/UMMA
      // friendly order — ops/b200.py::_qpack): the masked pairs come out already in K order, no PRMT needed
      o.x = x[0]; o.y = x[1]; o.z = x[2]; o.w = x[3];
      const int chunk = 4 * half + c;
      // 128B swizzle (Swizzle<3,4,3>): 16-byte chunk index XOR (row mod 8)
      *reinterpret_cast<uint4*>(row + ((chunk ^ (r & 7)) << 4)) = o;
    }
  } else {
    const uint4 v0 = reinterpret_cast<const uint4*>(packed_row)[2 * half], v1 = reinterpret_cast<const uint4*>(packed_row)[2 * half + 1];
    const uint32_t w[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};  // 8 words = 32 codes
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float f[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t x = w[2 * c + (i >> 2)];
        const float q = __uint_as_float(__byte_perm(x, 0x4B000000u, 0x7440u | (i & 3))) - 8388608.0f;
        f[i] = fmaf(s, q, b);
      }
      uint4 o;
      o.x = pack_bf16(f[0], f[1]); o.y = pack_bf16(f[2], f[3]); o.z = pack_bf16(f[4], f[5]); o.w = pack_bf16(f[6], f[7]);
      const int chunk = 4 * half + c;
      *reinterpret_cast<uint4*>(row + ((chunk ^ (r & 7)) << 4)) = o;
    }
  }
}


}  // namespace gemm

// Packed codes, scale and bias rows of each weight (the second set repeats the first without a pair) and the token tile.
struct QMaps { CUtensorMap wq, wq2, s, b, s2, b2, x; };
bool q_maps(const GemmArgs& a, int bn, QMaps* t);
cudaError_t gemm_q_persistent_launch(const GemmArgs& a, const GemmPlan& plan, cudaStream_t stream);

}  // namespace b200
