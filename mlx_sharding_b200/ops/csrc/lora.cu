// LoRA shrink for adapted quantised linears: u[T, R] = x[T, K] A[R, K]^T in fp32 (bf16 inputs).  The quantised GEMM then adds
// u[t, :] . (scale * B)[o, :] in its epilogue (gemm_common.cuh, lora_add16).
//
// One cluster per (8 tokens, 8 adapter rows).  Its `split` CTAs (cluster along z) take interleaved 2048-wide slices of K, so a
// decode-sized launch (T <= 8: R / 8 clusters) still spreads the K loop over up to 8 SMs instead of running it serially.  Within a
// CTA 8 warps split the slice, each lane reads 8 consecutive K values (16 bytes) of every token row and adapter row per step.
// Each warp reduces its partial dot products with shuffles, each CTA sums its 8 warps, and CTA 0 of the cluster sums the CTAs'
// partials through distributed shared memory: every reduction runs in a fixed order (deterministic).  A is R x K bf16 (at most
// a few MB) and stays in L2; x is re-read once per 8 adapter rows.
#include "gemm.h"
#include "gemm_cluster.cuh"
#include "launch.h"

namespace b200 {

namespace {

constexpr int kShrinkToks = 8, kShrinkRows = 8, kShrinkWarps = 8, kShrinkMaxSplit = 8;
constexpr int kShrinkSlice = kShrinkWarps * 256;   // K values one CTA covers per step

__device__ __forceinline__ void unpack8(const uint4 v, float (&f)[8]) {
  f[0] = bf16_lo(v.x); f[1] = bf16_hi(v.x); f[2] = bf16_lo(v.y); f[3] = bf16_hi(v.y);
  f[4] = bf16_lo(v.z); f[5] = bf16_hi(v.z); f[6] = bf16_lo(v.w); f[7] = bf16_hi(v.w);
}

__global__ void __launch_bounds__(kShrinkWarps * 32)
lora_shrink_kernel(const __nv_bfloat16* __restrict__ x, long long ld_x, const __nv_bfloat16* __restrict__ a, int T, int K, int R,
                   float* __restrict__ u) {
  __shared__ float part[kShrinkWarps][kShrinkToks * kShrinkRows];
  __shared__ float cta_sum[kShrinkToks * kShrinkRows];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int split = gridDim.z;
  const int rgroups = R / kShrinkRows;
  const int j0 = (blockIdx.x % rgroups) * kShrinkRows, t0 = (blockIdx.x / rgroups) * kShrinkToks;
  const int nt = min(kShrinkToks, T - t0);
  pdl_launch_dependents();
  pdl_wait();   // x comes from the kernel in front

  float acc[kShrinkToks][kShrinkRows];
#pragma unroll
  for (int t = 0; t < kShrinkToks; ++t)
#pragma unroll
    for (int r = 0; r < kShrinkRows; ++r) acc[t][r] = 0.f;

  for (int k = blockIdx.z * kShrinkSlice + (warp * 32 + lane) * 8; k < K; k += split * kShrinkSlice) {
    float xv[kShrinkToks][8];
#pragma unroll
    for (int t = 0; t < kShrinkToks; ++t) {
      if (t < nt) unpack8(__ldg(reinterpret_cast<const uint4*>(x + static_cast<size_t>(t0 + t) * ld_x + k)), xv[t]);
      else
#pragma unroll
        for (int i = 0; i < 8; ++i) xv[t][i] = 0.f;
    }
#pragma unroll
    for (int r = 0; r < kShrinkRows; ++r) {
      float av[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(a + static_cast<size_t>(j0 + r) * K + k)), av);
#pragma unroll
      for (int t = 0; t < kShrinkToks; ++t)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[t][r] = fmaf(xv[t][i], av[i], acc[t][r]);
    }
  }
  // per-warp butterfly sums, then the 8 warps in a fixed order
#pragma unroll
  for (int t = 0; t < kShrinkToks; ++t)
#pragma unroll
    for (int r = 0; r < kShrinkRows; ++r) {
      float v = acc[t][r];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) part[warp][t * kShrinkRows + r] = v;
    }
  __syncthreads();
  if (threadIdx.x < kShrinkToks * kShrinkRows) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kShrinkWarps; ++w) s += part[w][threadIdx.x];
    cta_sum[threadIdx.x] = s;
  }
  gemm::cluster_sync_all();   // every CTA's partial is in its shared memory
  if (blockIdx.z == 0 && threadIdx.x < kShrinkToks * kShrinkRows) {
    const int t = threadIdx.x / kShrinkRows, r = threadIdx.x % kShrinkRows;
    const uint32_t local = smem_u32(&cta_sum[threadIdx.x]);
    float s = 0.f;
    for (int c = 0; c < split; ++c) s += gemm::ld_dsmem_f32(gemm::mapa_shared(local, c));
    if (t < nt) u[static_cast<size_t>(t0 + t) * R + j0 + r] = s;
  }
  gemm::cluster_sync_all();   // the other CTAs keep their shared memory until CTA 0 has read it
}

}  // namespace

cudaError_t lora_shrink_launch(const void* x, long long ld_x, const void* a, int T, int K, int R, float* u, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (R <= 0 || R % kShrinkRows != 0 || K % 8 != 0 || ld_x % 8 != 0) return cudaErrorInvalidValue;
  const unsigned blocks = static_cast<unsigned>((T + kShrinkToks - 1) / kShrinkToks) * static_cast<unsigned>(R / kShrinkRows);
  // split K over a cluster while the launch would leave SMs idle; prefill-sized launches already fill the GPU
  unsigned split = static_cast<unsigned>((K + kShrinkSlice - 1) / kShrinkSlice);
  split = split > kShrinkMaxSplit ? kShrinkMaxSplit : split;
  if (blocks >= static_cast<unsigned>(sm_count())) split = 1;
  (void)launch_pdl_cluster(lora_shrink_kernel, dim3(blocks, 1, split), dim3(kShrinkWarps * 32), 0, stream, split,
                           static_cast<const __nv_bfloat16*>(x), ld_x, static_cast<const __nv_bfloat16*>(a), T, K, R, u);
  return cudaGetLastError();
}

}  // namespace b200
