// Expert-parallel MoE all-to-all over NVSwitch peer memory (SURVEY §2.4 "EP", §2.6 K11-EP, BASELINE config 5).
//
// The reference keeps all 64 routed experts of a layer on one stage (`mx.gather_qmm`); there is no
// collective anywhere in it.  Here the experts of every MoE layer can be sharded across the ranks of one
// NVSwitch domain and the token exchange is done by our own kernels — no NCCL call, no host hop.  One step is four launches:
//
//   dispatch  : every (token, k) pair reserves a row of its expert's segment in the owner's expert-major receive buffer with one
//               system-scope atomic, writes its token row there (peer memory, 16 B stores) together with the address its output
//               returns to; the last CTA publishes the step's sequence number to every destination with st.release.sys
//               (ep_dispatch.cuh).  This kernel, or the router with the dispatch folded in (moe.cu, EpDispatch).
//   gate/up   : the destination's grouped GEMM acquires every source's sequence number before it reads the rows and row counts
//               (gemm_persistent.cu, GemmParams::ep_arrive).
//   down      : the grouped down-projection's epilogue stores each fp32 output row straight to its return address and the CTA
//               completing the grid bumps every source's return flag (GemmParams::row_dst / signal_peers).
//   combine   : the source waits (in-kernel) for all W returns, then does the weighted combine (+ residual, + the next norm).
//
// Every wait is a bounded spin (ptx.cuh spin_acquire, wait_timeout_ns).  Sequence numbers / counting flags + device-resident
// expectations make every step CUDA-graph replay safe.  Buffer reuse is race-free by construction: a source only dispatches layer
// l+1 after it has combined layer l, which requires every destination to have consumed layer l and returned its rows.
#include "ep_dispatch.cuh"
#include "kernels.h"
#include "launch.h"
#include "ptx.cuh"

namespace b200 {

namespace {

// ---------------------------------------------------------------------------------------------- dispatch
// One warp per (token, k) pair: reserve its row on the owner, copy the token row there, then the step's publication.
__global__ void ep_dispatch_scatter_kernel(const __nv_bfloat16* __restrict__ x, long long ld_x, const int* __restrict__ idx, int npairs,
                                           int top_k, int H, const EpDispatch ep) {
  pdl_sync();
  const int warps_per_cta = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nvec = H / 8;
  const uint32_t seq = *reinterpret_cast<const volatile uint32_t*>(ep.send_seq) + 1u;   // this step (bumped by the last CTA)
  for (int p = blockIdx.x * warps_per_cta + warp; p < npairs; p += gridDim.x * warps_per_cta) {
    const int e = idx[p];
    const int dst = e / ep.experts_per_rank, le = e - dst * ep.experts_per_rank;
    int row = 0;
    if (lane == 0) row = ep_reserve_row(ep, seq, dst, le, (unsigned long long)p, H);
    row = __shfl_sync(0xffffffffu, row, 0);
    if (row >= 0) {
      const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)(p / top_k) * ld_x);
      uint4* drow = reinterpret_cast<uint4*>(ep.recv_x.p[dst]) + (size_t)row * nvec;
      for (int v = lane; v < nvec; v += 32) drow[v] = src[v];
    }
  }
  ep_publish(ep, seq);
}

// ---------------------------------------------------------------------------------------------- combine
// (the return all-to-all itself is the epilogue of the grouped down-projection: gemm_persistent.cu, GemmParams::row_dst)
// Source side: thread 0 waits until every rank's down-projection has stored its share of my pairs into my return buffer and bumped
// my flag.  `expected` was advanced by this step's dispatch (stream order).  The caller syncs the CTA before reading the rows.
__device__ __forceinline__ void wait_returns(const uint32_t* flag, const uint32_t* expected_ptr, uint32_t* error_flag,
                                             unsigned long long timeout_ns) {
  if (threadIdx.x == 0) {
    const uint32_t expected = *reinterpret_cast<const volatile uint32_t*>(expected_ptr);
    spin_acquire([&] { return (int32_t)(ld_acquire_sys(flag) - expected) >= 0; }, globaltimer_ns(), timeout_ns, error_flag);
    __threadfence_system();
  }
}

// Features 8v .. 8v+7 of token t: the returned rows of its top_k pairs weighted by w_row[k], summed in k order (+ residual), to bf16.
// Four pairs' loads are in flight before any is used.
__device__ __forceinline__ uint4 combine_chunk(const float* __restrict__ ret_y, const float* w_row, const __nv_bfloat16* __restrict__ residual,
                                               long long ld_res, int t, int top_k, int H, int v) {
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int k0 = 0; k0 < top_k; k0 += 4) {
    float4 a[4], b[4];
    float w[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int k = k0 + u < top_k ? k0 + u : top_k - 1;
      w[u] = k0 + u < top_k ? w_row[k] : 0.f;
      const float4* src = reinterpret_cast<const float4*>(ret_y + ((size_t)t * top_k + k) * H + v * 8);
      a[u] = __ldcv(src); b[u] = __ldcv(src + 1);   // rows were written by peers: never from a stale L1 line
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (k0 + u < top_k) {
        acc[0] += w[u] * a[u].x; acc[1] += w[u] * a[u].y; acc[2] += w[u] * a[u].z; acc[3] += w[u] * a[u].w;
        acc[4] += w[u] * b[u].x; acc[5] += w[u] * b[u].y; acc[6] += w[u] * b[u].z; acc[7] += w[u] * b[u].w;
      }
    }
  }
  if (residual != nullptr) {
    const uint4 r = reinterpret_cast<const uint4*>(residual + (size_t)t * ld_res)[v];
    const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc[2 * j] += bf16_lo(rr[j]); acc[2 * j + 1] += bf16_hi(rr[j]); }
  }
  return make_uint4(pack_bf16(acc[0], acc[1]), pack_bf16(acc[2], acc[3]), pack_bf16(acc[4], acc[5]), pack_bf16(acc[6], acc[7]));
}

// one thread per 8 features of a token
__global__ void ep_combine_kernel(const uint32_t* flag, const uint32_t* __restrict__ expected_ptr, uint32_t* error_flag,
                                  unsigned long long timeout_ns, const float* __restrict__ ret_y, const float* __restrict__ wts,
                                  const __nv_bfloat16* __restrict__ residual, long long ld_res, __nv_bfloat16* __restrict__ out,
                                  long long ld_out, int T, int top_k, int H) {
  pdl_sync();
  wait_returns(flag, expected_ptr, error_flag, timeout_ns);
  __syncthreads();
  const int nvec = H / 8;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)T * nvec) return;
  const int v = i % nvec;
  const int t = i / nvec;
  reinterpret_cast<uint4*>(out + (size_t)t * ld_out)[v] = combine_chunk(ret_y, wts + (size_t)t * top_k, residual, ld_res, t, top_k, H, v);
}

// Combine + the next layer's input RMSNorm (one CTA per token; same fusion as moe_combine_norm_kernel for the local MoE block)
constexpr int kEpCombThreads = 256;
constexpr int kEpCombMaxV = 4;   // H <= 8192
__global__ void __launch_bounds__(kEpCombThreads)
ep_combine_norm_kernel(const uint32_t* flag, const uint32_t* __restrict__ expected_ptr, uint32_t* error_flag, unsigned long long timeout_ns,
                       const float* __restrict__ ret_y, const float* __restrict__ wts, const __nv_bfloat16* __restrict__ residual,
                       long long ld_res, __nv_bfloat16* __restrict__ out, long long ld_out, int top_k, int H,
                       const __nv_bfloat16* __restrict__ norm_w, float norm_eps, __nv_bfloat16* __restrict__ normed, long long ld_normed) {
  pdl_sync();
  wait_returns(flag, expected_ptr, error_flag, timeout_ns);
  __shared__ float s_w[32];
  __shared__ float red[kEpCombThreads / 32];
  const int t = blockIdx.x;
  if (threadIdx.x < top_k) s_w[threadIdx.x] = wts[(size_t)t * top_k + threadIdx.x];
  __syncthreads();
  const int nvec = H / 8;
  uint4 keep[kEpCombMaxV];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < kEpCombMaxV; ++i) {
    const int v = threadIdx.x + i * kEpCombThreads;
    if (v < nvec) {
      const uint4 o = combine_chunk(ret_y, s_w, residual, ld_res, t, top_k, H, v);
      reinterpret_cast<uint4*>(out + (size_t)t * ld_out)[v] = o;
      keep[i] = o;
      const uint32_t oo[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) { const float a = bf16_lo(oo[j]), b = bf16_hi(oo[j]); ss += a * a + b * b; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < kEpCombThreads / 32; ++i) tot += red[i];
  const float inv = rsqrtf(tot / (float)H + norm_eps);
#pragma unroll
  for (int i = 0; i < kEpCombMaxV; ++i) {
    const int v = threadIdx.x + i * kEpCombThreads;
    if (v < nvec) {
      const uint4 g = __ldg(reinterpret_cast<const uint4*>(norm_w) + v);
      const uint32_t oo[4] = {keep[i].x, keep[i].y, keep[i].z, keep[i].w}, gg[4] = {g.x, g.y, g.z, g.w};
      uint32_t n[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) n[j] = pack_bf16(bf16_lo(oo[j]) * inv * bf16_lo(gg[j]), bf16_hi(oo[j]) * inv * bf16_hi(gg[j]));
      reinterpret_cast<uint4*>(normed + (size_t)t * ld_normed)[v] = make_uint4(n[0], n[1], n[2], n[3]);
    }
  }
}

}  // namespace

cudaError_t ep_dispatch_scatter_launch(const void* x, long long ld_x, const int* idx, int npairs, int top_k, int H, const EpDispatch& ep,
                                       cudaStream_t s) {
  if (ep.world > kEpMaxWorld || (H % 8)) return cudaErrorInvalidValue;
  int grid = (npairs + 7) / 8;
  if (grid < 1) grid = 1;
  if (grid > 592) grid = 592;
  (void)launch_pdl(ep_dispatch_scatter_kernel, dim3(grid), dim3(256), 0, s, static_cast<const __nv_bfloat16*>(x), ld_x, idx, npairs, top_k, H,
                   ep);
  return cudaGetLastError();
}

cudaError_t ep_combine_launch(const uint32_t* flag, const uint32_t* expected_ptr, uint32_t* error_flag, const float* ret_y,
                              const float* wts, const void* residual, long long ld_res, void* out, long long ld_out, int T, int top_k,
                              int H, cudaStream_t s, const void* norm_w, float norm_eps, void* normed, long long ld_normed) {
  if (T == 0) return cudaSuccess;
  if (H % 8) return cudaErrorInvalidValue;
  if (norm_w != nullptr) {
    if (normed == nullptr || top_k > 32 || H > kEpCombThreads * 8 * kEpCombMaxV) return cudaErrorInvalidValue;
    (void)launch_pdl(ep_combine_norm_kernel, dim3(T), dim3(kEpCombThreads), 0, s, flag, expected_ptr, error_flag, wait_timeout_ns(), ret_y, wts,
                     static_cast<const __nv_bfloat16*>(residual), ld_res, static_cast<__nv_bfloat16*>(out), ld_out, top_k, H,
                     static_cast<const __nv_bfloat16*>(norm_w), norm_eps, static_cast<__nv_bfloat16*>(normed), ld_normed);
    return cudaGetLastError();
  }
  const long long total = (long long)T * (H / 8);
  (void)launch_pdl(ep_combine_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, flag, expected_ptr, error_flag, wait_timeout_ns(),
                   ret_y, wts, static_cast<const __nv_bfloat16*>(residual), ld_res, static_cast<__nv_bfloat16*>(out), ld_out, T, top_k, H);
  return cudaGetLastError();
}

}  // namespace b200
