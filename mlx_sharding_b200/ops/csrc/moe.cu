// DeepSeek-V2 MoE support kernels (SURVEY §2.6 K10/K11): router (fp32 softmax + greedy / group-limited
// top-k), token permutation for the grouped GEMM, and the weighted combine fused with the residual and
// — on the last layer of a stage — with the P2P hand-off flag.  The reference gets this from
// mlx_lm's MoEGate + SwitchGLU (`mx.gather_qmm`, `(y * scores[..., None]).sum(-2)`); nothing is ported.
#include "ep_dispatch.cuh"
#include "kernels.h"
#include "launch.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kRouteThreads = 256;  // 8 warps
constexpr int kMaxEPerLane = 8;     // E <= 256

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// argmax with lowest-index tie-break
__device__ __forceinline__ void warp_argmax(float& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
  }
}

// TOKS tokens per CTA share every router-weight read: 8 for prefill-sized batches, 1 for decode batches
// (more CTAs; the 256 KB router matrix is L2 resident).
template <int kRouteToks>
__global__ void __launch_bounds__(kRouteToks == 1 ? 1024 : kRouteThreads)
moe_route_kernel(const __nv_bfloat16* __restrict__ x, long long ld_x, const __nv_bfloat16* __restrict__ gw, int T, int H,
                 int E, int top_k, int n_group, int topk_group, float scaling, int norm_topk, int extra, int* __restrict__ idx,
                 float* __restrict__ wts, int* __restrict__ sc_counts, int sc_stride, int* __restrict__ sc_pair_row,
                 __nv_bfloat16* __restrict__ sc_x, const __nv_bfloat16* __restrict__ norm_w, float norm_eps, const EpDispatch ep,
                 __nv_bfloat16* __restrict__ normed_out, long long ld_normed) {
  pdl_sync();  // PDL: predecessor's writes visible; let the successor start its prologue
  // expert-parallel dispatch fused into the router: this step's sequence number (bumped by the last CTA at the very end, after
  // every CTA has read it here)
  const uint32_t ep_seq = ep.enabled ? *reinterpret_cast<const volatile uint32_t*>(ep.send_seq) + 1u : 0u;
  extern __shared__ __align__(16) uint8_t smem[];
  __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(smem);                 // [kRouteToks][H]
  float* logits = reinterpret_cast<float*>(smem + (size_t)kRouteToks * H * 2);  // [kRouteToks][E]
  const int t0 = blockIdx.x * kRouteToks;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nvec = H / 8;
  for (int i = threadIdx.x; i < kRouteToks * nvec; i += blockDim.x) {
    const int tk = i / nvec, v = i % nvec;
    uint4 r = make_uint4(0, 0, 0, 0);
    if (t0 + tk < T) r = reinterpret_cast<const uint4*>(x + (size_t)(t0 + tk) * ld_x)[v];
    reinterpret_cast<uint4*>(xs + (size_t)tk * H)[v] = r;
  }
  __syncthreads();
  if (norm_w != nullptr) {
    // Fused pre-MoE RMSNorm: `x` is the un-normalised residual stream; warp `tk` normalises token `tk` in shared memory (same
    // arithmetic as rmsnorm_kernel: fp32 statistics, x * inv * w rounded to bf16), so the router logits AND the scattered expert
    // inputs below see exactly what a separate norm kernel would have written — without its launch and its HBM round trip.
    if (warp < kRouteToks) {
      uint4* row = reinterpret_cast<uint4*>(xs + (size_t)warp * H);
      float ss = 0.f;
      for (int v = lane; v < nvec; v += 32) {
        const uint4 r = row[v];
        const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float a = bf16_lo(rr[j]), b = bf16_hi(rr[j]); ss += a * a + b * b; }
      }
      ss = warp_sum(ss);
      const float inv = rsqrtf(ss / (float)H + norm_eps);
      for (int v = lane; v < nvec; v += 32) {
        const uint4 r = row[v];
        const uint4 g = __ldg(reinterpret_cast<const uint4*>(norm_w) + v);
        const uint32_t rr[4] = {r.x, r.y, r.z, r.w}, gg[4] = {g.x, g.y, g.z, g.w};
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = pack_bf16(bf16_lo(rr[j]) * inv * bf16_lo(gg[j]), bf16_hi(rr[j]) * inv * bf16_hi(gg[j]));
        row[v] = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
    __syncthreads();
  }
  if (normed_out != nullptr) {
    for (int i = threadIdx.x; i < kRouteToks * nvec; i += blockDim.x) {
      const int tk = i / nvec, v = i % nvec;
      if (t0 + tk < T) reinterpret_cast<uint4*>(normed_out + (size_t)(t0 + tk) * ld_normed)[v] = reinterpret_cast<const uint4*>(xs + (size_t)tk * H)[v];
    }
  }
  for (int e = warp; e < E; e += blockDim.x / 32) {
    float acc[kRouteToks];
#pragma unroll
    for (int k = 0; k < kRouteToks; ++k) acc[k] = 0.f;
    const uint4* wr = reinterpret_cast<const uint4*>(gw + (size_t)e * H);
    // the router row comes from L2: issue 8 independent 16 B loads per lane before using any of them (a plain loop
    // serialises one L2 round trip per iteration — 64 round trips per warp made this kernel 20 us for 64 tokens)
    for (int v0 = lane; v0 < nvec; v0 += 32 * 8) {
      uint4 wbuf[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int v = v0 + 32 * u;
        wbuf[u] = v < nvec ? __ldg(wr + v) : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int v = v0 + 32 * u;
        if (v >= nvec) break;
        const uint32_t ww[4] = {wbuf[u].x, wbuf[u].y, wbuf[u].z, wbuf[u].w};
#pragma unroll
        for (int k = 0; k < kRouteToks; ++k) {
          const uint4 x4 = reinterpret_cast<const uint4*>(xs + (size_t)k * H)[v];
          const uint32_t xx[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            acc[k] += bf16_lo(xx[j]) * bf16_lo(ww[j]);
            acc[k] += bf16_hi(xx[j]) * bf16_hi(ww[j]);
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < kRouteToks; ++k) {
      const float s = warp_sum(acc[k]);
      if (lane == 0) logits[k * E + e] = s;
    }
  }
  __syncthreads();
  // ---- one warp per token: softmax, (group mask), top-k
  const int tk = warp;
  const int t = t0 + tk;
  __shared__ int s_rows[32];
  __shared__ int s_dst[32];
  if (tk < kRouteToks && t < T) {
  float sc[kMaxEPerLane], sel[kMaxEPerLane];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < kMaxEPerLane; ++j) {
    const int e = lane + 32 * j;
    sc[j] = (e < E) ? logits[tk * E + e] : -INFINITY;
    mx = fmaxf(mx, sc[j]);
  }
  mx = warp_max(mx);
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < kMaxEPerLane; ++j) {
    const int e = lane + 32 * j;
    sc[j] = (e < E) ? __expf(sc[j] - mx) : 0.f;
    sum += sc[j];
  }
  sum = warp_sum(sum);
  const float inv = 1.0f / sum;
#pragma unroll
  for (int j = 0; j < kMaxEPerLane; ++j) {
    const int e = lane + 32 * j;
    sc[j] *= inv;
    sel[j] = (e < E) ? sc[j] : -1.0f;
  }
  if (n_group > 1 && topk_group < n_group) {
    const int gsz = E / n_group;
    // group id of each owned expert; choose topk_group groups by their max score
    unsigned chosen = 0u;  // bitmask over groups (n_group <= 32)
    for (int r = 0; r < topk_group; ++r) {
      float best = -1.0f;
      int bg = 0x7fffffff;
#pragma unroll
      for (int j = 0; j < kMaxEPerLane; ++j) {
        const int e = lane + 32 * j;
        if (e < E) {
          const int g = e / gsz;
          if (!((chosen >> g) & 1u) && (sc[j] > best || (sc[j] == best && g < bg))) { best = sc[j]; bg = g; }
        }
      }
      warp_argmax(best, bg);
      chosen |= (1u << bg);
    }
#pragma unroll
    for (int j = 0; j < kMaxEPerLane; ++j) {
      const int e = lane + 32 * j;
      if (e < E && !((chosen >> (e / gsz)) & 1u)) sel[j] = 0.0f;
    }
  }
  float wsum = 0.f;
  float my_w = 0.f;
  int my_i = 0;
  for (int r = 0; r < top_k; ++r) {
    float best = -2.0f;
    int bi = 0x7fffffff;
#pragma unroll
    for (int j = 0; j < kMaxEPerLane; ++j) {
      const int e = lane + 32 * j;
      if (e < E && (sel[j] > best || (sel[j] == best && e < bi))) { best = sel[j]; bi = e; }
    }
    warp_argmax(best, bi);
    // fetch the un-masked score of the winner from its owner lane
    float wv = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxEPerLane; ++j)
      if (lane + 32 * j == bi) { wv = sc[j]; sel[j] = -1.0f; }
    wv = __shfl_sync(0xffffffffu, wv, bi & 31);
    wsum += wv;
    if (lane == r) { my_w = wv; my_i = bi; }
  }
  // `extra` always-on experts (DeepSeek's shared experts appended to the routed bank as experts E .. E+extra-1, weight 1): they
  // ride the same permutation / grouped GEMMs / combine as the routed ones instead of two separate small dense GEMMs
  const int row = top_k + extra;
  if (lane < top_k) {
    const float w = (norm_topk && top_k > 1) ? my_w / (wsum + 1e-20f) : my_w * scaling;
    idx[(size_t)t * row + lane] = my_i;
    wts[(size_t)t * row + lane] = w;
  } else if (lane < row) {
    idx[(size_t)t * row + lane] = E + (lane - top_k);
    wts[(size_t)t * row + lane] = 1.0f;
  }
  // Scatter mode (decode batches, one token per CTA): claim a slot of the expert's fixed-stride segment with one atomic and record
  // the row — the counting sort (`moe_offsets_kernel`) and the gather (`moe_gather_kernel`) are folded into the router.  Slot order
  // within an expert is arbitrary; results do not depend on it (rows are independent GEMM columns, the combine gathers by pair).
  if (sc_counts != nullptr && lane < row) {
    const int e = lane < top_k ? my_i : E + (lane - top_k);
    const int r = e * sc_stride + atomicAdd(&sc_counts[e], 1);
    sc_pair_row[(size_t)t * row + lane] = r;
    s_rows[lane] = r;
  }
  if (kRouteToks == 1 && ep.enabled && lane < top_k) {
    // sender-side slot reservation in the owner's expert-major receive buffer (counters double-buffered by step parity) + the
    // address the owner's down-projection epilogue returns this pair's output row to (my return buffer as mapped by the owner)
    const int dst = my_i / ep.experts_per_rank, le = my_i - dst * ep.experts_per_rank;
    s_rows[lane] = ep_reserve_row(ep, ep_seq, dst, le, (unsigned long long)t * top_k + lane, H);
    s_dst[lane] = dst;
  }
  }
  if (kRouteToks == 1 && sc_counts != nullptr) {
    __syncthreads();
    if (t0 < T) {
      const int row = top_k + extra;
      for (int i = threadIdx.x; i < row * nvec; i += blockDim.x) {
        const int k = i / nvec, v = i % nvec;
        reinterpret_cast<uint4*>(sc_x + (size_t)s_rows[k] * H)[v] = reinterpret_cast<const uint4*>(xs)[v];
      }
    }
  }
  if (kRouteToks == 1 && ep.enabled) {
    __syncthreads();
    if (t0 < T) {
      for (int i = threadIdx.x; i < top_k * nvec; i += blockDim.x) {
        const int k = i / nvec, v = i % nvec;
        if (s_rows[k] >= 0)
          reinterpret_cast<uint4*>(ep.recv_x.p[s_dst[k]])[(size_t)s_rows[k] * nvec + v] = reinterpret_cast<const uint4*>(xs)[v];
      }
    }
    ep_publish(ep, ep_seq);
  }
}

// ------------------------------------------------------------------------------------------------ permutation
__global__ void __launch_bounds__(1024)
moe_offsets_kernel(const int* __restrict__ idx, int npairs, int E, int* __restrict__ expert_offsets,
                   int* __restrict__ pair_row) {
  pdl_sync();  // PDL: predecessor's writes visible; let the successor start its prologue
  __shared__ int cnt[256], cur[256];
  for (int e = threadIdx.x; e < E; e += blockDim.x) cnt[e] = 0;
  __syncthreads();
  for (int p = threadIdx.x; p < npairs; p += blockDim.x) atomicAdd(&cnt[idx[p]], 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int e = 0; e < E; ++e) { cur[e] = acc; expert_offsets[e] = acc; acc += cnt[e]; }
    expert_offsets[E] = acc;
  }
  __syncthreads();
  // Row placement inside an expert's segment is claimed with shared-memory atomics.  The order is arbitrary
  // but results do not depend on it: every permuted row is an independent GEMM column and the combine
  // gathers by (token, k) -> row, so outputs stay bit-identical run to run.
  for (int p = threadIdx.x; p < npairs; p += blockDim.x) pair_row[p] = atomicAdd(&cur[idx[p]], 1);
}

__global__ void moe_gather_kernel(const __nv_bfloat16* __restrict__ x, long long ld_x, const int* __restrict__ pair_row,
                                  __nv_bfloat16* __restrict__ x_perm, int H, int top_k, long long total) {
  pdl_sync();  // PDL: predecessor's writes visible; let the successor start its prologue
  const int nvec = H / 8;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int v = i % nvec;
  const long long p = i / nvec;
  const int t = p / top_k;
  reinterpret_cast<uint4*>(x_perm + (size_t)pair_row[p] * H)[v] =
      reinterpret_cast<const uint4*>(x + (size_t)t * ld_x)[v];
}

// ------------------------------------------------------------------------------------------------ combine
__global__ void moe_combine_kernel(const float* __restrict__ y_perm, const int* __restrict__ pair_row,
                                   const float* __restrict__ wts, const __nv_bfloat16* __restrict__ residual,
                                   long long ld_res, __nv_bfloat16* __restrict__ out, long long ld_out, int T, int top_k,
                                   int H, uint32_t* signal_flag, uint32_t signal_value, unsigned int* done_counter,
                                   int* __restrict__ zero_counts, int n_zero) {
  pdl_sync();  // PDL: predecessor's writes visible; let the successor start its prologue
  // scatter layout: the expert row counters were consumed by the grouped GEMMs before this kernel; reset them for the next layer
  if (zero_counts != nullptr && blockIdx.x == 0)
    for (int e = threadIdx.x; e < n_zero; e += blockDim.x) zero_counts[e] = 0;
  const int nvec = H / 8;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < (long long)T * nvec) {
    const int v = i % nvec;
    const int t = i / nvec;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    // the expert rows come from L2 / HBM: issue the loads of four pairs before using any (a plain k-loop serialises one round trip
    // per pair — 8 round trips for top-6 + 2 shared experts); the accumulation order stays k = 0, 1, 2, ...
    for (int k0 = 0; k0 < top_k; k0 += 4) {
      float4 a[4], b[4];
      float w[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int k = k0 + u < top_k ? k0 + u : top_k - 1;
        w[u] = k0 + u < top_k ? wts[(size_t)t * top_k + k] : 0.f;
        const float* src = y_perm + (size_t)pair_row[(size_t)t * top_k + k] * H + v * 8;
        a[u] = *reinterpret_cast<const float4*>(src);
        b[u] = *reinterpret_cast<const float4*>(src + 4);
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
    uint4 o;
    o.x = pack_bf16(acc[0], acc[1]); o.y = pack_bf16(acc[2], acc[3]);
    o.z = pack_bf16(acc[4], acc[5]); o.w = pack_bf16(acc[6], acc[7]);
    reinterpret_cast<uint4*>(out + (size_t)t * ld_out)[v] = o;
  }
  if (signal_flag != nullptr) {
    // fused stage boundary: `out` is the next stage's inbox (peer memory); the last CTA raises the flag
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned int done = atomicAdd(done_counter, 1u) + 1u;
      if (done == gridDim.x) {
        *done_counter = 0u;
        __threadfence_system();
        if (signal_value == 0u) atomicAdd_system(signal_flag, 1u);
        else st_release_sys(signal_flag, signal_value);
      }
    }
  }
}

// Combine + the NEXT layer's input RMSNorm, one CTA per token: the combined row is rounded to bf16 (that is the residual stream the
// un-fused graph stores), kept in registers, reduced to its mean square and written a second time normalised — the attention
// block of the next layer starts from `normed` without a norm kernel (launch + 2 x row traffic + one dependent-kernel gap saved).
constexpr int kCombThreads = 256;
constexpr int kCombMaxV = 4;   // H <= 256 * 8 * 4 = 8192
__global__ void __launch_bounds__(kCombThreads)
moe_combine_norm_kernel(const float* __restrict__ y_perm, const int* __restrict__ pair_row, const float* __restrict__ wts,
                        const __nv_bfloat16* __restrict__ residual, long long ld_res, __nv_bfloat16* __restrict__ out,
                        long long ld_out, int top_k, int H, int* __restrict__ zero_counts, int n_zero,
                        const __nv_bfloat16* __restrict__ norm_w, float norm_eps, __nv_bfloat16* __restrict__ normed,
                        long long ld_normed) {
  pdl_sync();
  if (zero_counts != nullptr && blockIdx.x == 0)
    for (int e = threadIdx.x; e < n_zero; e += blockDim.x) zero_counts[e] = 0;
  const int t = blockIdx.x;
  const int nvec = H / 8;
  __shared__ float s_w[32];
  __shared__ int s_row[32];
  __shared__ float red[kCombThreads / 32];
  if (threadIdx.x < top_k) {
    s_w[threadIdx.x] = wts[(size_t)t * top_k + threadIdx.x];
    s_row[threadIdx.x] = pair_row[(size_t)t * top_k + threadIdx.x];
  }
  __syncthreads();
  uint4 keep[kCombMaxV];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < kCombMaxV; ++i) {
    const int v = threadIdx.x + i * kCombThreads;
    if (v < nvec) {
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
      for (int k0 = 0; k0 < top_k; k0 += 4) {   // four pairs' loads in flight (see moe_combine_kernel)
        float4 a[4], b[4];
        float w[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int k = k0 + u < top_k ? k0 + u : top_k - 1;
          w[u] = k0 + u < top_k ? s_w[k] : 0.f;
          const float* src = y_perm + (size_t)s_row[k] * H + v * 8;
          a[u] = *reinterpret_cast<const float4*>(src);
          b[u] = *reinterpret_cast<const float4*>(src + 4);
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
      uint4 o;
      o.x = pack_bf16(acc[0], acc[1]); o.y = pack_bf16(acc[2], acc[3]);
      o.z = pack_bf16(acc[4], acc[5]); o.w = pack_bf16(acc[6], acc[7]);
      reinterpret_cast<uint4*>(out + (size_t)t * ld_out)[v] = o;
      keep[i] = o;
      const uint32_t oo[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) { const float a = bf16_lo(oo[j]), b = bf16_hi(oo[j]); ss += a * a + b * b; }
    }
  }
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < kCombThreads / 32; ++i) tot += red[i];
  const float inv = rsqrtf(tot / (float)H + norm_eps);
#pragma unroll
  for (int i = 0; i < kCombMaxV; ++i) {
    const int v = threadIdx.x + i * kCombThreads;
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

cudaError_t moe_route_launch(const void* x, long long ld_x, const void* gate_w, int T, int H, int E, int top_k, int n_group,
                             int topk_group, float scaling, bool norm_topk, int extra, int* idx, float* wts, int* sc_counts,
                             int sc_stride, int* sc_pair_row, void* sc_x, const void* norm_w, float norm_eps, cudaStream_t s,
                             const EpDispatch* ep_in, void* normed_out, long long ld_normed) {
  EpDispatch ep;
  if (ep_in != nullptr) ep = *ep_in;
  if (ep.enabled && (T == 0 || T > 1024 || ep.world > kEpMaxWorld || sc_counts != nullptr)) return cudaErrorInvalidValue;   // one-token-per-CTA variant only
  if (T == 0) return cudaSuccess;
  if (sc_counts != nullptr && (T > 1024 || sc_stride < T)) return cudaErrorInvalidValue;   // scatter: one-token-per-CTA variant only
  if (E > 32 * kMaxEPerLane || top_k + extra > 32 || extra < 0 || (H % 8) || n_group > 32 || (n_group > 1 && E % n_group)) return cudaErrorInvalidValue;
  auto xx = static_cast<const __nv_bfloat16*>(x);
  auto gw = static_cast<const __nv_bfloat16*>(gate_w);
  if (T <= 1024) {
    const size_t smem = (size_t)H * 2 + (size_t)E * 4;
    if (smem > 48 * 1024) return cudaErrorInvalidValue;
    // one token per CTA, 32 warps: each warp owns <= 2 experts, so the whole router row set costs two L2 round trips
    (void)launch_pdl(moe_route_kernel<1>, dim3(T), dim3(E >= 64 ? 1024 : (E >= 32 ? 512 : kRouteThreads)), smem, s, xx, ld_x, gw, T, H, E, top_k, n_group, topk_group, scaling,
                                                       norm_topk ? 1 : 0, extra, idx, wts, sc_counts, sc_stride, sc_pair_row, static_cast<__nv_bfloat16*>(sc_x),
                                                       static_cast<const __nv_bfloat16*>(norm_w), norm_eps, ep,
                                                       static_cast<__nv_bfloat16*>(normed_out), ld_normed);
  } else {
    constexpr int TOKS = 8;
    const size_t smem = (size_t)TOKS * H * 2 + (size_t)TOKS * E * 4;
    static size_t configured = 0;
    if (smem > 48 * 1024 && smem > configured) {
      cudaError_t e = cudaFuncSetAttribute(moe_route_kernel<TOKS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return e;
      configured = smem;
    }
    (void)launch_pdl(moe_route_kernel<TOKS>, dim3((T + TOKS - 1) / TOKS), dim3(kRouteThreads), smem, s, xx, ld_x, gw, T, H, E, top_k, n_group, topk_group,
                                                                           scaling, norm_topk ? 1 : 0, extra, idx, wts, sc_counts, sc_stride, sc_pair_row, static_cast<__nv_bfloat16*>(sc_x),
                                                                           static_cast<const __nv_bfloat16*>(norm_w), norm_eps, ep,
                                                                           static_cast<__nv_bfloat16*>(normed_out), ld_normed);
  }
  return cudaGetLastError();
}

cudaError_t moe_permute_launch(const int* idx, int T, int top_k, int E, int* expert_offsets, int* pair_row, int* counters,
                               const void* x, long long ld_x, void* x_perm, int H, cudaStream_t s) {
  (void)counters;
  if (T == 0) return cudaSuccess;
  if (E > 256 || (H % 8)) return cudaErrorInvalidValue;
  (void)launch_pdl(moe_offsets_kernel, dim3(1), dim3(1024), 0, s, idx, T * top_k, E, expert_offsets, pair_row);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const long long total = (long long)T * top_k * (H / 8);
  (void)launch_pdl(moe_gather_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, static_cast<const __nv_bfloat16*>(x), ld_x, pair_row,
                                                                    static_cast<__nv_bfloat16*>(x_perm), H, top_k, total);
  return cudaGetLastError();
}

cudaError_t moe_combine_launch(const void* y_perm, const int* pair_row, const float* wts, const void* residual,
                               long long ld_res, void* out, long long ld_out, int T, int top_k, int H,
                               uint32_t* signal_flag, uint32_t signal_value, unsigned int* done_counter, int* zero_counts,
                               int n_zero, const void* norm_w, float norm_eps, void* normed, long long ld_normed, cudaStream_t s) {
  if (T == 0) return cudaSuccess;
  if (H % 8) return cudaErrorInvalidValue;
  if (norm_w != nullptr) {
    // fused next-layer RMSNorm (never together with a stage hand-off: the last layer of a stage has no next layer to norm for)
    if (signal_flag != nullptr || normed == nullptr || top_k > 32 || H > kCombThreads * 8 * kCombMaxV) return cudaErrorInvalidValue;
    (void)launch_pdl(moe_combine_norm_kernel, dim3(T), dim3(kCombThreads), 0, s, static_cast<const float*>(y_perm), pair_row, wts,
                     static_cast<const __nv_bfloat16*>(residual), ld_res, static_cast<__nv_bfloat16*>(out), ld_out, top_k, H, zero_counts,
                     n_zero, static_cast<const __nv_bfloat16*>(norm_w), norm_eps, static_cast<__nv_bfloat16*>(normed), ld_normed);
    return cudaGetLastError();
  }
  const long long total = (long long)T * (H / 8);
  (void)launch_pdl(moe_combine_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, 
      static_cast<const float*>(y_perm), pair_row, wts, static_cast<const __nv_bfloat16*>(residual), ld_res,
      static_cast<__nv_bfloat16*>(out), ld_out, T, top_k, H, signal_flag, signal_value, done_counter, zero_counts, n_zero);
  return cudaGetLastError();
}

}  // namespace b200
