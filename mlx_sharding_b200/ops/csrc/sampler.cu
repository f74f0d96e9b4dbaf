// On-device sampler (SURVEY §2.6 K13): logit_bias + repetition penalty, log-softmax, argmax /
// temperature / nucleus (top-p) sampling and top-k logprobs — one CTA per sequence, everything stays on
// the last pipeline stage so only token ids (+ <=10 logprobs) travel back to stage 0 (SURVEY X3).
// Reference behaviour: shard/utils.py:126-139,166-177 and mlx_lm `top_p_sampling` (sort ascending,
// keep tokens whose cumulative mass exceeds 1 - top_p); here the nucleus is found without a sort by
// bisection on the logit threshold, and sampling inside it uses the Gumbel-max trick with a
// counter-based RNG (stateless: seed, step, row, token id).
// Optional per-row filters, in the order top-k -> top-p -> min-p: top-k keeps the logits >= the exact k-th largest (radix select,
// ties kept) and restricts the nucleus to that set; min-p is one logit threshold.  Presence / frequency penalties arrive folded
// into the additive bias table of apply_penalties_kernel.
// Optional token mask (structured output): one bit per vocabulary id; disallowed ids read as -inf everywhere the draw looks (greedy
// argmax, the temperature anchor, top-k, top-p sums, min-p, Gumbel) while the reported log-probs keep the full row.
#include "kernels.h"
#include "launch.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kSampThreads = 1024;

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// u = (k + 0.5) / 2^23 for the top 23 hash bits k, so 2^-24 <= u <= 1 - 2^-24.  Both u and u - 1 are exact in fp32 (a 24-bit k
// would round (2^24 - 1) + 0.5 up to 2^24, giving u = 1).
__device__ __forceinline__ float uniform01(uint64_t seed, uint64_t step, uint32_t row, uint32_t i) {
  const uint64_t h = mix64(mix64(seed ^ (step * 0xD1342543DE82EF95ull)) ^ ((uint64_t)row << 32 | i));
  return ((float)(uint32_t)(h >> 41) + 0.5f) * (1.0f / 8388608.0f);
}
// Gumbel noise g = -log(-log(u)), finite for every u above (-log(u) lies in [6e-8, 16.6], g in [-2.81, 16.6]).  The draw is
// decided by the ids with u near 1, where -log(u) is tiny: it comes from log1pf of the exact u - 1 at full precision
// (--use_fast_math compiles logf to __logf, whose absolute error near 1 is as large as -log(u) itself).  The outer __logf adds
// about 1e-7 absolute error to g.
__device__ __forceinline__ float gumbel(float u) { return -__logf(-log1pf(u - 1.0f)); }

struct ArgMax { float v; int i; };
__device__ __forceinline__ ArgMax better(ArgMax a, ArgMax b) {
  return (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a;
}
__device__ ArgMax block_argmax(ArgMax x, ArgMax* sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ArgMax y{__shfl_xor_sync(0xffffffffu, x.v, o), __shfl_xor_sync(0xffffffffu, x.i, o)};
    x = better(x, y);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) sm[warp] = x;
  __syncthreads();
  ArgMax r = sm[0];
  for (int w = 1; w < kSampThreads / 32; ++w) r = better(r, sm[w]);
  return r;
}
__device__ float block_sum(float x, float* sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) sm[warp] = x;
  __syncthreads();
  float r = 0.f;
  for (int w = 0; w < kSampThreads / 32; ++w) r += sm[w];
  return r;
}

// fp32 -> uint32 key with the same order (negative values flipped, positive ones offset above them); -inf is the smallest key
__device__ __forceinline__ uint32_t order_key(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Logit of id i as the draw sees it: -inf when the row has a mask (`al` != nullptr) and bit i & 31 of al[i >> 5] is clear.  The
// 32 ids a warp reads in one iteration share one mask word, so the mask costs one broadcast load per warp and pass.
template <bool kMask>
__device__ __forceinline__ float draw_logit(const float* __restrict__ lg, const uint32_t* __restrict__ al, int i) {
  const float x = lg[i];
  if constexpr (kMask) {
    if (al != nullptr && !((al[i >> 5] >> (i & 31)) & 1u)) return -INFINITY;
  }
  return x;
}

constexpr int kRadixBins = 2048;

// Exact k-th largest logit of a row (1 <= k < V) by radix select over `order_key`: three passes of 11, 11 and 10 bits, each a
// shared-memory histogram of the keys that match the digits chosen so far, then a suffix scan that finds the digit holding the
// k-th key. `hist` has kRadixBins words, `sm_u` 34.  Masked ids count as -inf (`draw_logit`).
template <bool kMask>
__device__ float radix_kth_largest(const float* __restrict__ lg, const uint32_t* __restrict__ al, int V, int k, uint32_t* hist,
                                   uint32_t* sm_u) {
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  uint32_t prefix = 0, mask = 0, rem = (uint32_t)k;  // rem: rank of the wanted key among the keys that match `prefix`
#pragma unroll 1
  for (int pass = 0; pass < 3; ++pass) {
    const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
    const uint32_t dmask = pass == 2 ? 1023u : 2047u;
    for (int i = t; i < kRadixBins; i += kSampThreads) hist[i] = 0u;
    __syncthreads();
    for (int i = t; i < V; i += kSampThreads) {
      const uint32_t key = order_key(draw_logit<kMask>(lg, al, i));
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & dmask], 1u);
    }
    __syncthreads();
    // thread t owns bins hi = 2047 - 2t and lo = 2046 - 2t: a scan in thread order counts keys from the top bin down
    const uint32_t ch = hist[kRadixBins - 1 - 2 * t], cl = hist[kRadixBins - 2 - 2 * t];
    uint32_t incl = ch + cl;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    if (lane == 31) sm_u[warp] = incl;
    __syncthreads();
    uint32_t above = incl - ch - cl;  // keys in bins above `hi`
    for (int w = 0; w < warp; ++w) above += sm_u[w];
    if (above < rem && above + ch >= rem) {
      sm_u[32] = kRadixBins - 1 - 2 * t;
      sm_u[33] = rem - above;
    } else if (above + ch < rem && above + ch + cl >= rem) {
      sm_u[32] = kRadixBins - 2 - 2 * t;
      sm_u[33] = rem - above - ch;
    }
    __syncthreads();
    prefix |= sm_u[32] << shift;
    mask |= dmask << shift;
    rem = sm_u[33];
  }
  return key_value(prefix);
}

// Temperature draw of one row inside the kept set.  kFilt == false is the plain top-p / categorical path; kFilt == true adds the
// top-k floor `kth` (the top-p mass sums run over x >= kth only) and keeps x >= floor = max(kth, min-p threshold) in the draw.
// kMask: ids masked off in `al` read as -inf, and `amv` is the max over the allowed ids.
template <bool kFilt, bool kMask>
__device__ __forceinline__ int draw_token(const float* __restrict__ lg, const uint32_t* __restrict__ al, int V, float amv,
                                          float temp, float tp, float kth,
                                          float floor, unsigned long long seed, unsigned long long step, uint32_t rng_row,
                                          ArgMax* sm_a, float* sm_f) {
  const float inv_t = 1.0f / temp;
  float thresh = -INFINITY;  // keep logits > thresh
  if (tp > 0.f && tp < 1.f) {
    // Z at temperature
    float zs = 0.f;
    for (int i = threadIdx.x; i < V; i += kSampThreads) {
      const float x = draw_logit<kMask>(lg, al, i);
      if (!kFilt || x >= kth) zs += __expf((x - amv) * inv_t);
    }
    zs = block_sum(zs, sm_f);
    // bisection on x in [lo, hi]: F(x) = mass{logit <= x}; find the smallest kept logit, i.e. the
    // infimum of x with F(x) > 1 - top_p
    float lo = amv - 80.f * temp, hi = amv;
    const float target = (1.0f - tp) * zs;
    for (int it = 0; it < 26; ++it) {
      const float mid = 0.5f * (lo + hi);
      float ms = 0.f;
      for (int i = threadIdx.x; i < V; i += kSampThreads) {
        const float x = draw_logit<kMask>(lg, al, i);
        if (x <= mid && (!kFilt || x >= kth)) ms += __expf((x - amv) * inv_t);
      }
      ms = block_sum(ms, sm_f);
      if (ms > target) hi = mid; else lo = mid;
    }
    thresh = lo;  // F(lo) <= target < F(hi): everything strictly above lo is in the nucleus
  }
  // Gumbel-max over the kept set: argmax (logit / T + g), g = -log(-log(u))
  ArgMax gm{-INFINITY, 0x7fffffff};
  for (int i = threadIdx.x; i < V; i += kSampThreads) {
    const float x = draw_logit<kMask>(lg, al, i);
    if (x > thresh && (!kFilt || x >= floor)) {
      gm = better(gm, ArgMax{(x - amv) * inv_t + gumbel(uniform01(seed, step, rng_row, i)), i});
    }
  }
  gm = block_argmax(gm, sm_a);
  return gm.i;
}

// kMask == false is the unmasked sampler; kMask == true reads a token mask `allow` of ceil(V / 32) words per row.
template <bool kMask>
__global__ void __launch_bounds__(kSampThreads, 1)
sample_kernel(const float* __restrict__ logits, int V, const float* __restrict__ temperature, const float* __restrict__ top_p,
              const int* __restrict__ keep_k, const float* __restrict__ min_p,
              unsigned long long seed, unsigned long long step, const unsigned long long* __restrict__ row_rng,
              long long* __restrict__ tokens, float* __restrict__ logprobs, int top_k, long long* __restrict__ top_ids,
              float* __restrict__ top_lp, const uint4* __restrict__ tag_src, uint4* __restrict__ tag_dst,
              const uint32_t* __restrict__ allow) {
  pdl_sync();  // PDL: predecessor's writes visible; let the successor start its prologue
  // Random stream of a row: (seed, step) launch scalars, or — for CUDA-graph replay, where scalars are frozen at capture — a
  // per-row (seed, step) pair in device memory (`row_rng[b]` = request seed, number of tokens that request has sampled so far:
  // a request's stream is then independent of which batch / row it decodes in).
  uint32_t rng_row = blockIdx.x;
  if (row_rng != nullptr) {
    seed = row_rng[2 * blockIdx.x];
    step = row_rng[2 * blockIdx.x + 1];
    rng_row = 0;
  }
  // 16-byte tag (step id of the scheduler) copied next to the results so the receiver can match result <-> step
  if (tag_dst != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *tag_dst = *tag_src;
  __shared__ ArgMax sm_a[kSampThreads / 32];
  __shared__ float sm_f[kSampThreads / 32];
  const int b = blockIdx.x;
  const float* lg = logits + (size_t)b * V;
  // pass 1: max / argmax of the row (`am`, for the reported log-probs) and of the ids the draw may pick (`dm`)
  ArgMax am{-INFINITY, 0x7fffffff};
  ArgMax dm{-INFINITY, 0x7fffffff};
  const uint32_t* al = nullptr;  // mask row, or nullptr when the row is sampled unmasked
  if constexpr (kMask) {
    const uint32_t* row = allow + (size_t)b * ((V + 31) >> 5);
    for (int i = threadIdx.x; i < V; i += kSampThreads) {
      const float x = lg[i];
      am = better(am, ArgMax{x, i});
      if ((row[i >> 5] >> (i & 31)) & 1u) dm = better(dm, ArgMax{x, i});
    }
    am = block_argmax(am, sm_a);
    dm = block_argmax(dm, sm_a);
    // a row without an allowed id of finite logit is sampled as if it had no mask (the engine refuses what it draws)
    if (dm.v > -INFINITY) al = row; else dm = am;
  } else {
    for (int i = threadIdx.x; i < V; i += kSampThreads) am = better(am, ArgMax{lg[i], i});
    am = block_argmax(am, sm_a);
    dm = am;
  }
  // pass 2: log-sum-exp (temperature is NOT applied to the reported logprobs, reference utils.py:131)
  float se = 0.f;
  for (int i = threadIdx.x; i < V; i += kSampThreads) se += __expf(lg[i] - am.v);
  se = block_sum(se, sm_f);
  const float lse = am.v + logf(se);

  const float temp = temperature[b];
  const float tp = top_p[b];
  int token = dm.i;
  if (temp > 0.f) {
    // optional per-row filters: keep_k[b] in [1, V) keeps the logits >= the k-th largest (ties kept), min_p[b] in (0, 1] keeps
    // p >= min_p * p_max at temperature T, i.e. logit >= max + T * ln(min_p); a row with neither runs the plain path.  Under a
    // mask, the k-th largest, the max and the top-p sums are taken over the allowed ids.
    const int kk = keep_k != nullptr ? keep_k[b] : 0;
    const float mp = min_p != nullptr ? min_p[b] : 0.f;
    const bool use_k = kk > 0 && kk < V;
    if (use_k || mp > 0.f) {
      __shared__ uint32_t sm_hist[kRadixBins];
      __shared__ uint32_t sm_u[34];
      const float kth = use_k ? radix_kth_largest<kMask>(lg, al, V, kk, sm_hist, sm_u) : -INFINITY;
      const float floor = mp > 0.f ? fmaxf(kth, dm.v + temp * logf(mp)) : kth;
      token = draw_token<true, kMask>(lg, al, V, dm.v, temp, tp, kth, floor, seed, step, rng_row, sm_a, sm_f);
    } else {
      token = draw_token<false, kMask>(lg, al, V, dm.v, temp, tp, -INFINITY, -INFINITY, seed, step, rng_row, sm_a, sm_f);
    }
  }
  if (threadIdx.x == 0) {
    tokens[b] = token;
    logprobs[b] = lg[token] - lse;
  }
  // top-k logprobs (k <= 10): k selection passes in (value desc, index asc) order
  ArgMax prev{INFINITY, -1};
  for (int r = 0; r < top_k; ++r) {
    ArgMax cur{-INFINITY, 0x7fffffff};
    for (int i = threadIdx.x; i < V; i += kSampThreads) {
      const float x = lg[i];
      if (x < prev.v || (x == prev.v && i > prev.i)) cur = better(cur, ArgMax{x, i});
    }
    cur = block_argmax(cur, sm_a);
    if (threadIdx.x == 0) {
      top_ids[(size_t)b * top_k + r] = cur.i;
      top_lp[(size_t)b * top_k + r] = cur.v - lse;
    }
    prev = cur;
  }
}

// repetition penalty over the (deduplicated) context, then logit_bias (reference order: utils.py:167-170 then :127-130)
__global__ void apply_penalties_kernel(float* __restrict__ logits, int V, const int* __restrict__ rep_ctx, int C,
                                       const float* __restrict__ penalty, const int* __restrict__ bias_idx,
                                       const float* __restrict__ bias_val, int NB) {
  pdl_sync();  // PDL: predecessor's writes visible; let the successor start its prologue
  const int b = blockIdx.x;
  float* lg = logits + (size_t)b * V;
  const float pen = penalty[b];
  if (pen != 1.0f) {
    for (int j = threadIdx.x; j < C; j += blockDim.x) {
      const int id = rep_ctx[(size_t)b * C + j];
      if (id < 0 || id >= V) continue;
      bool dup = false;
      for (int i = 0; i < j; ++i) dup |= (rep_ctx[(size_t)b * C + i] == id);
      if (dup) continue;
      const float x = lg[id];
      lg[id] = x < 0.f ? x * pen : x / pen;
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < NB; j += blockDim.x) {
    const int id = bias_idx[(size_t)b * NB + j];
    if (id >= 0 && id < V) atomicAdd(&lg[id], bias_val[(size_t)b * NB + j]);
  }
}

}  // namespace

cudaError_t apply_penalties_launch(float* logits, int B, int V, const int* rep_ctx, int C, const float* penalty,
                                   const int* bias_idx, const float* bias_val, int NB, cudaStream_t s) {
  if (B == 0) return cudaSuccess;
  (void)launch_pdl(apply_penalties_kernel, dim3(B), dim3(128), 0, s, logits, V, rep_ctx, C, penalty, bias_idx, bias_val, NB);
  return cudaGetLastError();
}

cudaError_t sample_launch(const float* logits, int B, int V, const float* temperature, const float* top_p, const int* keep_k,
                          const float* min_p, const uint32_t* allow, unsigned long long seed, unsigned long long step,
                          const unsigned long long* row_rng, long long* tokens, float* logprobs, int top_k, long long* top_ids,
                          float* top_lp, const void* tag_src, void* tag_dst, cudaStream_t s) {
  if (B == 0) return cudaSuccess;
  if (top_k > 32) return cudaErrorInvalidValue;
  if (allow != nullptr)
    (void)launch_pdl(sample_kernel<true>, dim3(B), dim3(kSampThreads), 0, s, logits, V, temperature, top_p, keep_k, min_p, seed,
                     step, row_rng, tokens, logprobs, top_k, top_ids, top_lp, static_cast<const uint4*>(tag_src),
                     static_cast<uint4*>(tag_dst), allow);
  else
    (void)launch_pdl(sample_kernel<false>, dim3(B), dim3(kSampThreads), 0, s, logits, V, temperature, top_p, keep_k, min_p, seed,
                     step, row_rng, tokens, logprobs, top_k, top_ids, top_lp, static_cast<const uint4*>(tag_src),
                     static_cast<uint4*>(tag_dst), static_cast<const uint32_t*>(nullptr));
  return cudaGetLastError();
}

}  // namespace b200
