// Absorbed-latent MLA decode attention on wgmma (SURVEY §2.6 K7, K5 "weight absorption"; VERDICT r1 item 6a).
//
// DeepSeek-V2's MLA caches one 512-dim latent c_t (+ a 64-dim roped key) per token.  The reference decompresses it to 16 heads of
// K 192 / V 128 and caches *that* (shard/server/model/deepseek_v2.py:120-125 -> 5120 values per token per layer).  With W_UK folded
// into the query and W_UV into the output projection, attention runs directly on the cached latent:
//
//     s[t, h] = q_abs[h] . c_t + q_pe[h] . k_pe_t            (576-dim dot, one shared "KV head")
//     o_lat[h] = sum_t softmax_t(s)[t, h] * c_t              (512-dim)
//
// i.e. 576 + 0 extra values per token instead of 5120: 8.9x fewer KV bytes, and both contractions are GEMM-shaped over the SAME
// shared-memory tile, so they run on the tensor cores:
//
//   * one CTA per (sequence, KV split); KV tile = one 64-token page = [64 x 576] bf16 fetched by TMA (9 boxes of 64 x 64, 128B
//     swizzle) into a double-buffered ring filled by a producer warp;
//   * S^T[64 tokens, 16 heads] = K_tile[64 x 576] . Q^T: wgmma M=64 (tokens), N=16 (heads), K-major operands, fp32 in registers;
//   * the same warpgroup does the online softmax on its S fragment (shuffles within a warp, shared memory across the 4 warps) and
//     writes P^T as bf16 into shared memory in the K-major swizzled layout;
//   * O^T[512 dims, 16 heads] = V^T . P^T where V^T is the *same* tile read as an MN-major operand (dims contiguous) — no
//     transpose, no second copy: 8 wgmma M-tiles of 64 dims x 4 k-steps of 16 tokens.  The running O stays in the wgmma
//     accumulator registers (64 fp32 per thread) and is rescaled in place before each PV;
//   * long contexts are split over CTAs (flash-decoding): partial (o, m, l) in fp32 + a small combine kernel.
//
// Decode only (one query token per sequence); prefill chunks take the decompressing path (models/deepseek_v2.py).
#include <cuda.h>

#include "gemm_tmap.h"
#include "kernels.h"
#include "launch.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kHeads = 16;
constexpr int kLat = 512;          // latent / value dim
constexpr int kRope = 64;
constexpr int kDk = kLat + kRope;  // 576
constexpr int kChunks = kDk / 64;  // 9 chunks of 64 dims (128 B rows)
constexpr int kTileTok = 64;       // tokens per tile = one KV page
constexpr int kChunkBytes = kTileTok * 128;          // 8 KB
constexpr int kTileBytes = kChunks * kChunkBytes;    // 72 KB
constexpr int kQChunkBytes = kHeads * 128;           // 2 KB
constexpr int kQBytes = kChunks * kQChunkBytes;      // 18 KB
constexpr int kPBytes = kHeads * 128;                // [16 heads x 64 tokens] bf16 = 2 KB
constexpr int kThreads = 160;                        // warps 0..3: QK / softmax / PV warpgroup, warp 4: TMA

B200_DEVICE void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

struct MlaParams {
  const int* block_tables; int max_blocks;
  const int* context_lens;                 // tokens in the cache per sequence (including the one written this step)
  int nsplit, tiles_per_split;
  float scale_log2;                        // softmax scale * log2(e)
  __nv_bfloat16* out; long long o_ld_t;    // [B, 16, 512] (row stride o_ld_t) when nsplit == 1
  float* part_o; float* part_ml;           // [B, nsplit, 16, 512], [B, nsplit, 16, 2]
  long long* dbg;                          // optional [6][16] clock64 timestamps of CTA (0,0) (MLXB200_MLA_TRACE, bench/mla_bench.py)
};

#define MLA_TRACE(ev, tile) \
  do { if (p.dbg != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && (tile) < 16) p.dbg[(ev) * 16 + (tile)] = clock64(); } while (0)

__global__ void __launch_bounds__(kThreads, 1)
mla_decode_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_kv, const MlaParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* kv_smem = smem;                                   // 2 x 72 KB
  uint8_t* q_smem = smem + 2 * kTileBytes;                   // 18 KB
  uint8_t* p_smem = q_smem + kQBytes;                        // 2 x 2 KB
  float* red = reinterpret_cast<float*>(p_smem + 2 * kPBytes);   // [2][4 warps][16 heads] cross-warp max / sum
  uint64_t* bars = reinterpret_cast<uint64_t*>(red + 2 * 4 * kHeads);
  uint64_t* kv_full = bars;          // [2]
  uint64_t* kv_free = bars + 2;      // [2]
  uint64_t* q_full = bars + 4;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int split = blockIdx.x, b = blockIdx.y;

  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_kv);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_free[i], 4);   // one arrival per consumer warp
    }
    mbar_init(q_full, 1);
    mbar_fence_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();  // q, the latent pool and the step metadata are written by predecessor kernels

  const int ctx = p.context_lens[b];
  const int ntiles_seq = (ctx + kTileTok - 1) / kTileTok;
  const int t_begin = split * p.tiles_per_split;
  int t_end = t_begin + p.tiles_per_split;
  if (t_end > ntiles_seq) t_end = ntiles_seq;
  const int n = t_end > t_begin ? t_end - t_begin : 0;

  if (warp == 4) {
    // ============================================================== TMA producer (whole warp waits, one elected lane issues)
    if (n > 0) {
      if (elect_one()) {
        mbar_arrive_expect_tx(q_full, kQBytes);
        for (int c = 0; c < kChunks; ++c) tma_load_3d(q_smem + c * kQChunkBytes, &tmap_q, q_full, c * 64, 0, b);
      }
      const int* bt = p.block_tables + (size_t)b * p.max_blocks;
      int page_next = bt[t_begin];
      for (int i = 0; i < n; ++i) {
        const int st = i & 1;
        const int page = page_next;
        if (i + 1 < n) page_next = bt[t_begin + i + 1];   // the dependent global load overlaps the wait below
        mbar_wait(&kv_free[st], ((i >> 1) & 1) ^ 1);
        if (elect_one()) {
          MLA_TRACE(0, i);
          uint8_t* dst = kv_smem + st * kTileBytes;
          mbar_arrive_expect_tx(&kv_full[st], kTileBytes);
#pragma unroll
          for (int c = 0; c < kChunks; ++c)
            tma_load_2d(dst + c * kChunkBytes, &tmap_kv, &kv_full[st], c * 64, page * kTileTok, kEvictFirst);
        }
        __syncwarp();
      }
    }
    return;
  }

  // ============================================================== QK, softmax and PV (one warpgroup)
  // wgmma fragment (ptx.cuh): element j of an m64n16 accumulator is row wg_row(j), column (head) wg_col(j).  Every thread holds 4
  // heads, hk(k) = 8 * (k >> 1) + 2 * (lane & 3) + (k & 1) for k = 0..3 (element j belongs to k = 2 * (j >> 2) + (j & 1)), and
  // two token rows of S.
  int hk[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) hk[k] = 8 * (k >> 1) + 2 * (lane & 3) + (k & 1);
  float m_run[4], l_run[4], o[8][8];
#pragma unroll
  for (int k = 0; k < 4; ++k) { m_run[k] = -INFINITY; l_run[k] = 0.f; }
#pragma unroll
  for (int m = 0; m < 8; ++m)
#pragma unroll
    for (int j = 0; j < 8; ++j) o[m][j] = 0.f;
  // byte offsets of this thread's P^T elements (K-major 128B-swizzled [16 heads][64 tokens] bf16)
  uint32_t p_off[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int t = wg_row(j), h = wg_col(j);
    p_off[j] = h * 128 + ((((t >> 3) ^ (h & 7)) & 7) << 4) + (t & 7) * 2;
  }

  if (n > 0) mbar_wait(q_full, 0);
  for (int i = 0; i < n; ++i) {
    const int st = i & 1;
    mbar_wait(&kv_full[st], (i >> 1) & 1);
    if (threadIdx.x == 0) MLA_TRACE(1, i);
    const uint32_t kv0 = smem_u32(kv_smem + st * kTileBytes), q0 = smem_u32(q_smem);
    float s[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
      const uint64_t ad = gmma_desc_sw128(kv0 + c * kChunkBytes), bd = gmma_desc_sw128(q0 + c * kQChunkBytes);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_bf16<16>(s, ad + 2 * kk, bd + 2 * kk);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(s);
    if (threadIdx.x == 0) MLA_TRACE(3, i);

    bool valid[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) valid[r] = ((t_begin + i) * kTileTok + wg_row(2 * r)) < ctx;
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = valid[(j >> 1) & 1] ? s[j] * p.scale_log2 : -INFINITY;
    // tile max per head: the thread's two rows, then the 8 lanes of the warp that hold the same heads, then the 4 warps
    float tm[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int j = 4 * (k >> 1) + (k & 1);
      float v = fmaxf(s[j], s[j + 2]);
      v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
      v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 8));
      v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 16));
      tm[k] = v;
    }
    float* rmax = red + (i & 1) * 64;   // [warp][head], double-buffered by tile parity
    if (lane < 4) {
#pragma unroll
      for (int k = 0; k < 4; ++k) rmax[warp * kHeads + hk[k]] = tm[k];
    }
    named_bar_sync(1, 128);
    float alpha[4], mn[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float t4 = fmaxf(fmaxf(rmax[hk[k]], rmax[kHeads + hk[k]]), fmaxf(rmax[2 * kHeads + hk[k]], rmax[3 * kHeads + hk[k]]));
      mn[k] = fmaxf(m_run[k], t4);
      alpha[k] = (mn[k] == -INFINITY) ? 1.f : exp2f(m_run[k] - mn[k]);
      m_run[k] = mn[k];
    }
    uint8_t* pb = p_smem + st * kPBytes;
    float psum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = 2 * (j >> 2) + (j & 1);
      const float pv = valid[(j >> 1) & 1] ? exp2f(s[j] - mn[k]) : 0.f;   // mn is finite whenever any row of the tile is valid
      psum[k] += pv;
      *reinterpret_cast<__nv_bfloat16*>(pb + p_off[j]) = __float2bfloat16_rn(pv);
    }
    // the row sum stays thread-private (all threads share m_run, so partial sums add linearly): reduced once at the end
#pragma unroll
    for (int k = 0; k < 4; ++k) l_run[k] = l_run[k] * alpha[k] + psum[k];
    fence_proxy_async_smem();   // generic-proxy P stores -> visible to the tensor core
    named_bar_sync(1, 128);
    if (threadIdx.x == 0) MLA_TRACE(4, i);

#pragma unroll
    for (int m = 0; m < 8; ++m)
#pragma unroll
      for (int j = 0; j < 8; ++j) o[m][j] *= alpha[2 * (j >> 2) + (j & 1)];
    const uint64_t pd = gmma_desc_sw128(smem_u32(pb));
    wgmma_fence();
#pragma unroll
    for (int m = 0; m < 8; ++m)
#pragma unroll
      for (int ks = 0; ks < kTileTok / 16; ++ks)
        wgmma_bf16_ta<16>(o[m], gmma_desc_mn_sw128(kv0 + m * kChunkBytes + ks * 2048, kChunkBytes, 1024), pd + 2 * ks);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int m = 0; m < 8; ++m) wgmma_fence_acc(o[m]);
    if (threadIdx.x == 0) MLA_TRACE(2, i);
    if (lane == 0) mbar_arrive(&kv_free[st]);   // QK and PV of this tile are done with the stage
  }

  // ---- row sums: thread-private partials -> CTA totals (once per kernel)
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float t = l_run[k];
    t += __shfl_xor_sync(0xffffffffu, t, 4);
    t += __shfl_xor_sync(0xffffffffu, t, 8);
    t += __shfl_xor_sync(0xffffffffu, t, 16);
    l_run[k] = t;
  }
  named_bar_sync(1, 128);   // the last tile's maxima have been read
  if (lane < 4) {
#pragma unroll
    for (int k = 0; k < 4; ++k) red[warp * kHeads + hk[k]] = l_run[k];
  }
  named_bar_sync(1, 128);
#pragma unroll
  for (int k = 0; k < 4; ++k)
    l_run[k] = (red[hk[k]] + red[kHeads + hk[k]]) + (red[2 * kHeads + hk[k]] + red[3 * kHeads + hk[k]]);

  // ---- write-out: element j of M-tile m is dim 64 * m + wg_row(j) of head wg_col(j)
  if (p.nsplit == 1) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = 2 * (j >> 2) + (j & 1);
      const float inv = l_run[k] > 0.f ? 1.0f / l_run[k] : 0.f;
      __nv_bfloat16* orow = p.out + (size_t)b * p.o_ld_t + (size_t)wg_col(j) * kLat + wg_row(j);
#pragma unroll
      for (int m = 0; m < 8; ++m) orow[m * 64] = __float2bfloat16_rn(o[m][j] * inv);
    }
  } else {
    float* po = p.part_o + ((size_t)b * p.nsplit + split) * kHeads * kLat;
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int m = 0; m < 8; ++m) po[(size_t)wg_col(j) * kLat + m * 64 + wg_row(j)] = o[m][j];
    if (warp == 0 && lane < 4) {   // lanes 0..3 of warp 0 hold all 16 heads between them
      float* ml = p.part_ml + ((size_t)b * p.nsplit + split) * kHeads * 2;
#pragma unroll
      for (int k = 0; k < 4; ++k) { ml[2 * hk[k]] = m_run[k]; ml[2 * hk[k] + 1] = l_run[k]; }
    }
  }
}

// LSE combine of the KV splits: out[b, h, :] = sum_s o_s * 2^(m_s - m) / sum_s l_s * 2^(m_s - m)
__global__ void mla_combine_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml, int nsplit,
                                   __nv_bfloat16* __restrict__ out, long long o_ld_t) {
  pdl_sync();
  const int b = blockIdx.x, h = blockIdx.y;
  float m = -INFINITY;
  for (int s = 0; s < nsplit; ++s) m = fmaxf(m, part_ml[(((size_t)b * nsplit + s) * kHeads + h) * 2]);
  float l = 0.f;
  for (int s = 0; s < nsplit; ++s) {
    const float* ml = part_ml + (((size_t)b * nsplit + s) * kHeads + h) * 2;
    l += (ml[0] == -INFINITY) ? 0.f : ml[1] * exp2f(ml[0] - m);
  }
  const float inv = l > 0.f ? 1.0f / l : 0.f;
  for (int d = threadIdx.x; d < kLat; d += blockDim.x) {
    float acc = 0.f;
    for (int s = 0; s < nsplit; ++s) {
      const float ms = part_ml[(((size_t)b * nsplit + s) * kHeads + h) * 2];
      if (ms == -INFINITY) continue;
      acc += part_o[(((size_t)b * nsplit + s) * kHeads + h) * kLat + d] * exp2f(ms - m);
    }
    out[(size_t)b * o_ld_t + (size_t)h * kLat + d] = __float2bfloat16_rn(acc * inv);
  }
}

// Prologue of the absorbed path, one CTA per token: latent = RMSNorm(c_kv) * w -> pool[slot][0:512]; rope(k_pe) -> pool[slot][512:576];
// rope(q_pe) in place for the 16 heads (q rows are [q_abs 512 | q_pe 64]).  Interleaved (traditional) rope pairs, YaRN frequencies.
__global__ void __launch_bounds__(128)
mla_absorbed_prologue_kernel(__nv_bfloat16* __restrict__ q, long long q_ld_t, const __nv_bfloat16* __restrict__ ckv, long long ckv_ld_t,
                             const __nv_bfloat16* __restrict__ kpe, long long pe_ld_t, const __nv_bfloat16* __restrict__ norm_w,
                             float eps, __nv_bfloat16* __restrict__ pool, const int* __restrict__ slots,
                             const int* __restrict__ positions, const float* __restrict__ inv_freq, float mscale) {
  pdl_sync();
  const int t = blockIdx.x, tid = threadIdx.x;
  __shared__ float red[4];
  __nv_bfloat16* dst = pool + (size_t)slots[t] * kDk;
  float f[8];
  float ss = 0.f;
  if (tid < kLat / 8) {
    const uint4 r = reinterpret_cast<const uint4*>(ckv + (size_t)t * ckv_ld_t)[tid];
    const uint32_t w4[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) { f[2 * j] = bf16_lo(w4[j]); f[2 * j + 1] = bf16_hi(w4[j]); }
#pragma unroll
    for (int j = 0; j < 8; ++j) ss += f[j] * f[j];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((tid & 31) == 0) red[tid >> 5] = ss;
  __syncthreads();
  const float rinv = rsqrtf((red[0] + red[1] + red[2] + red[3]) / (float)kLat + eps);
  if (tid < kLat / 8) {
    const uint4 wr = reinterpret_cast<const uint4*>(norm_w)[tid];
    const uint32_t w4[4] = {wr.x, wr.y, wr.z, wr.w};
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      // same rounding points as rmsnorm_kernel: (x * rinv) in fp32, times w, one bf16 rounding
      ow[j] = pack_bf16(f[2 * j] * rinv * bf16_lo(w4[j]), f[2 * j + 1] * rinv * bf16_hi(w4[j]));
    }
    reinterpret_cast<uint4*>(dst)[tid] = o;
  }
  const float pos = (float)positions[t];
  for (int i = tid; i < (kHeads + 1) * (kRope / 2); i += 128) {
    const int pair = i % (kRope / 2), hh = i / (kRope / 2);
    float sn, cs;
    sincosf(pos * inv_freq[pair], &sn, &cs);
    if (hh < kHeads) {
      uint32_t* w = reinterpret_cast<uint32_t*>(q + (size_t)t * q_ld_t + (size_t)hh * kDk + kLat) + pair;
      const uint32_t u = *w;
      const float a = bf16_lo(u) * mscale, bb = bf16_hi(u) * mscale;
      *w = pack_bf16(a * cs - bb * sn, a * sn + bb * cs);
    } else {
      const uint32_t u = reinterpret_cast<const uint32_t*>(kpe + (size_t)t * pe_ld_t)[pair];
      const float a = bf16_lo(u) * mscale, bb = bf16_hi(u) * mscale;
      reinterpret_cast<uint32_t*>(dst + kLat)[pair] = pack_bf16(a * cs - bb * sn, a * sn + bb * cs);
    }
  }
}

}  // namespace

cudaError_t mla_absorbed_prologue_launch(void* q, long long q_ld_t, const void* ckv, long long ckv_ld_t, const void* kpe,
                                         long long pe_ld_t, const void* norm_w, float eps, void* pool, const int* slots,
                                         const int* positions, const float* inv_freq, float mscale, int T, cudaStream_t s) {
  if (T == 0) return cudaSuccess;
  if ((q_ld_t % 8) || (ckv_ld_t % 8) || (pe_ld_t % 2)) return cudaErrorInvalidValue;
  (void)launch_pdl(mla_absorbed_prologue_kernel, dim3(T), dim3(128), 0, s, static_cast<__nv_bfloat16*>(q), q_ld_t,
                   static_cast<const __nv_bfloat16*>(ckv), ckv_ld_t, static_cast<const __nv_bfloat16*>(kpe), pe_ld_t,
                   static_cast<const __nv_bfloat16*>(norm_w), eps, static_cast<__nv_bfloat16*>(pool), slots, positions, inv_freq, mscale);
  return cudaGetLastError();
}

size_t mla_decode_workspace_floats(int B, int nsplit) {
  return nsplit > 1 ? (size_t)B * nsplit * kHeads * (kLat + 2) : 0;
}

cudaError_t mla_decode_launch(const void* q, long long q_ld_t, int B, const void* pool, long long num_pages, int page,
                              const int* block_tables, int max_blocks, const int* context_lens, int max_ctx, float scale,
                              int nsplit, float* workspace, void* out, long long o_ld_t, long long* dbg, cudaStream_t s) {
  if (B == 0) return cudaSuccess;
  if (page != kTileTok || (q_ld_t % 8) != 0) return cudaErrorInvalidValue;
  // q: [B tokens][16 heads][576] bf16, head stride 576, token stride q_ld_t -> boxes of [1][16][64]
  TmapSpec sq;
  sq.ptr = q; sq.rank = 3; sq.l2 = CU_TENSOR_MAP_L2_PROMOTION_L2_128B;
  sq.dims[0] = kDk; sq.dims[1] = kHeads; sq.dims[2] = B;
  sq.strides[0] = (uint64_t)kDk * 2; sq.strides[1] = (uint64_t)q_ld_t * 2;
  sq.box[0] = 64; sq.box[1] = kHeads; sq.box[2] = 1;
  // latent pool: [num_pages * page][576] bf16 -> boxes of [64 tokens][64]
  TmapSpec skv;
  skv.ptr = pool;
  skv.dims[0] = kDk; skv.dims[1] = (uint64_t)num_pages * page;
  skv.strides[0] = (uint64_t)kDk * 2;
  skv.box[0] = 64; skv.box[1] = kTileTok;
  CUtensorMap tq, tkv;
  if (!tmap_encode(&tq, sq) || !tmap_encode(&tkv, skv)) return cudaErrorInvalidValue;
  MlaParams p;
  p.block_tables = block_tables; p.max_blocks = max_blocks; p.context_lens = context_lens;
  const int max_tiles = (max_ctx + kTileTok - 1) / kTileTok;
  if (nsplit < 1) nsplit = 1;
  if (nsplit > max_tiles) nsplit = max_tiles > 0 ? max_tiles : 1;
  p.nsplit = nsplit;
  p.tiles_per_split = (max_tiles + nsplit - 1) / nsplit;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = static_cast<__nv_bfloat16*>(out); p.o_ld_t = o_ld_t;
  p.dbg = dbg;
  p.part_o = workspace;
  p.part_ml = workspace != nullptr ? workspace + (size_t)B * nsplit * kHeads * kLat : nullptr;
  if (nsplit > 1 && workspace == nullptr) return cudaErrorInvalidValue;
  constexpr int smem = 2 * kTileBytes + kQBytes + 2 * kPBytes + 2 * 4 * kHeads * 4 + 5 * 8 + 1024;
  static_assert(smem <= 227 * 1024, "shared memory budget exceeded");
  cudaError_t e = set_max_dynamic_smem_once<mla_decode_kernel>(smem);
  if (e != cudaSuccess) return e;
  (void)launch_pdl(mla_decode_kernel, dim3(nsplit, B), dim3(kThreads), smem, s, tq, tkv, p);
  e = cudaGetLastError();
  if (e != cudaSuccess || nsplit == 1) return e;
  (void)launch_pdl(mla_combine_kernel, dim3(B, kHeads), dim3(128), 0, s, (const float*)p.part_o, (const float*)p.part_ml, nsplit,
                   static_cast<__nv_bfloat16*>(out), o_ld_t);
  return cudaGetLastError();
}

}  // namespace b200
