// Causal flash-attention for prefill chunks against the paged KV cache (SURVEY §2.6 K7 "flash_prefill").
//
// The reference materialises a dense additive [T, T] mask and calls mx.fast.scaled_dot_product_attention
// on a contiguous cache (shard/server/model/llama.py:48-59, deepseek_v2.py:47-57).  Here causality is
// implicit, the cache is paged, batches are ragged (many sequences / chunks per launch) and the chunk may
// start at any context offset (chunked prefill).
//
// Tiling: CTA = 64 query rows of one (sequence, q-head), 4 warps x 16 rows; KV is walked in 64-key tiles,
// double buffered with cp.async straight from the page pool into padded (bank-conflict-free) shared memory.
// S = QK^T and O += PV run on the tensor cores through warp-level mma.m16n8k16 (bf16 in, fp32 accumulate) with
// the FA-2 register pipeline (S accumulators are re-used as the A operand of PV); softmax is online in
// registers with exp2.  NOTE: this is the legacy (HMMA) tensor path — a wgmma version of this
// kernel is the planned replacement; the GEMMs that dominate prefill FLOPs already run on wgmma.
#include "kernels.h"
#include "launch.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kBM = 64, kBN = 64, kWarps = 4, kThreads = 128;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(smem)));
}

template <int DK, int DV>
__global__ void __launch_bounds__(kThreads)
flash_prefill_kernel(const __nv_bfloat16* __restrict__ q, long long q_ld_t, long long q_ld_h,
                     const __nv_bfloat16* __restrict__ kpool, const __nv_bfloat16* __restrict__ vpool,
                     const int* __restrict__ block_tables, int max_blocks, const int* __restrict__ cu_seqlens,
                     const int* __restrict__ context_lens, int num_seqs, int q_heads, int kv_heads, int page, float scale_log2,
                     __nv_bfloat16* __restrict__ out, long long o_ld_t) {
  pdl_sync();  // PDL: predecessor's writes visible; let the successor start its prologue
  constexpr int KS = DK + 8, VS = DV + 8;  // padded row strides (elements): (stride/2) % 32 == 4 -> conflict free
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __nv_bfloat16* sK = reinterpret_cast<__nv_bfloat16*>(smem_raw);      // [2][kBN][KS]
  __nv_bfloat16* sV = sK + 2 * kBN * KS;                               // [2][kBN][VS]

  // ---- which (sequence, q tile) is this CTA?
  int tile = blockIdx.x, seq = 0, q0 = 0, qlen = 0;
  for (; seq < num_seqs; ++seq) {
    qlen = cu_seqlens[seq + 1] - cu_seqlens[seq];
    const int nt = (qlen + kBM - 1) / kBM;
    if (tile < nt) break;
    tile -= nt;
  }
  if (seq >= num_seqs) return;
  q0 = tile * kBM;
  const int hq = blockIdx.y;
  const int hk = hq / (q_heads / kv_heads);
  const int tok0 = cu_seqlens[seq] + q0;             // first token row of the tile
  const int rows = min(kBM, qlen - q0);
  const int ctx_after = context_lens[seq];
  const int pos0 = ctx_after - qlen + q0;            // absolute position of the tile's first query
  const int kv_end = min(ctx_after, pos0 + rows);    // causal: keys 0 .. last query position
  const int ntiles = (kv_end + kBN - 1) / kBN;
  const int* bt = block_tables + (size_t)seq * max_blocks;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r_lo = lane >> 2, c2 = (lane & 3) * 2;

  auto load_tile = [&](int j, int buf) {
    __nv_bfloat16* dK = sK + buf * kBN * KS;
    __nv_bfloat16* dV = sV + buf * kBN * VS;
    constexpr int KC = DK / 8, VC = DV / 8;
    for (int i = threadIdx.x; i < kBN * (KC + VC); i += kThreads) {
      const int r = i / (KC + VC), c = i % (KC + VC);
      int pos = j * kBN + r;
      if (pos >= kv_end) pos = kv_end - 1;  // clamp: masked later
      const size_t pg = bt[pos / page];
      const size_t row = (pg * kv_heads + hk) * page + (pos % page);
      if (c < KC) cp_async16(dK + r * KS + c * 8, kpool + row * DK + c * 8);
      else cp_async16(dV + r * VS + (c - KC) * 8, vpool + row * DV + (c - KC) * 8);
    }
    cp_async_commit();
  };

  // ---- Q fragments (A operand), straight from global memory
  uint32_t qa[DK / 16][4];
  {
    const int ra = warp * 16 + r_lo, rb = ra + 8;
    const __nv_bfloat16* qra = q + (size_t)(tok0 + ra) * q_ld_t + (size_t)hq * q_ld_h;
    const __nv_bfloat16* qrb = q + (size_t)(tok0 + rb) * q_ld_t + (size_t)hq * q_ld_h;
#pragma unroll
    for (int ks = 0; ks < DK / 16; ++ks) {
      qa[ks][0] = ra < rows ? *reinterpret_cast<const uint32_t*>(qra + ks * 16 + c2) : 0u;
      qa[ks][1] = rb < rows ? *reinterpret_cast<const uint32_t*>(qrb + ks * 16 + c2) : 0u;
      qa[ks][2] = ra < rows ? *reinterpret_cast<const uint32_t*>(qra + ks * 16 + 8 + c2) : 0u;
      qa[ks][3] = rb < rows ? *reinterpret_cast<const uint32_t*>(qrb + ks * 16 + 8 + c2) : 0u;
    }
  }
  float o[DV / 8][4];
#pragma unroll
  for (int i = 0; i < DV / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;
  const int qpos_a = pos0 + warp * 16 + r_lo, qpos_b = qpos_a + 8;

  load_tile(0, 0);
  for (int j = 0; j < ntiles; ++j) {
    const int buf = j & 1;
    if (j + 1 < ntiles) { load_tile(j + 1, buf ^ 1); cp_async_wait<1>(); }
    else cp_async_wait<0>();
    __syncthreads();
    const __nv_bfloat16* tK = sK + buf * kBN * KS;
    const __nv_bfloat16* tV = sV + buf * kBN * VS;
    // ---- S = Q K^T  (16 x 64 per warp)
    float s[kBN / 8][4];
#pragma unroll
    for (int nt = 0; nt < kBN / 8; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
      const __nv_bfloat16* kr = tK + (nt * 8 + r_lo) * KS + c2;
#pragma unroll
      for (int ks = 0; ks < DK / 16; ++ks) {
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(kr + ks * 16);
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(kr + ks * 16 + 8);
        mma_bf16(s[nt], qa[ks], b0, b1);
      }
    }
    // ---- scale, causal mask, online softmax (base 2)
    const int kbase = j * kBN;
    float mx_a = m_a, mx_b = m_b;
#pragma unroll
    for (int nt = 0; nt < kBN / 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int kpos = kbase + nt * 8 + c2 + e;
        s[nt][e] = (kpos <= qpos_a) ? s[nt][e] * scale_log2 : -INFINITY;
        s[nt][2 + e] = (kpos <= qpos_b) ? s[nt][2 + e] * scale_log2 : -INFINITY;
        mx_a = fmaxf(mx_a, s[nt][e]);
        mx_b = fmaxf(mx_b, s[nt][2 + e]);
      }
    }
    mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1)); mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
    mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1)); mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
    const float ca = (mx_a == -INFINITY) ? 1.f : exp2f(m_a - mx_a);
    const float cb = (mx_b == -INFINITY) ? 1.f : exp2f(m_b - mx_b);
    const float ba = (mx_a == -INFINITY) ? 0.f : mx_a, bb = (mx_b == -INFINITY) ? 0.f : mx_b;
    float sa = 0.f, sb = 0.f;
    uint32_t pa[kBN / 16][4];
#pragma unroll
    for (int nt = 0; nt < kBN / 8; ++nt) {
      const float p0 = exp2f(s[nt][0] - ba), p1 = exp2f(s[nt][1] - ba);
      const float p2 = exp2f(s[nt][2] - bb), p3 = exp2f(s[nt][3] - bb);
      sa += p0 + p1; sb += p2 + p3;
      pa[nt >> 1][(nt & 1) * 2 + 0] = pack_bf16(p0, p1);
      pa[nt >> 1][(nt & 1) * 2 + 1] = pack_bf16(p2, p3);
    }
    l_a = l_a * ca + sa; l_b = l_b * cb + sb;
    m_a = mx_a; m_b = mx_b;
#pragma unroll
    for (int i = 0; i < DV / 8; ++i) { o[i][0] *= ca; o[i][1] *= ca; o[i][2] *= cb; o[i][3] *= cb; }
    // ---- O += P V
#pragma unroll
    for (int kk = 0; kk < kBN / 16; ++kk) {
#pragma unroll
      for (int nt2 = 0; nt2 < DV / 16; ++nt2) {
        uint32_t vb[4];
        // lanes 0-15: rows kk*16 + (lane & 15) at column nt2*16; lanes 16-31: same rows at column +8
        ldmatrix_x4_trans(vb, tV + (kk * 16 + (lane & 15)) * VS + nt2 * 16 + ((lane >> 4) << 3));
        mma_bf16(o[nt2 * 2], pa[kk], vb[0], vb[1]);
        mma_bf16(o[nt2 * 2 + 1], pa[kk], vb[2], vb[3]);
      }
    }
    __syncthreads();
  }
  // ---- normalise and store
  l_a += __shfl_xor_sync(0xffffffffu, l_a, 1); l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 1); l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
  const float ia = l_a > 0.f ? 1.f / l_a : 0.f, ib = l_b > 0.f ? 1.f / l_b : 0.f;
  const int ra = warp * 16 + r_lo, rb = ra + 8;
#pragma unroll
  for (int i = 0; i < DV / 8; ++i) {
    if (ra < rows)
      *reinterpret_cast<uint32_t*>(out + (size_t)(tok0 + ra) * o_ld_t + (size_t)hq * DV + i * 8 + c2) = pack_bf16(o[i][0] * ia, o[i][1] * ia);
    if (rb < rows)
      *reinterpret_cast<uint32_t*>(out + (size_t)(tok0 + rb) * o_ld_t + (size_t)hq * DV + i * 8 + c2) = pack_bf16(o[i][2] * ib, o[i][3] * ib);
  }
}

template <int DK, int DV>
cudaError_t launch_prefill(const FlashPrefillArgs& a, cudaStream_t s) {
  constexpr int smem = 2 * kBN * ((DK + 8) + (DV + 8)) * 2;
  constexpr auto kern = flash_prefill_kernel<DK, DV>;
  cudaError_t e = set_max_dynamic_smem_once<kern>(smem);
  if (e != cudaSuccess) return e;
  dim3 grid(a.max_tiles, a.q_heads);
  (void)launch_pdl(kern, dim3(grid), dim3(kThreads), smem, s, static_cast<const __nv_bfloat16*>(a.q), a.q_ld_t, a.q_ld_h,
                                    static_cast<const __nv_bfloat16*>(a.kpool), static_cast<const __nv_bfloat16*>(a.vpool),
                                    a.block_tables, a.max_blocks, a.cu_seqlens, a.context_lens, a.num_seqs, a.q_heads, a.kv_heads,
                                    a.page, a.scale * 1.4426950408889634f, static_cast<__nv_bfloat16*>(a.out), a.o_ld_t);
  return cudaGetLastError();
}

}  // namespace

bool flash_prefill_supported(int dk, int dv) {
  return (dk == 192 && dv == 128) || (dk == 128 && dv == 128) || (dk == 64 && dv == 64);
}

cudaError_t flash_prefill_launch(const FlashPrefillArgs& a, cudaStream_t s) {
  if (a.num_seqs == 0 || a.max_tiles == 0) return cudaSuccess;
  if ((a.q_ld_t % 2) || (a.q_ld_h % 2)) return cudaErrorInvalidValue;
  if (a.dk_ == 192 && a.dv_ == 128) return launch_prefill<192, 128>(a, s);
  if (a.dk_ == 128 && a.dv_ == 128) return launch_prefill<128, 128>(a, s);
  if (a.dk_ == 64 && a.dv_ == 64) return launch_prefill<64, 64>(a, s);
  return cudaErrorNotSupported;
}

}  // namespace b200
