// Split-K reduction through distributed shared memory (thread-block cluster), used for decode-shaped GEMMs.
//
// With few output tiles (N/128 = 16..32) a skinny GEMM cannot fill 132 SMs unless K is split, but reducing the
// partials through global memory (workspace + fence + ticket + re-read) costs about as much as the decode GEMM itself.
// Here the `splits` CTAs that share an
// output tile form one cluster (cluster dims {1,1,splits}):
//   phase A  every CTA stores its register accumulator into its *own* shared memory as fp32 [cols][128];
//   barrier.cluster (release/acquire);
//   phase B  CTA r sums token columns [r*BN/S, (r+1)*BN/S) over all S CTAs with ld.shared::cluster (DSMEM),
//            in split order (deterministic), applies the epilogue and stores its rows;
//   barrier.cluster so no CTA retires while a peer still reads its shared memory.
// No workspace, no atomics, no global round trip.
#pragma once
#include "gemm_common.cuh"

namespace b200 {
namespace gemm {

B200_DEVICE uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
B200_DEVICE void cluster_arrive_release() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
B200_DEVICE void cluster_wait_acquire() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
B200_DEVICE void cluster_sync_all() { cluster_arrive_release(); cluster_wait_acquire(); }
B200_DEVICE uint32_t mapa_shared(uint32_t local_addr, uint32_t cta_rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(cta_rank));
  return r;
}
B200_DEVICE float ld_dsmem_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}

// Phase B (MMA warpgroup): reduce this CTA's slice of token columns over the cluster, epilogue, store.
template <int BN, bool DUAL, typename OutT>
__device__ __forceinline__ void cluster_epilogue_reduce_store(const GemmParams& p, uint8_t* smem, const TileInfo& ti) {
  const int S = p.splits;
  const int r = static_cast<int>(cluster_ctarank());
  const int f_local = threadIdx.x;  // 0..127: one feature per thread -> 256 B coalesced rows
  const int f_glob = ti.n0 + f_local;
  const int per = (BN + S - 1) / S;
  const int t0 = r * per;
  int t1 = t0 + per;
  if (t1 > ti.rows_valid) t1 = ti.rows_valid;
  const float bias = feature_bias(p, f_glob);
  const uint32_t local = smem_u32(smem);
  uint32_t peer[8];
#pragma unroll
  for (int s = 0; s < 8; ++s) peer[s] = mapa_shared(local, s < S ? s : 0);
  for (int t = t0; t < t1; ++t) {
    float g = 0.f, u = 0.f;
    float gv[8], uv[8];
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      if (s < S) {
        gv[s] = ld_dsmem_f32(peer[s] + static_cast<uint32_t>((t * kTileM + f_local) * 4));
        if (DUAL) uv[s] = ld_dsmem_f32(peer[s] + static_cast<uint32_t>(((BN + t) * kTileM + f_local) * 4));
      }
    }
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      if (s < S) {
        g += gv[s];
        if (DUAL) u += uv[s];
      }
    }
    float y = epi_value<DUAL>(p, g, u, bias);
    if (f_glob < p.n) {
      const size_t row = static_cast<size_t>(ti.row_base + t);
      if (sizeof(OutT) == 2) {
        // as write_rows: round the GEMM result to bf16 first, then add the residual
        float o = __bfloat162float(__float2bfloat16_rn(y));
        if (p.residual != nullptr) o += __bfloat162float(p.residual[row * p.ld_res + f_glob]);
        reinterpret_cast<__nv_bfloat16*>(p.out)[row * p.ld_out + f_glob] = __float2bfloat16_rn(o);
      } else {
        if (p.residual != nullptr) y += __bfloat162float(p.residual[row * p.ld_res + f_glob]);
        reinterpret_cast<float*>(p.out)[row * p.ld_out + f_glob] = y;
      }
    }
  }
  if (p.signal_flag != nullptr) __threadfence_system();
}

// After the final cluster barrier: one thread of cluster rank 0 reports the tile as stored.
__device__ __forceinline__ void cluster_signal(const GemmParams& p) {
  if (p.signal_flag == nullptr) return;
  if (cluster_ctarank() == 0 && threadIdx.x == 0) {
    __threadfence_system();
    publish_tiles_done(p, 1u);
  }
}

}  // namespace gemm
}  // namespace b200
