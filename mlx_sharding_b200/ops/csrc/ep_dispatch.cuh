// Device side of one expert-parallel dispatch step: the slot reservation of a (token, k) pair and the step's publication.  Both
// dispatch kernels use it: ep_dispatch_scatter_kernel (ep.cu) and the router with the dispatch folded in (moe.cu).  The destination's
// grouped gate/up GEMM acquires what ep_publish releases (gemm_persistent.cu, GemmParams::ep_arrive).
#pragma once
#include "kernels.h"
#include "ptx.cuh"

namespace b200 {

// Reserves the next row of local expert `le` in destination `dst`'s expert-major receive buffer with one system-scope atomic on its
// row counter (double-buffered by the parity of step `seq`), and stores next to the row where its output returns to: pair `pair`'s
// row of this rank's return buffer, as `dst` maps it.  Returns the row (le * cap_e + slot), or -1 when the expert's segment is full.
B200_DEVICE int ep_reserve_row(const EpDispatch& ep, uint32_t seq, int dst, int le, unsigned long long pair, int H) {
  const int slot = atomicAdd_system(reinterpret_cast<int*>(ep.recv_cnt.p[dst]) + (int)(seq & 1u) * ep.experts_per_rank + le, 1);
  const int r = slot < ep.cap_e ? le * ep.cap_e + slot : -1;
  if (r >= 0) reinterpret_cast<unsigned long long*>(ep.recv_dst.p[dst])[r] = ep.my_ret.p[dst] + pair * H * sizeof(float);
  return r;
}

// Publication, called by every thread of every CTA after its row stores: each CTA fences them at system scope, the last CTA to arrive
// writes `seq` to this rank's arrival word at every destination with st.release.sys, then advances the step state (sequence number,
// arrival counter, and the return arrivals the combine of this step waits for).
B200_DEVICE void ep_publish(const EpDispatch& ep, uint32_t seq) {
  __threadfence_system();
  __syncthreads();
  __shared__ bool last;
  if (threadIdx.x == 0) last = (atomicAdd(ep.done_counter, 1u) + 1u == gridDim.x);
  __syncthreads();
  if (last) {
    __threadfence_system();
    for (int r = threadIdx.x; r < ep.world; r += blockDim.x)
      st_release_sys_u64(reinterpret_cast<unsigned long long*>(ep.recv_seq.p[r]) + ep.my_rank, (unsigned long long)seq);
    __syncthreads();
    if (threadIdx.x == 0) {
      *ep.send_seq = seq;
      *ep.done_counter = 0u;
      if (ep.ret_expected != nullptr) *ep.ret_expected += (uint32_t)ep.world;
    }
  }
}

}  // namespace b200
