// Kernel launch helper with Programmatic Dependent Launch (PDL).
//
// A decode step is ~430 small kernels inside one CUDA graph; at that granularity launch latency and each
// kernel's prologue (barrier init, descriptor fetch) are a visible fraction of the step.
// Every kernel in this directory therefore
//   * is launched with cudaLaunchAttributeProgrammaticStreamSerialization, and
//   * executes `griddepcontrol.launch_dependents` as early as possible and `griddepcontrol.wait` before it touches any
//     global memory a predecessor may have written (or writes anything at all),
// so kernel N+1's blocks are scheduled and run their pre-wait part while kernel N is still running.  For the GEMMs the
// pre-wait part is barrier init *and the first ring-full of weight TMA loads* (weights are never
// produced by a predecessor), so the HBM latency of a small GEMM hides behind the kernel in front of it.
// (launch_dependents only takes effect once *every* block of N has issued it, i.e. once all of N's blocks are
// resident, so the waiting blocks of N+1 can never starve N; completion of N+1 implies completion of N, so N+2's
// wait on N+1 transitively orders it after N.)
#pragma once
#include <cuda_runtime.h>

namespace b200 {

// One-shot opt-out for the next launch of this host thread: the first kernel after a cross-stream fork / join has a
// dependency that is not its same-stream predecessor, so it is launched with plain (full) dependencies.
inline bool& pdl_skip_next_flag() {
  static thread_local bool skip = false;
  return skip;
}
inline bool pdl_use_now() {
  bool& skip = pdl_skip_next_flag();
  const bool use = !skip;
  skip = false;
  return use;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_use_now() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace b200

namespace b200 {

// Same, with a thread-block cluster of {1, 1, cluster_z} CTAs (DSMEM split-K reduction).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                      unsigned cluster_z, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  unsigned n = 0;
  if (cluster_z > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = 1;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = cluster_z;
    ++n;
  }
  if (pdl_use_now()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace b200
