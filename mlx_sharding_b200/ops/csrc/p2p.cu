// Device-side primitives of the fused P2P stage boundary (SURVEY §5.8 tier T0, call sites X1/X3):
// flag wait (bounded spin, acquire.sys), flag set (release.sys), copy-with-signal for hand-offs that
// cannot ride a GEMM epilogue, and the on-device step-metadata advance that lets a CUDA-graphed decode
// step re-run without any host -> device traffic.  The reference's equivalent is a blocking gRPC unary
// call per stage per token with host staging (shard/utils.py:71-90,162-164).
#include "kernels.h"
#include "launch.h"
#include "ptx.cuh"

namespace b200 {

namespace {

// Spin until *flag >= expected (monotonic step counters).  Bounded: after ~timeout the kernel records an
// error and returns instead of hanging the GPU (a dead peer must never wedge the box).
__global__ void wait_flag_kernel(const uint32_t* flag, uint32_t expected, uint32_t* error_flag, unsigned long long timeout_ns) {
  pdl_sync();  // PDL: predecessor's writes visible; let the successor start its prologue
  const unsigned long long t0 = globaltimer_ns();
  while (true) {
    const uint32_t v = ld_acquire_sys(flag);
    if ((int32_t)(v - expected) >= 0) break;
    if (globaltimer_ns() - t0 > timeout_ns) {
      if (error_flag != nullptr) atomicExch(error_flag, 1u);
      break;
    }
    __nanosleep(64);
  }
}

// Counting variant for CUDA-graph replay: the expected value is this consumer's own arrival count, kept in
// device memory (`local_counter`), so the same captured node is correct on every replay.
__global__ void wait_flag_counter_kernel(const uint32_t* flag, uint32_t* local_counter, uint32_t* error_flag,
                                         uint32_t* error_host, unsigned long long timeout_ns) {
  pdl_sync();  // PDL: predecessor's writes visible; let the successor start its prologue
  const uint32_t expected = atomicAdd(local_counter, 1u) + 1u;
  const unsigned long long t0 = globaltimer_ns();
  while (true) {
    const uint32_t v = ld_acquire_sys(flag);
    if ((int32_t)(v - expected) >= 0) break;
    // a wait that already timed out on this device poisons the following ones: they return at once instead of
    // serialising one full timeout per queued step (the host reads the error word and fails the requests)
    if (error_flag != nullptr && *reinterpret_cast<volatile uint32_t*>(error_flag) != 0u) break;
    if (globaltimer_ns() - t0 > timeout_ns) {
      if (error_flag != nullptr) atomicExch(error_flag, 1u);
      // mirror in mapped pinned host memory: the host learns about the timeout with a plain load, without a device sync
      if (error_host != nullptr) { *reinterpret_cast<volatile uint32_t*>(error_host) = 1u; __threadfence_system(); }
      break;
    }
    __nanosleep(32);
  }
}

__global__ void set_flag_kernel(uint32_t* flag, uint32_t value) {
  pdl_sync();  // PDL: predecessor's writes visible; let the successor start its prologue
  __threadfence_system();
  st_release_sys(flag, value);
}

// dst may be peer memory: stream src -> dst with 16 B stores, then publish the flag from the last CTA.
__global__ void copy_signal_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, size_t nvec, uint32_t* flag,
                                   uint32_t value, unsigned int* done_counter) {
  pdl_sync();  // PDL: predecessor's writes visible; let the successor start its prologue
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) dst[i] = src[i];
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int done = atomicAdd(done_counter, 1u) + 1u;
    if (done == gridDim.x) {
      *done_counter = 0u;
      __threadfence_system();
      if (value == 0u) atomicAdd_system(flag, 1u);
      else st_release_sys(flag, value);
    }
  }
}

// decode step k -> k+1 for every sequence of a micro-batch: position, context length, KV slot
__global__ void advance_meta_kernel(int* positions, int* context_lens, int* slots, const int* block_tables, int max_blocks,
                                    int page, int B) {
  pdl_sync();  // PDL: predecessor's writes visible; let the successor start its prologue
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int p = positions[b] + 1;
  positions[b] = p;
  context_lens[b] = p + 1;
  slots[b] = block_tables[(size_t)b * max_blocks + p / page] * page + p % page;
}

}  // namespace

cudaError_t wait_flag_launch(const uint32_t* flag, uint32_t expected, uint32_t* error_flag, cudaStream_t s) {
  (void)launch_pdl(wait_flag_kernel, dim3(1), dim3(1), 0, s, flag, expected, error_flag, wait_timeout_ns());
  return cudaGetLastError();
}

cudaError_t wait_flag_counter_launch(const uint32_t* flag, uint32_t* local_counter, uint32_t* error_flag, uint32_t* error_host,
                                     cudaStream_t s) {
  (void)launch_pdl(wait_flag_counter_kernel, dim3(1), dim3(1), 0, s, flag, local_counter, error_flag, error_host, wait_timeout_ns());
  return cudaGetLastError();
}

cudaError_t set_flag_launch(uint32_t* flag, uint32_t value, cudaStream_t s) {
  (void)launch_pdl(set_flag_kernel, dim3(1), dim3(1), 0, s, flag, value);
  return cudaGetLastError();
}

cudaError_t copy_signal_launch(const void* src, void* dst, size_t bytes, uint32_t* flag, uint32_t value,
                               unsigned int* done_counter, cudaStream_t s) {
  if (bytes % 16) return cudaErrorInvalidValue;
  const size_t nvec = bytes / 16;
  int grid = (int)((nvec + 255) / 256);
  if (grid > 296) grid = 296;
  if (grid < 1) grid = 1;
  (void)launch_pdl(copy_signal_kernel, dim3(grid), dim3(256), 0, s, static_cast<const uint4*>(src), static_cast<uint4*>(dst), nvec, flag, value, done_counter);
  return cudaGetLastError();
}

cudaError_t advance_meta_launch(int* positions, int* context_lens, int* slots, const int* block_tables, int max_blocks,
                                int page, int B, cudaStream_t s) {
  if (B == 0) return cudaSuccess;
  (void)launch_pdl(advance_meta_kernel, dim3((B + 127) / 128), dim3(128), 0, s, positions, context_lens, slots, block_tables, max_blocks, page, B);
  return cudaGetLastError();
}

void pdl_skip_next() { pdl_skip_next_flag() = true; }

}  // namespace b200
