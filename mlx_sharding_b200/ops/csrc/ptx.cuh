// Thin inline-PTX wrappers for the sm_90a features used by the kernels in this directory:
// mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA (wgmma), and the system-scope release/acquire
// primitives of the fused P2P stage boundary.
//
// Nothing here comes from the reference (it has no native code, SURVEY §2.3); descriptor bit layouts follow
// the PTX ISA ("Matrix Descriptor Format" of the wgmma section).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

#define B200_DEVICE __device__ __forceinline__

B200_DEVICE uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
B200_DEVICE uint32_t lane_id() { return threadIdx.x & 31; }

// One elected lane of a fully converged warp.  Unlike `if (lane == 0)`, nvcc knows the branch is warp-uniform-with-one-thread, so
// TMA / mbarrier instructions inside it compile to plain uniform-datapath code instead of an ELECT / BRA.U.ANY loop per instruction.
B200_DEVICE bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------------------------- mbarrier
B200_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
B200_DEVICE void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
B200_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
B200_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
B200_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must trap (kernel error), never hang the GPU.
B200_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 24)) __trap();
  }
}

// ---------------------------------------------------------------------------------------------- TMA
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

B200_DEVICE void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tile load global -> shared, completion signalled on an mbarrier (complete_tx::bytes)
B200_DEVICE void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
      : "memory");
}
B200_DEVICE void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------- wgmma
// Warpgroup MMA (sm_90a): the four warps of an aligned warpgroup issue together, the fp32 accumulator lives in their registers.
// Fragment of an m64nN tile: thread t = 32 * w + l holds rows 16 * w + l / 4 + 8 * r and columns 8 * i + 2 * (l % 4) + e in
// element [4 * i + 2 * r + e] (see wg_row / wg_col).
B200_DEVICE void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
B200_DEVICE void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
B200_DEVICE void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int N>
B200_DEVICE void wgmma_fence_acc(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
B200_DEVICE int wg_row(int j) { return 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2) + 8 * ((j >> 1) & 1); }
B200_DEVICE int wg_col(int j) { return 8 * (j >> 2) + 2 * (threadIdx.x & 3) + (j & 1); }

// K-major, 128B-swizzled shared-memory operand descriptor (sm_90 GMMA layout):
//   [0,14) start>>4 | [16,30) LBO>>4 (=1, ignored for swizzled K-major) | [32,46) SBO>>4 (8 rows * 128 B) | [62,64) 1 = SWIZZLE_128B
// Advancing 16 bf16 (32 B) along K inside the swizzle atom is +2 in the address field.
B200_DEVICE uint64_t gmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// MN-major, 128B-swizzled operand: 64 MN-elements per 128 B line, 8 K rows 128 B apart, groups of 8 K rows `sbo_bytes` apart,
// 64-element MN blocks `lbo_bytes` apart.
B200_DEVICE uint64_t gmma_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(lbo_bytes >> 4) << 16;
  d |= static_cast<uint64_t>(sbo_bytes >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// D (+)= A[smem desc] * B[smem desc], m64nNk16, bf16 inputs, fp32 accumulate; both operands K-major (the _ta form: A MN-major)
template <int N> B200_DEVICE void wgmma_bf16(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc);
template <>
B200_DEVICE void wgmma_bf16<16>(float (&d)[8], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, 1, 1, 1, 0, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc));
}

template <>
B200_DEVICE void wgmma_bf16<32>(float (&d)[16], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, 1, 1, 1, 0, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc));
}

template <>
B200_DEVICE void wgmma_bf16<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, 1, 1, 1, 0, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc));
}

// N = 128 as two N = 64 halves: columns 64.. are elements 32.. of the fragment and token rows 64.. of the B tile (+8 KB)
template <>
B200_DEVICE void wgmma_bf16<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  wgmma_bf16<64>(*reinterpret_cast<float(*)[32]>(&d[0]), adesc, bdesc);
  wgmma_bf16<64>(*reinterpret_cast<float(*)[32]>(&d[32]), adesc, bdesc + ((64 * 128) >> 4));
}

template <int N> B200_DEVICE void wgmma_bf16_ta(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc);
template <>
B200_DEVICE void wgmma_bf16_ta<16>(float (&d)[8], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, 1, 1, 1, 1, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc));
}

template <int N> B200_DEVICE void wgmma_e4m3(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc);  // D = A * B (no accumulate)
template <>
B200_DEVICE void wgmma_e4m3<16>(float (&d)[8], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n16k32.f32.e4m3.e4m3 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, 0, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc));
}

template <>
B200_DEVICE void wgmma_e4m3<32>(float (&d)[16], uint64_t adesc, uint64_t bdesc) {   // two N = 16 halves (see wgmma_bf16<128>)
  wgmma_e4m3<16>(*reinterpret_cast<float(*)[8]>(&d[0]), adesc, bdesc);
  wgmma_e4m3<16>(*reinterpret_cast<float(*)[8]>(&d[8]), adesc, bdesc + ((16 * 128) >> 4));
}

template <>
B200_DEVICE void wgmma_e4m3<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc) {   // two N = 32 halves (see wgmma_bf16<128>)
  wgmma_e4m3<32>(*reinterpret_cast<float(*)[16]>(&d[0]), adesc, bdesc);
  wgmma_e4m3<32>(*reinterpret_cast<float(*)[16]>(&d[16]), adesc, bdesc + ((32 * 128) >> 4));
}


// ---------------------------------------------------------------------------------------------- scopes
B200_DEVICE void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
B200_DEVICE uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
B200_DEVICE void st_release_sys_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
B200_DEVICE unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
B200_DEVICE uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
B200_DEVICE void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Programmatic dependent launch (see launch.h): wait for the predecessor grid's memory, then let the successor's
// blocks be scheduled while this grid is still running.
B200_DEVICE void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
B200_DEVICE void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// Small kernels: release the successor first (its CTAs become resident and run their pre-wait prologue — for the GEMMs that is
// barrier init and the first ring-full of *weight* TMA loads), then wait for the predecessor.  Nothing before the
// wait may touch memory a predecessor writes; completion of grid i+1 implies completion of grid i, so the chain stays ordered.
B200_DEVICE void pdl_sync() { pdl_launch_dependents(); pdl_wait(); }

B200_DEVICE float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
B200_DEVICE float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xFFFF0000u); }
B200_DEVICE uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

}  // namespace b200
