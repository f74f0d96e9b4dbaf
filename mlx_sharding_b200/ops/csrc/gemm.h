// Host API of the swap-AB wgmma GEMM (see gemm_splitk.cu and gemm_persistent.cu).  Plain CUDA, no torch dependency.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace b200 {

enum : int { kActNone = 0, kActSilu = 1, kActGeluTanh = 2 };

// Device-side parameter block (passed by value).
struct GemmParams {
  int m, n, k, splits;
  const int* expert_offsets;
  // block-scaled FP8 (gemm_fp8.cu): ue8m0 scale words (4 scales = one 128-element k-block per uint32), row-major [rows, K / 128]
  const uint32_t* w_sf; const uint32_t* w2_sf; const uint32_t* x_sf;
  int sf_ld_w, sf_ld_x;
  // Expert-parallel receive side (ep.cu, gemm_persistent.cu only): before touching tokens / counts the kernel waits until every
  // source rank has published this step's sequence number (ep_arrive[r], acquire.sys), for at most ep_timeout_ns (wait_timeout_ns);
  // counts are double-buffered by step parity
  const unsigned long long* ep_arrive; const uint32_t* ep_seq; uint32_t* ep_error; unsigned long long ep_timeout_ns;
  int ep_world; int ep_zero_other;
  int expert_stride;  // > 0: experts live at fixed row stride, expert_offsets[e] is the row COUNT of expert e (scatter layout)
  void* out;
  long long ld_out;
  const __nv_bfloat16* residual;
  long long ld_res;
  const __nv_bfloat16* bias;
  int act;
  float softcap;
  float* workspace;
  unsigned int* tile_counters;
  uint32_t* signal_flag;
  uint32_t signal_value;
  unsigned int* done_counter;
  unsigned int signal_tiles;
  int cluster_splitk;  // 1: the `splits` CTAs of a tile form a cluster and reduce through DSMEM
  // Expert-parallel return path fused into the grouped down-projection (gemm_persistent.cu only):
  const unsigned long long* row_dst;       // per output row: address of its destination row (may be peer memory); overrides out
  const unsigned long long* signal_peers;  // `num_signal_peers` flag addresses, each bumped (+1, .sys) after ALL tiles are stored
  int num_signal_peers;
};

// Host-side launch description.  Y[rows, n] = X[rows, k] * W[n, k]^T, bf16 in, fp32 accumulate.
struct GemmArgs {
  const void* x = nullptr;        // bf16 [x_rows, k], row stride ld_x
  long long x_rows = 0, ld_x = 0;
  const void* w = nullptr;        // bf16 [(num_experts *) n, k], row stride ld_w
  const void* w2 = nullptr;       // optional second weight (gate/up pair): out = act(x w^T) * (x w2^T)
  long long ld_w = 0;
  int m = 0;                      // rows when not grouped
  int n = 0, k = 0;
  int max_rows = 0;               // upper bound of rows per (expert) problem: sizes the grid
  int num_experts = 0;            // grouped: number of experts (0: dense)
  long long expected_rows = 0;    // grouped: rows expected over all experts, sizes the token tile (0: sized for max_rows)
  const int* expert_offsets = nullptr;  // grouped: int32 [num_experts + 1] row offsets into x / out (device)
  const unsigned long long* ep_arrive = nullptr; const uint32_t* ep_seq = nullptr; uint32_t* ep_error = nullptr;
  int ep_world = 0; bool ep_zero_other = false;   // EP receive side: arrival wait fused into the grouped GEMM (see GemmParams)
  int expert_stride = 0;                // > 0: expert e owns rows [e * stride, e * stride + expert_offsets[e]) (counts, not offsets)
  void* out = nullptr;            // bf16 (or fp32 if out_fp32) [rows, n], row stride ld_out; may be a peer pointer
  long long ld_out = 0;
  bool out_fp32 = false;
  const void* residual = nullptr; // bf16 [rows, n] added in the epilogue
  long long ld_res = 0;
  const void* bias = nullptr;     // bf16 [n]
  int act = kActNone;             // used with w2
  float softcap = 0.f;            // y = cap * tanh(y / cap) (Gemma-2 final logits)
  int splits = 0;                 // split-K factor (0 = chosen by gemm_plan)
  float* workspace = nullptr;     // fp32, GemmPlan::workspace_floats elements (workspace split-K route only)
  unsigned int* tile_counters = nullptr;  // zero-initialised, >= number of output tiles (workspace split-K route only)
  uint32_t* signal_flag = nullptr;        // fused stage boundary: raised (release.sys) when every tile is stored
  uint32_t signal_value = 0;
  unsigned int* done_counter = nullptr;   // zero-initialised device counter
  const unsigned long long* row_dst = nullptr;       // EP return: per-row destination addresses (device array)
  const unsigned long long* signal_peers = nullptr;  // EP return: device table of peer flag addresses
  int num_signal_peers = 0;
  // MLX affine-quantised weights (gemm_q_launch): w / w2 point at the packed uint32 codes [rows, k*bits/32];
  // scales / biases are pre-transposed to [k/group, rows] bf16 at load time (TMA-friendly)
  // block-scaled FP8 (gemm_fp8_launch): w / w2 / x point at e4m3 bytes, *_sf at their ue8m0 scales [rows, k / 32]
  const void* w_sf = nullptr; const void* w2_sf = nullptr; const void* x_sf = nullptr;
  int q_bits = 0, q_group = 64;
  const void* q_scales_t = nullptr; const void* q_biases_t = nullptr;
  const void* q_scales2_t = nullptr; const void* q_biases2_t = nullptr;
  // LoRA adapter of a quantised launch (gemm_q_launch, bf16 output): the epilogue adds sum_j u[row, j] * lora_b[o, j] to the
  // accumulator of feature o.  u = x A^T is fp32 [rows, lora_r] (lora_shrink_launch), for a pair [rows, 2 * lora_r] with the
  // second weight's adapter in columns lora_r..; lora_b / lora_b2 are bf16 scale * B, [n, lora_r].  lora_r is a multiple of 8
  // (0: no adapter).
  const float* lora_u = nullptr;
  const void* lora_b = nullptr; const void* lora_b2 = nullptr;
  int lora_r = 0;
};

// Weight format of a launch: bf16, MLX affine int4 / int8 (dequantised in the kernel), MXFP8.
enum GemmKind : int { kGemmBf16 = 0, kGemmQuant = 1, kGemmFp8 = 2 };

enum GemmRoute : int {
  kRoutePersistent = 0,       // no split-K: one CTA per SM walks the tile list (gemm_persistent.cu, gemm_q_persistent.cu, gemm_fp8.cu)
  kRouteClusterSplitK = 1,    // the `splits` CTAs of a tile form a cluster and reduce through DSMEM (bf16 only)
  kRouteWorkspaceSplitK = 2,  // partial tiles go through an fp32 workspace, the last CTA of a tile reduces them
};

// Every host-side choice of a launch, made once by gemm_plan and read by the binding (workspace) and the launcher.
struct GemmPlan {
  GemmRoute route = kRoutePersistent;
  int bn = 0;                  // token tile
  int splits = 1;              // split-K factor, <= the k-block count
  int tiles_n = 0, tiles_m = 0, num_tiles = 0;  // 128-feature tiles, token tiles per expert, tiles of all experts
  dim3 grid;
  unsigned cluster_z = 1;      // CTAs per cluster along z
  size_t workspace_floats = 0;  // fp32 workspace the route reads
};

// Pure function of the launch shape (rows, n, k, pair, experts, expected rows, requested splits) and the SM count.
GemmPlan gemm_plan(const GemmArgs& a, GemmKind kind, int sm_count);
// Kernel parameters shared by every route: zero-initialised, then the launch's common fields and the plan's split-K choice.
GemmParams gemm_params(const GemmArgs& a, const GemmPlan& plan);
int sm_count();  // of the current device, read once

cudaError_t gemm_launch(const GemmArgs& a, const GemmPlan& plan, cudaStream_t stream);
cudaError_t gemm_persistent_launch(const GemmArgs& a, const GemmPlan& plan, cudaStream_t stream);
bool gemm_q_supported(int bits, int group, int k);
cudaError_t gemm_q_launch(const GemmArgs& a, const GemmPlan& plan, cudaStream_t stream);
cudaError_t gemm_fp8_launch(const GemmArgs& a, const GemmPlan& plan, cudaStream_t stream);   // MXFP8 x MXFP8 -> bf16 / fp32 (gemm_fp8.cu)
// LoRA shrink (lora.cu): u[T, R] = x[T, K] a[R, K]^T in fp32, bf16 inputs; R and K multiples of 8, rows 16-byte aligned
cudaError_t lora_shrink_launch(const void* x, long long ld_x, const void* a, int T, int K, int R, float* u, cudaStream_t stream);

}  // namespace b200
