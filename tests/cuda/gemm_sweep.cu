// Split-K / tile sweep for the decode-shaped GEMMs: device time per launch measured by replaying a CUDA graph
// of launches that rotate over enough weight copies to defeat the 50 MB L2 (weights are streamed from HBM,
// as in a real decode step).  Prints one line per (shape, splits).
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../mlx_sharding_b200/ops/csrc/gemm.h"
using namespace b200;
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(2); } } while (0)

struct Shape { const char* name; int m, n, k; bool dual; bool res; };

int main() {
  std::vector<Shape> shapes = {
    {"o_proj      64x2048x2048", 64, 2048, 2048, false, true},
    {"qkv_a       64x3648x2048", 64, 3648, 2048, false, false},
    {"kv_b        64x4096x512 ", 64, 4096, 512, false, false},
    {"shared_gu   64x2816x2048", 64, 2816, 2048, true, false},
    {"shared_down 64x2048x2816", 64, 2048, 2816, false, true},
    {"llama_qkv   64x6144x4096", 64, 6144, 4096, false, false},
    {"llama_o     64x4096x4096", 64, 4096, 4096, false, true},
    {"o_abs       64x2048x8192", 64, 2048, 8192, false, true},
    {"qkv_abs     64x9792x2048", 64, 9792, 2048, false, false},
    {"o_proj m8    8x2048x2048", 8, 2048, 2048, false, true},
    {"o_proj m256 256x2048x2048", 256, 2048, 2048, false, true},
  };
  cudaStream_t st; CK(cudaStreamCreate(&st));
  constexpr size_t kWsFloats = 64u << 20;   // 256 MB
  float* ws; unsigned int* ctr;
  CK(cudaMalloc(&ws, kWsFloats * 4)); CK(cudaMalloc(&ctr, 65536 * 4)); CK(cudaMemset(ctr, 0, 65536 * 4));
  for (auto& s : shapes) {
    const size_t wbytes = (size_t)s.n * s.k * 2 * (s.dual ? 2 : 1);
    int nrot = (int)((300ull << 20) / wbytes) + 1; if (nrot > 64) nrot = 64;
    __nv_bfloat16 *x, *res, *out; std::vector<__nv_bfloat16*> w(nrot), w2(nrot);
    CK(cudaMalloc(&x, (size_t)s.m * s.k * 2)); CK(cudaMalloc(&res, (size_t)s.m * s.n * 2)); CK(cudaMalloc(&out, (size_t)s.m * s.n * 2));
    CK(cudaMemset(x, 0, (size_t)s.m * s.k * 2)); CK(cudaMemset(res, 0, (size_t)s.m * s.n * 2));
    for (int i = 0; i < nrot; ++i) {
      CK(cudaMalloc(&w[i], (size_t)s.n * s.k * 2)); CK(cudaMemset(w[i], 0, (size_t)s.n * s.k * 2));
      if (s.dual) { CK(cudaMalloc(&w2[i], (size_t)s.n * s.k * 2)); CK(cudaMemset(w2[i], 0, (size_t)s.n * s.k * 2)); }
    }
    for (int splits : {1, 2, 4, 8, 16}) {
      if ((s.k / 64) / splits < 2) continue;
      GemmArgs a; a.x = x; a.x_rows = s.m; a.ld_x = s.k; a.ld_w = s.k; a.m = s.m; a.n = s.n; a.k = s.k; a.max_rows = s.m;
      a.out = out; a.ld_out = s.n; if (s.res) { a.residual = res; a.ld_res = s.n; } a.act = kActSilu; a.splits = splits;
      a.workspace = ws; a.tile_counters = ctr; a.w2 = s.dual ? w2[0] : nullptr;
      const GemmPlan plan = gemm_plan(a, kGemmBf16, sm_count());
      if (plan.workspace_floats > kWsFloats) { printf("workspace of %zu floats does not fit\n", plan.workspace_floats); exit(3); }
      auto launch = [&](int i) { a.w = w[i % nrot]; a.w2 = s.dual ? w2[i % nrot] : nullptr; cudaError_t e = gemm_launch(a, plan, st); if (e != cudaSuccess) { printf("launch err %s\n", cudaGetErrorString(e)); exit(3); } };
      for (int i = 0; i < nrot; ++i) launch(i);   // warm: descriptors cached, attributes set
      CK(cudaStreamSynchronize(st));
      const int iters = 2 * nrot;
      cudaGraph_t g; cudaGraphExec_t ge;
      CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeGlobal));
      for (int i = 0; i < iters; ++i) launch(i);
      CK(cudaStreamEndCapture(st, &g)); CK(cudaGraphInstantiate(&ge, g, 0));
      CK(cudaGraphLaunch(ge, st)); CK(cudaStreamSynchronize(st));
      cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
      cudaEventRecord(e0, st); CK(cudaGraphLaunch(ge, st)); cudaEventRecord(e1, st); CK(cudaEventSynchronize(e1));
      float ms; cudaEventElapsedTime(&ms, e0, e1);
      const double us = ms * 1000.0 / iters;
      printf("%-28s splits=%2d  ctas=%4d  %7.2f us  %6.0f GB/s\n", s.name, splits, ((s.n + 127) / 128) * splits, us, wbytes / us * 1e-3);
      cudaGraphExecDestroy(ge); cudaGraphDestroy(g);
    }
    for (int i = 0; i < nrot; ++i) { cudaFree(w[i]); if (s.dual) cudaFree(w2[i]); }
    cudaFree(x); cudaFree(res); cudaFree(out);
  }
  return 0;
}
