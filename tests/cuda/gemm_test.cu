// Standalone correctness + timing harness for the wgmma GEMM (no torch): compares against a naive
// fp32 CUDA reference on the shapes the models use.  Build: see tests/cuda/build.sh; run on an H100.
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <vector>
#include <string>
#include "../../mlx_sharding_b200/ops/csrc/gemm.h"

using namespace b200;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(2); } } while (0)

__global__ void init_bf16(__nv_bfloat16* p, size_t n, uint32_t seed, float scale) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) {
    uint32_t h = (uint32_t)i * 2654435761u ^ seed;
    h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
    float u = (h & 0xFFFFFF) / float(0x1000000) - 0.5f;
    p[i] = __float2bfloat16(u * scale);
  }
}

// naive reference: one thread per output element
__global__ void ref_gemm(const __nv_bfloat16* x, long long ldx, const __nv_bfloat16* w, const __nv_bfloat16* w2, long long ldw,
                         const int* offs, int E, int m, int n, int k, const __nv_bfloat16* res, long long ldr,
                         const __nv_bfloat16* bias, int act, float softcap, float* out, int total_rows) {
  int col = blockIdx.x * blockDim.x + threadIdx.x;
  int row = blockIdx.y;
  if (col >= n || row >= total_rows) return;
  int e = 0;
  if (offs) { while (e < E && row >= offs[e + 1]) ++e; if (e >= E) { out[(size_t)row * n + col] = 0.f; return; } }
  const __nv_bfloat16* wr = w + ((size_t)e * n + col) * ldw;
  float acc = 0.f, acc2 = 0.f;
  for (int i = 0; i < k; ++i) {
    float xv = __bfloat162float(x[(size_t)row * ldx + i]);
    acc += xv * __bfloat162float(wr[i]);
    if (w2) acc2 += xv * __bfloat162float(w2[((size_t)e * n + col) * ldw + i]);
  }
  if (bias) acc += __bfloat162float(bias[col]);
  if (w2) {
    float g = acc;
    if (act == kActSilu) g = g / (1.f + expf(-g));
    else if (act == kActGeluTanh) g = 0.5f * g * (1.f + tanhf(0.7978845608028654f * (g + 0.044715f * g * g * g)));
    acc = g * acc2;
  }
  if (softcap > 0.f) acc = softcap * tanhf(acc / softcap);
  if (res) acc += __bfloat162float(res[(size_t)row * ldr + col]);
  out[(size_t)row * n + col] = acc;
}

struct Case {
  std::string name; int m, n, k; bool dual = false, res = false, bias = false, fp32 = false; int splits = 1;
  int E = 0; float softcap = 0.f; int act = kActSilu; int ldx_pad = 0; int iters = 0;
};

static int run_case(const Case& c) {
  const int E = c.E > 0 ? c.E : 1;
  // grouped: uneven rows per expert, some empty
  std::vector<int> offs(E + 1, 0);
  int total_rows = c.m;
  if (c.E > 0) {
    int acc = 0;
    for (int e = 0; e < E; ++e) { int r = (e % 5 == 3) ? 0 : (1 + (e * 7 + 3) % (2 * c.m / E + 1)); offs[e] = acc; acc += r; }
    offs[E] = acc; total_rows = acc;
  }
  int max_rows = c.m;
  if (c.E > 0) { max_rows = 0; for (int e = 0; e < E; ++e) max_rows = std::max(max_rows, offs[e + 1] - offs[e]); }
  const long long ldx = c.k + c.ldx_pad;
  __nv_bfloat16 *x, *w, *w2 = nullptr, *res = nullptr, *bias = nullptr; void* out; float* ref; int* d_offs = nullptr;
  CK(cudaMalloc(&x, (size_t)total_rows * ldx * 2));
  CK(cudaMalloc(&w, (size_t)E * c.n * c.k * 2));
  if (c.dual) CK(cudaMalloc(&w2, (size_t)E * c.n * c.k * 2));
  if (c.res) CK(cudaMalloc(&res, (size_t)total_rows * c.n * 2));
  if (c.bias) CK(cudaMalloc(&bias, (size_t)c.n * 2));
  CK(cudaMalloc(&out, (size_t)total_rows * c.n * 4));
  CK(cudaMalloc(&ref, (size_t)total_rows * c.n * 4));
  CK(cudaMemset(out, 0xFF, (size_t)total_rows * c.n * (c.fp32 ? 4 : 2)));
  auto init = [&](__nv_bfloat16* p, size_t n, uint32_t seed, float s) { init_bf16<<<(unsigned)((n + 255) / 256), 256>>>(p, n, seed, s); };
  init(x, (size_t)total_rows * ldx, 1, 2.0f);
  init(w, (size_t)E * c.n * c.k, 2, 0.2f);
  if (c.dual) init(w2, (size_t)E * c.n * c.k, 3, 0.2f);
  if (c.res) init(res, (size_t)total_rows * c.n, 4, 2.0f);
  if (c.bias) init(bias, c.n, 5, 1.0f);
  if (c.E > 0) { CK(cudaMalloc(&d_offs, (E + 1) * 4)); CK(cudaMemcpy(d_offs, offs.data(), (E + 1) * 4, cudaMemcpyHostToDevice)); }

  GemmArgs a;
  a.x = x; a.x_rows = total_rows; a.ld_x = ldx; a.w = w; a.w2 = w2; a.ld_w = c.k;
  a.m = c.m; a.n = c.n; a.k = c.k; a.max_rows = max_rows; a.num_experts = c.E; a.expert_offsets = d_offs;
  a.out = out; a.ld_out = c.n; a.out_fp32 = c.fp32; a.residual = res; a.ld_res = c.n; a.bias = bias;
  a.act = c.act; a.softcap = c.softcap; a.splits = c.splits;
  const GemmPlan plan = gemm_plan(a, kGemmBf16, sm_count());
  const int bn = plan.bn;
  float* ws = nullptr; unsigned int* ctr = nullptr;
  if (plan.workspace_floats > 0) {
    CK(cudaMalloc(&ws, plan.workspace_floats * 4)); CK(cudaMalloc(&ctr, 65536 * 4)); CK(cudaMemset(ctr, 0, 65536 * 4));
    a.workspace = ws; a.tile_counters = ctr;
  }
  cudaError_t le = gemm_launch(a, plan, 0);
  if (le != cudaSuccess) { printf("[%s] launch failed: %s\n", c.name.c_str(), cudaGetErrorString(le)); return 1; }
  cudaError_t se = cudaDeviceSynchronize();
  if (se != cudaSuccess) { printf("[%s] kernel failed: %s\n", c.name.c_str(), cudaGetErrorString(se)); exit(3); }
  dim3 rg((c.n + 127) / 128, total_rows);
  ref_gemm<<<rg, 128>>>(x, ldx, w, w2, c.k, d_offs, E, c.m, c.n, c.k, res, c.n, bias, c.act, c.softcap, ref, total_rows);
  CK(cudaDeviceSynchronize());
  std::vector<float> h_ref((size_t)total_rows * c.n), h_out((size_t)total_rows * c.n);
  CK(cudaMemcpy(h_ref.data(), ref, h_ref.size() * 4, cudaMemcpyDeviceToHost));
  if (c.fp32) CK(cudaMemcpy(h_out.data(), out, h_out.size() * 4, cudaMemcpyDeviceToHost));
  else {
    std::vector<__nv_bfloat16> hb(h_out.size());
    CK(cudaMemcpy(hb.data(), out, hb.size() * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < hb.size(); ++i) h_out[i] = __bfloat162float(hb[i]);
  }
  double max_err = 0, max_ref = 0; size_t bad = 0, nan = 0;
  for (size_t i = 0; i < h_ref.size(); ++i) {
    float r = h_ref[i], o = h_out[i];
    if (!(o == o)) { ++nan; continue; }
    double err = fabs((double)r - o), tol = (c.fp32 ? 2e-3 : 2e-2) * fmax(1.0, fabs((double)r));
    if (err > tol) { if (bad < 5) printf("   mismatch @%zu (row %zu col %zu): ref %f got %f\n", i, i / c.n, i % c.n, r, o); ++bad; }
    max_err = fmax(max_err, err); max_ref = fmax(max_ref, fabs((double)r));
  }
  int fail = (bad || nan) ? 1 : 0;
  double us = 0;
  if (!fail && c.iters > 0) {
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int i = 0; i < 3; ++i) gemm_launch(a, plan, 0);
    cudaEventRecord(e0);
    for (int i = 0; i < c.iters; ++i) gemm_launch(a, plan, 0);
    cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
    float ms; cudaEventElapsedTime(&ms, e0, e1); us = ms * 1000.0 / c.iters;
  }
  double wbytes = (double)E * c.n * c.k * 2 * (c.dual ? 2 : 1);
  double flops = 2.0 * total_rows * c.n * (double)c.k * (c.dual ? 2 : 1);
  printf("[%-28s] rows=%d n=%d k=%d bn=%d splits=%d %s max_err=%.4g (max_ref %.3g) bad=%zu nan=%zu", c.name.c_str(), total_rows,
         c.n, c.k, bn, plan.splits, fail ? "FAIL" : "ok", max_err, max_ref, bad, nan);
  if (us > 0) printf("  %.1f us  %.0f GB/s(w)  %.1f TFLOP/s", us, wbytes / us * 1e-3, flops / us * 1e-6);
  printf("\n");
  cudaFree(x); cudaFree(w); if (w2) cudaFree(w2); if (res) cudaFree(res); if (bias) cudaFree(bias);
  cudaFree(out); cudaFree(ref); if (d_offs) cudaFree(d_offs); if (ws) cudaFree(ws); if (ctr) cudaFree(ctr);
  return fail;
}

int main(int argc, char** argv) {
  bool quick = argc > 1 && std::string(argv[1]) == "quick";
  std::vector<Case> cases;
  { Case c; c.name = "tiny_m16"; c.m = 16; c.n = 128; c.k = 64; cases.push_back(c); }
  { Case c; c.name = "tiny_m16_k256"; c.m = 16; c.n = 128; c.k = 256; cases.push_back(c); }
  { Case c; c.name = "m1_n256_k512"; c.m = 1; c.n = 256; c.k = 512; cases.push_back(c); }
  { Case c; c.name = "m7_partialN"; c.m = 7; c.n = 200; c.k = 192; cases.push_back(c); }
  { Case c; c.name = "m64_deep_k"; c.m = 64; c.n = 384; c.k = 2048; cases.push_back(c); }
  { Case c; c.name = "m40_bn64_ldx"; c.m = 40; c.n = 256; c.k = 512; c.ldx_pad = 64; cases.push_back(c); }
  { Case c; c.name = "m128"; c.m = 128; c.n = 256; c.k = 512; cases.push_back(c); }
  { Case c; c.name = "m300_bn256"; c.m = 300; c.n = 384; c.k = 1024; cases.push_back(c); }
  { Case c; c.name = "res_bias"; c.m = 33; c.n = 256; c.k = 512; c.res = true; c.bias = true; cases.push_back(c); }
  { Case c; c.name = "fp32_out_softcap"; c.m = 9; c.n = 512; c.k = 256; c.fp32 = true; c.softcap = 30.f; cases.push_back(c); }
  { Case c; c.name = "dual_silu"; c.m = 20; c.n = 256; c.k = 512; c.dual = true; cases.push_back(c); }
  { Case c; c.name = "dual_gelu_m200"; c.m = 200; c.n = 256; c.k = 512; c.dual = true; c.act = kActGeluTanh; cases.push_back(c); }
  { Case c; c.name = "splitk4"; c.m = 8; c.n = 256; c.k = 2048; c.splits = 4; c.res = true; cases.push_back(c); }
  { Case c; c.name = "splitk3_dual"; c.m = 24; c.n = 128; c.k = 1408; c.splits = 3; c.dual = true; cases.push_back(c); }
  { Case c; c.name = "grouped"; c.m = 48; c.n = 256; c.k = 512; c.E = 8; cases.push_back(c); }
  { Case c; c.name = "grouped_dual"; c.m = 96; c.n = 384; c.k = 512; c.E = 16; c.dual = true; cases.push_back(c); }
  { Case c; c.name = "grouped_big_rows"; c.m = 2000; c.n = 256; c.k = 256; c.E = 4; cases.push_back(c); }
  if (!quick) {
    // model shapes (DeepSeek-V2-Lite / Llama-3-8B), with timing
    { Case c; c.name = "dsv2_qkv_a_m64"; c.m = 64; c.n = 3648; c.k = 2048; c.iters = 20; cases.push_back(c); }
    { Case c; c.name = "dsv2_qkv_a_m64_sk4"; c.m = 64; c.n = 3648; c.k = 2048; c.splits = 4; c.iters = 20; cases.push_back(c); }
    { Case c; c.name = "dsv2_o_m64_sk8"; c.m = 64; c.n = 2048; c.k = 2048; c.splits = 8; c.res = true; c.iters = 20; cases.push_back(c); }
    { Case c; c.name = "dsv2_lmhead_m64"; c.m = 64; c.n = 102400; c.k = 2048; c.fp32 = true; c.iters = 10; cases.push_back(c); }
    { Case c; c.name = "dsv2_experts_gateup"; c.m = 384; c.n = 1408; c.k = 2048; c.E = 64; c.dual = true; c.iters = 10; cases.push_back(c); }
    { Case c; c.name = "dsv2_experts_down"; c.m = 384; c.n = 2048; c.k = 1408; c.E = 64; c.iters = 10; cases.push_back(c); }
    { Case c; c.name = "llama_gateup_m64"; c.m = 64; c.n = 14336; c.k = 4096; c.dual = true; c.iters = 10; cases.push_back(c); }
    { Case c; c.name = "llama_down_m64"; c.m = 64; c.n = 4096; c.k = 14336; c.res = true; c.splits = 4; c.iters = 10; cases.push_back(c); }
    { Case c; c.name = "prefill_m1024_qkv"; c.m = 1024; c.n = 3648; c.k = 2048; c.iters = 10; cases.push_back(c); }
    { Case c; c.name = "prefill_m4096_gateup"; c.m = 4096; c.n = 14336; c.k = 4096; c.dual = true; c.iters = 5; cases.push_back(c); }
    { Case c; c.name = "square_8192"; c.m = 8192; c.n = 8192; c.k = 8192; c.iters = 5; cases.push_back(c); }
  }
  int fails = 0;
  for (auto& c : cases) fails += run_case(c);
  printf("%s: %d/%zu cases failed\n", fails ? "FAILED" : "PASSED", fails, cases.size());
  return fails ? 1 : 0;
}
