// Shared device pieces of the swap-AB wgmma GEMM family: tile constants, the warpgroup main loop, the tile decode, the
// epilogue (bias / activation-gating / soft-cap value, staging tile -> global rows with residual, workspace split-K reduction)
// and the fused completion signal.  Used by the bf16 (gemm_splitk.cu, gemm_persistent.cu), quantised (gemm_q_splitk.cu,
// gemm_q_persistent.cu) and MXFP8 (gemm_fp8.cu) kernels.
#pragma once
#include "gemm.h"
#include "ptx.cuh"

namespace b200 {
namespace gemm {

constexpr int kTileM = 128;      // output features per CTA (two wgmma M = 64 halves)
constexpr int kBlockK = 64;      // bf16 elements per k-block = one 128B swizzle row
constexpr int kMmaK = 16;
constexpr int kNumThreads = 160;  // warps 0..3: MMA warpgroup + epilogue, warp 4: TMA
constexpr int kEpiThreads = 128;
constexpr int kProducerWarp = 4;
constexpr int kATileBytes = kTileM * kBlockK * 2;  // 16 KB
// Register accumulators bound the token tile: 128 x BN fp32 over 128 threads is BN registers per weight matrix.
constexpr int kMaxBN = 128, kMaxBNDual = 64;
// MXFP8 (gemm_fp8.cu): the per-block product needs a second register tile next to the accumulator
constexpr int kFp8MaxBN = 64, kFp8MaxBNDual = 32;

__host__ __device__ constexpr int acc_bytes(int BN, bool dual) { return BN * (dual ? 2 : 1) * kTileM * 4; }
__host__ __device__ constexpr int stage_bytes(int BN, bool dual) {
  return kATileBytes * (dual ? 2 : 1) + BN * kBlockK * 2;
}
__host__ __device__ constexpr int num_stages(int BN, bool dual, int out_bytes) {
  // leave room for barriers; the accumulator and the epilogue staging buffer alias the (by then idle) stage ring
  int s = (200 * 1024) / stage_bytes(BN, dual);
  s = s > 8 ? 8 : s;
  while (s * stage_bytes(BN, dual) < acc_bytes(BN, dual) + BN * kTileM * out_bytes) ++s;
  return s;
}

// One k-block (64 deep) of a 128 x BN tile: two M = 64 halves of the weight tile against the token tile, both K-major.
template <int BN>
__device__ __forceinline__ void mma_kblock(float (&acc)[2][BN / 2], uint32_t a_addr, uint32_t b_addr) {
  const uint64_t bdesc = gmma_desc_sw128(b_addr);
#pragma unroll
  for (int kk = 0; kk < kBlockK / kMmaK; ++kk)
#pragma unroll
    for (int h = 0; h < 2; ++h) wgmma_bf16<BN>(acc[h], gmma_desc_sw128(a_addr + h * 64 * 128) + 2 * kk, bdesc + 2 * kk);
}

template <int BN>
__device__ __forceinline__ void acc_zero(float (&acc)[2][BN / 2]) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[h][j] = 0.f;
}

// MMA warpgroup main loop of one tile over ring iterations [it0, it0 + num_kb): `ready(stage, phase)` waits until the stage is
// filled; a stage is released (one arrival per warp, empty barriers count 4) once the MMAs reading it have completed.
template <int BN, bool DUAL, int STAGES, int STAGE_BYTES, int OFF_B, typename Ready>
__device__ __forceinline__ void mma_mainloop(float (&acc)[2][BN / 2], float (&acc2)[2][BN / 2], uint8_t* smem, uint64_t* empty_bar,
                                             uint32_t it0, int num_kb, Ready ready) {
  const bool leader = (threadIdx.x & 31) == 0;
  for (int i = 0; i < num_kb; ++i) {
    const uint32_t it = it0 + i, s = it % STAGES;
    ready(s, (it / STAGES) & 1);
    const uint32_t a_addr = smem_u32(smem + s * STAGE_BYTES);
    wgmma_fence();
    mma_kblock<BN>(acc, a_addr, a_addr + OFF_B);
    if (DUAL) mma_kblock<BN>(acc2, a_addr + kATileBytes, a_addr + OFF_B);
    wgmma_commit();
    wgmma_wait<1>();  // the previous k-block's MMAs are done: its stage can be refilled
    if (i > 0 && leader) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
  }
  wgmma_wait<0>();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    wgmma_fence_acc(acc[h]);
    if (DUAL) wgmma_fence_acc(acc2[h]);
  }
  if (num_kb > 0 && leader) mbar_arrive(&empty_bar[(it0 + num_kb - 1) % STAGES]);
}

// Register accumulator -> shared memory fp32 [col][128 features] (column offset `c0`: the second matrix of a DUAL pair at BN).
template <int BN>
__device__ __forceinline__ void acc_store_smem(const float (&acc)[2][BN / 2], float* buf, int c0) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) buf[(c0 + wg_col(j)) * kTileM + h * 64 + wg_row(j)] = acc[h][j];
}

__device__ __forceinline__ float apply_act(int act, float g) {
  if (act == kActSilu) return g / (1.0f + __expf(-g));
  if (act == kActGeluTanh) {
    const float k0 = 0.7978845608028654f, k1 = 0.044715f;
    float u = k0 * (g + k1 * g * g * g);
    float t = 1.0f - 2.0f / (1.0f + __expf(2.0f * u));  // tanh(u)
    return 0.5f * g * (1.0f + t);
  }
  return g;
}

template <typename OutT>
__device__ __forceinline__ void stage_store(OutT* p, float v);
template <>
__device__ __forceinline__ void stage_store<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
template <>
__device__ __forceinline__ void stage_store<float>(float* p, float v) { *p = v; }


__device__ __forceinline__ float feature_bias(const GemmParams& p, int f_glob) {
  return (p.bias != nullptr && f_glob < p.n) ? __bfloat162float(p.bias[f_glob]) : 0.0f;
}

// The output value of one (feature, token) before rounding: + bias, then act(g) * u for a gate/up pair, then the soft-cap.  Every
// route computes it in this order, so their outputs agree bit for bit; rounding to OutT and the residual add follow in the store.
template <bool DUAL>
__device__ __forceinline__ float epi_value(const GemmParams& p, float g, float u, float bias) {
  float y = g + bias;
  if (DUAL) y = apply_act(p.act, y) * u;
  if (p.softcap > 0.f) y = p.softcap * tanhf(y / p.softcap);
  return y;
}

// ---- LoRA term (adapted quantised launches)
// A kernel parameter of its own, next to GemmParams, so the launches without an adapter keep their parameter layout.
struct LoraParams {
  const float* u;            // fp32 [rows, ld_u] = x A^T; a pair's second adapter starts at column r
  const __nv_bfloat16* b;    // bf16 [n, r]: scale * B, one row per output feature
  const __nv_bfloat16* b2;   // the pair's second weight
  int r, ld_u;               // r: multiple of 8
};

__device__ __forceinline__ void lora_dot8(const float* u, const uint4 bw, float& acc) {
  const float4 u0 = __ldg(reinterpret_cast<const float4*>(u)), u1 = __ldg(reinterpret_cast<const float4*>(u) + 1);
  acc = fmaf(u0.x, bf16_lo(bw.x), acc); acc = fmaf(u0.y, bf16_hi(bw.x), acc);
  acc = fmaf(u0.z, bf16_lo(bw.y), acc); acc = fmaf(u0.w, bf16_hi(bw.y), acc);
  acc = fmaf(u1.x, bf16_lo(bw.z), acc); acc = fmaf(u1.y, bf16_hi(bw.z), acc);
  acc = fmaf(u1.z, bf16_lo(bw.w), acc); acc = fmaf(u1.w, bf16_hi(bw.w), acc);
}

// Epilogue thread of feature f_glob, token rows row0 .. row0 + rows - 1 (rows <= 16): g[j] += sum_i u[row0 + j, i] * b[f_glob, i]
// (and u / b2 for a pair's second accumulator).  Each thread streams its own contiguous row of B; the u loads are the same
// address across the warp (broadcast).
template <bool DUAL>
__device__ __forceinline__ void lora_add16(const LoraParams& l, int n, int f_glob, int row0, int rows, float (&g)[16], float (&u)[16]) {
  if (f_glob >= n) return;
  const size_t fo = static_cast<size_t>(f_glob) * l.r;
#pragma unroll 1
  for (int i = 0; i < l.r; i += 8) {
    const uint4 bw = __ldg(reinterpret_cast<const uint4*>(l.b + fo + i));
    uint4 bw2;
    if (DUAL) bw2 = __ldg(reinterpret_cast<const uint4*>(l.b2 + fo + i));
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      if (j < rows) {
        const float* ur = l.u + static_cast<size_t>(row0 + j) * l.ld_u + i;
        lora_dot8(ur, bw, g[j]);
        if (DUAL) lora_dot8(ur + l.r, bw2, u[j]);
      }
    }
  }
}

// ---- tile walk
struct TileInfo {
  int n0, w_row, row_base, rows_valid, mt;   // rows_valid <= 0: the tile holds no token rows
};

// Token tile `mt` of 128-feature tile `nt` of `expert`: the token rows of a dense launch, or of the expert in one of the grouped
// layouts.  Offsets: expert_offsets[e] .. [e + 1].  Scatter (expert_stride > 0): expert e owns rows from e * stride, and
// expert_offsets[e] is its row count, written by atomics (no __ldg).
__device__ __forceinline__ TileInfo tile_at(const GemmParams& p, int nt, int mt, int expert, int BN) {
  TileInfo ti;
  ti.mt = mt;
  ti.n0 = nt * kTileM;
  ti.row_base = 0;
  ti.rows_valid = p.m;
  if (p.expert_offsets != nullptr) {
    if (p.expert_stride > 0) {
      ti.row_base = expert * p.expert_stride;
      ti.rows_valid = __ldcg(p.expert_offsets + expert);
    } else {
      const int lo = __ldg(p.expert_offsets + expert), hi = __ldg(p.expert_offsets + expert + 1);
      ti.row_base = lo;
      ti.rows_valid = hi - lo;
    }
  }
  ti.rows_valid -= mt * BN;
  ti.row_base += mt * BN;
  if (ti.rows_valid > BN) ti.rows_valid = BN;
  ti.w_row = expert * p.n + ti.n0;
  return ti;
}

// Tile t of the persistent kernels' list: feature tile fastest, then token tile, then expert.
__device__ __forceinline__ TileInfo decode_tile(const GemmParams& p, int t, int tiles_n, int tiles_m, int BN) {
  const int rest = t / tiles_n;
  return tile_at(p, t % tiles_n, rest % tiles_m, rest / tiles_m, BN);
}

// The split-K kernels' CTA: blockIdx = (feature tile, expert, token tile * splits + split); it reduces k-blocks
// [kb_begin, kb_begin + num_kb), and num_kb may be 0 or less for a trailing split, which then contributes zeros.
struct SplitTile {
  TileInfo ti;
  int split, kb_begin, num_kb;
};

__device__ __forceinline__ SplitTile splitk_tile(const GemmParams& p, int BN) {
  SplitTile st;
  st.split = blockIdx.z % p.splits;
  st.ti = tile_at(p, blockIdx.x, blockIdx.z / p.splits, blockIdx.y, BN);
  const int kb_total = (p.k + kBlockK - 1) / kBlockK;
  const int kb_per = (kb_total + p.splits - 1) / p.splits;
  st.kb_begin = st.split * kb_per;
  st.num_kb = min(kb_per, kb_total - st.kb_begin);
  return st;
}

// ---- epilogue stores
// Output staging tile of the persistent kernels: up to 64 token rows of 128 features, `ld` elements apart.
__host__ __device__ constexpr int stg_rows(int BN) { return BN < 64 ? BN : 64; }
__host__ __device__ constexpr int staging_bytes(int BN, int ld, int out_bytes) { return stg_rows(BN) * ld * out_bytes; }

// MMA warpgroup (thread `et` of 128): staging rows [0, rows) of pitch `ld_stg` -> output rows row0.. of features n0..n0+127, as
// 16-byte chunks of 8 features (16 chunks per row, 8 rows per pass).  The residual is added to the staged (already rounded)
// value and the sum is rounded again.  A row goes to `out` + row * ld_out, or (EP return) to row_dst[row], possibly peer memory.
template <typename OutT>
__device__ __forceinline__ void write_rows(const GemmParams& p, const OutT* stg, int ld_stg, int et, int n0, int row0, int rows) {
  constexpr int kVec = 8;
  constexpr int kChunks = kTileM / kVec;                  // 16
  constexpr int kRowsPerIter = kEpiThreads / kChunks;     // 8
  const int ch = et % kChunks;
  const int f0 = n0 + ch * kVec;
  if (f0 >= p.n) return;
  for (int r = et / kChunks; r < rows; r += kRowsPerIter) {
    const size_t row = static_cast<size_t>(row0 + r);
    float vals[kVec];
    if (sizeof(OutT) == 2) {
      const uint4 raw = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(stg) + r * ld_stg + ch * kVec);
      const uint32_t w4[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) { vals[2 * j] = bf16_lo(w4[j]); vals[2 * j + 1] = bf16_hi(w4[j]); }
    } else {
      const float4 a = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(stg) + r * ld_stg + ch * kVec);
      const float4 b = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(stg) + r * ld_stg + ch * kVec + 4);
      vals[0] = a.x; vals[1] = a.y; vals[2] = a.z; vals[3] = a.w;
      vals[4] = b.x; vals[5] = b.y; vals[6] = b.z; vals[7] = b.w;
    }
    if (p.residual != nullptr) {
      const uint4 rr = *reinterpret_cast<const uint4*>(p.residual + row * p.ld_res + f0);
      const uint32_t w4[4] = {rr.x, rr.y, rr.z, rr.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) { vals[2 * j] += bf16_lo(w4[j]); vals[2 * j + 1] += bf16_hi(w4[j]); }
    }
    OutT* orow = p.row_dst != nullptr ? reinterpret_cast<OutT*>(__ldg(p.row_dst + row)) : reinterpret_cast<OutT*>(p.out) + row * p.ld_out;
    if (sizeof(OutT) == 2) {
      uint4 o;
      o.x = pack_bf16(vals[0], vals[1]); o.y = pack_bf16(vals[2], vals[3]);
      o.z = pack_bf16(vals[4], vals[5]); o.w = pack_bf16(vals[6], vals[7]);
      *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(orow) + f0) = o;
    } else {
      float* o = reinterpret_cast<float*>(orow) + f0;
      *reinterpret_cast<float4*>(o) = make_float4(vals[0], vals[1], vals[2], vals[3]);
      *reinterpret_cast<float4*>(o + 4) = make_float4(vals[4], vals[5], vals[6], vals[7]);
    }
  }
}

// MMA warpgroup, one feature per thread: the tile's fp32 accumulator in shared memory (`acc`, [col][128 features], a pair's
// second matrix at column BN) -> epilogue values -> staging tile [stg_rows(BN)][128] -> global, one staging tile of token rows
// at a time.  Ends with the staging tile and the accumulator free again.  LORA: the adapter term joins the accumulator first.
template <int BN, bool DUAL, typename OutT, bool LORA = false>
__device__ __forceinline__ void store_acc_tile(const GemmParams& p, const float* acc, OutT* stg, const TileInfo& ti,
                                               const LoraParams* lora = nullptr) {
  constexpr int STG_ROWS = stg_rows(BN);
  const int f_local = threadIdx.x;
  const float bias = feature_bias(p, ti.n0 + f_local);
#pragma unroll 1
  for (int c0 = 0; c0 < BN; c0 += STG_ROWS) {
    if (c0 >= ti.rows_valid) break;
#pragma unroll 1
    for (int c = c0; c < c0 + STG_ROWS; c += 16) {
      if (c >= ti.rows_valid) break;
      float g[16], u[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        g[j] = acc[(c + j) * kTileM + f_local];
        if (DUAL) u[j] = acc[(BN + c + j) * kTileM + f_local];
      }
      if constexpr (LORA) lora_add16<DUAL>(*lora, p.n, ti.n0 + f_local, ti.row_base + c, ti.rows_valid - c, g, u);
#pragma unroll
      for (int j = 0; j < 16; ++j) stage_store<OutT>(&stg[(c - c0 + j) * kTileM + f_local], epi_value<DUAL>(p, g[j], u[j], bias));
    }
    named_bar_sync(1, kEpiThreads);
    write_rows<OutT>(p, stg, kTileM, f_local, ti.n0, ti.row_base + c0, min(STG_ROWS, ti.rows_valid - c0));
    named_bar_sync(1, kEpiThreads);
  }
}

// ---- completion signal
// One thread, after the stores it reports are fenced with system scope: `n` more tiles of the grid are stored.  The arrival that
// completes signal_tiles resets the counter and raises the consumer flag(s) with system scope: every peer flag of the EP return,
// else the fused stage boundary's flag, counting (+1, graph-replay safe) when signal_value is 0 and set to signal_value otherwise.
__device__ __forceinline__ void publish_tiles_done(const GemmParams& p, unsigned int n) {
  const unsigned int done = atomicAdd(p.done_counter, n) + n;
  if (done != p.signal_tiles) return;
  *p.done_counter = 0u;
  __threadfence_system();
  if (p.signal_peers != nullptr) {
    for (int i = 0; i < p.num_signal_peers; ++i) atomicAdd_system(reinterpret_cast<unsigned int*>(__ldg(p.signal_peers + i)), 1u);
  } else if (p.signal_value == 0u) {
    atomicAdd_system(p.signal_flag, 1u);
  } else {
    st_release_sys(p.signal_flag, p.signal_value);
  }
}

// Workspace split-K route, on the MMA warpgroup once the tile's accumulator is in shared memory (`acc`, fp32 [col][128 features],
// a pair's second matrix at column BN): write the raw partial, take the tile's ticket, and the last of its `splits` CTAs sums the
// partials in split order, runs the epilogue through the staging tile `stg` [BN][128] and reports the tile as stored.  LORA: the
// adapter term joins the reduced sum (once per tile, not per split).
template <int BN, bool DUAL, typename OutT, bool LORA = false>
__device__ __forceinline__ void run_epilogue(const GemmParams& p, const float* acc, OutT* stg, uint32_t* flag_smem, const TileInfo& ti,
                                             int split, const LoraParams* lora = nullptr) {
  constexpr int kTileFloats = BN * (DUAL ? 2 : 1) * kTileM;
  const int f_local = threadIdx.x;   // 0..127: feature within the tile
  const int tile = (blockIdx.y * gridDim.x + blockIdx.x) * (gridDim.z / p.splits) + ti.mt;
  const float* ws0 = p.workspace + static_cast<size_t>(tile) * p.splits * kTileFloats;
  float* ws = p.workspace + (static_cast<size_t>(tile) * p.splits + split) * kTileFloats;
#pragma unroll 1
  for (int c = 0; c < BN * (DUAL ? 2 : 1); ++c) ws[c * kTileM + f_local] = acc[c * kTileM + f_local];
  __threadfence();
  named_bar_sync(1, kEpiThreads);
  if (f_local == 0) {
    unsigned int* ctr = p.tile_counters + tile;
    const unsigned int old = atomicAdd(ctr, 1u);
    const bool last = (old == static_cast<unsigned int>(p.splits - 1));
    if (last) *ctr = 0u;  // self-reset for the next launch
    *flag_smem = last ? 1u : 0u;
  }
  named_bar_sync(1, kEpiThreads);
  const bool last = *flag_smem != 0u;
  if (last) {
    __threadfence();
    const float bias = feature_bias(p, ti.n0 + f_local);
#pragma unroll 1
    for (int c = 0; c < BN; c += 16) {
      if (c >= ti.rows_valid) break;
      float g[16], u[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) { g[j] = 0.f; u[j] = 0.f; }
      // deterministic split order, but 2 splits x 16 columns of independent L2 loads are in flight
      // per thread before they are consumed (the reduction is latency-, not bandwidth-bound)
      for (int s = 0; s < p.splits; s += 2) {
        const float* w0 = ws0 + static_cast<size_t>(s) * kTileFloats;
        const bool two = (s + 1) < p.splits;
        const float* w1 = two ? w0 + kTileFloats : w0;
        float a0[16], a1[16], b0[16], b1[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          a0[j] = __ldcg(&w0[(c + j) * kTileM + f_local]);
          a1[j] = two ? __ldcg(&w1[(c + j) * kTileM + f_local]) : 0.f;
          if (DUAL) {
            b0[j] = __ldcg(&w0[(BN + c + j) * kTileM + f_local]);
            b1[j] = two ? __ldcg(&w1[(BN + c + j) * kTileM + f_local]) : 0.f;
          }
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          g[j] = (g[j] + a0[j]) + a1[j];
          if (DUAL) u[j] = (u[j] + b0[j]) + b1[j];
        }
      }
      if constexpr (LORA) lora_add16<DUAL>(*lora, p.n, ti.n0 + f_local, ti.row_base + c, ti.rows_valid - c, g, u);
#pragma unroll
      for (int j = 0; j < 16; ++j) stage_store<OutT>(&stg[(c + j) * kTileM + f_local], epi_value<DUAL>(p, g[j], u[j], bias));
    }
    named_bar_sync(1, kEpiThreads);
    write_rows<OutT>(p, stg, kTileM, f_local, ti.n0, ti.row_base, ti.rows_valid);
  }
  // fused stage boundary: the tile's last CTA reports it once its rows are fenced
  if (p.signal_flag != nullptr) {
    __threadfence_system();
    named_bar_sync(1, kEpiThreads);
    if (f_local == 0 && last) publish_tiles_done(p, 1u);
  }
}

// ---- host: token tile x pair x output type -> kernel instance
template <int BN_, bool DUAL_, typename OutT_>
struct TileCfg {
  static constexpr int BN = BN_;
  static constexpr bool DUAL = DUAL_;
  using OutT = OutT_;
};

template <bool DUAL, typename OutT, int MaxBN, typename F>
cudaError_t dispatch_bn(int bn, F& launch) {
  switch (bn) {
    case 16: return launch(TileCfg<16, DUAL, OutT>{});
    case 32: return launch(TileCfg<32, DUAL, OutT>{});
    case 64:
      if constexpr (MaxBN >= 64) return launch(TileCfg<64, DUAL, OutT>{});
      break;
    case 128:
      if constexpr (MaxBN >= 128) return launch(TileCfg<128, DUAL, OutT>{});
      break;
  }
  return cudaErrorInvalidValue;
}

// Calls launch(TileCfg<BN, DUAL, OutT>{}) for the family's kernel instance: fp32 output (single matrix only), gate/up pair
// into bf16, or a single matrix into bf16.  A family compiles token tiles up to MaxBN (MaxBNDual for a pair); any other bn
// has no instance and returns cudaErrorInvalidValue.
template <int MaxBN, int MaxBNDual, typename F>
cudaError_t dispatch_tile(int bn, bool dual, bool out_fp32, F launch) {
  if (out_fp32) return dispatch_bn<false, float, MaxBN>(bn, launch);
  if (dual) return dispatch_bn<true, __nv_bfloat16, MaxBNDual>(bn, launch);
  return dispatch_bn<false, __nv_bfloat16, MaxBN>(bn, launch);
}

}  // namespace gemm
}  // namespace b200
