"""Launch routes chosen by the GEMM planner (``gemm_plan`` in ops/csrc/gemm_host.cu), pinned at the shapes the models run.

The planner is a pure host function of the launch shape and the SM count, so these tests call it through the extension's
``gemm_plan`` binding without a GPU.  Arguments are the planner's inputs as the bindings fill them: ``max_rows`` is the token
count of a dense launch (``linear``, ``linear_q``, dense ``linear_fp8``) and the per-expert row bound of a grouped one;
``expected_rows`` is the grouped launches' row estimate (``T * top_k``, or the permuted row count).

Each expected tuple is ``(route, bn, splits, grid, cluster, workspace_floats)``.  The rules they follow:
  * token tile ``pick(r)`` = 16 / 32 / 64 / 128 for r <= 16 / 32 / 64 / more; grouped launches use
    ``pick(min(max_rows, max(64, 2 * ceil(expected_rows / experts))))``; capped at 64 for a gate/up pair (MXFP8: 64, pair 32);
  * automatic split-K (bf16 up to 256 rows, quantised up to 32, never grouped or MXFP8): double ``s`` while
    ``tiles_n * 2s <= SMs``, ``k_blocks / 2s >= 8`` and ``s < 4``; explicit splits are clamped to the k-block count;
  * splits = 1: persistent, ``min(tiles, SMs)`` CTAs; bf16 with splits <= 8 and ``bn * (1 + pair) <= 128``: cluster
    split-K with ``splits`` CTAs per cluster; otherwise the fp32 workspace split-K.
"""
import os

import pytest

from mlx_sharding_b200.ops import b200

pytestmark = pytest.mark.skipif(not os.path.exists(b200._SO), reason="_b200_C.so is not built")

P, C, W = "persistent", "cluster", "workspace"

# [N, K] of the projections (pair: gate/up streamed together)
DSV2_LITE = {"qkv_a": (3648, 2048), "kv_b": (4096, 512), "o": (2048, 2048), "shared_gate_up": (2816, 2048, True),
             "shared_down": (2048, 2816), "lm_head": (102400, 2048)}
LLAMA3_8B = {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (14336, 4096, True), "down": (4096, 14336),
             "lm_head": (128256, 4096)}


def plan(kind, max_rows, shape, sm_count=132, **kw):
    n, k, pair = (shape + (False,))[:3]
    p = b200.load_extension().gemm_plan(kind, max_rows, n, k, pair=pair, sm_count=sm_count, **kw)
    return p["route"], p["bn"], p["splits"], tuple(p["grid"]), p["cluster"], p["workspace_floats"]


@pytest.mark.parametrize("T, name, expected", [
    # T = 1 and 16: 16-token tile; every projection but kv_b (8 k-blocks) and the LM head (800 tiles) splits K four ways
    (1, "qkv_a", (C, 16, 4, (29, 1, 4), 4, 0)),
    (1, "kv_b", (P, 16, 1, (32, 1, 1), 1, 0)),
    (1, "o", (C, 16, 4, (16, 1, 4), 4, 0)),
    (1, "shared_gate_up", (C, 16, 4, (22, 1, 4), 4, 0)),
    (1, "shared_down", (C, 16, 4, (16, 1, 4), 4, 0)),
    (1, "lm_head", (P, 16, 1, (132, 1, 1), 1, 0)),
    (16, "qkv_a", (C, 16, 4, (29, 1, 4), 4, 0)),
    (16, "o", (C, 16, 4, (16, 1, 4), 4, 0)),
    (16, "shared_gate_up", (C, 16, 4, (22, 1, 4), 4, 0)),
    (16, "lm_head", (P, 16, 1, (132, 1, 1), 1, 0)),
    # T = 64: the pair's two 64-token partial tiles still fit the cluster reduction (64 * 2 <= 128)
    (64, "qkv_a", (C, 64, 4, (29, 1, 4), 4, 0)),
    (64, "kv_b", (P, 64, 1, (32, 1, 1), 1, 0)),
    (64, "o", (C, 64, 4, (16, 1, 4), 4, 0)),
    (64, "shared_gate_up", (C, 64, 4, (22, 1, 4), 4, 0)),
    (64, "shared_down", (C, 64, 4, (16, 1, 4), 4, 0)),
    # T = 256: the last automatic split-K batch; 128-token tiles (64 for the pair) in 2 (4) token tiles
    (256, "qkv_a", (C, 128, 4, (29, 1, 8), 4, 0)),
    (256, "kv_b", (P, 128, 1, (64, 1, 1), 1, 0)),
    (256, "o", (C, 128, 4, (16, 1, 8), 4, 0)),
    (256, "shared_gate_up", (C, 64, 4, (22, 1, 16), 4, 0)),
    (256, "lm_head", (P, 128, 1, (132, 1, 1), 1, 0)),
])
def test_deepseek_v2_lite_decode(T, name, expected):
    assert plan("bf16", T, DSV2_LITE[name]) == expected


@pytest.mark.parametrize("sm_count, name, expected", [
    (132, "qkv", (C, 16, 2, (48, 1, 2), 2, 0)),
    (132, "o", (C, 16, 4, (32, 1, 4), 4, 0)),
    (132, "gate_up", (P, 16, 1, (112, 1, 1), 1, 0)),
    (132, "down", (C, 16, 4, (32, 1, 4), 4, 0)),
    (132, "lm_head", (P, 16, 1, (132, 1, 1), 1, 0)),
    # 114 SMs: four splits of o would need 128 CTAs
    (114, "qkv", (C, 16, 2, (48, 1, 2), 2, 0)),
    (114, "o", (C, 16, 2, (32, 1, 2), 2, 0)),
    (114, "gate_up", (P, 16, 1, (112, 1, 1), 1, 0)),
    (114, "lm_head", (P, 16, 1, (114, 1, 1), 1, 0)),
])
def test_llama3_8b_decode(sm_count, name, expected):
    assert plan("bf16", 16, LLAMA3_8B[name], sm_count=sm_count) == expected


def test_sm_count_changes_the_split():
    assert plan("bf16", 1, DSV2_LITE["qkv_a"], sm_count=114) == (C, 16, 2, (29, 1, 2), 2, 0)
    assert plan("bf16", 1, DSV2_LITE["o"], sm_count=114) == (C, 16, 4, (16, 1, 4), 4, 0)


@pytest.mark.parametrize("sm_count", [132, 114])
def test_prefill(sm_count):
    assert plan("bf16", 2048, DSV2_LITE["o"], sm_count) == (P, 128, 1, (sm_count, 1, 1), 1, 0)
    assert plan("bf16", 2048, DSV2_LITE["shared_gate_up"], sm_count) == (P, 64, 1, (sm_count, 1, 1), 1, 0)
    assert plan("bf16", 2048, LLAMA3_8B["down"], sm_count) == (P, 128, 1, (sm_count, 1, 1), 1, 0)
    # one row above the automatic split-K range
    assert plan("bf16", 257, DSV2_LITE["o"], sm_count) == (P, 128, 1, (min(48, sm_count), 1, 1), 1, 0)


def test_explicit_splits():
    # more than 8 splits: only the workspace reduction takes them (the 16-way split of the GEMM sweep)
    assert plan("bf16", 64, DSV2_LITE["o"], splits=16) == (W, 64, 16, (16, 1, 16), 1, 16 * 16 * 64 * 128)
    assert plan("bf16", 64, DSV2_LITE["o"], splits=8) == (C, 64, 8, (16, 1, 8), 8, 0)
    assert plan("bf16", 24, (128, 1408, True), splits=3) == (C, 32, 3, (1, 1, 3), 3, 0)
    # clamped to the k-block count (4), and splits = 1 forces the persistent kernel
    assert plan("bf16", 8, (256, 256), splits=8) == (C, 16, 4, (2, 1, 4), 4, 0)
    assert plan("bf16", 8, DSV2_LITE["o"], splits=1) == (P, 16, 1, (16, 1, 1), 1, 0)


# DeepSeek-V2-Lite experts: 64 experts, top-6; scatter layout = fixed row stride per expert, max_rows = stride
@pytest.mark.parametrize("kind", ["bf16", "q"])
@pytest.mark.parametrize("stride, T, bn, tiles_m", [(64, 1, 64, 1), (64, 16, 64, 1), (128, 128, 64, 2)])
def test_grouped_scatter(kind, stride, T, bn, tiles_m):
    g = dict(num_experts=64, expected_rows=6 * T)
    assert plan(kind, stride, (1408, 2048, True), **g) == (P, bn, 1, (min(11 * tiles_m * 64, 132), 1, 1), 1, 0)
    assert plan(kind, stride, (2048, 1408), **g) == (P, bn, 1, (132, 1, 1), 1, 0)


def test_grouped_token_tile():
    g = dict(num_experts=64)
    # 2 * ceil(3072 / 64) = 96 rows -> 128-token tile, 64 for the pair
    assert plan("bf16", 512, (2048, 1408), expected_rows=3072, **g) == (P, 128, 1, (132, 1, 1), 1, 0)
    assert plan("bf16", 512, (1408, 2048, True), expected_rows=3072, **g) == (P, 64, 1, (132, 1, 1), 1, 0)
    # a small max_rows caps the tile; grouped launches never split K
    assert plan("bf16", 4, (2048, 1408), expected_rows=24, splits=0, **g) == (P, 16, 1, (132, 1, 1), 1, 0)
    assert plan("q", 16, (1408, 2048, True), expected_rows=96, **g) == (P, 16, 1, (132, 1, 1), 1, 0)
    # without expected rows the tile is sized for max_rows (the standalone GEMM harness)
    assert plan("bf16", 48, (256, 512), num_experts=8) == (P, 64, 1, (16, 1, 1), 1, 0)


@pytest.mark.parametrize("T, name, expected", [
    # up to 32 rows the quantised GEMM takes the bf16 split rule, reduced through the workspace (no cluster variant)
    (16, "o", (W, 16, 4, (32, 1, 4), 1, 32 * 4 * 16 * 128)),
    (16, "gate_up", (P, 16, 1, (112, 1, 1), 1, 0)),
    (64, "o", (P, 64, 1, (32, 1, 1), 1, 0)),
    (64, "gate_up", (P, 64, 1, (112, 1, 1), 1, 0)),
    (64, "down", (P, 64, 1, (32, 1, 1), 1, 0)),
])
def test_quantised(T, name, expected):
    assert plan("q", T, LLAMA3_8B[name]) == expected


def test_quantised_pair_workspace():
    assert plan("q", 16, DSV2_LITE["shared_gate_up"]) == (W, 16, 4, (22, 1, 4), 1, 22 * 4 * 16 * 2 * 128)
    assert plan("q", 33, DSV2_LITE["o"]) == (P, 64, 1, (16, 1, 1), 1, 0)
    assert plan("q", 16, DSV2_LITE["o"], splits=2) == (W, 16, 2, (16, 1, 2), 1, 16 * 2 * 16 * 128)


def test_fp8():
    # dense: pick(T), at most 64 (32 for the pair); never split
    assert plan("fp8", 16, DSV2_LITE["o"]) == (P, 16, 1, (16, 1, 1), 1, 0)
    assert plan("fp8", 16, DSV2_LITE["o"], splits=4) == (P, 16, 1, (16, 1, 1), 1, 0)
    assert plan("fp8", 200, DSV2_LITE["o"]) == (P, 64, 1, (64, 1, 1), 1, 0)
    assert plan("fp8", 200, DSV2_LITE["shared_gate_up"]) == (P, 32, 1, (132, 1, 1), 1, 0)
    # grouped scatter layout, stride 64: the grouped tile (64), capped
    g = dict(num_experts=64, expected_rows=96)
    assert plan("fp8", 64, (1408, 2048, True), **g) == (P, 32, 1, (132, 1, 1), 1, 0)
    assert plan("fp8", 64, (2048, 1408), **g) == (P, 64, 1, (132, 1, 1), 1, 0)
    assert plan("fp8", 64, (2048, 1408), sm_count=114, **g) == (P, 64, 1, (114, 1, 1), 1, 0)
