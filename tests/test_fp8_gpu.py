"""Block-scaled FP8 (MXFP8) on sm_90a: the activation quantiser, the wgmma e4m3 GEMM with per-32 block scales (dense, DUAL,
grouped with offsets, grouped scatter layout) against fp32 matmuls of the *same* MXFP8 operands, and the error budget of
FP8 expert banks against the bf16 / MLX-affine oracle."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, device=DEV, generator=g) * scale).to(torch.bfloat16)


def test_quant_kernel_matches_host_conversion():
    from mlx_sharding_b200.ops import b200
    from mlx_sharding_b200.utils.quant import from_mxfp8, to_mxfp8

    x = rnd(37, 1408 - 1408 % 128 + 128, scale=2.0)
    x[3, :64] = 0
    x[5] *= 1e-3
    q, sf = b200.quant_mxfp8(x)
    q2, sf2 = to_mxfp8(x)
    assert torch.equal(sf, sf2)
    assert torch.equal(q, q2)
    rel = (from_mxfp8(q, sf) - x.float()).abs().max() / x.float().abs().max()
    assert rel < 0.07


@pytest.mark.parametrize("T,N,K,dual", [(64, 256, 512, False), (5, 1408, 2048, True), (200, 2048, 1408 + 128, False)])
def test_fp8_gemm_dense(T, N, K, dual):
    from mlx_sharding_b200.ops import b200
    from mlx_sharding_b200.utils.quant import from_mxfp8, to_mxfp8

    C = b200.load_extension()
    N = (N + 127) // 128 * 128
    x, w, w2 = rnd(T, K, seed=1), rnd(N, K, scale=0.05, seed=2), rnd(N, K, scale=0.05, seed=3)
    xq, xsf = C.quant_mxfp8(x)
    wq, wsf = to_mxfp8(w)
    xd, wd = from_mxfp8(xq, xsf), from_mxfp8(wq, wsf)
    if dual:
        w2q, w2sf = to_mxfp8(w2)
        got = C.linear_fp8(xq, xsf, wq, wsf, w2q, w2sf, None, 0, None, 1, False)
        g = xd @ wd.t()
        ref = torch.nn.functional.silu(g) * (xd @ from_mxfp8(w2q, w2sf).t())
    else:
        res = rnd(T, N, seed=4)
        got = C.linear_fp8(xq, xsf, wq, wsf, None, None, None, 0, res, 0, False)
        ref = xd @ wd.t() + res.float()
    err = (got.float() - ref).abs().max().item()
    assert err < 2e-2 * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize("scatter", [False, True])
def test_fp8_gemm_grouped(scatter):
    from mlx_sharding_b200.ops import b200
    from mlx_sharding_b200.utils.quant import from_mxfp8, to_mxfp8

    C = b200.load_extension()
    E, N, K, stride = 6, 256, 512, 64
    counts = torch.tensor([3, 0, 64, 17, 1, 40], dtype=torch.int32, device=DEV)
    w = rnd(E, N, K, scale=0.05, seed=2)
    wq, wsf = to_mxfp8(w)
    if scatter:
        x = rnd(E * stride, K, seed=1)
        xq, xsf = C.quant_mxfp8(x)
        got = C.linear_fp8(xq, xsf, wq, wsf, None, None, counts, stride, None, 0, True, int(counts.sum()), stride)
        rows = [(e * stride, int(counts[e])) for e in range(E)]
    else:
        offs = torch.cat([torch.zeros(1, dtype=torch.int32, device=DEV), counts.cumsum(0).to(torch.int32)])
        R = int(offs[-1])
        x = rnd(R, K, seed=1)
        xq, xsf = C.quant_mxfp8(x)
        got = C.linear_fp8(xq, xsf, wq, wsf, None, None, offs, 64, None, 0, True, 0, 0)
        rows = [(int(offs[e]), int(counts[e])) for e in range(E)]
    xd, wd = from_mxfp8(xq, xsf), from_mxfp8(wq, wsf)
    for e, (r0, n) in enumerate(rows):
        if n:
            ref = xd[r0:r0 + n] @ wd[e].t()
            err = (got[r0:r0 + n] - ref).abs().max().item()
            assert err < 1e-2 * max(1.0, ref.abs().max().item()), (e, err)


def test_fp8_expert_bank_error_budget():
    """MoE block with the expert banks converted to MXFP8 (from bf16 here; the same conversion runs on dequantised MLX int4/int8
    banks) vs the bf16 block: relative error of the block output (before the residual) stays within the documented budget."""
    from mlx_sharding_b200.ops import b200
    from mlx_sharding_b200.ops.weights import LinearWeight

    H, I, E, k = 2048, 1408, 16, 4
    gw = rnd(E, H, scale=0.05)
    bank = (LinearWeight(weight=rnd(E, I, H, scale=0.03, seed=1)), LinearWeight(weight=rnd(E, I, H, scale=0.03, seed=2)),
            LinearWeight(weight=rnd(E, H, I, scale=0.03, seed=3)))
    fp8 = tuple(W.to_mxfp8() for W in bank)
    rk = dict(top_k=k, method="greedy", n_group=1, topk_group=1, scaling=1.0, norm_topk=False)
    for T in (64, 300):       # scatter path and permutation path
        x = rnd(T, H)
        ref = b200.moe_block(x, gw, rk, *bank, "silu")
        got = b200.moe_block(x, gw, rk, *fp8, "silu")
        rel = ((got.float() - ref.float()).norm() / ref.float().norm()).item()
        assert rel < 0.09, rel     # e4m3 operands on both sides, two chained GEMMs: ~6.5 % of the block output norm
