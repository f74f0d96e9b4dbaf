"""CPU checks of the fp64 MoE oracle in ``moe_oracle.py`` (the helpers ``test_moe_block_gpu.py`` trusts): the tie-aware top-k
check, group masking, the routing-weight rules, the rounding checks and the expert-output allowance."""
import torch

import moe_oracle as O
from mlx_sharding_b200.utils.quant import from_mxfp8, to_mxfp8


def _l(*rows):
    return torch.tensor(rows, dtype=torch.float64)


def test_exact_tie_accepts_either_order():
    l = _l([1.0, 1.0, 0.0, -1.0])
    eps = torch.zeros_like(l)
    for sel in ([[0]], [[1]]):
        ok, clear, same = O.check_topk(l, eps, torch.tensor(sel), 1)
        assert ok.all()
        assert not clear.any()      # a tie is never "clear", so neither order is demanded
    ok, _, _ = O.check_topk(l, eps, torch.tensor([[2]]), 1)
    assert not ok.any()


def test_selection_off_by_more_than_eps_is_rejected():
    l = _l([1.0, 1.0 + 3e-4, 0.0, -1.0])
    eps = torch.full_like(l, 1e-4)
    ok, clear, same = O.check_topk(l, eps, torch.tensor([[0]]), 1)
    assert not ok.any()             # 3e-4 apart, each side known to 1e-4
    ok, clear, same = O.check_topk(l, eps, torch.tensor([[1]]), 1)
    assert ok.all() and clear.all() and same.all()
    # within the error both are fine and neither is demanded
    eps = torch.full_like(l, 2e-4)
    assert O.check_topk(l, eps, torch.tensor([[0]]), 1)[0].all()
    assert not O.check_topk(l, eps, torch.tensor([[1]]), 1)[1].any()


def test_duplicate_experts_are_rejected():
    l = _l([3.0, 2.0, 1.0, 0.0])
    assert not O.check_topk(l, torch.zeros_like(l), torch.tensor([[0, 0]]), 2)[0].any()
    assert O.check_topk(l, torch.zeros_like(l), torch.tensor([[1, 0]]), 2)[0].all()


def test_group_masking():
    # 4 groups of 2, keep the top 2 groups by their maximum: groups 0 (max 5) and 2 (max 4)
    l = _l([5.0, -9.0, 3.5, 3.4, 4.0, 0.0, 1.0, 1.0])
    eps = torch.zeros_like(l)
    kw = dict(n_group=4, topk_group=2)
    assert O.check_topk(l, eps, torch.tensor([[0, 4, 5]]), 3, **kw)[0].all()
    # 2 and 3 are the next-best experts but their group (max 3.5) is masked
    assert not O.check_topk(l, eps, torch.tensor([[0, 4, 2]]), 3, **kw)[0].any()
    # unselected experts of an unchosen group do not count against the selection
    ok, clear, same = O.check_topk(l, eps, torch.tensor([[0, 4, 1]]), 3, **kw)
    assert not ok.any()             # 1 (score -9) was chosen over 5 (score 0) of a chosen group
    ok, clear, same = O.check_topk(l, eps, torch.tensor([[4, 0, 5]]), 3, **kw)
    assert ok.all() and clear.all() and same.all()
    # a group tie within the error: either group may be chosen, and its experts are then the valid picks
    l = _l([5.0, -9.0, 4.0 - 1e-6, 3.4, 4.0, 0.0, 1.0, 1.0])
    eps = torch.full_like(l, 1e-5)
    assert O.check_topk(l, eps, torch.tensor([[0, 4, 5]]), 3, **kw)[0].all()
    ok, clear, _ = O.check_topk(l, eps, torch.tensor([[0, 2, 3]]), 3, **kw)
    assert ok.all() and not clear.any()
    # a group that cannot be among the top two is never valid
    assert not O.check_topk(l, eps, torch.tensor([[0, 6, 7]]), 3, **kw)[0].any()


def test_routing_weights_scaling_and_norm_topk():
    l = _l([2.0, 1.0, 0.0, -1.0], [0.0, 0.0, 0.0, 0.0])
    idx = torch.tensor([[0, 2, 4], [3, 1, 4]])
    p = torch.softmax(l, -1)
    w = O.routing_weights(l, idx, 2, 1, 16.0, False)
    assert torch.allclose(w[:, :2], torch.stack([p[0, [0, 2]], p[1, [3, 1]]]) * 16.0)
    assert (w[:, 2] == 1).all()
    w = O.routing_weights(l, idx, 2, 1, 16.0, True)      # renormalised; the scaling is not applied on top
    assert torch.allclose(w[:, :2].sum(-1), torch.ones(2, dtype=torch.float64))
    assert torch.allclose(w[0, 0] / w[0, 1], p[0, 0] / p[0, 2])
    w = O.routing_weights(l, idx[:, :1], 1, 0, 2.0, True)  # top-1: norm_topk does not apply
    assert torch.allclose(w[:, 0], torch.stack([p[0, 0], p[1, 3]]) * 2.0)


def test_route_logit_bound_covers_fp32_sums():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(16, 2048, generator=g).to(torch.bfloat16)
    gw = (torch.randn(64, 2048, generator=g) * 0.05).to(torch.bfloat16)
    l, eps = O.route_logits(x, gw)
    # the kernel's accumulation order: 32 lanes, each adding its 8-wide vectors in turn, then a shuffle tree
    p = x.float()[:, None, :] * gw.float()[None, :, :]
    lanes = p.view(16, 64, 2048 // 256, 32, 8).permute(0, 1, 3, 2, 4).reshape(16, 64, 32, -1)
    acc = torch.zeros(16, 64, 32)
    for i in range(lanes.shape[-1]):
        acc = acc + lanes[..., i]
    while acc.shape[-1] > 1:
        acc = acc[..., : acc.shape[-1] // 2] + acc[..., acc.shape[-1] // 2:]
    err = (acc[..., 0].double() - l).abs()
    assert (err <= eps).all()
    assert (err.max() < eps.min())      # the bound is not vacuous either: the real error is far below it


def test_assert_rounded_admits_only_the_straddled_neighbour():
    one = torch.tensor([1.0], dtype=torch.float64)
    mid = one + 2.0 ** -8              # exactly between 1 and the next bf16
    dv = torch.tensor([1e-6], dtype=torch.float64)
    for got in (1.0, 1.0 + 2.0 ** -7):
        assert O.assert_rounded(torch.tensor([got], dtype=torch.bfloat16), mid, dv, "tie") == 1
    try:
        O.assert_rounded(torch.tensor([1.0 + 2.0 ** -7], dtype=torch.bfloat16), one + 2.0 ** -10, dv, "clear")
    except AssertionError:
        pass
    else:
        raise AssertionError("a value that is not a rounding of the reference was accepted")


def test_bf16_ulp():
    v = torch.tensor([1.0, 1.5, 0.75, -3.0, 2.0 ** -20], dtype=torch.float64)
    assert O.bf16_ulp(v).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -8, 2.0 ** -6, 2.0 ** -27]


def _bank(E, I, H, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(E, *s, generator=g) * 0.03).to(torch.bfloat16) for s in ((I, H), (I, H), (H, I))]


def _fp32_block(x, idx, w, bank, fp8):
    """The block the way the kernels store it: fp32 GEMMs, bf16 h, MXFP8 operands when ``fp8``, fp32 combine."""
    q = (lambda v: from_mxfp8(*to_mxfp8(v))) if fp8 else (lambda v: v.float())
    Wg, Wu, Wd = (q(b) for b in bank)
    xs = q(x)
    y = torch.zeros(x.shape, dtype=torch.float32)
    for t in range(x.shape[0]):
        for s in range(idx.shape[1]):
            e = int(idx[t, s])
            h = (torch.nn.functional.silu(xs[t] @ Wg[e].t()) * (xs[t] @ Wu[e].t())).to(torch.bfloat16)
            y[t] += float(w[t, s]) * (q(h[None])[0] @ Wd[e].t())
    return y.to(torch.bfloat16)


def test_expert_oracle_admits_an_fp32_block_and_its_controls_fail():
    torch.manual_seed(0)
    T, H, I, E, k = 3, 256, 128, 8, 3
    bank = _bank(E, I, H, 1)
    x = torch.randn(T, H).to(torch.bfloat16)
    idx = torch.tensor([[0, 3, 5], [1, 3, 7], [5, 2, 0]])
    w = torch.tensor([[0.5, 0.2, 0.05], [0.3, 0.3, 0.1], [0.6, 0.02, 0.01]], dtype=torch.float64)
    for fmt in ("bf16", "mxfp8"):
        fp8 = fmt == "mxfp8"
        if fp8:
            wts = lambda e: tuple(from_mxfp8(*to_mxfp8(b[e]), dtype=torch.float64) for b in bank)
        else:
            wts = lambda e: tuple(b[e].double() for b in bank)
        ref, allow, _, kept = O.expert_oracle(x, idx, w, wts, fmt, keep=O.control_pairs(w))
        got = _fp32_block(x, idx, w.float(), bank, fp8)
        tol = O.tolerance(ref, allow)
        assert O.err_ratio(got, ref, tol) <= 1
        O.assert_controls_fail(got, ref, tol, w, kept)
