"""The MoE block (``ops/b200.py::moe_block``: router, grouped gate/up, grouped down, combine) and its three support kernels against
the fp64 oracle of ``moe_oracle.py``, for every expert-bank format (bf16, MXFP8, packed MLX-affine), both row layouts (scatter
for decode batches, counting-sort permutation otherwise), greedy and group-limited routing, and at the batch sizes where the code
changes course: scatter stride 64 / 128 (T = 64 / 65), scatter / permutation (T = 128 / 129), one- / eight-token router CTAs
(T = 1024 / 1025).  Every comparison is made on the kernel's own routing, after checking that routing is a valid top-k, so
near-ties cannot fail a correct kernel; each block comparison is repeated without the residual, where a dropped or mis-weighted
expert is visible, and three perturbed oracles must fail it.  Each test also asserts which row layout it ran."""
import functools

import pytest
import torch

import moe_oracle as O
from mlx_sharding_b200.ops.weights import LinearWeight
from mlx_sharding_b200.utils import quant
from mlx_sharding_b200.utils.quant import from_mxfp8

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 1e-6

GREEDY = dict(method="greedy", n_group=1, topk_group=1, scaling=1.0, norm_topk=False)
# DeepSeek-Coder-V2-Lite: 64 routed experts, top-6, 2 shared experts appended to the bank
LITE = dict(H=2048, I=1408, E=64, extra=2, rk=dict(GREEDY, top_k=6))
# DeepSeek-V2 routing geometry (160 experts in 8 groups, 3 groups kept, routed scaling 16) at I = 512 to bound the bank size
V2 = dict(H=5120, I=512, E=160, extra=2, rk=dict(top_k=6, method="group_limited_greedy", n_group=8, topk_group=3, scaling=16.0,
                                                 norm_topk=False))
LITE_NORM_TOPK = dict(H=2048, I=1408, E=64, extra=0, rk=dict(GREEDY, top_k=4, norm_topk=True))


@pytest.fixture(scope="module")
def B():
    from mlx_sharding_b200.ops import b200

    b200.load_extension()
    return b200


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, device=DEV, generator=g) * scale).to(torch.bfloat16)


@functools.lru_cache(maxsize=None)
def bank(H, I, Et, fmt):
    """Expert bank ``(Wg, Wu, Wd)`` of ``Et`` experts in ``fmt`` and ``weights(e)``: expert ``e``'s three matrices in fp64, as
    the GEMMs see them.  Weight scale 0.03 keeps h and the expert outputs O(1)."""
    if fmt == "mxfp8":
        W = tuple(w.to_mxfp8() for w in bank(H, I, Et, "bf16")[0])
        return W, lambda e: tuple(from_mxfp8(w.mxfp8[0][e], w.mxfp8[1][e], torch.float64) for w in W)
    if fmt == "bf16":
        W = tuple(LinearWeight(weight=w) for w in (rnd(Et, I, H, scale=0.03, seed=1), rnd(Et, I, H, scale=0.03, seed=2),
                                                    rnd(Et, H, I, scale=0.03, seed=3)))
        return W, lambda e: tuple(w.weight[e].double() for w in W)
    bits = int(fmt[len("affine"):])

    def pack(w):   # 8 experts at a time: bounds the fp32 temporaries of the quantiser
        parts = [quant.quantize(c, 64, bits, out_dtype=torch.bfloat16) for c in w.weight.split(8)]
        wq, scales, biases = (torch.cat(p) for p in zip(*parts))
        return LinearWeight(wq=wq, scales=scales, biases=biases, group_size=64, bits=bits)
    W = tuple(pack(w) for w in bank(H, I, Et, "bf16")[0])

    def weights(e):
        # the producer warps dequantise in fp32 and round to bf16
        return tuple(LinearWeight(wq=w.wq[e], scales=w.scales[e], biases=w.biases[e], group_size=64, bits=bits).dense(torch.bfloat16)
                     .double() for w in W)
    return W, weights


def block_inputs(shape, T, seed=0, hot=False):
    """Residual stream ``x`` (the block input before its norm), router gate (scale 0.02: logits of spread ~1, so the smallest
    routed weights of a batch stay near 1e-2 and a dropped pair is visible), and the two norm weights."""
    H, E = shape["H"], shape["E"]
    x = rnd(1 if hot else T, H, seed=100 + seed).expand(T, H).contiguous()
    gw = rnd(E, H, scale=0.02, seed=4)
    n1, n2 = 1.0 + rnd(H, scale=0.1, seed=5), 1.0 + rnd(H, scale=0.1, seed=6)
    return x, gw, n1, n2


def scatter_stride(B, fmt, T):
    """The row layout ``moe_block`` must take: the scatter stride, or 0 for the permutation."""
    if fmt.startswith("affine") or T > B.SCATTER_MAX_TOKENS:
        return 0
    return 64 if T <= 64 else B.SCATTER_MAX_TOKENS


def replay_route(B, x, gw, rk, extra, Et, n1, stride):
    """The router call ``moe_block`` makes, on buffers of our own: the kernel's selection, weights and the normed rows the
    experts read.  The router is deterministic, so this is the block's own routing.  On the scatter layout the normed rows are
    the scattered copies (all copies of a token must agree); on the permutation the block runs the norm kernel first."""
    T, H = x.shape
    if stride:
        counts = torch.zeros(Et, dtype=torch.int32, device=DEV)
        xs = torch.empty(Et * stride, H, dtype=torch.bfloat16, device=DEV)
        idx, w, pair_row = B.moe_route(x, gw, extra=extra, scatter=(counts, stride, xs, n1, EPS), **rk)
        rows = xs[pair_row.long()]
        assert torch.equal(rows, rows[:, :1].expand_as(rows))
        return rows[:, 0], idx, w
    xn = B.rmsnorm(x, n1, EPS)
    idx, w = B.moe_route(xn, gw, extra=extra, **rk)
    return xn, idx, w


def checked_routing(x, xn, gw, n1, idx, w, shape, min_clear):
    """The pre-MoE norm and the routing checked against fp64; returns the fp64 weights and their relative tolerance."""
    rk = shape["rk"]
    O.assert_rounded(xn, *O.rmsnorm64(x, n1, EPS), "pre-MoE norm")
    l, eps = O.route_logits(xn, gw)
    rtol = O.weight_rtol(xn, gw)
    ref_w = O.assert_valid_routing(l, eps, idx, w, rk["top_k"], shape["extra"], shape["E"], rk["scaling"], rk["norm_topk"],
                                   rk["n_group"], rk["topk_group"], rtol=rtol, min_clear=min_clear)
    return ref_w, rtol


def counters_zero(B):
    torch.cuda.synchronize()
    return all(int(c.abs().sum()) == 0 for c, _ in B._scatter_bufs.values())


def check_block(B, shape, fmt, T, x, gw, n1, n2, label, clear_bufs=True, min_clear=None):
    """``moe_block`` as the model calls it (residual = block input, fused pre-MoE and next-layer norms) and again without the
    residual, against the oracle on the kernel's own routing.  Returns the two error-to-tolerance ratios."""
    H, I, E, extra, rk = shape["H"], shape["I"], shape["E"], shape["extra"], shape["rk"]
    Et = E + extra
    (Wg, Wu, Wd), weights = bank(H, I, Et, fmt)
    stride = scatter_stride(B, fmt, T)
    xn, idx, w = replay_route(B, x, gw, rk, extra, Et, n1, stride)
    ref_w, rtol = checked_routing(x, xn, gw, n1, idx, w, shape, (0.8 if T >= 32 else 0.0) if min_clear is None else min_clear)
    routed, allow, mag, kept = O.expert_oracle(xn, idx, ref_w, weights, "mxfp8" if fmt == "mxfp8" else "bf16",
                                               keep=O.control_pairs(ref_w))
    allow = allow + rtol[:, None] * mag                  # the kernel's weights are fp32 roundings of ref_w
    k = idx.shape[1]
    ratios = []
    for residual in (x, None):
        if clear_bufs:
            B._scatter_bufs.clear()
        out, normed = B.moe_block(x, gw, rk, Wg, Wu, Wd, "silu", residual=residual, extra=extra, pre_norm=(n1, EPS),
                                  next_norm=(n2, EPS))
        if stride:
            assert (x.device.index, Et, H, stride) in B._scatter_bufs, "expected the scatter layout"
        else:
            assert not clear_bufs or not B._scatter_bufs, "expected the permutation layout"
        assert counters_zero(B), "the combine left scatter counters non-zero"
        ref, al = (routed, allow) if residual is None else O.with_residual(routed, allow, residual, k)
        tol = O.tolerance(ref, al)
        r = O.err_ratio(out, ref, tol)
        assert r <= 1, f"{label}: block output off by {r:.3g} x tolerance (residual={'none' if residual is None else 'h'})"
        O.assert_rounded(normed, *O.rmsnorm64(out, n2, EPS), "next-layer norm")
        if residual is None:
            c = O.assert_controls_fail(out, ref, tol, ref_w, kept)
            print(f"MOE {label} fmt={fmt} T={T}: controls (drop, scale, swap) {c[0]:.2f} {c[1]:.2f} {c[2]:.2f}")
        ratios.append(r)
    print(f"MOE {label} fmt={fmt} T={T} stride={stride}: error/tolerance {ratios[0]:.3f} with residual, {ratios[1]:.3f} routed only")
    return ratios


# ------------------------------------------------------------------------------------------------ the block
@pytest.mark.parametrize("fmt,T", [(f, T) for f in ("bf16", "mxfp8") for T in (1, 7, 64, 65, 128, 129, 1024, 1025, 8192)
                                   if not (f == "mxfp8" and T == 8192)])
def test_block_lite(B, fmt, T):
    x, gw, n1, n2 = block_inputs(LITE, T)
    check_block(B, LITE, fmt, T, x, gw, n1, n2, "lite")


@pytest.mark.parametrize("fmt,T", [(f, T) for f in ("bf16", "mxfp8") for T in (1, 64, 65, 1025)])
def test_block_v2_group_limited(B, fmt, T):
    x, gw, n1, n2 = block_inputs(V2, T, seed=1)
    check_block(B, V2, fmt, T, x, gw, n1, n2, "v2")


@pytest.mark.parametrize("T", [1, 64, 300])
def test_block_norm_topk(B, T):
    x, gw, n1, n2 = block_inputs(LITE_NORM_TOPK, T, seed=2)
    check_block(B, LITE_NORM_TOPK, "bf16", T, x, gw, n1, n2, "norm-topk")


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("T", [1, 64, 300])
def test_block_affine(B, bits, T):
    """Packed MLX-affine banks (group 64) always take the permutation layout; ``moe_experts`` is checked on the same routing."""
    fmt = f"affine{bits}"
    x, gw, n1, n2 = block_inputs(LITE, T, seed=3)
    check_block(B, LITE, fmt, T, x, gw, n1, n2, "affine")
    H, I, E, extra, rk = LITE["H"], LITE["I"], LITE["E"], LITE["extra"], LITE["rk"]
    (Wg, Wu, Wd), weights = bank(H, I, E + extra, fmt)
    xn, idx, w = replay_route(B, x, gw, rk, extra, E + extra, n1, 0)
    ref_w, rtol = checked_routing(x, xn, gw, n1, idx, w, LITE, 0.8 if T >= 32 else 0.0)
    routed, allow, mag, _ = O.expert_oracle(xn, idx, ref_w, weights, "bf16")
    got = B.moe_experts(xn, idx, w, Wg, Wu, Wd, "silu")
    r = O.err_ratio(got, routed, O.tolerance(routed, allow + rtol[:, None] * mag))
    print(f"MOE moe_experts fmt={fmt} T={T}: error/tolerance {r:.3f}")
    assert r <= 1


@pytest.mark.parametrize("T", [64, 128])
def test_block_hot_experts(B, T):
    """All rows identical: the 6 routed and 2 shared experts each get exactly ``stride`` rows, filling their segments."""
    x, gw, n1, n2 = block_inputs(LITE, T, seed=4, hot=True)
    Et = LITE["E"] + LITE["extra"]
    stride = scatter_stride(B, "bf16", T)
    assert stride == T
    counts = torch.zeros(Et, dtype=torch.int32, device=DEV)
    xs = torch.empty(Et * stride, LITE["H"], dtype=torch.bfloat16, device=DEV)
    B.moe_route(x, gw, extra=LITE["extra"], scatter=(counts, stride, xs, n1, EPS), **LITE["rk"])
    assert sorted(counts.tolist(), reverse=True)[:8] == [stride] * 8 and int(counts.sum()) == 8 * T
    check_block(B, LITE, "bf16", T, x, gw, n1, n2, "hot", min_clear=0.0)


def test_block_buffer_reuse(B):
    """Consecutive blocks of different sizes share the persistent scatter buffers: T = 64, 65, 1, 64 (strides 64, 128, 64,
    64); the counters are zero after each, and each result matches its oracle."""
    B._scatter_bufs.clear()
    for i, T in enumerate((64, 65, 1, 64)):
        x, gw, n1, n2 = block_inputs(LITE, T, seed=10 + i)
        check_block(B, LITE, "bf16", T, x, gw, n1, n2, "reuse", clear_bufs=False)
    assert {k[3] for k in B._scatter_bufs} == {64, 128}


def test_block_cuda_graph_replay(B):
    """Decode runs the block inside a CUDA graph: warm up at T = 64, capture, then replay on two different inputs copied into the
    static input.  Each replay matches its oracle and leaves the counters at zero (the captured combine resets them)."""
    T = 64
    H, I, E, extra, rk = LITE["H"], LITE["I"], LITE["E"], LITE["extra"], LITE["rk"]
    Et = E + extra
    (Wg, Wu, Wd), weights = bank(H, I, Et, "bf16")
    x0, gw, n1, n2 = block_inputs(LITE, T, seed=20)
    static_x = x0.clone()
    run = lambda: B.moe_block(static_x, gw, rk, Wg, Wu, Wd, "silu", residual=static_x, extra=extra, pre_norm=(n1, EPS),
                              next_norm=(n2, EPS))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            run()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out, normed = run()
    assert counters_zero(B)
    for seed in (21, 22):
        x = block_inputs(LITE, T, seed=seed)[0]
        static_x.copy_(x)
        graph.replay()
        assert counters_zero(B), "a graph replay left scatter counters non-zero"
        xn, idx, w = replay_route(B, x, gw, rk, extra, Et, n1, 64)
        ref_w, rtol = checked_routing(x, xn, gw, n1, idx, w, LITE, 0.8)
        routed, allow, mag, _ = O.expert_oracle(xn, idx, ref_w, weights, "bf16")
        ref, al = O.with_residual(routed, allow + rtol[:, None] * mag, x, idx.shape[1])
        r = O.err_ratio(out, ref, O.tolerance(ref, al))
        print(f"MOE graph replay seed={seed}: error/tolerance {r:.3f}")
        assert r <= 1
        O.assert_rounded(normed, *O.rmsnorm64(out, n2, EPS), "next-layer norm")


# ------------------------------------------------------------------------------------------------ the support kernels
@pytest.mark.parametrize("E,H,top_k,extra,n_group,topk_group,T,norm", [
    (64, 2048, 6, 2, 1, 1, 37, False),
    (64, 2048, 6, 2, 1, 1, 128, True),
    (160, 5120, 6, 2, 8, 3, 64, True),
    (256, 2048, 30, 2, 1, 1, 100, False),      # top-k + extra = 32: every lane of the selection warp
    (256, 7168, 8, 1, 8, 4, 65, True),
])
def test_route_scatter(B, E, H, top_k, extra, n_group, topk_group, T, norm):
    """The router's scatter layout: per-expert counts equal the selection's histogram, every pair's row lies in its expert's
    segment and no two coincide, and every scattered row is bitwise the token's (normed) row; the routing is a valid top-k."""
    x = rnd(T, H, seed=30)
    gw = rnd(E, H, scale=0.02, seed=31)
    nw = (1.0 + rnd(H, scale=0.1, seed=32)) if norm else None
    Et, stride = E + extra, 64 if T <= 64 else 128
    counts = torch.zeros(Et, dtype=torch.int32, device=DEV)
    xs = torch.zeros(Et * stride, H, dtype=torch.bfloat16, device=DEV)
    method = "group_limited_greedy" if n_group > 1 else "greedy"
    idx, w, pair_row = B.moe_route(x, gw, top_k, method, n_group, topk_group, 2.5, False, extra=extra,
                                   scatter=(counts, stride, xs, nw, EPS))
    hist = torch.bincount(idx.long().flatten(), minlength=Et)
    assert torch.equal(counts.long(), hist)
    seg = pair_row.long() // stride
    assert torch.equal(seg, idx.long())
    assert bool((pair_row.long() % stride < counts.long()[idx.long()]).all())
    assert pair_row.unique().numel() == pair_row.numel()
    rows = xs[pair_row.long()]
    if norm:
        assert torch.equal(rows, rows[:, :1].expand_as(rows))
        xn = rows[:, 0]
        O.assert_rounded(xn, *O.rmsnorm64(x, nw, EPS), "fused router norm")
    else:
        xn = x
        assert torch.equal(rows, x[:, None].expand_as(rows))
    l, eps = O.route_logits(xn, gw)
    O.assert_valid_routing(l, eps, idx, w, top_k, extra, E, 2.5, False, n_group, topk_group, rtol=O.weight_rtol(xn, gw))


@pytest.mark.parametrize("E,H,top_k,n_group,topk_group,T,norm_topk", [
    (64, 2048, 6, 8, 3, 1024, False),         # one token per CTA
    (64, 2048, 6, 8, 3, 1025, False),         # eight tokens per CTA
    (256, 2048, 8, 8, 4, 1025, True),
    (160, 5120, 6, 1, 1, 1031, True),         # eight-token CTAs at 80 KB of shared memory
])
def test_route_prefill(B, E, H, top_k, n_group, topk_group, T, norm_topk):
    x = rnd(T, H, seed=40)
    gw = rnd(E, H, scale=0.02, seed=41)
    method = "group_limited_greedy" if n_group > 1 else "greedy"
    idx, w = B.moe_route(x, gw, top_k, method, n_group, topk_group, 1.5, norm_topk)
    l, eps = O.route_logits(x, gw)
    O.assert_valid_routing(l, eps, idx, w, top_k, 0, E, 1.5, norm_topk, n_group, topk_group, rtol=O.weight_rtol(x, gw))


@pytest.mark.parametrize("T,k,E", [(1, 8, 66), (300, 6, 64), (1025, 32, 256)])
def test_permute(B, T, k, E):
    """Counting-sort permutation: offsets are the exclusive prefix sum of the histogram, ``pair_row`` is a bijection onto
    [0, T k) that keeps every pair in its expert's segment, and the gathered rows are bitwise their tokens' rows."""
    g = torch.Generator(device=DEV).manual_seed(50)
    idx = torch.rand(T, E, device=DEV, generator=g).argsort(-1)[:, :k].to(torch.int32).contiguous()
    x = rnd(T, 2048, seed=51)
    offs, pair_row, xp = B.C().moe_permute(idx, x, E)
    hist = torch.bincount(idx.long().flatten(), minlength=E)
    assert offs.tolist() == [0] + hist.cumsum(0).tolist()
    pr = pair_row.long()
    assert torch.equal(pr.sort().values, torch.arange(T * k, device=DEV))
    e = idx.long().flatten()
    assert bool(((pr >= offs.long()[e]) & (pr < offs.long()[e + 1])).all())
    assert torch.equal(xp[pr], x.repeat_interleave(k, 0))


@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("H", [2048, 5120, 8192])
def test_combine(B, H, norm):
    """Weighted combine (+ residual, + the fused next-layer norm) of random fp32 expert rows against fp64: within half a bf16
    spacing plus the fp32 sum's error, so never more than one spacing; the fused norm is a correct rounding of the fp64 norm of
    the stored row; the scatter counters handed to it are zeroed."""
    T, k = 33, 8
    g = torch.Generator(device=DEV).manual_seed(60)
    y = torch.randn(T * k, H, device=DEV, generator=g)
    pair_row = torch.randperm(T * k, device=DEV, generator=g).to(torch.int32).view(T, k)
    w = torch.rand(T, k, device=DEV, generator=g)
    res = rnd(T, H, seed=61)
    counts = torch.arange(1, 67, dtype=torch.int32, device=DEV)
    nw = 1.0 + rnd(H, scale=0.1, seed=62)
    normed = torch.empty(T, H, dtype=torch.bfloat16, device=DEV)
    args = (counts, nw, EPS, normed) if norm else (counts,)
    out = B.C().moe_combine(y, pair_row, w, res, None, k, 0, 0, *args)
    torch.cuda.synchronize()
    assert int(counts.abs().sum()) == 0
    terms = w.double()[:, :, None] * y.double()[pair_row.long()]
    ref = terms.sum(1) + res.double()
    allow = (k + 4) * O.U32 * (terms.abs().sum(1) + res.double().abs())
    err = (out.double() - ref).abs()
    assert O.err_ratio(out, ref, O.tolerance(ref, allow)) <= 1
    assert bool((err <= O.bf16_ulp(ref)).all())
    if norm:
        O.assert_rounded(normed, *O.rmsnorm64(out, nw, EPS), "fused combine norm")
