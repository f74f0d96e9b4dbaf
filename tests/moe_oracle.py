"""fp64 oracle of the MoE block (router, pre-MoE norm, grouped gate/up + down expert GEMMs, weighted combine, next-layer norm)
shared by ``test_moe_block_gpu.py`` and its CPU self-test ``test_moe_oracle.py``.

The oracle rounds only where the kernels store data (normed rows and ``h = act(g) * u`` in bf16, MXFP8 operands in e4m3 with
per-32 block scales, the block output in bf16) and carries, next to every fp64 value, a bound on how far the kernels' fp32
arithmetic may move it.  Where that bound straddles a bf16 (or e4m3) rounding point the kernel may legitimately store either
neighbour: those elements are *ambiguous*, and the tolerances below admit exactly that and nothing more.  Routing is never compared
set-to-set: a selection is checked to be *a* valid top-k of the fp64 probabilities within the fp32 logit error, and the expert
oracle is evaluated on the kernel's own selection, so near-ties cannot make a correct kernel fail.
"""
import torch

from mlx_sharding_b200.utils.quant import from_mxfp8, to_mxfp8

U32 = 2.0 ** -24          # unit roundoff of fp32
# Half-width of the admitted spread of the ambiguous h elements (in standard deviations of a sum of independent +-d terms).
C_FLIP = 3.0
# FP8 wgmma adds the 32 e4m3 products of one scale block with a short internal accumulator before the fp32 add: bound on that
# error relative to the sum of |products|.  Measured on an H100 SXM (80 GB HBM3, 700 W limit) with the MXFP8 cases of
# test_moe_block_gpu.py: at 2^-20 the kernel exceeds its tolerance up to 28-fold (so the block sums are not exact); at 2^-18 its
# largest error-to-tolerance ratio is 0.80 and the 1.01-weight control still fails by 1.8x or more; at 2^-16 that control
# passes.  2^-18 is the value that admits the kernel and still rejects a 1 % weight error.
FP8_ACC = 2.0 ** -18


def bf16_ulp(v: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 values in the binade of ``v`` (fp64); the subnormal floor for zero."""
    _, e = torch.frexp(v.double().abs())
    return torch.where(v == 0, torch.full_like(v.double(), 2.0 ** -133), torch.ldexp(torch.ones_like(v.double()), e - 8))


def rounding_set(v: torch.Tensor, dv: torch.Tensor, dtype=torch.bfloat16):
    """The two values a store of ``v +- dv`` (fp64) may round to: rounding is monotone, so every value in the interval rounds
    to one of ``lo``, ``hi`` or a value between them; for ``dv`` below one spacing that is at most two neighbours."""
    return (v - dv).to(dtype), (v + dv).to(dtype)


def assert_rounded(got: torch.Tensor, v: torch.Tensor, dv: torch.Tensor, what: str) -> int:
    """``got`` (bf16) is a correct rounding of ``v`` computed with an error of at most ``dv``: equal to round(v), or on an
    element whose interval straddles a rounding point, to the other neighbour.  Returns the number of such elements."""
    lo, hi = rounding_set(v, dv)
    ok = (got == lo) | (got == hi)
    bad = (~ok).nonzero()
    assert bad.numel() == 0, (f"{what}: {bad.shape[0]} elements off; first {bad[0].tolist()}: got {got[tuple(bad[0])].item()!r} "
                              f"for {v[tuple(bad[0])].item()!r} +- {dv[tuple(bad[0])].item():.3g}")
    return int((lo != hi).sum())


def rmsnorm64(x: torch.Tensor, w: torch.Tensor, eps: float):
    """fp64 RMSNorm of the bf16 rows ``x`` times ``w``, and the bound on the kernels' fp32 version of it: the mean square is a
    sum of H squares over 32 lanes (H/32 sequential adds and a 5-level shuffle tree), halved through the square root, plus
    rsqrtf (2 ulp) and the two products."""
    xd = x.double()
    H = x.shape[-1]
    v = xd * torch.rsqrt(xd.square().mean(-1, keepdim=True) + eps) * w.double()
    return v, v.abs() * ((H / 64 + 8) * U32)


def route_logits(x: torch.Tensor, gw: torch.Tensor):
    """fp64 router logits of bf16 rows ``x`` and gate ``gw``, and a bound on the router kernel's fp32 logits: every product of
    two bf16 values is exact in fp32, and each lane adds H/32 of them before a 5-level shuffle tree, so the error is at most
    (H/32 + 5) u sum|x w| (first order; +3 for slack).  The softmax is taken with __expf (relative error below
    (2 + 1.2 |l - max|) fp32 ulps) and one product, which moves a comparison of probabilities like a logit shift of that size."""
    xd, wd = x.double(), gw.double()
    H = x.shape[-1]
    l = xd @ wd.t()
    eps = (H / 32 + 8) * U32 * (xd.abs() @ wd.abs().t())
    eps = eps + (4 + 2 * (l.amax(-1, keepdim=True) - l)) * 2 * U32
    return l, eps


def weight_rtol(x: torch.Tensor, gw: torch.Tensor) -> torch.Tensor:
    """Per-token relative tolerance of the routing weights: a probability's relative error is the difference of two logit
    errors.  The fp32 logit error is a sum of H/32 + 5 roundings of partial sums; its spread is about u ||x * w||_2 sqrt(H) / 4,
    eight times that bounds each logit here, plus 1e-5 for __expf and the normalisation."""
    H = x.shape[-1]
    l2 = (x.double().square() @ gw.double().square().t()).sqrt().amax(-1)
    return 1e-5 + 2 * 8 * U32 * H ** 0.5 * l2 / 4


def routing_weights(l: torch.Tensor, idx: torch.Tensor, top_k: int, extra: int, scaling: float, norm_topk: bool):
    """The weights the router returns for the selection ``idx`` (the kernel's own), in fp64: softmax probability of each chosen
    expert, renormalised over the chosen ones (``norm_topk`` with top_k > 1) or times ``scaling``; 1.0 for appended experts."""
    p = torch.softmax(l, -1)
    w = p.gather(1, idx[:, :top_k].long())
    w = w / w.sum(-1, keepdim=True) if (norm_topk and top_k > 1) else w * scaling
    return torch.cat([w, torch.ones(w.shape[0], extra, dtype=w.dtype, device=w.device)], 1)


def check_topk(l: torch.Tensor, eps: torch.Tensor, sel: torch.Tensor, top_k: int, n_group: int = 1, topk_group: int = 1):
    """Is ``sel[:, :top_k]`` a valid (group-limited) top-k of the logits ``l`` for every token, given that each logit is known
    only to within ``eps``?  Returns ``(ok, clear, same)`` per token: ``ok`` = valid; ``clear`` = the fp64 top-k is unique
    beyond the error (its group and expert margins exceed the errors on both sides); ``same`` = ``sel`` equals the fp64 top-k
    as a set.  Valid means: the experts are distinct; every chosen group could be among the top ``topk_group`` groups by their
    maximum; every selected expert scores at least every unselected expert of an allowed group, within the errors.  Allowed
    groups are the selected experts' groups and every group that is surely among the top ``topk_group``."""
    T, E = l.shape
    sel = sel[:, :top_k].long()
    chosen = torch.zeros(T, E, dtype=torch.bool, device=l.device).scatter_(1, sel, True)
    ok = chosen.sum(-1) == top_k
    clear = torch.ones(T, dtype=torch.bool, device=l.device)
    allowed = torch.ones_like(chosen)
    ref_allowed = allowed
    if n_group > 1 and topk_group < n_group:
        gsz = E // n_group
        gmax = l.view(T, n_group, gsz).amax(-1)
        geps = eps.view(T, n_group, gsz).amax(-1)
        hi, lo = gmax + geps, gmax - geps
        surely_beats = lo[:, :, None] > hi[:, None, :]                    # [t, g', g]: g' is above g whatever the errors
        eye = torch.eye(n_group, dtype=torch.bool, device=l.device)
        maybe_beats = (hi[:, :, None] >= lo[:, None, :]) & ~eye
        possible = surely_beats.sum(1) < topk_group
        certain = maybe_beats.sum(1) < topk_group
        sel_groups = torch.zeros(T, n_group, dtype=torch.bool, device=l.device).scatter_(1, sel // gsz, True)
        ok &= (sel_groups & ~possible).sum(-1) == 0
        ok &= sel_groups.sum(-1) <= topk_group
        allowed = (sel_groups | certain).repeat_interleave(gsz, 1)
        top_groups = gmax.topk(topk_group, -1).indices
        ref_allowed = torch.zeros(T, n_group, dtype=torch.bool, device=l.device).scatter_(1, top_groups, True)
        clear &= certain.sum(-1) == topk_group
        ref_allowed = ref_allowed.repeat_interleave(gsz, 1)
    inf = torch.full_like(l, float("inf"))
    lo_sel = torch.where(chosen, l + eps, inf).amin(-1)
    hi_rest = torch.where(allowed & ~chosen, l - eps, -inf).amax(-1)
    ok &= lo_sel >= hi_rest
    lm = torch.where(ref_allowed, l, -inf)
    ref = lm.topk(top_k, -1).indices
    ref_set = torch.zeros_like(chosen).scatter_(1, ref, True)
    lo_ref = torch.where(ref_set, l - eps, inf).amin(-1)
    hi_out = torch.where(ref_allowed & ~ref_set, l + eps, -inf).amax(-1)
    clear &= lo_ref > hi_out
    same = (ref_set == chosen).all(-1)
    return ok, clear, same


def assert_valid_routing(l, eps, idx, w, top_k, extra, E, scaling=1.0, norm_topk=False, n_group=1, topk_group=1, rtol=None,
                         min_clear=0.8):
    """Everything the router promises, checked against fp64: a valid top-k (tie-aware), the fp64 top-k exactly wherever it is
    clear, appended experts ``E .. E+extra-1`` with weight 1, and the weights of the fp64 softmax on the kernel's selection."""
    T = l.shape[0]
    assert idx.shape == (T, top_k + extra) and w.shape == (T, top_k + extra)
    ok, clear, same = check_topk(l, eps, idx, top_k, n_group, topk_group)
    assert bool(ok.all()), f"invalid top-k for tokens {(~ok).nonzero().flatten()[:8].tolist()}"
    assert bool(same[clear].all()), f"clear tokens routed off the fp64 top-k: {(clear & ~same).nonzero().flatten()[:8].tolist()}"
    assert clear.double().mean() >= min_clear, f"only {clear.double().mean():.2f} of the tokens have a clear top-k"
    if extra:
        assert (idx[:, top_k:] == torch.arange(E, E + extra, device=idx.device, dtype=idx.dtype)).all()
        assert (w[:, top_k:] == 1).all()
    ref = routing_weights(l, idx, top_k, extra, scaling, norm_topk)
    rel = ((w.double() - ref).abs() / ref.abs()).amax(-1)
    if rtol is not None:
        assert bool((rel <= rtol).all()), f"routing weights off by {rel.max().item():.3g} (tolerance {rtol.min().item():.3g})"
    return ref


def _silu(g):
    return g * torch.sigmoid(g)


def _dsilu(g):
    s = torch.sigmoid(g)
    return s * (1 + g * (1 - s))


def _fp8_roundtrip(v):
    return from_mxfp8(*to_mxfp8(v), dtype=torch.float64)


def _dot_err(a, w, fp8: bool):
    """Bound on the fp32 accumulation error of ``a @ w.T`` as the GEMM kernels compute it.  bf16 wgmma: the spread of a sum of
    K roundings of partial sums is about u ||a * w||_2 sqrt(K); eight times that.  FP8 wgmma: FP8_ACC of sum|a w|."""
    if fp8:
        return FP8_ACC * (a.abs() @ w.abs().t())
    return 8 * U32 * a.shape[-1] ** 0.5 * (a.square() @ w.square().t()).sqrt()


def expert_oracle(x: torch.Tensor, idx: torch.Tensor, w: torch.Tensor, weights, fmt: str, keep=()):
    """fp64 value and error allowance of ``sum_k w[t, k] * down_e(act(gate_e x_t) * up_e x_t)`` (the routed contribution, before
    the residual and the kernel's final bf16 store), on the kernel's selection ``idx`` and fp64 routing weights ``w``.

    ``weights(e)`` -> the three fp64 matrices ``(Wg [I, H], Wu [I, H], Wd [H, I])`` of expert ``e`` as the GEMMs see them.
    ``fmt``: 'bf16' (also packed affine: its producer warps round to bf16), or 'mxfp8' (x and h quantised per 32-wide block).
    ``keep``: (token, slot) pairs whose fp64 expert output rows are returned too (the negative controls perturb with them).

    The allowance is: the down GEMM's and the combine's accumulation error, plus C_FLIP standard deviations of the spread of
    the ambiguous h elements (those whose stored bf16 / e4m3 value may differ from the oracle's because the gate/up GEMM's
    fp32 error straddles a rounding point).  Returns ``(value, allowance, sum_k |w y_k|, kept rows)``: the caller adds the
    routing weights' relative tolerance times that sum."""
    fp8 = fmt == "mxfp8"
    T, k = idx.shape
    H = x.shape[1]
    dev = x.device
    out = torch.zeros(T, H, dtype=torch.float64, device=dev)
    lin = torch.zeros_like(out)
    var = torch.zeros_like(out)
    mag = torch.zeros_like(out)
    kept = {}
    xs = _fp8_roundtrip(x) if fp8 else x.double()
    flat = idx.long().flatten()
    order = torch.argsort(flat, stable=True)
    counts = torch.bincount(flat, minlength=int(flat.max()) + 1).tolist()
    start = 0
    for e, n in enumerate(counts):
        if n == 0:
            continue
        pairs = order[start:start + n]
        start += n
        tok, slot = pairs // k, pairs % k
        Wg, Wu, Wd = weights(e)
        a = xs[tok]
        g, u = a @ Wg.t(), a @ Wu.t()
        dg, du = _dot_err(a, Wg, fp8), _dot_err(a, Wu, fp8)
        h = _silu(g) * u
        dh = (_dsilu(g) * u).abs() * dg + _silu(g).abs() * du + 8 * U32 * h.abs() * (1 + g.abs())
        ho = h.to(torch.bfloat16).double()
        lo, hi = (v.double() for v in rounding_set(h, dh))
        if fp8:
            hq, lo, hi = _fp8_roundtrip(ho), _fp8_roundtrip(lo), _fp8_roundtrip(hi)
        else:
            hq = ho
        d = torch.maximum((lo - hq).abs(), (hi - hq).abs())
        y = hq @ Wd.t()
        ww = w[tok, slot].double()[:, None]
        out.index_add_(0, tok, ww * y)
        lin.index_add_(0, tok, ww.abs() * _dot_err(hq, Wd, fp8))
        var.index_add_(0, tok, ww.square() * (d.square() @ Wd.square().t()))
        mag.index_add_(0, tok, (ww * y).abs())
        for t, s in keep:
            m = (tok == t) & (slot == s)
            if bool(m.any()):
                kept[(t, s)] = y[m.nonzero()[0, 0]]
    allow = lin + C_FLIP * var.sqrt() + (k + 4) * U32 * mag
    return out, allow, mag, kept


def with_residual(ref, allow, residual, k: int):
    """The oracle of the block with ``residual`` added in the combine's fp32 sum (one more term of k + 1)."""
    r = residual.double()
    return ref + r, allow + (k + 4) * U32 * r.abs()


def tolerance(ref: torch.Tensor, allow: torch.Tensor) -> torch.Tensor:
    """Admitted |kernel - ref| for a bf16 store of a value within ``allow`` of ``ref``: half a bf16 spacing at that value
    plus ``allow``."""
    return 0.5 * bf16_ulp(ref.abs() + allow) + allow


def err_ratio(got: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor) -> float:
    """Largest |got - ref| / tol over all elements (<= 1 passes)."""
    return ((got.double() - ref).abs() / tol).max().item()


def control_pairs(w: torch.Tensor):
    """(token, slot) pairs the negative controls perturb: the smallest and the largest weight of the batch, and token 0's
    largest- and smallest-weight pairs."""
    k = w.shape[1]
    lo, hi = divmod(int(w.flatten().argmin()), k), divmod(int(w.flatten().argmax()), k)
    return lo, hi, (0, int(w[0].argmax())), (0, int(w[0].argmin()))


def assert_controls_fail(got, ref, tol, w, kept):
    """A tolerance that admits ``got`` must reject three oracles that are wrong the way a kernel could be wrong: the batch's
    smallest-weight pair dropped, the largest weight scaled by 1.01, and token 0's largest- and smallest-weight experts' outputs
    swapped.  Returns the three ratios."""
    lo, hi, a, b = control_pairs(w)
    drop, scale, swap = ref.clone(), ref.clone(), ref.clone()
    drop[lo[0]] -= w[lo] * kept[lo]
    scale[hi[0]] += 0.01 * w[hi] * kept[hi]
    swap[0] += (w[a] - w[b]) * (kept[b] - kept[a])
    ratios = [err_ratio(got, r, tol) for r in (drop, scale, swap)]
    assert min(ratios) > 1, f"a perturbed oracle passes (drop, scale, swap ratios {ratios})"
    return ratios
