"""The sm_90a sampler's draws against an exact host replay of its Gumbel-max draw.

``sample_kernel`` (``ops/csrc/sampler.cu``) draws a temperature token as ``argmax((x - max) / T + g)`` over the kept ids, with
Gumbel noise ``g`` from a stateless hash of (seed, step, row, id).  The replay below is a plain fp64 / integer model of that
draw: a numpy port of the hash, the noise through the mapping documented at ``gumbel``, the kept set in the kernel's order
(mask, top-k, top-p, min-p) and the argmax.  The GPU tests compare the kernel's token with the replay's on every row at real
vocabulary sizes, pin the noise at the top of the uniform range, check the tail mass of a full-vocabulary draw against the fp64
softmax without the replay, and check the reported log-probs against fp64 ``log_softmax``.  The CPU tests check the replay
itself: the noise over every bit pattern, Gumbel-max frequencies against the softmax, and the kept set against
``reference.filter_keep``."""
import functools

import numpy as np
import pytest
import torch

from mlx_sharding_b200.ops import reference as R

DEV = "cuda"
VOCABS = [1000, 32000, 50257, 102400, 128256, 256000]     # 50257 % 32 != 0: the last mask word is partial
ROWS = 128                                                # rows per launch, two launches per vocabulary size
TIE = 1e-4          # rows whose best and second-best replay scores are closer than this may flip under fp32 rounding
MARGIN = 1e-3       # no kept id sits closer than this (in logits) to a top-p or min-p boundary

# ------------------------------------------------------------------------------------------------ hash and noise
_U64 = np.uint64


def mix64(z):
    """splitmix64 finaliser, as ``mix64`` in sampler.cu (uint64 arithmetic wraps)."""
    z = z + _U64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> _U64(30))) * _U64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> _U64(27))) * _U64(0x94D049BB133111EB)
    return z ^ (z >> _U64(31))


def hash_bits(seed, step, row, ids):
    """64-bit hash of (seed, step, row, id), as ``uniform01`` computes it; the arguments broadcast."""
    with np.errstate(over="ignore"):
        base = mix64(_U64(seed) ^ (_U64(step) * _U64(0xD1342543DE82EF95)))
        return mix64(base ^ ((_U64(row) << _U64(32)) | np.asarray(ids, dtype=np.uint64)))


def uniform(h):
    """The uniform of a hash: u = (k + 0.5) / 2^23 for the top 23 bits k, so 2^-24 <= u <= 1 - 2^-24, each value exact in fp32."""
    return ((h >> _U64(41)).astype(np.float64) + 0.5) / 2.0 ** 23


def gumbel(h):
    """Gumbel noise g = -log(-log(u)) in fp64, with -log(u) as -log1p(u - 1) so that it stays accurate near u = 1."""
    return -np.log(-np.log1p(uniform(h) - 1.0))


# ------------------------------------------------------------------------------------------------ replay
def draw_row(x, allow):
    """The logits the draw sees (fp64): ids the mask disallows read -inf; a row without an allowed finite id is drawn unmasked."""
    d = x.astype(np.float64)
    if allow is not None:
        m = np.where(allow, d, -np.inf)
        if np.isfinite(m).any():
            d = m
    return d


def bounds(d, t, top_p, top_k, min_p):
    """(kth, top-p threshold, floor) of a temperature draw: ids with ``x >= kth`` form the top-k set, ``x > threshold`` the
    nucleus of that set at temperature ``t``, and ``x >= floor`` passes top-k and min-p together."""
    V, M = d.size, d.max()
    kth = np.partition(d, V - top_k)[V - top_k] if 0 < top_k < V else -np.inf
    thr = -np.inf
    if 0 < top_p < 1:
        xs = np.sort(d[(d >= kth) & np.isfinite(d)])
        cw = np.cumsum(np.exp((xs - M) / t))
        F = cw[np.searchsorted(xs, xs, side="right") - 1]          # mass{logit <= x}, ties included
        drop = F <= (1.0 - top_p) * cw[-1]
        if drop.any():
            thr = xs[drop][-1]
    floor = max(kth, M + t * np.log(min_p)) if min_p > 0 else kth
    return kth, thr, floor


def kept_ids(d, t, top_p, top_k, min_p):
    _, thr, floor = bounds(d, t, top_p, top_k, min_p)
    return np.isfinite(d) & (d > thr) & (d >= floor)


def replay(x, allow, t, top_p, top_k, min_p, seed, step, row):
    """Token of one row, and the gap between the best and second-best scores (inf for a greedy or one-id draw)."""
    d = draw_row(x, allow)
    if t == 0:
        return int(np.argmax(d)), np.inf
    ids = np.nonzero(kept_ids(d, t, top_p, top_k, min_p))[0]
    s = (d[ids] - d.max()) / t + gumbel(hash_bits(seed, step, row, ids))
    b = int(np.argmax(s))                    # first of equal scores: the lower id, as ``better`` in sampler.cu
    gap = s[b] - np.max(np.delete(s, b)) if ids.size > 1 else np.inf
    return int(ids[b]), gap


# ------------------------------------------------------------------------------------------------ designed batches
PLAIN = [dict(t=0.5), dict(t=1.0), dict(t=1.7), dict(t=0.0),
         dict(t=1.0, top_p=0.9), dict(t=0.8, top_p=0.5),
         dict(t=1.0, top_k=40), dict(t=1.2, top_k=1000), dict(t=1.0, min_p=0.05),
         dict(t=1.0, top_k=40, top_p=0.9, min_p=0.05), dict(t=0.7, top_k=1000, top_p=0.5, min_p=0.02),
         dict(t=1.0, top_k=40, sparse=True)]
MASKED = [dict(mask=0.01, t=1.0), dict(mask=0.5, t=0.7), dict(mask=0.01, t=0.0), dict(mask=0.5, t=0.0),
          dict(mask=0.01, t=1.0, top_k=40), dict(mask=0.5, t=1.0, top_p=0.9, min_p=0.05),
          dict(mask=0.5, t=1.3, top_k=1000, top_p=0.5), dict(mask=0.01, t=1.0, top_k=40, top_p=0.9, min_p=0.05),
          dict(mask="no finite", t=1.0), dict(mask="no finite", t=0.0), dict(mask="empty", t=1.0, top_p=0.9)]


def _params(c):
    return c["t"], c.get("top_p", 1.0), c.get("top_k", 0), c.get("min_p", 0.0)


def _design(x, allow, c):
    """Move the ids within MARGIN of a top-p or min-p boundary out of it (in place): up past the top-p threshold, down
    below the min-p floor, until none is left.  fp32 sums and thresholds in the kernel cannot flip such an id.  A tie at
    the smallest kept logit is broken too: the kernel keeps or drops the tied ids together, ``filter_keep`` splits them in
    id order."""
    t, top_p, top_k, min_p = _params(c)
    if t == 0 or not (0 < top_p < 1 or min_p > 0):
        return
    for _ in range(50):
        d = draw_row(x, allow)
        kth, thr, _ = bounds(d, t, top_p, top_k, min_p)
        fin = np.isfinite(d)
        up = np.zeros_like(fin)
        if np.isfinite(thr):
            above = fin & (d >= kth) & (d > thr)
            up = above & (d < thr + MARGIN)
            up[np.nonzero(above & (d == d[above].min()))[0][1:]] = True
        down = fin & (np.abs(d - (d.max() + t * np.log(min_p))) < MARGIN) if min_p > 0 else np.zeros_like(fin)
        if not (up.any() or down.any()):
            return
        x[up] += np.float32(MARGIN)
        x[down] -= np.float32(2 * MARGIN)
    raise AssertionError("row design did not converge")


@functools.lru_cache(maxsize=None)
def batch(V, masked):
    """One launch: ROWS rows of ``randn * scale`` logits cycling through the configurations, each with 32 ``-inf`` entries
    (logit_bias), the row max tied on two more ids and the 10th largest logit tied with the 11th; masks where configured.
    The launch scalars (``sample``) or the per-row state (``sample_into``) feed the RNG, alternating with V."""
    cfgs = MASKED if masked else PLAIN
    g = np.random.default_rng([V, int(masked)])
    x = np.empty((ROWS, V), np.float32)
    allow = np.ones((ROWS, V), bool) if masked else None
    for b in range(ROWS):
        c = cfgs[b % len(cfgs)]
        r = (g.standard_normal(V) * (1.5, 2.5, 3.5)[(b // len(cfgs)) % 3]).astype(np.float32)
        if c.get("sparse"):                                   # 5 finite logits: top-k 40 reaches -inf
            keep = g.choice(V, 5, replace=False)
            r = np.full(V, -np.inf, np.float32)
            r[keep] = g.standard_normal(5)
        else:
            r[g.choice(V, 32, replace=False)] = -np.inf
            top = np.argpartition(-r, 11)[:11]
            order = top[np.argsort(-r[top])]
            r[order[1:3]] = r[order[0]]                       # three-way tie at the max
            r[order[10]] = r[order[9]]                        # tie across the 10th / 11th place
        if masked:
            m = c["mask"]
            if m == "no finite":
                allow[b] = ~np.isfinite(r)                    # only -inf ids allowed: drawn unmasked
            elif m == "empty":
                allow[b] = False
            else:
                allow[b] = g.random(V) < m
        _design(r, None if allow is None else allow[b], c)
        x[b] = r
    t, top_p, top_k, min_p = (np.array(v) for v in zip(*(_params(cfgs[b % len(cfgs)]) for b in range(ROWS))))
    per_row = (VOCABS.index(V) + int(masked)) % 2 == 1
    if per_row:
        seeds = 2000 + 7919 * np.arange(ROWS, dtype=np.int64) + V
        steps = 3 + np.arange(ROWS, dtype=np.int64)
        rows = np.zeros(ROWS, np.int64)
    else:
        seeds = np.full(ROWS, 1000 + V, np.int64)
        steps = np.full(ROWS, 7 + int(masked), np.int64)
        rows = np.arange(ROWS, dtype=np.int64)
    return dict(V=V, cfgs=[cfgs[b % len(cfgs)] for b in range(ROWS)], x=x, allow=allow, t=t.astype(np.float32),
                top_p=top_p.astype(np.float32), top_k=top_k.astype(np.int32), min_p=min_p.astype(np.float32),
                per_row=per_row, seeds=seeds, steps=steps, rows=rows)


def pack_allow(allow):
    """bool [B, V] -> int32 [B, ceil(V/32)] token mask; the bits past V are set, and the kernel must not read them."""
    B, V = allow.shape
    W = (V + 31) // 32
    bits = np.ones((B, W * 32), np.uint64)
    bits[:, :V] = allow
    words = (bits.reshape(B, W, 32) << np.arange(32, dtype=np.uint64)).sum(-1)
    return words.astype(np.uint32).view(np.int32)


# ------------------------------------------------------------------------------------------------ CPU: the oracle
def test_noise_is_finite_for_every_bit_pattern():
    h = np.arange(1 << 24, dtype=np.uint64) << _U64(40)              # every value of the top 24 hash bits
    u = uniform(h)
    assert u.min() > 0 and u.max() < 1
    assert u.min() == 2.0 ** -24 and u.max() == 1 - 2.0 ** -24
    # the kernel's fp32 arithmetic gives the same u, exactly, and an exact u - 1
    u32 = ((h >> _U64(41)).astype(np.float32) + np.float32(0.5)) * np.float32(1 / 8388608)
    assert np.array_equal(u32.astype(np.float64), u)
    assert np.array_equal((u32 - np.float32(1)).astype(np.float64), u - 1)
    g = gumbel(h)
    assert np.isfinite(g).all()
    assert g.max() == pytest.approx(-np.log(2.0 ** -24 * (1 + 2.0 ** -25)), rel=1e-12)     # -log(-log(1 - 2^-24))
    assert g.min() == pytest.approx(-np.log(24 * np.log(2)), rel=1e-12)
    # an fp32 evaluation of the same formula stays within fp32 accuracy of it over the whole range
    g32 = -np.log(-np.log1p(u32 - np.float32(1)))
    assert g32.dtype == np.float32 and np.isfinite(g32).all()
    assert np.abs(g32 - g).max() < 4e-6


@pytest.mark.parametrize("t", [1.0, 0.5])
def test_replayed_gumbel_max_frequencies(t):
    V, n = 16, 200_000
    x = np.linspace(1.5, -2.0, V)
    h = hash_bits(42, 9 + int(10 * t), np.arange(n, dtype=np.uint64)[:, None], np.arange(V))
    toks = np.argmax(x / t + gumbel(h), axis=1)
    p = np.exp(x / t - np.logaddexp.reduce(x / t))
    chi2 = (((np.bincount(toks, minlength=V) - n * p) ** 2) / (n * p)).sum()
    assert chi2 < 44.26, chi2                      # chi-square, 15 degrees of freedom, p = 1e-4


def test_replay_kept_set_matches_filter_keep():
    checked = 0
    for V in VOCABS:
        for masked in (False, True):
            bt = batch(V, masked)
            for b, c in enumerate(bt["cfgs"]):
                t, top_p, top_k, min_p = _params(c)
                if t == 0 or (top_p, top_k, min_p) == (1.0, 0, 0.0):
                    continue
                d = draw_row(bt["x"][b], None if bt["allow"] is None else bt["allow"][b])
                want = R.filter_keep(torch.from_numpy(d), t, top_p, top_k, min_p).numpy() & np.isfinite(d)
                got = kept_ids(d, t, top_p, top_k, min_p)
                assert np.array_equal(got, want), (V, masked, b, c, np.nonzero(got != want)[0][:10])
                checked += 1
    assert checked > 500


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def C():
    from mlx_sharding_b200.ops import b200

    return b200.load_extension()


def launch(C, bt, top_logprobs=10):
    """Run one batch through ``sample`` (launch scalars) or ``sample_into`` (per-row state); returns numpy outputs."""
    n = ROWS
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    logits = dev(bt["x"])
    kw = dict(keep_k=dev(bt["top_k"]), min_p=dev(bt["min_p"]))
    if bt["allow"] is not None:
        kw["allow"] = dev(pack_allow(bt["allow"]))
    if bt["per_row"]:
        rng = dev(np.stack([bt["seeds"], bt["steps"]], 1))
        toks = torch.empty(n, dtype=torch.int64, device=DEV)
        lp = torch.empty(n, device=DEV)
        ti = torch.empty(n, top_logprobs, dtype=torch.int64, device=DEV)
        tl = torch.empty(n, top_logprobs, device=DEV)
        C.sample_into(logits, dev(bt["t"]), dev(bt["top_p"]), rng, top_logprobs, toks, lp, ti, tl, **kw)
    else:
        toks, lp, ti, tl = C.sample(logits, dev(bt["t"]), dev(bt["top_p"]), int(bt["seeds"][0]), int(bt["steps"][0]),
                                    top_logprobs, **kw)
    torch.cuda.synchronize()
    return toks.cpu().numpy(), lp.cpu().numpy(), ti.cpu().numpy(), tl.cpu().numpy()


@pytest.fixture(scope="module", params=VOCABS, ids=lambda v: f"V{v}")
def draws(request, C):
    """Both launches of one vocabulary size: the kernel's outputs next to the batch."""
    return [(bt, launch(C, bt)) for bt in (batch(request.param, False), batch(request.param, True))]


@pytest.mark.gpu
def test_tokens_match_the_replay(draws):
    for bt, (toks, _, _, _) in draws:
        ties, wrong = 0, []
        for b, c in enumerate(bt["cfgs"]):
            allow = None if bt["allow"] is None else bt["allow"][b]
            want, gap = replay(bt["x"][b], allow, float(bt["t"][b]), float(bt["top_p"][b]), int(bt["top_k"][b]),
                               float(bt["min_p"][b]), bt["seeds"][b], bt["steps"][b], bt["rows"][b])
            ties += gap < TIE
            if toks[b] != want and not gap < TIE:
                wrong.append((b, c, int(toks[b]), want, gap))
        rng = "per-row state" if bt["per_row"] else "launch scalars"
        assert not wrong, (bt["V"], rng, len(wrong), wrong[:8])
        assert ties < 0.01 * ROWS, ties


@pytest.mark.gpu
def test_logprobs_match_fp64(draws):
    """The drawn token's log-prob and the 10 top log-probs (value descending, then id ascending) are those of the full row,
    masked or not, against fp64 log_softmax."""
    for bt, (toks, lp, ti, tl) in draws:
        x = bt["x"].astype(np.float64)
        lsm = x - np.logaddexp.reduce(x, axis=1, keepdims=True)
        np.testing.assert_allclose(lp, lsm[np.arange(ROWS), toks], rtol=0, atol=2e-4)
        for b in range(ROWS):
            r = bt["x"][b]
            cand = np.nonzero(r >= np.partition(r, r.size - 10)[r.size - 10])[0]      # the 10 largest, and ties of the 10th
            order = cand[np.argsort(-r[cand], kind="stable")][:10]                   # value descending, then id ascending
            assert np.array_equal(ti[b], order), (bt["V"], b, ti[b], order)
            np.testing.assert_allclose(tl[b], lsm[b, order], rtol=0, atol=2e-4)


TAIL_V = 102400


@functools.lru_cache(maxsize=None)
def _tail_rows():
    """(seed, step) pairs for ``sample_into`` (row 0) whose hash puts some id at the top uniform value, and another whose
    largest value is in the 64 quanta below the top (and no id at the top), with that id."""
    ids = np.arange(TAIL_V, dtype=np.uint64)
    found = {}
    for step in range(1, 20000):
        k = hash_bits(5, step, 0, ids) >> _U64(40)                     # 24 bits: 2^24 - 1 is the top under 23 bits too
        top = int(k.max())
        if top == (1 << 24) - 1 and "top" not in found:
            found["top"] = (step, int(np.argmax(k)))
        elif (1 << 24) - 130 <= top < (1 << 24) - 2 and "near" not in found:
            found["near"] = (step, int(np.argmax(k)))
        if len(found) == 2:
            return found
    raise AssertionError(found)


def _pinned_row(where, side):
    step, j = _tail_rows()[where]
    x = (np.random.default_rng(11).standard_normal(TAIL_V) * 2).astype(np.float32)
    g = gumbel(hash_bits(5, step, 0, np.arange(TAIL_V)))
    s = x.astype(np.float64) + g
    best_other = np.max(np.delete(s, j))
    x[j] = np.float32(best_other - g[j] + (0.5 if side == "above" else -0.5))
    return step, j, x


@pytest.mark.gpu
@pytest.mark.parametrize("side", ["below", "above"])
@pytest.mark.parametrize("where", ["top", "near"])
def test_pinned_tail_noise(C, where, side):
    """An id whose uniform is the largest one the hash can give ("top"), or within 64 quanta of it ("near"), with its logit
    placed so its replay score is 0.5 below / above the best other score: the kernel must agree with the replay."""
    step, j, x = _pinned_row(where, side)
    want, gap = replay(x, None, 1.0, 1.0, 0, 0.0, 5, step, 0)
    assert (want == j) == (side == "above") and gap > 0.4
    toks = torch.empty(1, dtype=torch.int64, device=DEV)
    lp = torch.empty(1, device=DEV)
    C.sample_into(torch.from_numpy(x[None]).to(DEV), torch.ones(1, device=DEV), torch.ones(1, device=DEV),
                  torch.tensor([[5, step]], dtype=torch.int64, device=DEV), 0, toks, lp)
    assert int(toks.item()) == want, (where, side, j, int(toks.item()), want)


@pytest.mark.gpu
def test_tail_mass_of_a_full_vocabulary_draw(C):
    """Eight head ids hold 1 - 1e-6 of the mass at T = 1; 16 x 1024 draws put about 0.016 on the tail.  Checked against the
    fp64 softmax only, so a defect the replay shares with the kernel still shows."""
    V, n, launches = TAIL_V, 1024, 16
    rng = np.random.default_rng(3)
    head = rng.choice(V, 8, replace=False)
    hp = np.array([0.3, 0.2, 0.15, 0.1, 0.1, 0.07, 0.05, 0.03]) * (1 - 1e-6)
    x = np.full(V, np.log(1e-6 / (V - 8)), np.float32)
    x[head] = np.log(hp)
    p = np.exp(x.astype(np.float64) - np.logaddexp.reduce(x.astype(np.float64)))
    assert abs(p[head].sum() - (1 - 1e-6)) < 1e-9
    logits = torch.from_numpy(x).to(DEV).expand(n, V).contiguous()
    ones = torch.ones(n, device=DEV)
    toks = np.concatenate([C.sample(logits, ones, ones, 77, step, 0)[0].cpu().numpy() for step in range(1, launches + 1)])
    N = n * launches
    assert (~np.isin(toks, head)).sum() <= 3, np.unique(toks[~np.isin(toks, head)])[:20]
    f = np.array([(toks == h).sum() for h in head]) / N
    sigma = np.sqrt(p[head] * (1 - p[head]) / N)
    assert (np.abs(f - p[head]) < 5 * sigma).all(), (f, p[head])
