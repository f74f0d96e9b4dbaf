"""GPU: the sm_90a sampler's top-k / min-p filters against the reference kept sets, the unchanged default path, and the
filters and presence / frequency penalties through the graph-replayed step block."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import GPU_LLAMA
from mlx_sharding_b200.engine.sampler import OutputCounts, SamplingParams, folded_bias
from mlx_sharding_b200.ops import reference as R

DEV = "cuda"
V = 102400


@pytest.fixture(scope="module")
def B():
    from mlx_sharding_b200.ops import b200

    b200.load_extension()
    return b200


def _row(seed=0, scale=2.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(V, generator=g) * scale


def _draw(B, row, n=4096, t=1.0, top_p=1.0, top_k=0, min_p=0.0, seed=1):
    logits = row.to(DEV).repeat(n, 1).contiguous()
    g = torch.Generator(device=DEV).manual_seed(seed)
    toks, _, _, _ = B.sample(logits, torch.full((n,), t, device=DEV), torch.full((n,), top_p, device=DEV), generator=g,
                             top_k=torch.full((n,), top_k, dtype=torch.int32, device=DEV),
                             min_p=torch.full((n,), min_p, device=DEV))
    return toks.cpu()


def _assert_within(toks, keep):
    kept = set(torch.nonzero(keep).flatten().tolist())
    got = set(toks.tolist())
    assert got <= kept, sorted(got - kept)[:10]
    return got


@pytest.mark.parametrize("k", [1, 50, 1000])
def test_top_k_support(B, k):
    row = _row(k)
    row[torch.randperm(V, generator=torch.Generator().manual_seed(3))[:100]] = float("-inf")   # logit_bias -inf entries
    keep = R.filter_keep(row, 1.0, 1.0, k, 0.0)
    assert int(keep.sum()) == k
    got = _assert_within(_draw(B, row, top_k=k), keep)
    assert len(got) >= min(k, 20)
    if k == 1:
        assert got == {int(row.argmax())}


def test_top_k_keeps_ties_at_the_boundary(B):
    row = _row(5).clamp(max=8.0)                      # every other logit stays below the designed ones
    idx = torch.randperm(V, generator=torch.Generator().manual_seed(4))[:55]
    row[idx[:45]] = 10.0 + 0.01 * torch.arange(45, dtype=torch.float32)   # ranks 1..45
    row[idx[45:]] = 9.0                                                   # ranks 46..55 tie; k = 50 falls inside the tie
    keep = R.filter_keep(row, 1.0, 1.0, 50, 0.0)
    assert int(keep.sum()) == 55
    got = _assert_within(_draw(B, row, top_k=50, n=8192), keep)
    assert len(got & set(idx[50:].tolist())) > 0      # tied tokens past rank 50 are drawn too


def test_top_k_beyond_the_finite_logits(B):
    row = torch.full((V,), float("-inf"))
    fin = torch.randperm(V, generator=torch.Generator().manual_seed(6))[:30]
    row[fin] = torch.randn(30, generator=torch.Generator().manual_seed(7))
    got = set(_draw(B, row, top_k=50).tolist())       # k-th largest is -inf: every finite token stays
    assert got <= set(fin.tolist()) and len(got) > 10


@pytest.mark.parametrize("t", [0.7, 1.5])
def test_min_p_support(B, t):
    row = _row(8)
    mp = 0.05
    th = float(row.max()) + t * torch.log(torch.tensor(mp)).item()
    near = (row - th).abs() < 1e-2
    row[near] -= 2e-2                                 # keep the designed logits away from the min-p boundary
    keep = R.filter_keep(row, t, 1.0, 0, mp)
    assert 1 < int(keep.sum()) < V // 10
    got = _assert_within(_draw(B, row, t=t, min_p=mp), keep)
    assert len(got) > 1


def test_top_k_and_top_p_support(B):
    row = _row(9)
    keep = R.filter_keep(row, 1.0, 0.5, 1000, 0.0)
    alone = R.filter_keep(row, 1.0, 0.5, 0, 0.0)
    assert int(keep.sum()) < int(alone.sum())         # the nucleus of the top-k set is narrower than top-p alone
    _assert_within(_draw(B, row, top_p=0.5, top_k=1000), keep)
    # all three together
    keep = R.filter_keep(row, 1.0, 0.9, 1000, 0.02)
    _assert_within(_draw(B, row, top_p=0.9, top_k=1000, min_p=0.02), keep)


def test_filtered_frequencies(B):
    Vs, n = 64, 4000
    base = torch.tensor([4.0, 3.0, 2.0, 1.0] + [-4.0] * (Vs - 4), device=DEV)
    logits = base.repeat(n, 1).contiguous()
    g = torch.Generator(device=DEV).manual_seed(1234)
    ones = torch.ones(n, device=DEV)

    def freq(**kw):
        filt = dict(top_k=torch.full((n,), kw.get("top_k", 0), dtype=torch.int32, device=DEV),
                    min_p=torch.full((n,), kw.get("min_p", 0.0), device=DEV))
        toks, _, _, _ = B.sample(logits, ones * kw.get("t", 1.0), ones * kw.get("top_p", 1.0), generator=g, **filt)
        return torch.bincount(toks, minlength=Vs).float().cpu() / n

    def renorm(idx, t=1.0):
        p = torch.softmax(base.cpu()[idx] / t, 0)
        out = torch.zeros(Vs)
        out[idx] = p
        return out

    f = freq(top_k=3)
    assert (f - renorm([0, 1, 2])).abs().max() < 0.03, f[:4]
    f = freq(min_p=0.3)                               # ratios 1, 0.37, 0.14: keeps {0, 1}
    assert (f - renorm([0, 1])).abs().max() < 0.03, f[:4]
    f = freq(min_p=0.3, t=2.0)                        # ratios 1, 0.61, 0.37, 0.22: keeps {0, 1, 2}
    assert (f - renorm([0, 1, 2], 2.0)).abs().max() < 0.03, f[:4]
    f = freq(top_k=3, top_p=0.7)                      # renormalised (0.67, 0.24, 0.09): nucleus 0.7 keeps {0, 1}
    assert (f - renorm([0, 1])).abs().max() < 0.03, f[:4]


@pytest.mark.parametrize("t,top_p", [(0.0, 1.0), (1.0, 1.0), (1.0, 0.9)])
def test_default_path_unchanged(B, t, top_p):
    """Null filter pointers and filter arrays that are off give bitwise the same tokens and log-probs."""
    n = 64
    g = torch.Generator(device=DEV).manual_seed(11)
    logits = (torch.randn(n, V, device=DEV, generator=g) * 3).contiguous()
    temps, tps = torch.full((n,), t, device=DEV), torch.full((n,), top_p, device=DEV)
    rng = torch.stack([torch.arange(n) + 100, torch.full((n,), 7)], 1).to(torch.int64).to(DEV).contiguous()
    outs = []
    for filt in ({}, dict(keep_k=torch.zeros(n, dtype=torch.int32, device=DEV), min_p=torch.zeros(n, device=DEV)),
                 dict(keep_k=torch.full((n,), V, dtype=torch.int32, device=DEV), min_p=torch.zeros(n, device=DEV))):
        toks = torch.empty(n, dtype=torch.int64, device=DEV)
        lp = torch.empty(n, device=DEV)
        B.C().sample_into(logits, temps, tps, rng, 0, toks, lp, **filt)
        outs.append((toks.cpu(), lp.cpu()))
    for toks, lp in outs[1:]:
        assert torch.equal(toks, outs[0][0]) and torch.equal(lp.view(torch.int32), outs[0][1].view(torch.int32))


def test_penalty_table_same_greedy_tokens_on_both_backends(B):
    n = 8
    g = torch.Generator().manual_seed(12)
    logits = torch.randn(n, V, generator=g) * 2
    prm = SamplingParams(logit_bias={3: 1.0}, frequency_penalty=1.5, presence_penalty=0.5)
    tables = []
    for b in range(n):
        top = torch.topk(logits[b], 4).indices.tolist()        # penalise the current leaders so the argmax moves
        tables.append(folded_bias(prm, OutputCounts.of([top[0]] * 3 + [top[1], 3, 3])))
    NB = max(len(ids) for ids, _ in tables)
    bidx = torch.full((n, NB), -1, dtype=torch.int32)
    bval = torch.zeros(n, NB)
    for b, (ids, vals) in enumerate(tables):
        bidx[b, :len(ids)], bval[b, :len(ids)] = torch.from_numpy(ids), torch.from_numpy(vals)
    ctx, pen = torch.full((n, 1), -1, dtype=torch.int32), torch.ones(n)
    zeros, ones = torch.zeros(n), torch.ones(n)
    a = logits.to(DEV).contiguous()
    B.apply_penalties_(a, ctx.to(DEV), pen.to(DEV), bidx.to(DEV), bval.to(DEV))
    ta, _, _, _ = B.sample(a, zeros.to(DEV), ones.to(DEV))
    r = logits.clone()
    R.apply_penalties_(r, ctx, pen, bidx, bval)
    tr, _, _, _ = R.sample(r, zeros, ones)
    assert torch.equal(ta.cpu(), tr)
    assert not torch.equal(tr, logits.argmax(-1))             # the table changed some greedy tokens


def test_graph_replay_mixed_batch():
    from mlx_sharding_b200.engine.core import LLMEngine
    from mlx_sharding_b200.parallel.pipeline import LocalPipeline
    from mlx_sharding_b200.utils.loader import random_model

    model = random_model(GPU_LLAMA, dtype=torch.bfloat16, device="cuda:0", backend="b200", seed=0)
    prompts = [[5, 6, 7, 8], [100, 50, 3], list(range(20, 40)), [42] * 9, [7, 300, 12], [9, 9, 1]]
    default = [SamplingParams(), SamplingParams(logprobs=2), SamplingParams(temperature=0.8, top_p=0.9, seed=5)]
    controls = [SamplingParams(temperature=1.0, top_k=20, min_p=0.05, seed=7),
                SamplingParams(frequency_penalty=2.0, presence_penalty=1.0),
                SamplingParams(temperature=0.9, top_k=40, top_p=0.8, frequency_penalty=0.4, logit_bias={11: -1.0}, seed=9)]
    off = [SamplingParams(temperature=1.0, seed=7), SamplingParams(), SamplingParams(temperature=0.9, top_p=0.8, seed=9)]

    def run(params):
        pipe = LocalPipeline.from_models([model], num_pages=64, page_size=16)
        eng = LLMEngine(pipe, num_pages=64, page_size=16)
        reqs = [eng.submit(p, prm, max_tokens=40) for p, prm in zip(prompts, params)]
        eng.drain()
        assert all(r.finished and len(r.output) == 40 for r in reqs)
        assert pipe.gcache.replays >= 20, pipe.gcache.replays
        return [r.output for r in reqs], pipe

    mixed, pipe = run(default + controls)
    keys = {k[1] for k in pipe.gcache.entries}
    assert any(k[-1] == 1 for k in keys)                          # the filter section is part of the graph key
    assert len({k[4] for k in keys}) >= 2                         # the bias table crossed an NB bucket
    assert len(set(mixed[4])) > 16                                # the penalised greedy request keeps moving on
    plain, _ = run(default + off)
    assert mixed[:3] == plain[:3]                                 # default rows do not see the other rows' controls
    again, _ = run(default + controls)
    assert again == mixed                                         # seeded filtered requests reproduce
