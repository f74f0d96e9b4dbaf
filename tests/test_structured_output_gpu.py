"""GPU: the sm_90a sampler's token mask (structured output) against the reference — support of greedy, temperature and filtered
draws at V = 102400, masked frequencies, bitwise-unchanged log-probs and unmasked rows — and a graph-replayed engine batch that
mixes constrained, filtered and default requests."""
import json

import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import GPU_LLAMA
from mlx_sharding_b200.engine.grammar import mask_words
from mlx_sharding_b200.engine.sampler import SamplingParams
from mlx_sharding_b200.ops import reference as R

DEV = "cuda"
V = 102400
NB = 64


@pytest.fixture(scope="module")
def B():
    from mlx_sharding_b200.ops import b200

    b200.load_extension()
    return b200


def pack_allow(ok: torch.Tensor) -> torch.Tensor:
    """bool [B, V] -> int32 [B, ceil(V/32)] token mask (inverse of ``reference.unpack_allow``)."""
    b, v = ok.shape
    W = mask_words(v)
    bits = torch.zeros(b, W * 32, dtype=torch.int64)
    bits[:, :v] = ok.long()
    words = (bits.view(b, W, 32) << torch.arange(32)).sum(-1)
    return torch.where(words >= 1 << 31, words - (1 << 32), words).to(torch.int32)


def _logits(seed, n=NB, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, V, generator=g) * scale


def _mask(kind, lf, seed):
    g = torch.Generator().manual_seed(seed)
    n = lf.shape[0]
    if kind == "one":
        ok = torch.zeros(n, V, dtype=torch.bool)
        ok[torch.arange(n), torch.randint(0, V, (n,), generator=g)] = True
        return ok
    if kind == "far":                                   # allowed ids sit 100 logits below the row max
        ok = torch.rand(n, V, generator=g) < 0.01
        lf[ok] -= 100.0
        return ok
    frac = {"1%": 0.01, "50%": 0.5}[kind]
    return torch.rand(n, V, generator=g) < frac


def _sample(B, lf, t, allow=None, top_p=1.0, top_k=0, min_p=0.0, seed=1, k=0):
    n = lf.shape[0]
    g = torch.Generator(device=DEV).manual_seed(seed)
    extra = {} if allow is None else dict(allow=allow.to(DEV))
    return B.sample(lf.to(DEV).contiguous(), torch.full((n,), t, device=DEV), torch.full((n,), top_p, device=DEV), generator=g,
                    top_logprobs=k, top_k=torch.full((n,), top_k, dtype=torch.int32, device=DEV),
                    min_p=torch.full((n,), min_p, device=DEV), **extra)


@pytest.mark.parametrize("kind", ["1%", "50%", "one", "far"])
def test_masked_greedy_and_draws(B, kind):
    lf = _logits(1)
    ok = _mask(kind, lf, 2)
    allow = pack_allow(ok)
    toks = _sample(B, lf, 0.0, allow)[0].cpu()
    assert torch.equal(toks, lf.masked_fill(~ok, float("-inf")).argmax(-1))
    rows = torch.arange(NB)
    for seed in range(8):
        for t, p in ((1.0, 1.0), (0.7, 0.9), (1.5, 0.5)):
            toks = _sample(B, lf, t, allow, top_p=p, seed=100 + seed)[0].cpu()
            assert ok[rows, toks].all(), (kind, seed, t, p)


@pytest.mark.parametrize("kind", ["1%", "50%", "far"])
@pytest.mark.parametrize("top_k,top_p,min_p", [(20, 1.0, 0.0), (0, 0.5, 0.0), (0, 1.0, 0.1), (200, 0.9, 0.02)])
def test_masked_filter_support_is_the_reference_kept_set(B, kind, top_k, top_p, min_p):
    n, t = 4096, 1.0
    lf = _logits(3, n=1, scale=2.0)
    ok = _mask(kind, lf, 4)
    masked = lf[0].masked_fill(~ok[0], float("-inf"))
    keep = R.filter_keep(masked, t, top_p, top_k, min_p)
    kept = set(torch.nonzero(keep & ok[0]).flatten().tolist())
    probs = torch.softmax((masked / t).masked_fill(~keep, float("-inf")), 0)
    likely = set(torch.nonzero(probs > 5e-3).flatten().tolist())
    got = set(_sample(B, lf.repeat(n, 1), t, pack_allow(ok.repeat(n, 1)), top_p, top_k, min_p, seed=5)[0].cpu().tolist())
    assert got <= kept, sorted(got - kept)[:10]
    assert likely <= got, sorted(likely - got)[:10]


def test_masked_frequencies(B):
    Vs, n = 64, 4000
    base = torch.tensor([4.0, 3.0, 2.0, 1.0] + [-4.0] * (Vs - 4))
    ok = torch.zeros(Vs, dtype=torch.bool)
    ok[[1, 2, 5, 9]] = True
    logits = base.to(DEV).repeat(n, 1).contiguous()
    allow = pack_allow(ok.repeat(n, 1)).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(77)
    ones = torch.ones(n, device=DEV)

    def freq(t=1.0, top_p=1.0, top_k=0):
        toks, _, _, _ = B.sample(logits, ones * t, ones * top_p, generator=g, allow=allow,
                                 top_k=torch.full((n,), top_k, dtype=torch.int32, device=DEV), min_p=ones * 0)
        return torch.bincount(toks, minlength=Vs).float().cpu() / n

    def renorm(idx, t=1.0):
        p = torch.softmax(base[idx] / t, 0)
        out = torch.zeros(Vs)
        out[idx] = p
        return out

    f = freq()
    assert (f - renorm([1, 2, 5, 9])).abs().max() < 0.03, f[:10]
    f = freq(t=2.0)
    assert (f - renorm([1, 2, 5, 9], 2.0)).abs().max() < 0.03, f[:10]
    f = freq(top_k=2)                                  # the 2 largest allowed: {1, 2}
    assert (f - renorm([1, 2])).abs().max() < 0.03, f[:10]


@pytest.mark.parametrize("t,top_p", [(0.0, 1.0), (1.0, 1.0), (1.0, 0.9)])
def test_unmasked_outputs_unchanged(B, t, top_p):
    """All-ones and empty masks give bitwise the tokens and log-probs of no mask; a real mask leaves the log-probs and top
    log-probs bitwise alone."""
    n, k = 64, 5
    g = torch.Generator(device=DEV).manual_seed(11)
    logits = (torch.randn(n, V, device=DEV, generator=g) * 3).contiguous()
    temps, tps = torch.full((n,), t, device=DEV), torch.full((n,), top_p, device=DEV)
    rng = torch.stack([torch.arange(n) + 100, torch.full((n,), 7)], 1).to(torch.int64).to(DEV).contiguous()
    W = mask_words(V)

    def run(allow):
        toks = torch.empty(n, dtype=torch.int64, device=DEV)
        lp = torch.empty(n, device=DEV)
        ti = torch.empty(n, k, dtype=torch.int64, device=DEV)
        tl = torch.empty(n, k, device=DEV)
        B.C().sample_into(logits, temps, tps, rng, k, toks, lp, ti, tl, allow=allow)
        return toks.cpu(), lp.cpu().view(torch.int32), ti.cpu(), tl.cpu().view(torch.int32)

    base = run(None)
    for allow in (torch.full((n, W), -1, dtype=torch.int32, device=DEV), torch.zeros(n, W, dtype=torch.int32, device=DEV)):
        got = run(allow)
        assert all(torch.equal(a, b) for a, b in zip(got, base))
    ok = torch.rand(n, V, generator=torch.Generator().manual_seed(12)) < 0.01
    toks, lp, ti, tl = run(pack_allow(ok).to(DEV))
    assert ok[torch.arange(n), toks].all()
    assert torch.equal(ti, base[2]) and torch.equal(tl, base[3])
    want = (logits - torch.logsumexp(logits, -1, keepdim=True)).cpu().gather(1, toks[:, None])[:, 0]
    assert torch.allclose(lp.view(torch.float32), want, atol=1e-4)
    # the chosen token's log-prob is the unmasked row's, exactly as an unmasked draw of the same token reports it
    same = toks == base[0]
    assert torch.equal(lp[same], base[1][same])


def test_graph_replay_mixed_constrained_batch(tmp_path):
    pytest.importorskip("xgrammar")
    from mlx_sharding_b200.engine.core import LLMEngine
    from mlx_sharding_b200.engine.grammar import GrammarBackend, canonical_format
    from mlx_sharding_b200.engine.tokenizer import load_tokenizer, write_byte_tokenizer
    from mlx_sharding_b200.parallel.pipeline import LocalPipeline
    from mlx_sharding_b200.utils.loader import random_model

    tok = load_tokenizer(write_byte_tokenizer(str(tmp_path / "tok"), vocab_size=GPU_LLAMA["vocab_size"]))
    eos = tok.eos_token_id
    grammar = GrammarBackend(tok, GPU_LLAMA["vocab_size"])
    model = random_model(GPU_LLAMA, dtype=torch.bfloat16, device="cuda:0", backend="b200", seed=0)
    schema = {"type": "object", "properties": {"c": {"enum": ["red", "green"]}}, "required": ["c"], "additionalProperties": False}
    enum_fmt = canonical_format({"type": "json_schema", "json_schema": {"name": "c", "schema": schema}})
    obj_fmt = canonical_format({"type": "json_object"})
    prompts = [[5, 6, 7, 8], [100, 50, 3], list(range(20, 40)), [42] * 9, [7, 300, 12], [9, 9, 1]]
    others = [SamplingParams(), SamplingParams(temperature=0.8, top_p=0.9, seed=5, logprobs=2),
              SamplingParams(temperature=1.0, top_k=20, min_p=0.05, seed=7), SamplingParams(frequency_penalty=1.0)]
    constrained = [SamplingParams(response_format=enum_fmt), SamplingParams(temperature=1.0, seed=3, response_format=obj_fmt)]

    def run(params, max_tokens):
        pipe = LocalPipeline.from_models([model], num_pages=64, page_size=16)
        eng = LLMEngine(pipe, num_pages=64, page_size=16)
        eng.grammar = grammar
        reqs = [eng.submit(p, prm, max_tokens=m, eos_token_id=eos if prm.response_format else None)
                for p, prm, m in zip(prompts, params, max_tokens)]
        eng.drain()
        assert all(r.finished and r.error is None for r in reqs), [r.error for r in reqs]
        return reqs, pipe

    reqs, pipe = run(others + constrained, [40] * 6)
    assert pipe.gcache.replays > 0
    assert any(k[1][6] == mask_words(GPU_LLAMA["vocab_size"]) for k in pipe.gcache.entries)     # masked graphs were replayed
    enum, obj = reqs[4], reqs[5]
    assert enum.finish_reason == "stop" and enum.output[-1] == eos
    assert json.loads(tok.decode(enum.output[:-1]))["c"] in ("red", "green")
    m = grammar.matcher(obj_fmt)
    assert obj.output[0] == ord("{") and all(m.accept_token(t) for t in obj.output)
    # the same batch with the constrained requests replaced by unconstrained ones of the same lengths: the other rows' tokens
    # do not change
    plain, _ = run(others + [SamplingParams(), SamplingParams(temperature=1.0, seed=3)],
                   [40] * 4 + [len(enum.output), len(obj.output)])
    assert [r.output for r in plain[:4]] == [r.output for r in reqs[:4]]
