"""top-k, min-p, presence and frequency penalties on the CPU reference path: sampler semantics, step-block wire format, engine
and HTTP server."""
import http.client
import json
import os
import threading
from collections import Counter

import numpy as np
import pytest
import torch

from helpers import TINY_LLAMA
from mlx_sharding_b200.config import ModelConfig
from mlx_sharding_b200.engine.core import LLMEngine
from mlx_sharding_b200.engine.kv_cache import PagedKVCache
from mlx_sharding_b200.engine.sampler import OutputCounts, SamplingParams, folded_bias
from mlx_sharding_b200.models import build_stage
from mlx_sharding_b200.ops import reference as R
from mlx_sharding_b200.ops.meta import BatchMeta
from mlx_sharding_b200.parallel.graph_decode import HEADER_WORDS, StepViews, pack_step, unpack_header
from mlx_sharding_b200.parallel.pipeline import LocalPipeline
from mlx_sharding_b200.server import openai_api
from mlx_sharding_b200.utils.checkpoint import random_state_dict, write_synthetic_checkpoint


# ------------------------------------------------------------------------------------------------ reference semantics
def _draws(x, n=600, t=1.0, top_p=1.0, top_k=0, min_p=0.0, seed=0):
    """Tokens of ``n`` identical rows through ``reference.sample`` with the given controls."""
    logits = torch.tensor(x, dtype=torch.float32).repeat(n, 1)
    g = torch.Generator().manual_seed(seed)
    toks, lp, _, _ = R.sample(logits, torch.full((n,), t), torch.full((n,), top_p), generator=g,
                              top_k=torch.full((n,), top_k, dtype=torch.int32), min_p=torch.full((n,), min_p))
    return toks, lp


def test_top_k_keeps_ties_at_the_kth_value():
    x = [5.0, 4.0, 4.0, 4.0, 1.0, 0.0, float("-inf")]
    keep = R.filter_keep(torch.tensor(x), 1.0, 1.0, 2, 0.0)
    assert keep.tolist() == [True, True, True, True, False, False, False]
    toks, _ = _draws(x, top_k=2)
    assert set(toks.tolist()) == {0, 1, 2, 3}
    # k = 1 with a unique max is greedy; k >= V is off
    assert set(_draws(x, top_k=1)[0].tolist()) == {0}
    assert R.filter_keep(torch.tensor(x), 1.0, 1.0, len(x), 0.0).all()


def test_top_k_then_top_p_differs_from_top_p_alone():
    x = torch.tensor([0.4, 0.3, 0.2, 0.1]).log().tolist()
    # top-p 0.5 alone: ascending cumulative mass 0.1, 0.3, 0.6, 1.0 > 0.5 keeps {0, 1}
    assert R.filter_keep(torch.tensor(x), 1.0, 0.5, 0, 0.0).tolist() == [True, True, False, False]
    # top-k 2 renormalises to (4/7, 3/7): cumulative 3/7, 1.0 > 0.5 keeps {0} only
    assert R.filter_keep(torch.tensor(x), 1.0, 0.5, 2, 0.0).tolist() == [True, False, False, False]
    assert set(_draws(x, top_p=0.5)[0].tolist()) == {0, 1}
    assert set(_draws(x, top_p=0.5, top_k=2)[0].tolist()) == {0}


def test_min_p_is_taken_at_the_request_temperature():
    x = [2.0, 1.0, 0.0, -1.0]
    # T = 2: p_i / p_max = exp((x_i - 2) / 2) = 1, 0.61, 0.37, 0.22 -> min_p 0.5 keeps {0, 1}
    assert R.filter_keep(torch.tensor(x), 2.0, 1.0, 0, 0.5).tolist() == [True, True, False, False]
    # T = 1: ratios 1, 0.37, 0.14, 0.05 -> only {0}
    assert R.filter_keep(torch.tensor(x), 1.0, 1.0, 0, 0.5).tolist() == [True, False, False, False]
    toks, _ = _draws(x, n=4000, t=2.0, min_p=0.5)
    assert set(toks.tolist()) == {0, 1}
    f0 = (toks == 0).float().mean().item()
    assert abs(f0 - 1 / (1 + np.exp(-0.5))) < 0.03
    assert set(_draws(x, t=1.0, min_p=0.5)[0].tolist()) == {0}


def test_filters_leave_greedy_and_logprobs_alone():
    x = [0.5, 3.0, 2.0, -1.0]
    toks, lp = _draws(x, n=8, t=0.0, top_k=3, min_p=0.9)
    assert set(toks.tolist()) == {1}
    lf = torch.tensor(x)
    ref = (lf - torch.logsumexp(lf, 0))[1]
    assert torch.allclose(lp, ref.expand(8))
    # a sampled token's log-prob is still logit - logsumexp(logit): no temperature, no filter
    toks, lp = _draws(x, n=64, t=0.7, top_k=2)
    assert torch.allclose(lp, (lf - torch.logsumexp(lf, 0))[toks])


# ------------------------------------------------------------------------------------------------ step block
def _meta(B):
    return BatchMeta.build([1] * B, [3] * B, [[1 + b] for b in range(B)], 16, pad_blocks_to=8)


def _pack(params, counts=None):
    B = len(params)
    wire, lay = pack_step(7, _meta(B), torch.arange(B, dtype=torch.int64), params, [[]] * B, [(1, 0)] * B, False, counts=counts)
    return wire, lay


def _views(wire):
    lay, _ = unpack_header(wire)
    blk = torch.from_numpy(np.ascontiguousarray(wire[HEADER_WORDS:HEADER_WORDS + lay.size]))
    return lay, StepViews(blk, lay, 16, 16)


def test_default_wire_has_no_filter_section_and_no_bias_table():
    wire, lay = _pack([SamplingParams(), SamplingParams(temperature=0.8, top_p=0.9)])
    assert wire[7] == 0 and lay.F == 0 and lay.keep_k == -1 and lay.min_p == -1
    assert lay.C == 0 and lay.NB == 0 and lay.bidx == -1
    # greedy requests ignore top-k / min-p, and a penalised request that has generated nothing has nothing to fold: the wire
    # is the default one, byte for byte
    same, _ = _pack([SamplingParams(top_k=5, min_p=0.2, presence_penalty=1.0),
                     SamplingParams(temperature=0.8, top_p=0.9, frequency_penalty=0.5)], counts=[OutputCounts(), OutputCounts()])
    assert np.array_equal(same, wire)
    _, sv = _views(wire)
    assert not sv.has_filter and sv.keep_k is None and sv.min_p is None and not sv.has_pen


def test_filter_section_round_trip():
    params = [SamplingParams(temperature=1.0, top_k=50), SamplingParams(temperature=0.7, min_p=0.1),
              SamplingParams(temperature=0.0, top_k=9), SamplingParams(temperature=1.0, top_k=-1, top_p=0.9)]
    wire, lay = _pack(params)
    assert wire[7] == 1 and lay.F == 1 and lay.key[-1] == 1
    lay2, sv = _views(wire)
    assert lay2.key == lay.key and sv.has_filter and not sv.has_pen
    assert sv.keep_k.tolist() == [50, 0, 0, 0]
    assert sv.min_p.tolist() == pytest.approx([0.0, 0.1, 0.0, 0.0])
    assert sv.temps.tolist() == pytest.approx([1.0, 0.7, 0.0, 1.0]) and sv.top_p.tolist() == pytest.approx([1, 1, 1, 0.9])
    assert sv.tokens.tolist() == [0, 1, 2, 3]


def test_folded_table_for_output_5_5_7():
    f, p = 0.5, 0.3
    prm = SamplingParams(temperature=0.0, logit_bias={7: 1.0}, frequency_penalty=f, presence_penalty=p)
    counts = OutputCounts.of([5, 5, 7])
    ids, vals = folded_bias(prm, counts)
    assert ids.dtype == np.int32 and vals.dtype == np.float32
    assert dict(zip(ids.tolist(), vals.tolist())) == pytest.approx({7: 1.0 - (f + p), 5: -(2 * f + p)})
    wire, lay = _pack([prm, SamplingParams()], counts=[counts, None])
    assert lay.NB == 16 and wire[7] == 0
    _, sv = _views(wire)
    ids = sv.bidx[0].tolist()
    got = {i: v for i, v in zip(ids, sv.bval[0].tolist()) if i >= 0}
    assert sorted(i for i in ids if i >= 0) == [5, 7]            # one entry per token id
    assert got == pytest.approx({5: -(2 * f + p), 7: 1.0 - (f + p)})
    assert all(i == -1 for i in sv.bidx[1].tolist())


def test_merged_bias_and_penalty_round_trip():
    prm = SamplingParams(temperature=1.0, logit_bias={7: 1.0, 9: -2.0}, frequency_penalty=0.5, presence_penalty=0.25,
                         top_k=3)
    counts = OutputCounts.of([5, 5, 7])
    wire, lay = _pack([prm], counts=[counts])
    assert lay.F == 1 and lay.NB == 16 and lay.C == 32
    _, sv = _views(wire)
    assert sv.has_pen and sv.has_filter and sv.keep_k.tolist() == [3]
    ids = [i for i in sv.bidx[0].tolist() if i >= 0]
    assert len(ids) == len(set(ids)) == 3
    got = dict(zip(sv.bidx[0].tolist(), sv.bval[0].tolist()))
    assert got[7] == pytest.approx(0.25) and got[9] == pytest.approx(-2.0) and got[5] == pytest.approx(-1.25)
    # the reference sampler applies the folded table exactly like separate bias + penalty terms
    lf = torch.randn(1, 16)
    out = lf.clone()
    R.apply_penalties_(out, sv.rep, sv.penalty, sv.bidx, sv.bval)
    want = lf.clone()[0]
    want[7] += 1.0
    want[9] -= 2.0
    for t, c in ((5, 2), (7, 1)):
        want[t] -= 0.5 * c + 0.25
    assert torch.allclose(out[0], want, atol=1e-6)


def test_bias_table_grows_to_the_next_bucket():
    prm = SamplingParams(temperature=1.0, presence_penalty=0.5)
    _, lay = _pack([prm], counts=[OutputCounts.of(range(16))])
    assert lay.NB == 16
    _, lay = _pack([prm], counts=[OutputCounts.of(range(17))])
    assert lay.NB == 32


def test_largest_penalised_decode_step_fits_the_control_ring():
    """A max-batch decode step where every row has a penalty table at its limit (plus a repetition context, top-k / min-p and
    top log-probs) fits one slot of the multi-process control ring."""
    from mlx_sharding_b200.engine.sampler import MAX_PENALTY_TABLE
    from mlx_sharding_b200.parallel.pipeline import control_slot_bytes
    from mlx_sharding_b200.parallel.shm_ring import KIND_STEP, ShmControl

    B, n_bias = 64, 24
    prm = SamplingParams(temperature=1.0, top_k=40, min_p=0.05, logprobs=5, repetition_penalty=1.1,
                         frequency_penalty=0.5, presence_penalty=0.5, logit_bias={100000 + i: 1.0 for i in range(n_bias)})
    counts = OutputCounts.of([t for t in range(MAX_PENALTY_TABLE - n_bias) for _ in range(1 + t % 3)])
    meta = BatchMeta.build([1] * B, [4000] * B, [list(range(1 + 63 * b, 64 + 63 * b)) for b in range(B)], 64, pad_blocks_to=64)
    wire, lay = pack_step(3, meta, torch.arange(B, dtype=torch.int64), [prm] * B, [list(range(20))] * B, [(1, 5)] * B,
                          False, counts=[counts] * B)
    assert lay.NB == MAX_PENALTY_TABLE and lay.F == 1
    assert wire.nbytes > 256 << 10                     # more than the ring's 256 KiB floor
    ctl = ShmControl.create(1, slots=2, slot_bytes=control_slot_bytes(2048, B))
    try:
        assert wire.size <= ctl.max_payload_words
        ctl.publish(KIND_STEP, 0, wire)
    finally:
        ctl.unlink()


def test_penalised_request_over_the_table_limit_is_refused():
    from mlx_sharding_b200.engine.sampler import MAX_PENALTY_TABLE

    _, eng = _engine()
    with pytest.raises(ValueError, match="max_tokens"):
        eng.submit([1, 2, 3], SamplingParams(frequency_penalty=0.5), max_tokens=MAX_PENALTY_TABLE + 1)
    with pytest.raises(ValueError, match="logit_bias"):
        eng.submit([1, 2, 3], SamplingParams(presence_penalty=0.5, logit_bias={1: 1.0, 2: 1.0}), max_tokens=MAX_PENALTY_TABLE - 1)
    # at the limit, and without a penalty, long generations are accepted
    eng.submit([1, 2, 3], SamplingParams(presence_penalty=0.5, logit_bias={1: 1.0}), max_tokens=MAX_PENALTY_TABLE - 1).cancel()
    eng.submit([1, 2, 3], SamplingParams(logit_bias={1: 1.0}), max_tokens=4 * MAX_PENALTY_TABLE).cancel()
    eng.drain()


def test_sampling_params_validation():
    for bad in (dict(top_k=-2), dict(top_k=1.5), dict(top_k=True), dict(min_p=1.5), dict(min_p=-0.1),
                dict(presence_penalty=2.5), dict(frequency_penalty=-3.0)):
        with pytest.raises(ValueError):
            SamplingParams(**bad).validate()
    SamplingParams(top_k=-1, min_p=1.0, presence_penalty=-2.0, frequency_penalty=2.0).validate()


# ------------------------------------------------------------------------------------------------ engine
def _engine(**kw):
    cfg = ModelConfig.from_dict(TINY_LLAMA)
    sd = dict(random_state_dict(cfg, dtype=torch.float32))
    models = [build_stage(cfg, cfg.shard(0, cfg.num_hidden_layers), torch.float32).load_state(sd)]
    pipe = LocalPipeline.from_models(models, num_pages=64, page_size=16)
    return models, LLMEngine(pipe, num_pages=64, page_size=16, **kw)


def _penalised_oracle(models, prompt, n, frequency, presence, page_size=16):
    """Greedy decode of one sequence with ``logit[j] -= frequency * c[j] + presence * (c[j] > 0)`` over its own output."""
    npages = (len(prompt) + n + page_size - 1) // page_size + 2
    kvs = [PagedKVCache.for_model(m, npages, page_size) for m in models]
    pages = list(range(1, npages))

    def step(ids, c0):
        meta = BatchMeta.build([len(ids)], [c0], [pages], page_size)
        x = torch.tensor(ids, dtype=torch.int64)
        for m, kv in zip(models, kvs):
            x = m(x, meta, kv)
        return x[-1].float()

    logits, out, counts = step(list(prompt), 0), [], Counter()
    for i in range(n):
        lg = logits.clone()
        for t, c in counts.items():
            lg[t] -= frequency * c + presence * (c > 0)
        tok = int(lg.argmax())
        out.append(tok)
        counts[tok] += 1
        if i + 1 < n:
            logits = step([tok], len(prompt) + i)
    return out


def test_engine_presence_and_frequency_penalties_match_oracle():
    models, eng = _engine()
    prompt = [3, 9, 27, 81]
    plain = eng.generate(prompt, SamplingParams(), max_tokens=12)
    prm = SamplingParams(temperature=0.0, frequency_penalty=1.5, presence_penalty=0.5)
    r = eng.submit(prompt, prm, max_tokens=12)
    eng.drain()
    want = _penalised_oracle(models, prompt, 12, 1.5, 0.5)
    assert r.output == want
    assert r.output != plain              # the penalty changes this greedy continuation
    assert dict(zip(r.counts.ids[:len(r.counts)].tolist(), r.counts.cnt[:len(r.counts)].tolist())) == Counter(r.output)
    assert eng._penalised == 0
    # negative penalties reward repetition; a default request next to a penalised one is unaffected
    a = eng.submit(prompt, SamplingParams(frequency_penalty=-1.0, presence_penalty=-0.5), max_tokens=8)
    b = eng.submit(prompt, SamplingParams(), max_tokens=8)
    eng.drain()
    assert a.output == _penalised_oracle(models, prompt, 8, -1.0, -0.5)
    assert b.output == plain[:8] and b.counts is None


def test_engine_filters_on_reference_backend():
    models, eng = _engine()
    prompt = [5, 6, 7]
    greedy = eng.generate(prompt, SamplingParams(), max_tokens=6)
    # top-k 1 and min-p 1 keep only the argmax: sampled requests decode greedily
    assert eng.generate(prompt, SamplingParams(temperature=1.0, top_k=1, seed=3), max_tokens=6) == greedy
    assert eng.generate(prompt, SamplingParams(temperature=1.5, min_p=1.0, seed=4), max_tokens=6) == greedy
    a = eng.generate(prompt, SamplingParams(temperature=1.0, top_k=20, top_p=0.9, min_p=0.05, seed=11), max_tokens=8)
    b = eng.generate(prompt, SamplingParams(temperature=1.0, top_k=20, top_p=0.9, min_p=0.05, seed=11), max_tokens=8)
    assert a == b and len(a) == 8


# ------------------------------------------------------------------------------------------------ HTTP
@pytest.fixture(scope="module")
def server(tmp_path_factory):
    d = tmp_path_factory.mktemp("ckpt")
    path = write_synthetic_checkpoint(str(d / "tiny"), TINY_LLAMA, dtype=torch.float32)
    cwd = os.getcwd()
    os.chdir(d)
    args = openai_api.build_arg_parser().parse_args(["--model", path, "--port", "0", "--kv-pages", "128", "--page-size", "16"])
    args.static_dir = os.path.join(os.path.dirname(openai_api.__file__), "static")
    provider = openai_api.ModelProvider(args, [])
    httpd = openai_api.make_server("127.0.0.1", 0, provider, args.static_dir)
    t = threading.Thread(target=httpd.serve_forever, daemon=True)
    t.start()
    yield httpd.server_address[1], provider
    httpd.shutdown()
    provider.engine.shutdown()
    os.chdir(cwd)


def _post(port, path, body):
    c = http.client.HTTPConnection("127.0.0.1", port, timeout=60)
    c.request("POST", path, json.dumps(body), {"Content-Type": "application/json"})
    r = c.getresponse()
    data = r.read()
    c.close()
    return r, json.loads(data)


@pytest.mark.parametrize("field,value", [("top_k", -2), ("top_k", 2.5), ("top_k", "5"), ("top_k", True), ("min_p", 1.5),
                                         ("min_p", -0.1), ("min_p", "0.1"), ("presence_penalty", 2.5),
                                         ("presence_penalty", [1]), ("frequency_penalty", -2.1), ("frequency_penalty", False)])
def test_bad_values_are_rejected(server, field, value):
    port, _ = server
    for path in ("/v1/completions", "/v1/chat/completions"):
        body = {"prompt": "hi", "messages": [{"role": "user", "content": "hi"}], "max_tokens": 2, field: value}
        r, j = _post(port, path, body)
        assert r.status == 400 and field in j["error"]["message"], (path, j)


def test_http_refuses_penalised_request_over_the_table_limit(server):
    port, _ = server
    r, j = _post(port, "/v1/completions", {"prompt": "hi", "max_tokens": 2000, "frequency_penalty": 0.5})
    assert r.status == 400 and "max_tokens" in j["error"]["message"]


def test_http_penalties_and_filters(server):
    port, provider = server
    body = {"prompt": "hello there", "max_tokens": 10, "temperature": 0, "frequency_penalty": 1.5, "presence_penalty": 0.5}
    r, j = _post(port, "/v1/completions", body)
    assert r.status == 200
    toks = j["choices"][0]["logprobs"]["tokens"]
    prompt = list(provider.tokenizer.encode("hello there"))
    want = _penalised_oracle([provider.model], prompt, 10, 1.5, 0.5)
    assert toks and toks == want[:len(toks)]
    assert len(toks) == 10 or j["choices"][0]["finish_reason"] == "stop"
    # top_k 1 at temperature 1 is greedy; nulls mean "default"
    plain = {"messages": [{"role": "user", "content": "x"}], "max_tokens": 6, "temperature": 0}
    _, g = _post(port, "/chat/completions", plain)
    _, k1 = _post(port, "/v1/chat/completions", dict(plain, temperature=1.0, top_k=1, min_p=None, presence_penalty=None))
    assert k1["choices"][0]["logprobs"]["tokens"] == g["choices"][0]["logprobs"]["tokens"]
