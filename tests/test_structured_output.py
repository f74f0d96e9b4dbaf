"""Structured output (``response_format``) on the CPU reference path: masked sampler semantics, the token-mask section of the step
block, the engine's grammar bookkeeping, the gloo chain and the HTTP server."""
import http.client
import json
import os
import socket
import threading
import types

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from helpers import TINY_LLAMA
from mlx_sharding_b200.config import ModelConfig
from mlx_sharding_b200.engine.core import LLMEngine
from mlx_sharding_b200.engine.grammar import canonical_format, mask_words
from mlx_sharding_b200.engine.sampler import SamplingParams
from mlx_sharding_b200.models import build_stage
from mlx_sharding_b200.ops import reference as R
from mlx_sharding_b200.ops.meta import BatchMeta
from mlx_sharding_b200.parallel.graph_decode import HEADER_WORDS, StepViews, pack_step, unpack_header
from mlx_sharding_b200.parallel.pipeline import LocalPipeline
from mlx_sharding_b200.utils.checkpoint import random_state_dict

ENUM_SCHEMA = {"type": "object", "properties": {"c": {"enum": ["red", "green"]}}, "required": ["c"],
               "additionalProperties": False}
ENUM_FORMAT = {"type": "json_schema", "json_schema": {"name": "c", "schema": ENUM_SCHEMA}}
ENUM_TEXTS = ('{"c": "red"}', '{"c": "green"}')
EOS = 257          # <|eos|> of the byte tokenizer (engine/tokenizer.py::write_byte_tokenizer)


def pack_allow(ok: torch.Tensor) -> torch.Tensor:
    """bool [B, V] -> int32 [B, ceil(V/32)] token mask (inverse of ``reference.unpack_allow``)."""
    B, V = ok.shape
    W = mask_words(V)
    bits = torch.zeros(B, W * 32, dtype=torch.int64)
    bits[:, :V] = ok.long()
    words = (bits.view(B, W, 32) << torch.arange(32)).sum(-1)
    return torch.where(words >= 1 << 31, words - (1 << 32), words).to(torch.int32)


# ------------------------------------------------------------------------------------------------ oracle
def _rows(B, V, seed):
    g = torch.Generator().manual_seed(seed)
    lf = torch.randn(B, V, generator=g) * 3
    ok = torch.rand(B, V, generator=g) < 0.3
    ok[:, 0] = False
    ok[torch.arange(B), torch.randint(1, V, (B,), generator=g)] = True      # at least one allowed id per row
    return lf, ok


def test_unpack_allow_round_trip_and_ignores_bits_past_v():
    lf, ok = _rows(3, 70, 0)
    allow = pack_allow(ok)
    assert allow.shape == (3, 3)
    assert torch.equal(R.unpack_allow(allow, 70), ok)
    allow[:, 2] = -1                                                         # ids 64..69 plus 26 bits past V
    assert R.unpack_allow(allow, 70)[:, 64:].all() and R.unpack_allow(allow, 70).shape == (3, 70)


def test_masked_greedy_and_draws_stay_allowed():
    B, V = 16, 200
    lf, ok = _rows(B, V, 1)
    allow = pack_allow(ok)
    toks, lp, ti, tl = R.sample(lf, torch.zeros(B), torch.ones(B), top_logprobs=5, allow=allow)
    assert torch.equal(toks, lf.masked_fill(~ok, float("-inf")).argmax(-1))
    want_lp = lf - torch.logsumexp(lf, -1, keepdim=True)
    assert torch.equal(lp, want_lp.gather(1, toks[:, None])[:, 0])
    # log-probs and top log-probs are those of the unmasked call
    t0, lp0, ti0, tl0 = R.sample(lf, torch.zeros(B), torch.ones(B), top_logprobs=5)
    assert torch.equal(ti, ti0) and torch.equal(tl, tl0)
    g = torch.Generator().manual_seed(3)
    for t, p in ((1.0, 1.0), (0.7, 0.9), (2.0, 0.5)):
        toks, _, _, _ = R.sample(lf, torch.full((B,), t), torch.full((B,), p), generator=g, allow=allow)
        assert ok[torch.arange(B), toks].all()


@pytest.mark.parametrize("top_k,top_p,min_p", [(5, 1.0, 0.0), (0, 0.8, 0.0), (0, 1.0, 0.2), (8, 0.9, 0.05), (10_000, 1.0, 0.0)])
def test_masked_filters_keep_filter_keep_of_the_masked_row(top_k, top_p, min_p):
    V, n, t = 40, 3000, 1.3
    lf, ok = _rows(1, V, 5)
    masked = lf[0].masked_fill(~ok[0], float("-inf"))
    keep = R.filter_keep(masked, t, top_p, top_k, min_p) & ok[0]
    g = torch.Generator().manual_seed(9)
    toks, lp, _, _ = R.sample(lf.repeat(n, 1), torch.full((n,), t), torch.full((n,), top_p), generator=g,
                              top_k=torch.full((n,), top_k, dtype=torch.int32), min_p=torch.full((n,), min_p),
                              allow=pack_allow(ok.repeat(n, 1)))
    got = set(toks.tolist())
    assert got <= set(torch.nonzero(keep).flatten().tolist())
    probs = torch.softmax((masked / t).masked_fill(~keep, float("-inf")), 0)
    likely = {int(j) for j in torch.nonzero(probs > 0.01).flatten()}
    assert likely <= got
    assert torch.allclose(lp, (lf[0] - torch.logsumexp(lf[0], 0))[toks])


def test_empty_mask_and_all_ones_mask_behave_as_no_mask():
    B, V = 8, 100
    lf, _ = _rows(B, V, 7)
    for fill in (0, -1):
        allow = torch.full((B, mask_words(V)), fill, dtype=torch.int32)
        for t in (0.0, 1.0):
            a = R.sample(lf, torch.full((B,), t), torch.full((B,), 0.9), generator=torch.Generator().manual_seed(1),
                         top_logprobs=3, allow=allow)
            b = R.sample(lf, torch.full((B,), t), torch.full((B,), 0.9), generator=torch.Generator().manual_seed(1),
                         top_logprobs=3)
            assert all(torch.equal(x, y) for x, y in zip(a, b))
    # an allowed set whose logits are all -inf is no allowed set either
    lf2 = lf.clone()
    lf2[:, :10] = float("-inf")
    allow = pack_allow(torch.arange(V).expand(B, V) < 10)
    assert torch.equal(R.sample(lf2, torch.zeros(B), torch.ones(B), allow=allow)[0], lf2.argmax(-1))


# ------------------------------------------------------------------------------------------------ step block
def _meta(B):
    return BatchMeta.build([1] * B, [3] * B, [[1 + b] for b in range(B)], 16, pad_blocks_to=8)


def _pack(params, allow=None, pad_decode=False):
    B = len(params)
    return pack_step(7, _meta(B), torch.arange(B, dtype=torch.int64), params, [[]] * B, [(1, 0)] * B, False,
                     pad_decode=pad_decode, allow=allow)


def _views(wire):
    lay, _ = unpack_header(wire)
    blk = torch.from_numpy(np.ascontiguousarray(wire[HEADER_WORDS:HEADER_WORDS + lay.size]))
    return lay, StepViews(blk, lay, 16, 16)


def test_unconstrained_batch_packs_the_same_bytes():
    params = [SamplingParams(), SamplingParams(temperature=0.8, top_k=5), SamplingParams(temperature=1.0, top_p=0.9)]
    B = len(params)
    old, lay = pack_step(7, _meta(B), torch.arange(B, dtype=torch.int64), params, [[]] * B, [(1, 0)] * B, False)
    new, lay2 = _pack(params, allow=None)
    assert np.array_equal(old, new) and lay2.W == 0 and lay2.allow == -1
    assert new[7] == lay.F == 1
    _, sv = _views(new)
    assert sv.allow is None


def test_mask_section_round_trip_and_padding_rows():
    V = 1000
    W = mask_words(V)
    rng = np.random.default_rng(0)
    allow = rng.integers(-(1 << 31), 1 << 31, size=(3, W), dtype=np.int64).astype(np.int32)
    allow[1] = -1
    params = [SamplingParams(response_format='{"type":"json_object"}'), SamplingParams(), SamplingParams(temperature=1.0, top_k=3)]
    wire, lay = _pack(params, allow=allow, pad_decode=True)          # 3 decode rows -> bucket of 4
    assert lay.B == 4 and lay.W == W and lay.F == 1
    assert wire[7] == 1 | (W << 1) and lay.allow % 4 == 0
    lay2, sv = _views(wire)
    assert lay2.key == lay.key and lay2.W == W
    assert np.array_equal(sv.allow[:3].numpy(), allow)
    assert (sv.allow[3] == -1).all()                                  # the padding row may draw anything
    assert sv.keep_k.tolist() == [0, 0, 3, 0] and sv.tokens.tolist()[:3] == [0, 1, 2]
    # the mask is part of the layout key, hence of the graph key
    _, lay3 = _pack(params[1:], allow=None)
    assert lay3.key != lay2.key


def test_largest_masked_decode_step_fits_the_control_ring():
    from mlx_sharding_b200.parallel.pipeline import control_slot_bytes
    from mlx_sharding_b200.parallel.shm_ring import KIND_STEP, ShmControl

    from mlx_sharding_b200.engine.sampler import MAX_PENALTY_TABLE, OutputCounts

    B, V = 64, 102400
    prm = SamplingParams(temperature=1.0, top_k=40, min_p=0.05, logprobs=5, repetition_penalty=1.1, frequency_penalty=0.5,
                         response_format='{"type":"json_object"}')
    counts = OutputCounts.of(range(MAX_PENALTY_TABLE))
    meta = BatchMeta.build([1] * B, [4000] * B, [list(range(1 + 63 * b, 64 + 63 * b)) for b in range(B)], 64, pad_blocks_to=64)
    allow = np.zeros((B, mask_words(V)), np.int32)
    wire, lay = pack_step(3, meta, torch.arange(B, dtype=torch.int64), [prm] * B, [list(range(20))] * B, [(1, 5)] * B,
                          False, counts=[counts] * B, allow=allow)
    assert lay.W == 3200 and lay.NB == MAX_PENALTY_TABLE
    ctl = ShmControl.create(1, slots=2, slot_bytes=control_slot_bytes(2048, B, V))
    try:
        assert wire.size <= ctl.max_payload_words
        ctl.publish(KIND_STEP, 0, wire)
    finally:
        ctl.unlink()
    assert control_slot_bytes(2048, B, V) - control_slot_bytes(2048, B) >= 4 * B * 3200


# ------------------------------------------------------------------------------------------------ formats
def test_canonical_format_shapes():
    assert canonical_format(None) is None and canonical_format({"type": "text"}) is None
    assert json.loads(canonical_format({"type": "json_object"})) == {"type": "json_object"}
    c = canonical_format(dict(ENUM_FORMAT, json_schema=dict(ENUM_FORMAT["json_schema"], strict=True)))
    assert json.loads(c) == {"type": "json_schema", "schema": ENUM_SCHEMA}
    assert c == canonical_format(ENUM_FORMAT)                         # name / strict do not change what is compiled
    for bad in ("json", [], {"type": "xml"}, {"type": "json_schema"}, {"type": "json_schema", "json_schema": {"schema": 3}},
                {"type": "json_schema", "json_schema": {"name": 1, "schema": {}}},
                {"type": "json_schema", "json_schema": {"schema": {}, "strict": "yes"}}):
        with pytest.raises(ValueError, match="response_format"):
            canonical_format(bad)
    with pytest.raises(ValueError):
        SamplingParams(response_format="{not json").validate()
    with pytest.raises(ValueError):
        SamplingParams(response_format='{"type":"text"}').validate()
    SamplingParams(response_format=canonical_format(ENUM_FORMAT)).validate()


def test_expert_parallel_group_refuses_response_format():
    from mlx_sharding_b200.parallel.ep_serving import LockstepGroup

    group = LockstepGroup.__new__(LockstepGroup)          # rank 0's submit path only: no process group needed
    group.rank, group.engine = 0, types.SimpleNamespace(max_model_len=1000)
    with pytest.raises(ValueError, match="response_format"):
        group.submit([1, 2, 3], SamplingParams(response_format=canonical_format({"type": "json_object"})), max_tokens=4)


# ------------------------------------------------------------------------------------------------ engine
@pytest.fixture(scope="module")
def grammar(tmp_path_factory):
    pytest.importorskip("xgrammar")
    from mlx_sharding_b200.engine.grammar import GrammarBackend
    from mlx_sharding_b200.engine.tokenizer import load_tokenizer, write_byte_tokenizer

    d = write_byte_tokenizer(str(tmp_path_factory.mktemp("tok")), vocab_size=TINY_LLAMA["vocab_size"])
    tok = load_tokenizer(d)
    assert tok.eos_token_id == EOS
    return GrammarBackend(tok, TINY_LLAMA["vocab_size"])


def _engine(grammar=None, **kw):
    cfg = ModelConfig.from_dict(TINY_LLAMA)
    sd = dict(random_state_dict(cfg, dtype=torch.float32))
    models = [build_stage(cfg, cfg.shard(0, cfg.num_hidden_layers), torch.float32).load_state(sd)]
    eng = LLMEngine(LocalPipeline.from_models(models, num_pages=64, page_size=16), num_pages=64, page_size=16, **kw)
    eng.grammar = grammar
    return eng


def _text(tokens):
    return bytes(t for t in tokens if t < 256).decode()


def test_grammar_backend_errors_and_cache(grammar):
    with pytest.raises(ValueError, match="invalid JSON schema"):
        grammar.matcher(canonical_format({"type": "json_schema", "json_schema": {"schema": {"type": 5}}}))
    fmt = canonical_format(ENUM_FORMAT)
    assert grammar.compile(fmt) is grammar.compile(fmt)
    allow = np.zeros((3, grammar.words), np.int32)
    grammar.fill([grammar.matcher(fmt)], allow, [1])
    assert R.unpack_allow(torch.from_numpy(allow), 320)[1].nonzero().flatten().tolist() == [ord("{")]
    assert (allow[0] == 0).all() and (allow[2] == 0).all()


def test_engine_enum_schema(grammar):
    eng = _engine(grammar)
    fmt = canonical_format(ENUM_FORMAT)
    outs = []
    for prm in (SamplingParams(response_format=fmt), SamplingParams(temperature=1.0, seed=5, response_format=fmt),
                SamplingParams(temperature=1.5, top_k=3, top_p=0.9, seed=2, response_format=fmt)):
        r = eng.submit([5, 6, 7], prm, max_tokens=40, eos_token_id=EOS)
        eng.drain()
        assert r.error is None and r.finish_reason == "stop" and r.output[-1] == EOS
        assert _text(r.output[:-1]) in ENUM_TEXTS
        outs.append(r)
    assert eng._constrained == 0


def test_engine_json_object_tokens_are_accepted_by_a_fresh_matcher(grammar):
    eng = _engine(grammar, mixed_batches=True)
    fmt = canonical_format({"type": "json_object"})
    reqs = [eng.submit([9, 10 + i, 11], SamplingParams(temperature=1.0, seed=i, response_format=fmt), max_tokens=30,
                       eos_token_id=EOS) for i in range(3)]
    eng.drain()
    for r in reqs:
        assert r.error is None and r.output[0] == ord("{")
        m = grammar.matcher(fmt)
        assert all(m.accept_token(t) for t in r.output)
        if r.finish_reason == "stop":
            json.loads(_text(r.output[:-1]))
        else:
            assert r.finish_reason == "length" and len(r.output) == 30


def test_unconstrained_neighbour_is_unchanged(grammar):
    prm = SamplingParams(temperature=1.0, top_p=0.9, seed=42)
    alone = _engine(grammar).generate([3, 4, 5], prm, max_tokens=12)
    eng = _engine(grammar)
    a = eng.submit([3, 4, 5], SamplingParams(temperature=1.0, top_p=0.9, seed=42), max_tokens=12)
    b = eng.submit([8, 8], SamplingParams(response_format=canonical_format(ENUM_FORMAT)), max_tokens=20, eos_token_id=EOS)
    eng.drain()
    assert a.output == alone and b.error is None and _text(b.output[:-1]) in ENUM_TEXTS


def test_rejected_token_fails_only_that_request(grammar):
    eng = _engine(grammar)
    words = grammar.words
    eng.grammar = types.SimpleNamespace(words=words, fill=lambda matchers, allow, rows: None, matcher=lambda fmt: object(),
                                        accept=lambda matchers, tokens: [False] * len(matchers))
    bad = eng.submit([1, 2], SamplingParams(response_format=canonical_format({"type": "json_object"})), max_tokens=5)
    ok = eng.submit([1, 2], SamplingParams(), max_tokens=5)
    eng.drain()
    assert isinstance(bad.error, RuntimeError) and "response_format" in str(bad.error) and bad.output == []
    with pytest.raises(RuntimeError):
        list(bad)
    assert ok.error is None and len(ok.output) == 5
    assert eng._constrained == 0 and eng.table.alloc.num_free == 63


def test_engine_without_grammar_refuses_response_format():
    eng = _engine(None)
    with pytest.raises(ValueError, match="response_format"):
        eng.submit([1, 2], SamplingParams(response_format=canonical_format({"type": "json_object"})), max_tokens=3)


def test_grpc_relay_sampler_honours_the_mask():
    from mlx_sharding_b200.engine.sampler import Sampler

    lf, ok = _rows(4, 90, 11)
    so = Sampler(R)(lf, [SamplingParams(), SamplingParams(temperature=1.0), SamplingParams(), SamplingParams()],
                    allow=pack_allow(ok).numpy())
    assert ok[torch.arange(4), so.tokens].all()


# ------------------------------------------------------------------------------------------------ gloo chain
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _chain_worker(rank, world, port, tok_dir, q):
    import torch.distributed as dist

    from mlx_sharding_b200.config import ShardSpec
    from mlx_sharding_b200.engine.grammar import GrammarBackend
    from mlx_sharding_b200.engine.tokenizer import load_tokenizer
    from mlx_sharding_b200.parallel.pipeline import ChainPipeline, StageExecutor, build_chain, worker_loop

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    cfg = ModelConfig.from_dict(dict(TINY_LLAMA, num_hidden_layers=2))
    spec = ShardSpec.even_split(cfg.num_hidden_layers, world)[rank]
    model = build_stage(cfg, spec, torch.float32).load_state(dict(random_state_dict(cfg, spec, dtype=torch.float32)))
    stage = StageExecutor(model, num_pages=32, page_size=16)
    ctl, plane = build_chain(stage, num_groups=world, max_tokens=64, max_seqs=8, control="shm")
    if rank == 0:
        pipe = ChainPipeline(stage, ctl, plane)
        eng = LLMEngine(pipe, num_pages=32, page_size=16, num_groups=world)
        eng.grammar = GrammarBackend(load_tokenizer(tok_dir), cfg.vocab_size)
        c = eng.submit([5, 6, 7], SamplingParams(temperature=1.0, seed=3, response_format=canonical_format(ENUM_FORMAT)),
                       max_tokens=30, eos_token_id=EOS)
        u = eng.submit([5, 6, 7], SamplingParams(), max_tokens=6)
        eng.drain()
        pipe.shutdown()
        q.put((c.output, c.finish_reason, repr(c.error), u.output))
    else:
        worker_loop(stage, ctl, plane)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(180)
def test_gloo_chain_carries_the_mask(tmp_path):
    pytest.importorskip("xgrammar")
    from mlx_sharding_b200.engine.tokenizer import write_byte_tokenizer

    tok_dir = write_byte_tokenizer(str(tmp_path / "tok"), vocab_size=TINY_LLAMA["vocab_size"])
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_chain_worker, args=(r, 2, port, tok_dir, q)) for r in range(2)]
    for p in procs:
        p.start()
    out, reason, err, plain = q.get(timeout=150)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert err == "None" and reason == "stop" and out[-1] == EOS and _text(out[:-1]) in ENUM_TEXTS
    assert len(plain) == 6


# ------------------------------------------------------------------------------------------------ HTTP
@pytest.fixture(scope="module")
def server(tmp_path_factory):
    pytest.importorskip("xgrammar")
    from mlx_sharding_b200.server import openai_api
    from mlx_sharding_b200.server.frontend import FrontEnd
    from mlx_sharding_b200.utils.checkpoint import write_synthetic_checkpoint

    d = tmp_path_factory.mktemp("ckpt")
    path = write_synthetic_checkpoint(str(d / "tiny"), TINY_LLAMA, dtype=torch.float32)
    cwd = os.getcwd()
    os.chdir(d)
    args = openai_api.build_arg_parser().parse_args(["--model", path, "--port", "0", "--kv-pages", "128", "--page-size", "16"])
    args.static_dir = os.path.join(os.path.dirname(openai_api.__file__), "static")
    provider = openai_api.ModelProvider(args, [])
    httpd = openai_api.make_server("127.0.0.1", 0, provider, args.static_dir)
    threading.Thread(target=httpd.serve_forever, daemon=True).start()
    wport = _free_port()
    front = FrontEnd(provider.engine, 1, "127.0.0.1", wport, args.static_dir, path, "default_model", {}, "WARNING").start()
    yield httpd.server_address[1], wport, provider
    front.stop()
    httpd.shutdown()
    provider.engine.shutdown()
    os.chdir(cwd)


def _post(port, path, body, raw=False):
    c = http.client.HTTPConnection("127.0.0.1", port, timeout=120)
    c.request("POST", path, json.dumps(body), {"Content-Type": "application/json"})
    r = c.getresponse()
    data = r.read()
    c.close()
    return r, (data if raw else json.loads(data))


def _content(path, j):
    ch = j["choices"][0]
    return ch["message"]["content"] if "chat" in path else ch["text"]


@pytest.mark.parametrize("path", ["/v1/completions", "/v1/chat/completions", "/chat/completions"])
def test_http_enum_schema(server, path):
    port, _, _ = server
    body = {"prompt": "colour?", "messages": [{"role": "user", "content": "colour?"}], "max_tokens": 40, "temperature": 1.0,
            "seed": 1, "response_format": ENUM_FORMAT}
    r, j = _post(port, path, body)
    assert r.status == 200 and j["choices"][0]["finish_reason"] == "stop"
    assert json.loads(_content(path, j))["c"] in ("red", "green")
    r, raw = _post(port, path, dict(body, stream=True), raw=True)
    ev = [e[6:] for e in raw.decode().split("\n\n") if e.startswith("data: ")]
    assert r.status == 200 and ev[-1] == "[DONE]"
    chunks = [json.loads(e)["choices"][0] for e in ev[:-1]]
    text = "".join(c["delta"]["content"] if "chat" in path else c["text"] for c in chunks)
    assert json.loads(text) == json.loads(_content(path, j)) and chunks[-1]["finish_reason"] == "stop"


def test_http_text_and_null_formats_are_unconstrained(server):
    port, _, _ = server
    body = {"messages": [{"role": "user", "content": "x"}], "max_tokens": 6, "temperature": 0}
    _, plain = _post(port, "/v1/chat/completions", body)
    for rf in (None, {"type": "text"}):
        r, j = _post(port, "/v1/chat/completions", dict(body, response_format=rf))
        assert r.status == 200 and j["choices"][0]["logprobs"]["tokens"] == plain["choices"][0]["logprobs"]["tokens"]


BAD_FORMATS = ["json", {"type": "xml"}, {"type": "json_schema"}, {"type": "json_schema", "json_schema": {"name": "x"}},
               {"type": "json_schema", "json_schema": {"name": "x", "schema": [1]}},
               {"type": "json_schema", "json_schema": {"name": "x", "schema": {"type": 5}}}]


@pytest.mark.parametrize("fmt", BAD_FORMATS)
def test_http_malformed_formats_answer_400(server, fmt):
    iport, wport, _ = server
    for port in (iport, wport):              # in-process server and the --api-workers front end
        for path in ("/v1/completions", "/v1/chat/completions"):
            body = {"prompt": "hi", "messages": [{"role": "user", "content": "hi"}], "max_tokens": 2, "response_format": fmt}
            r, j = _post(port, path, body)
            assert r.status == 400 and j["error"]["type"] == "invalid_request_error", (port, path, j)
            assert "response_format" in j["error"]["message"]


def test_http_enum_schema_through_api_workers(server):
    _, wport, _ = server
    body = {"messages": [{"role": "user", "content": "colour?"}], "max_tokens": 40, "response_format": ENUM_FORMAT}
    r, j = _post(wport, "/v1/chat/completions", body)
    assert r.status == 200 and json.loads(j["choices"][0]["message"]["content"])["c"] in ("red", "green")
