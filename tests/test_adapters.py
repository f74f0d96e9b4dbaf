"""mlx_lm LoRA adapters on the CPU path: parsing and refusals, stage filtering, folding into dense weights, the unfused term on
packed weights (reference backend), block-diagonal concatenation, and ``--adapter-path`` through the CLI and the HTTP server."""
import http.client
import json
import os
import threading

import pytest
import torch

from helpers import TINY_LLAMA, run_sequence
from mlx_sharding_b200.config import ShardSpec
from mlx_sharding_b200.ops import LinearWeight, reference
from mlx_sharding_b200.utils import quant
from mlx_sharding_b200.utils.adapters import CONFIG_FILE, WEIGHTS_FILE, attach, load_adapter
from mlx_sharding_b200.utils.checkpoint import save_safetensors, write_synthetic_adapter, write_synthetic_checkpoint
from mlx_sharding_b200.utils.loader import load_model, random_model

Q4 = {"group_size": 64, "bits": 4}
L = TINY_LLAMA["num_hidden_layers"]


def _edit_config(d, **kw):
    p = os.path.join(d, CONFIG_FILE)
    with open(p) as f:
        c = json.load(f)
    for k, v in kw.items():
        if v is None:
            c.pop(k, None)
        else:
            c[k] = v
    with open(p, "w") as f:
        json.dump(c, f)


def _edit_tensors(d, fn):
    from safetensors.torch import load_file

    p = os.path.join(d, WEIGHTS_FILE)
    t = load_file(p)
    fn(t)
    save_safetensors(p, t)


# ------------------------------------------------------------------------------------------------ parsing
def test_config_parsing_and_legacy_lora_layers(tmp_path):
    d = write_synthetic_adapter(str(tmp_path / "a"), TINY_LLAMA, rank=4, scale=2.5, num_layers=2, seed=1)
    ad = load_adapter(d)
    assert (ad.rank, ad.scale, ad.num_layers) == (4, 2.5, 2)
    assert sorted(ad) == sorted(f"model.layers.{i}.{m}" for i in (2, 3) for m in
                                ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj",
                                 "mlp.gate_proj", "mlp.up_proj", "mlp.down_proj"))
    A, B = ad["model.layers.3.self_attn.q_proj"]
    assert A.shape == (64, 4) and B.shape == (4, 64) and A.dtype == torch.float32
    _edit_config(d, num_layers=None, lora_layers=2, fine_tune_type=None)   # older mlx_lm config
    ad2 = load_adapter(d)
    assert ad2.num_layers == 2 and sorted(ad2) == sorted(ad)


@pytest.mark.parametrize("edit,match", [
    (dict(fine_tune_type="dora"), "fine_tune_type 'dora'"),
    (dict(fine_tune_type="full"), "fine_tune_type 'full'"),
    (dict(fine_tune_type=None, use_dora=True), "fine_tune_type 'dora'"),
])
def test_refuses_dora_and_full(tmp_path, edit, match):
    d = write_synthetic_adapter(str(tmp_path / "a"), TINY_LLAMA, rank=4, num_layers=1)
    _edit_config(d, **edit)
    with pytest.raises(ValueError, match=match) as e:
        load_adapter(d)
    assert CONFIG_FILE in str(e.value)


@pytest.mark.parametrize("drop", ["lora_a", "lora_b"])
def test_refuses_tensor_without_partner(tmp_path, drop):
    d = write_synthetic_adapter(str(tmp_path / "a"), TINY_LLAMA, rank=4, num_layers=1)
    _edit_tensors(d, lambda t: t.pop(f"model.layers.3.self_attn.v_proj.{drop}"))
    keep = "lora_b" if drop == "lora_a" else "lora_a"
    with pytest.raises(ValueError, match=f"'model.layers.3.self_attn.v_proj.{keep}' has no partner") as e:
        load_adapter(d)
    assert WEIGHTS_FILE in str(e.value)


def test_refuses_rank_mismatch(tmp_path):
    d = write_synthetic_adapter(str(tmp_path / "a"), TINY_LLAMA, rank=4, num_layers=1)
    _edit_config(d, lora_parameters={"rank": 8, "scale": 1.0, "dropout": 0.0})
    with pytest.raises(ValueError, match=r"model\.layers\.3\..*does not match the config's rank 8") as e:
        load_adapter(d)
    assert WEIGHTS_FILE in str(e.value)


@pytest.mark.parametrize("module", ["mlp.switch_mlp.gate_proj", "mlp.experts.3.up_proj"])
def test_refuses_routed_experts(tmp_path, module):
    d = write_synthetic_adapter(str(tmp_path / "a"), TINY_LLAMA, rank=4, num_layers=1)
    _edit_tensors(d, lambda t: t.update({f"model.layers.3.{module}.lora_a": torch.zeros(64, 4),
                                         f"model.layers.3.{module}.lora_b": torch.zeros(4, 32)}))
    with pytest.raises(ValueError, match="routed experts") as e:
        load_adapter(d)
    assert module in str(e.value)


def test_refuses_layer_outside_num_layers(tmp_path):
    d = write_synthetic_adapter(str(tmp_path / "a"), TINY_LLAMA, rank=4, num_layers=2)
    _edit_config(d, num_layers=1)
    with pytest.raises(ValueError, match=r"'model\.layers\.2\.[a-z_.]+\.lora_a' is in layer 2, outside the adapted layers \[3, 4\) \(num_layers=1\)") as e:
        random_model(TINY_LLAMA, dtype=torch.float32, adapter=load_adapter(d))
    assert WEIGHTS_FILE in str(e.value)


@pytest.mark.parametrize("num_layers", [-1, L, L + 3])
def test_num_layers_minus_one_or_more_than_the_model_means_all_layers(tmp_path, num_layers):
    # mlx_lm.lora --num-layers -1 adapts every block and writes -1 into adapter_config.json
    d = write_synthetic_adapter(str(tmp_path / "a"), TINY_LLAMA, rank=4, num_layers=L, seed=2)
    _edit_config(d, num_layers=num_layers)
    ad = load_adapter(d)
    m = random_model(TINY_LLAMA, dtype=torch.float32, seed=1, quantization=Q4, adapter=ad)
    assert all(m.layer_weights[i]["qkv"].has_lora and m.layer_weights[i]["down"].has_lora for i in range(L))


def test_refuses_unknown_module_and_shape_mismatch(tmp_path):
    d = write_synthetic_adapter(str(tmp_path / "a"), TINY_LLAMA, rank=4, num_layers=1)
    _edit_tensors(d, lambda t: t.update({"model.layers.3.self_attn.x_proj.lora_a": torch.zeros(64, 4),
                                         "model.layers.3.self_attn.x_proj.lora_b": torch.zeros(4, 64)}))
    with pytest.raises(ValueError, match=r"match no linear weight.*self_attn\.x_proj\.lora_a"):
        random_model(TINY_LLAMA, dtype=torch.float32, adapter=load_adapter(d))
    d2 = write_synthetic_adapter(str(tmp_path / "b"), TINY_LLAMA, rank=4, num_layers=1)
    _edit_tensors(d2, lambda t: t.update({"model.layers.3.mlp.down_proj.lora_a": torch.zeros(64, 4)}))   # in is 128
    with pytest.raises(ValueError, match=r"'model\.layers\.3\.mlp\.down_proj\.lora_a' \(64, 4\).*do not fit"):
        random_model(TINY_LLAMA, dtype=torch.float32, adapter=load_adapter(d2))


# ------------------------------------------------------------------------------------------------ stage filtering
def test_stage_filtering_half_layer_split(tmp_path):
    d = write_synthetic_adapter(str(tmp_path / "a"), TINY_LLAMA, rank=4, num_layers=L, seed=3)
    ad = load_adapter(d)
    full = random_model(TINY_LLAMA, dtype=torch.float32, seed=5, adapter=ad)
    # boundary inside layer 1: its attention on stage 0, its MLP on stage 1
    s0 = random_model(TINY_LLAMA, dtype=torch.float32, seed=5, adapter=ad, spec=ShardSpec(0, 2, L, defer_last_mlp=True))
    s1 = random_model(TINY_LLAMA, dtype=torch.float32, seed=5, adapter=ad, spec=ShardSpec(1, L, L, skip_first_attn=True))
    assert "qkv" in s0.layer_weights[1] and "gate" not in s0.layer_weights[1]
    assert "gate" in s1.layer_weights[1] and "qkv" not in s1.layer_weights[1]
    for i in range(L):
        for k, w in full.layer_weights[i].items():
            if isinstance(w, LinearWeight):
                part = (s0 if i == 0 or (i == 1 and k in ("qkv", "o")) else s1).layer_weights[i][k]
                assert torch.equal(part.weight, w.weight), (i, k)
    assert len(ad) == 7 * L   # the stages only read the adapter, they do not consume it
    toks = [3, 9, 27, 81, 5]
    ref = run_sequence([full], toks, n_decode=2)
    got = run_sequence([s0, s1], toks, n_decode=2)
    for a, b in zip(ref, got):
        torch.testing.assert_close(a, b, rtol=0, atol=0)


# ------------------------------------------------------------------------------------------------ folding
def test_fold_matches_fp64():
    g = torch.Generator().manual_seed(0)
    W = torch.randn(96, 64, generator=g).to(torch.bfloat16)
    A, B = torch.randn(64, 8, generator=g) * 0.1, torch.randn(8, 96, generator=g) * 0.1
    got = attach(LinearWeight(weight=W.clone()), "p", A, B, 3.0).weight
    want = (W.double() + 3.0 * (A.double() @ B.double()).t()).to(torch.bfloat16)
    # one rounding of an fp32 sum: equal to the rounded fp64 value except at rare bf16 ties
    assert (got.float() - want.float()).abs().max() <= 2 ** -7 * want.float().abs().max()
    assert (got != want).float().mean() < 0.01


def test_bf16_adapter_equals_hand_fused_checkpoint(tmp_path):
    from safetensors.torch import load_file

    base = write_synthetic_checkpoint(str(tmp_path / "base"), TINY_LLAMA, dtype=torch.bfloat16, seed=2)
    ad_dir = write_synthetic_adapter(str(tmp_path / "ad"), TINY_LLAMA, rank=8, scale=4.0, num_layers=3, seed=7)
    ad = load_adapter(ad_dir)
    fused = write_synthetic_checkpoint(str(tmp_path / "fused"), TINY_LLAMA, dtype=torch.bfloat16, seed=2)
    sd = load_file(os.path.join(fused, "model.safetensors"))
    for prefix, (A, B) in ad.items():     # mlx_lm.fuse: W + scale * (A B)^T in fp32, rounded once
        w = sd[prefix + ".weight"]
        sd[prefix + ".weight"] = (w.float() + (A @ B).t() * ad.scale).to(w.dtype)
    save_safetensors(os.path.join(fused, "model.safetensors"), sd)
    m_ad = load_model(base, dtype=torch.bfloat16, device="cpu", backend="reference", adapter_path=ad_dir)
    m_fu = load_model(fused, dtype=torch.bfloat16, device="cpu", backend="reference")
    m_base = load_model(base, dtype=torch.bfloat16, device="cpu", backend="reference")
    toks = [11, 12, 13, 200, 7, 1]
    a, f, b = (run_sequence([m], toks, n_decode=3) for m in (m_ad, m_fu, m_base))
    for x, y in zip(a, f):
        torch.testing.assert_close(x, y, rtol=0, atol=0)
    assert not torch.allclose(a[0], b[0])


# ------------------------------------------------------------------------------------------------ packed weights
def _dense_oracle(model):
    """A copy of the stage with every adapted packed weight replaced by fp64-built dense weights, W + B_s A."""
    import copy

    m = copy.copy(model)
    m.layer_weights = {}
    for i, w in model.layer_weights.items():
        m.layer_weights[i] = dict(w)
        for k, W in w.items():
            if isinstance(W, LinearWeight) and W.has_lora:
                d = quant.dequantize(W.wq, W.scales, W.biases, W.group_size, W.bits, torch.float64)
                d = d + W.lora_b_scaled.double() @ W.lora_a.double()
                m.layer_weights[i][k] = LinearWeight(weight=d.float(), bias=W.bias)
    return m


def test_4bit_adapter_matches_fp64_unfused_oracle(tmp_path):
    d = write_synthetic_adapter(str(tmp_path / "a"), TINY_LLAMA, rank=8, scale=8.0, num_layers=2, seed=4)
    m = random_model(TINY_LLAMA, dtype=torch.float32, seed=1, quantization=Q4, backend="reference", adapter=load_adapter(d))
    qkv = m.layer_weights[3]["qkv"]
    assert qkv.is_quantized and qkv.has_lora and qkv.lora_a.shape == (24, 64) and qkv.lora_b_scaled.shape == (128, 24)
    assert not m.layer_weights[0]["qkv"].has_lora
    base = random_model(TINY_LLAMA, dtype=torch.float32, seed=1, quantization=Q4, backend="reference")
    toks = [5, 6, 7, 8, 9, 10, 11]
    got = run_sequence([m], toks, n_decode=3)
    want = run_sequence([_dense_oracle(m)], toks, n_decode=3)
    b = run_sequence([base], toks, n_decode=3)
    for x, y in zip(got, want):
        torch.testing.assert_close(x, y, rtol=1e-4, atol=1e-4)
    assert (got[0] - b[0]).abs().max() > 1e-2


def test_packed_adapter_tensors_match_the_adapter_file(tmp_path):
    """The unfused tensors against (A, B, scale) read straight from the file, not from what ``attach`` stored."""
    from safetensors.torch import load_file

    d = write_synthetic_adapter(str(tmp_path / "a"), TINY_LLAMA, rank=8, scale=6.0, num_layers=1, seed=4)
    raw = load_file(os.path.join(d, WEIGHTS_FILE))
    with open(os.path.join(d, CONFIG_FILE)) as f:
        scale = json.load(f)["lora_parameters"]["scale"]
    m = random_model(TINY_LLAMA, dtype=torch.float32, seed=1, quantization=Q4, adapter=load_adapter(d))
    for key in ("mlp.down_proj", "mlp.gate_proj"):
        W = m.layer_weights[3][key.split(".")[1].replace("_proj", "")]
        A, B = raw[f"model.layers.3.{key}.lora_a"].double(), raw[f"model.layers.3.{key}.lora_b"].double()
        want = scale * (A @ B).t()
        torch.testing.assert_close(W.lora_b_scaled.double() @ W.lora_a.double(), want, rtol=0, atol=2e-2 * want.abs().max().item())
    qkv = m.layer_weights[3]["qkv"]   # q | k | v rows of the block-diagonal product
    delta = qkv.lora_b_scaled.double() @ qkv.lora_a.double()
    n0 = 0
    for mod in ("q_proj", "k_proj", "v_proj"):
        A, B = raw[f"model.layers.3.self_attn.{mod}.lora_a"].double(), raw[f"model.layers.3.self_attn.{mod}.lora_b"].double()
        want = scale * (A @ B).t()
        torch.testing.assert_close(delta[n0:n0 + B.shape[1]], want, rtol=0, atol=2e-2 * want.abs().max().item())
        n0 += B.shape[1]


def test_zero_b_gives_base_logits_exactly(tmp_path):
    d = write_synthetic_adapter(str(tmp_path / "a"), TINY_LLAMA, rank=8, num_layers=L, seed=4, zero_b=True)
    for q in (None, Q4):
        m = random_model(TINY_LLAMA, dtype=torch.float32, seed=1, quantization=q, adapter=load_adapter(d))
        base = random_model(TINY_LLAMA, dtype=torch.float32, seed=1, quantization=q)
        assert m.layer_weights[2]["down"].has_lora == (q is not None)
        for x, y in zip(run_sequence([m], [1, 2, 3], n_decode=2), run_sequence([base], [1, 2, 3], n_decode=2)):
            assert torch.equal(x, y)


def test_block_diagonal_concat_with_missing_adapter():
    g = torch.Generator().manual_seed(0)
    K = 128

    def packed(n):
        wq, s, b = quant.quantize(torch.randn(n, K, generator=g) * 0.02, 64, 4, out_dtype=torch.bfloat16)
        return LinearWeight(wq=wq.view(torch.int32), scales=s, biases=b, group_size=64, bits=4)

    q, k, v = packed(128), packed(64), packed(64)
    attach(q, "q", torch.randn(K, 8, generator=g) * 0.1, torch.randn(8, 128, generator=g) * 0.1, 2.0)
    attach(v, "v", torch.randn(K, 4, generator=g) * 0.1, torch.randn(4, 64, generator=g) * 0.1, 2.0)
    cat = LinearWeight.concat([q, k, v])
    assert cat.lora_a.shape == (16, K) and cat.lora_b_scaled.shape == (256, 16)   # v's rank 4 padded to 8
    assert cat.lora_b_scaled[:128, 8:].abs().sum() == 0 and cat.lora_b_scaled[128:192].abs().sum() == 0
    assert cat.lora_b_scaled[192:, :8].abs().sum() == 0
    x = torch.randn(5, K, generator=g)
    want = torch.cat([x.double() @ w.dense(torch.float64).t() for w in (q, k, v)], 1)   # fp64, each module folded alone
    torch.testing.assert_close(reference.linear(x, cat).double(), want, rtol=1e-5, atol=1e-5)
    sl = cat.slice_out(128, 256)     # k | v rows keep their adapter rows
    torch.testing.assert_close(reference.linear(x, sl).double(), want[:, 128:], rtol=1e-5, atol=1e-5)
    assert cat.to(dtype=torch.float32).lora_b_scaled.dtype == torch.bfloat16


def test_packed_weight_turned_dense_folds_adapter():
    g = torch.Generator().manual_seed(1)
    wq, s, b = quant.quantize(torch.randn(64, 128, generator=g) * 0.02, 64, 4, out_dtype=torch.bfloat16)
    W = attach(LinearWeight(wq=wq.view(torch.int32), scales=s, biases=b, group_size=64, bits=4), "w",
               torch.randn(128, 8, generator=g), torch.randn(8, 64, generator=g) * 0.01, 1.5)
    base = W.dense(torch.float64, fold_lora=False)
    torch.testing.assert_close(W.dense(torch.float64), base + W.lora_b_scaled.double() @ W.lora_a.double())


# ------------------------------------------------------------------------------------------------ CLI / HTTP
def test_api_cli_passes_adapter_path_to_load_model(tmp_path, monkeypatch):
    from mlx_sharding_b200.server import openai_api
    from mlx_sharding_b200.utils import loader

    seen = {}

    def fake_load_model(path, **kw):
        seen.update(kw, path=path)
        raise RuntimeError("stop here")

    monkeypatch.setattr(loader, "load_model", fake_load_model)
    ckpt = write_synthetic_checkpoint(str(tmp_path / "m"), TINY_LLAMA, dtype=torch.float32)
    monkeypatch.chdir(tmp_path)
    args = openai_api.build_arg_parser().parse_args(["--model", ckpt, "--adapter-path", "my_adapter"])
    with pytest.raises(RuntimeError, match="stop here"):
        openai_api.ModelProvider(args, [])
    assert seen["path"] == ckpt and seen["adapter_path"] == "my_adapter"


def test_http_chat_completion_with_adapter_equals_engine(tmp_path, monkeypatch):
    from mlx_sharding_b200.engine.sampler import SamplingParams
    from mlx_sharding_b200.server import openai_api

    ckpt = write_synthetic_checkpoint(str(tmp_path / "m"), TINY_LLAMA, dtype=torch.float32, seed=3)
    ad = write_synthetic_adapter(str(tmp_path / "ad"), TINY_LLAMA, rank=8, scale=10.0, num_layers=2, seed=9)
    monkeypatch.chdir(tmp_path)
    args = openai_api.build_arg_parser().parse_args(["--model", ckpt, "--adapter-path", ad, "--kv-pages", "64",
                                                      "--page-size", "16"])
    args.static_dir = os.path.join(os.path.dirname(openai_api.__file__), "static")
    provider = openai_api.ModelProvider(args, [])
    httpd = openai_api.make_server("127.0.0.1", 0, provider, args.static_dir)
    t = threading.Thread(target=httpd.serve_forever, daemon=True)
    t.start()
    try:
        body = {"messages": [{"role": "user", "content": "hi"}], "max_tokens": 6, "temperature": 0.8, "seed": 1234}
        c = http.client.HTTPConnection("127.0.0.1", httpd.server_address[1], timeout=60)
        c.request("POST", "/v1/chat/completions", json.dumps(body), {"Content-Type": "application/json"})
        j = json.loads(c.getresponse().read())
        c.close()
        got = j["choices"][0]["logprobs"]["tokens"]
        tok = provider.tokenizer
        prompt = tok.apply_chat_template(body["messages"], tokenize=True, add_generation_prompt=True)
        if hasattr(prompt, "keys"):
            prompt = prompt["input_ids"]
        req = provider.engine.submit(list(prompt), SamplingParams(temperature=0.8, seed=1234), max_tokens=6,
                                     eos_token_id=tok.eos_token_id)
        assert got == [ev.token for ev in req]
        # the adapter changed the model: the base checkpoint's layers differ
        base = load_model(ckpt, dtype=torch.float32, device="cpu")
        assert not torch.equal(base.layer_weights[3]["qkv"].weight, provider.model.layer_weights[3]["qkv"].weight)
        assert torch.equal(base.layer_weights[1]["qkv"].weight, provider.model.layer_weights[1]["qkv"].weight)
    finally:
        httpd.shutdown()
        provider.engine.shutdown()
