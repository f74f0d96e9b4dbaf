"""LoRA adapters on the sm_90a kernels: the shrink launch plus the adapter term in the quantised GEMM epilogue, on both quantised
routes (persistent, workspace split-K), against fp64; B = 0 is bitwise the adapter-free launch; end to end on a 4-bit Llama
(reference backend, CUDA-graph replay) and on a bf16 DeepSeek-V2-Lite-shaped model whose absorbed attention uses folded weights."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import GPU_LLAMA, run_sequence
from mlx_sharding_b200.ops import LinearWeight, b200, reference
from mlx_sharding_b200.utils import quant
from mlx_sharding_b200.utils.adapters import attach, load_adapter
from mlx_sharding_b200.utils.checkpoint import write_synthetic_adapter
from mlx_sharding_b200.utils.loader import random_model

DEV = "cuda"
TS = [1, 7, 64, 130, 1000]


def _packed(n, k, bits, seed, rank=None, scale=2.0, zero_b=False, bias=False):
    g = torch.Generator().manual_seed(seed)
    wq, s, b = quant.quantize(torch.randn(n, k, generator=g) * 0.02, 64, bits, out_dtype=torch.bfloat16)
    W = LinearWeight(wq=wq.view(torch.int32).to(DEV), scales=s.to(DEV), biases=b.to(DEV), group_size=64, bits=bits,
                     bias=(torch.randn(n, generator=g) * 0.1).to(DEV, torch.bfloat16) if bias else None)
    if rank:
        A = torch.randn(k, rank, generator=g) / k ** 0.5
        B = torch.zeros(rank, n) if zero_b else torch.randn(rank, n, generator=g) * 0.05
        attach(W, "w", A, B, scale)
    return W


def _oracle(x, W):
    """fp64: x W^T + (x A^T) B_s^T with the stored (bf16) adapter tensors."""
    xd = x.double()
    y = xd @ W.dense(torch.float64, fold_lora=False).t()
    if W.has_lora:
        y = y + (xd @ W.lora_a.double().t()) @ W.lora_b_scaled.double().t()
    return y


def _route(T, n, k, pair=False):
    return b200.C().gemm_plan("q", T, n, k, pair=pair, sm_count=torch.cuda.get_device_properties(0).multi_processor_count)["route"]


def _close(got, want, rel=2e-2):
    err = (got.double() - want).abs().max().item()
    assert err <= rel * max(1.0, want.abs().max().item()), err


# single weights: (n, k) = (384, 512) plans persistent at every T; (512, 4096) plans workspace split-K for T < 64
@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("nk", [(384, 512), (512, 4096)], ids=["n384k512", "n512k4096"])
@pytest.mark.parametrize("rank", [8, 12, 16, 64, "3x8"])
@pytest.mark.parametrize("bits", [4, 8])
def test_linear_with_adapter_matches_fp64(T, nk, rank, bits):
    n, k = nk
    g = torch.Generator().manual_seed(T)
    x = (torch.randn(T, k, generator=g)).to(DEV, torch.bfloat16)
    if rank == "3x8":   # block-diagonal q | k | v adapter
        parts = [_packed(n // 4 * 2, k, bits, 1, 8), _packed(n // 4, k, bits, 2, 8), _packed(n // 4, k, bits, 3, 8)]
        W = LinearWeight.concat(parts)
        assert W.lora_a.shape[0] == 24
    else:
        W = _packed(n, k, bits, 1, rank)
    y = b200.linear(x, W)
    _close(y, _oracle(x, W))
    assert (y.double() - _oracle(x, W)).abs().max() < (y.double() - (x.double() @ W.dense(torch.float64, False).t())).abs().max()


def test_shapes_cover_both_quantised_routes():
    routes = {_route(T, n, k) for T in TS for n, k in ((384, 512), (512, 4096))}
    routes_pair = {_route(T, 256, 1024, True) for T in TS}
    assert routes == {"persistent", "workspace"} and routes_pair == {"persistent", "workspace"}


@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("nk", [(384, 512), (512, 4096)], ids=["n384k512", "n512k4096"])
@pytest.mark.parametrize("epi", ["bias", "residual", "bias+residual", "softcap", "bias+softcap"])
def test_linear_adapter_epilogue_combinations(T, nk, epi):
    n, k = nk
    # the k4096 shape takes the workspace split-K route below 64 tokens: the term joins the reduced sum there
    assert _route(T, n, k) == ("workspace" if k == 4096 and T < 64 else "persistent")
    W = _packed(n, k, 4, 5, 16, bias="bias" in epi)
    g = torch.Generator().manual_seed(100 + T)
    x = torch.randn(T, k, generator=g).to(DEV, torch.bfloat16)
    res = torch.randn(T, n, generator=g).to(DEV, torch.bfloat16) if "residual" in epi else None
    cap = 0.5 if "softcap" in epi else 0.0
    y = b200.linear(x, W, residual=res, softcap=cap)
    want = _oracle(x, W)
    if W.bias is not None:
        want = want + W.bias.double()
    if cap:
        want = cap * torch.tanh(want / cap)
    if res is not None:
        want = want + res.double()
    _close(y, want)


@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("act", ["silu", "gelu_tanh"])
@pytest.mark.parametrize("which", ["both", "gate_only", "up_only"])
def test_gated_up_with_adapters_matches_fp64(T, act, which):
    n, k = 256, 1024
    Wg = _packed(n, k, 4, 7, 16 if which != "up_only" else None)
    Wu = _packed(n, k, 4, 8, 8 if which != "gate_only" else None)
    g = torch.Generator().manual_seed(T)
    x = torch.randn(T, k, generator=g).to(DEV, torch.bfloat16)
    y = b200.gated_up(x, Wg, Wu, act)
    gd, ud = _oracle(x, Wg), _oracle(x, Wu)
    want = reference.act_fn(act, gd) * ud
    _close(y, want, rel=3e-2)


@pytest.mark.parametrize("T", TS)
def test_zero_b_is_bitwise_the_plain_launch(T):
    g = torch.Generator().manual_seed(T)
    for n, k in ((384, 512), (512, 4096)):
        x = torch.randn(T, k, generator=g).to(DEV, torch.bfloat16)
        res = torch.randn(T, n, generator=g).to(DEV, torch.bfloat16)
        plain, ad = _packed(n, k, 4, 9, bias=True), _packed(n, k, 4, 9, 16, zero_b=True, bias=True)
        assert torch.equal(b200.linear(x, plain, residual=res), b200.linear(x, ad, residual=res))
    xg = torch.randn(T, 1024, generator=g).to(DEV, torch.bfloat16)
    pg, pu = _packed(256, 1024, 8, 10), _packed(256, 1024, 8, 11)
    ag, au = _packed(256, 1024, 8, 10, 8, zero_b=True), _packed(256, 1024, 8, 11, 8, zero_b=True)
    assert torch.equal(b200.gated_up(xg, pg, pu), b200.gated_up(xg, ag, au))


Q4 = {"group_size": 64, "bits": 4}


def _adapted_llama(tmp_path, backend, rank=16):
    d = write_synthetic_adapter(str(tmp_path / f"ad{backend}"), GPU_LLAMA, rank=rank, scale=8.0, num_layers=3, seed=3)
    return random_model(GPU_LLAMA, dtype=torch.bfloat16, device=DEV, backend=backend, seed=1, quantization=Q4,
                        adapter=load_adapter(d))


def test_4bit_llama_with_adapter_matches_reference(tmp_path):
    fast, ref = _adapted_llama(tmp_path, "b200"), _adapted_llama(tmp_path, "reference")
    assert fast.layer_weights[3]["qkv"].has_lora and fast.layer_weights[3]["down"].has_lora
    base = random_model(GPU_LLAMA, dtype=torch.bfloat16, device=DEV, backend="reference", seed=1, quantization=Q4)
    toks = [5, 17, 200, 31, 8, 99, 100, 42]
    a, b, c = (run_sequence([m], toks, 4, page_size=16) for m in (fast, ref, base))
    for x, y in zip(a, b):
        assert (x - y).abs().max().item() < 0.05 * max(1.0, y.abs().max().item())
    assert [int(x.argmax()) for x in a] == [int(y.argmax()) for y in b]
    assert (b[0] - c[0]).abs().max().item() > 0.05 * max(1.0, c[0].abs().max().item())   # the adapter matters


def test_4bit_llama_with_adapter_graph_decode_matches_eager(tmp_path):
    from mlx_sharding_b200.engine.core import LLMEngine
    from mlx_sharding_b200.engine.sampler import SamplingParams
    from mlx_sharding_b200.parallel.pipeline import LocalPipeline

    fast = _adapted_llama(tmp_path, "b200")
    prompts = [[5, 6, 7, 8, 9, 10, 11], [100, 50], list(range(20, 60)), [42] * 9]
    outs = []
    for use_graphs in (True, False):
        pipe = LocalPipeline.from_models([fast], num_pages=64, page_size=16)
        if not use_graphs:
            pipe.gcache.enabled = False
        eng = LLMEngine(pipe, num_pages=64, page_size=16)
        reqs = [eng.submit(p, SamplingParams(), max_tokens=12) for p in prompts]
        eng.drain()
        outs.append([r.output for r in reqs])
        if use_graphs:
            assert pipe.gcache.captures >= 1 and pipe.gcache.replays >= 5
    assert outs[0] == outs[1]


def test_deepseek_lite_attention_adapter_absorbs_folded_weights(tmp_path):
    from mlx_sharding_b200.config import deepseek_v2_lite_config

    cfg = dict(deepseek_v2_lite_config(), num_hidden_layers=3, vocab_size=8192)
    d = write_synthetic_adapter(str(tmp_path / "ds"), cfg, rank=8, scale=16.0, num_layers=2, seed=5,
                                modules=["self_attn.q_proj", "self_attn.kv_a_proj_with_mqa", "self_attn.kv_b_proj",
                                         "self_attn.o_proj"])
    ad = load_adapter(d)
    fast = random_model(cfg, dtype=torch.bfloat16, device=DEV, backend="b200", seed=0, adapter=ad)
    ref = random_model(cfg, dtype=torch.bfloat16, device=DEV, backend="reference", seed=0, adapter=ad)
    base = random_model(cfg, dtype=torch.bfloat16, device=DEV, backend="reference", seed=0)
    assert fast.absorbed_mla and "qkv_abs" in fast.layer_weights[2]
    toks = list(range(5, 5 + 9))
    a, b, c = (run_sequence([m], toks, 3, page_size=64) for m in (fast, ref, base))
    for x, y in zip(a, b):
        assert (x - y).abs().max().item() < 0.1 * max(1.0, y.abs().max().item())
    assert (b[0] - c[0]).abs().max().item() > 0.1 * max(1.0, c[0].abs().max().item())
