"""GPU end-to-end: stage models on the b200 (sm_90a kernels) backend vs the PyTorch reference backend
with identical bf16 weights — logits agree, greedy tokens agree, engine runs batched requests."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import GPU_DSV2, GPU_GEMMA2, GPU_LLAMA, run_sequence
from mlx_sharding_b200.config import ModelConfig
from mlx_sharding_b200.models import build_stage
from mlx_sharding_b200.utils.checkpoint import random_state_dict


def _pair(C, ranges=None, quantization=None):
    if quantization:
        C = dict(C, quantization=quantization)
    cfg = ModelConfig.from_dict(C)
    sd = dict(random_state_dict(cfg, dtype=torch.bfloat16, device="cuda", quantization=quantization))
    ranges = ranges or [(0, cfg.num_hidden_layers)]
    mk = lambda be: [build_stage(cfg, cfg.shard(s, e), torch.bfloat16, "cuda", be).load_state(dict(sd)) for s, e in ranges]
    return mk("b200"), mk("reference")


@pytest.mark.parametrize("C", [GPU_LLAMA, GPU_GEMMA2, GPU_DSV2], ids=lambda c: c["model_type"])
def test_b200_backend_matches_reference(C):
    fast, ref = _pair(C)
    toks = [5, 17, 200, 31, 8, 99, 100, 42, 7, 300, 301, 302, 11]
    a = run_sequence(fast, toks, 4, page_size=16)
    b = run_sequence(ref, toks, 4, page_size=16)
    for x, y in zip(a, b):
        err = (x - y).abs().max().item()
        assert err < 0.15 * max(1.0, y.abs().max().item()), err
    assert int(a[0].argmax()) == int(b[0].argmax())


def test_b200_sharded_and_chunked(C=GPU_DSV2):
    fast, _ = _pair(C)
    parts, _ = _pair(C, ranges=[(0, 1), (1, 3), (3, 4)])
    toks = list(range(3, 40))
    a = run_sequence(fast, toks, 3, page_size=16)
    b = run_sequence(parts, toks, 3, page_size=16, chunk=16)
    for x, y in zip(a, b):
        assert (x - y).abs().max().item() < 0.1 * max(1.0, y.abs().max().item())


def test_b200_quantized_checkpoint():
    fast, ref = _pair(GPU_LLAMA, quantization=dict(group_size=64, bits=4))
    toks = [5, 17, 200, 31, 8]
    a, b = run_sequence(fast, toks, 2, page_size=16), run_sequence(ref, toks, 2, page_size=16)
    for x, y in zip(a, b):
        assert (x - y).abs().max().item() < 0.15 * max(1.0, y.abs().max().item())


def test_engine_on_gpu_batched():
    from mlx_sharding_b200.engine.core import LLMEngine
    from mlx_sharding_b200.engine.sampler import SamplingParams
    from mlx_sharding_b200.parallel.pipeline import LocalPipeline

    fast, _ = _pair(GPU_DSV2)
    pipe = LocalPipeline.from_models(fast, num_pages=64, page_size=16)
    eng = LLMEngine(pipe, num_pages=64, page_size=16, max_prefill_tokens=24)
    prompts = [[5, 6, 7, 8, 9, 10, 11], [100, 50], list(range(20, 60)), [42] * 9]
    reqs = [eng.submit(p, SamplingParams(logprobs=2), max_tokens=6) for p in prompts]
    eng.drain()
    for p, r in zip(prompts, reqs):
        assert r.finished and len(r.output) == 6
        solo = [int(o.argmax()) for o in run_sequence(fast, p, 5, page_size=16)]
        # batch invariance of the kernels: same tokens as a solo run (allow one near-tie flip)
        assert sum(int(x != y) for x, y in zip(solo, r.output)) <= 1, (solo, r.output)
    hot = eng.generate([1, 2, 3], SamplingParams(temperature=1.0, top_p=0.9), max_tokens=8)
    assert len(hot) == 8


def test_engine_graph_decode_matches_eager():
    """Steady-state decode steps run as captured CUDA graphs (parallel/graph_decode.py) — same tokens as eager."""
    from mlx_sharding_b200.engine.core import LLMEngine
    from mlx_sharding_b200.engine.sampler import SamplingParams
    from mlx_sharding_b200.parallel.pipeline import LocalPipeline

    fast, _ = _pair(GPU_DSV2)
    prompts = [[5, 6, 7, 8, 9, 10, 11], [100, 50], list(range(20, 60)), [42] * 9]
    outs = []
    for use_graphs in (True, False):
        pipe = LocalPipeline.from_models(fast, num_pages=64, page_size=16)
        if not use_graphs:
            pipe.gcache.enabled = False
        eng = LLMEngine(pipe, num_pages=64, page_size=16)
        reqs = [eng.submit(p, SamplingParams(), max_tokens=12) for p in prompts]
        eng.drain()
        outs.append([r.output for r in reqs])
        if use_graphs:
            assert pipe.gcache.captures >= 1 and pipe.gcache.replays >= 5
    assert outs[0] == outs[1]
