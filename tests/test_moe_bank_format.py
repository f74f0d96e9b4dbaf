"""Load-time weight formats of a DeepSeek MoE stage on the CUDA backend (``models/deepseek_v2.py::_choose_weight_formats``).

``MLXB200_FP8_EXPERTS`` and the checkpoint format decide, once at load, whether the expert banks are bf16, block-scaled MXFP8 or
packed MLX-affine, whether the shared experts ride in the routed bank, and whether attention runs on the absorbed latent weights.
Loading needs no GPU: the stage is built on the CPU with ``backend="b200"``."""
import pytest
import torch

from mlx_sharding_b200.config import ModelConfig
from mlx_sharding_b200.models import build_stage
from mlx_sharding_b200.utils.checkpoint import random_state_dict
from mlx_sharding_b200.utils.loader import random_model

# layer 0 dense, layer 1 MoE; attention at the shapes of the absorbed-latent MLA kernel (16 heads, kv_lora_rank 512, rope 64)
CFG = dict(model_type="deepseek_v2", vocab_size=256, hidden_size=256, intermediate_size=256, moe_intermediate_size=128,
           num_hidden_layers=2, num_attention_heads=16, num_key_value_heads=16, n_shared_experts=2, n_routed_experts=8,
           routed_scaling_factor=1.0, kv_lora_rank=512, q_lora_rank=None, qk_rope_head_dim=64, v_head_dim=32, qk_nope_head_dim=32,
           topk_method="greedy", n_group=1, topk_group=1, num_experts_per_tok=2, moe_layer_freq=1, first_k_dense_replace=1,
           norm_topk_prob=False, rms_norm_eps=1e-6, rope_theta=10000.0, max_position_embeddings=512, tie_word_embeddings=False)
E, NS = 8, 2


def load(monkeypatch, bits, env, edit=None, expert_shard=None, **cfg):
    if env is None:
        monkeypatch.delenv("MLXB200_FP8_EXPERTS", raising=False)
    else:
        monkeypatch.setenv("MLXB200_FP8_EXPERTS", env)
    cfg = dict(CFG, **cfg)
    quant = dict(group_size=64, bits=bits) if bits else None
    if edit is None:
        return random_model(cfg, backend="b200", seed=3, quantization=quant, expert_shard=expert_shard)
    if quant:
        cfg["quantization"] = quant
    c = ModelConfig.from_dict(cfg)
    model = build_stage(c, c.shard(), torch.bfloat16, "cpu", "b200")
    sd = dict(random_state_dict(c, seed=3, quantization=quant))
    edit(sd)
    return model.load_state(sd)


def fmt(W):
    return "mxfp8" if W.mxfp8 is not None else "affine" if W.is_quantized else "bf16"


def experts(W):
    return (W.mxfp8[0] if W.mxfp8 is not None else W.wq if W.is_quantized else W.weight).shape[0]


def check(m, bank, fused, absorbed, attention, n_experts=E):
    w = m.layer_weights[1]
    assert [fmt(w[k]) for k in ("e_gate", "e_up", "e_down")] == [bank] * 3
    assert all(experts(w[k]) == n_experts + (NS if fused else 0) for k in ("e_gate", "e_up", "e_down"))
    assert ("n_fused_shared" in w) == fused and w.get("n_fused_shared", NS) == NS
    assert all((k in w) != fused for k in ("s_gate", "s_up", "s_down"))
    assert m.absorbed_mla == absorbed
    assert all(("qkv_abs" in m.layer_weights[i]) == absorbed for i in (0, 1))
    assert all(fmt(m.layer_weights[i][k]) == attention for i in (0, 1) for k in ("qkv_a", "kv_b", "o"))
    assert fmt(m.layer_weights[0]["gate"]) == ("affine" if m.qcfg else "bf16")


@pytest.mark.parametrize("bits,env,bank,fused,absorbed", [
    (0, None, "bf16", True, True),
    (0, "0", "bf16", True, True),
    (0, "1", "mxfp8", True, True),
    (4, None, "mxfp8", True, True),
    (4, "1", "mxfp8", True, True),
    (8, None, "mxfp8", True, True),
    (8, "1", "mxfp8", True, True),
    (4, "0", "affine", False, False),
    (8, "0", "affine", False, False),
])
def test_bank_format_policy(monkeypatch, bits, env, bank, fused, absorbed):
    """Quantised attention is promoted to bf16 exactly where the banks become MXFP8; the dense layer-0 MLP stays packed."""
    check(load(monkeypatch, bits, env), bank, fused, absorbed, "affine" if bits and not absorbed else "bf16")


@pytest.mark.parametrize("env", [None, "0", "1"])
@pytest.mark.parametrize("bits", [0, 4])
def test_expert_shard_keeps_weights_as_loaded(monkeypatch, bits, env):
    m = load(monkeypatch, bits, env, expert_shard=(0, 2))
    check(m, "affine" if bits else "bf16", False, not bits, "affine" if bits else "bf16", n_experts=E // 2)


@pytest.mark.parametrize("shape", [dict(moe_intermediate_size=64), dict(hidden_size=192)])
@pytest.mark.parametrize("bits,env", [(0, "1"), (4, None)])
def test_bank_not_multiple_of_128_keeps_its_format(monkeypatch, shape, bits, env):
    """The FP8 GEMM's k-block is 128 wide: such a bank stays as loaded (a bf16 one still takes the shared experts), while the
    attention promotion of a quantised checkpoint still applies."""
    check(load(monkeypatch, bits, env, **shape), "affine" if bits else "bf16", not bits, True, "bf16")


@pytest.mark.parametrize("env", [None, "1"])
def test_shared_experts_of_another_width_stay_apart(monkeypatch, env):
    p = "model.layers.1.mlp.shared_experts."

    def narrow(sd):
        for n in ("gate_proj", "up_proj"):
            sd[p + n + ".weight"] = sd[p + n + ".weight"][:128].contiguous()
        sd[p + "down_proj.weight"] = sd[p + "down_proj.weight"][:, :128].contiguous()

    check(load(monkeypatch, 0, env, edit=narrow), "mxfp8" if env == "1" else "bf16", False, True, "bf16")


def test_shared_experts_with_bias_stay_apart(monkeypatch):
    def bias(sd):
        sd["model.layers.1.mlp.shared_experts.gate_proj.bias"] = torch.ones(NS * 128, dtype=torch.bfloat16)

    m = load(monkeypatch, 0, None, edit=bias)
    check(m, "bf16", False, True, "bf16")
    assert m.layer_weights[1]["s_gate"].bias is not None
