"""Absorbed-latent MLA on sm_90a (ops/csrc/mla_decode.cu): the wgmma multi-query decode kernel over the cached 576-dim latent,
its fused prologue, and the whole DeepSeek stage on the folded weights — each against a plain PyTorch fp32 reference."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

NH, LAT, ROPE, PAGE = 16, 512, 64, 64


def _ref_attention(q, pool, block_tables, ctx_lens, scale):
    """fp32 oracle: q [B,16,576], pool [P,1,64,576] -> [B,16,512]."""
    B = q.shape[0]
    out = torch.zeros(B, NH, LAT, dtype=torch.float32, device=q.device)
    flat = pool.view(-1, PAGE, LAT + ROPE).float()
    for b in range(B):
        n = int(ctx_lens[b])
        pages = block_tables[b, : (n + PAGE - 1) // PAGE].long()
        kv = flat[pages].reshape(-1, LAT + ROPE)[:n]                  # [n, 576]
        s = (q[b].float() @ kv.t()) * scale                           # [16, n]
        p = torch.softmax(s, -1)
        out[b] = p @ kv[:, :LAT]
    return out


@pytest.mark.parametrize("B,ctxs,nsplit", [(3, [1, 64, 65], 0), (4, [128, 37, 200, 129], 0), (2, [1000, 517], 0), (2, [1000, 517], 4),
                                           (1, [8200], 0), (64, None, 0)])
def test_mla_decode_matches_fp32(B, ctxs, nsplit):
    from mlx_sharding_b200.ops import b200

    C = b200.load_extension()
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(B * 7 + (nsplit or 0))
    ctxs = ctxs or [128] * B
    max_ctx = max(ctxs)
    mb = (max_ctx + PAGE - 1) // PAGE
    npages = B * mb + 3
    pool = (torch.randn(npages, 1, PAGE, LAT + ROPE, device=dev, generator=g) * 0.5).to(torch.bfloat16)
    perm = torch.randperm(npages - 1, device=dev, generator=g)[: B * mb] + 1          # scattered pages, page 0 unused
    bt = perm.view(B, mb).to(torch.int32).contiguous()
    # q lives inside a wider row (the fused qkv GEMM output): token stride != 16 * 576
    wide = (torch.randn(B, NH * (LAT + ROPE) + 576, device=dev, generator=g) * 0.3).to(torch.bfloat16)
    q = wide[:, : NH * (LAT + ROPE)].unflatten(1, (NH, LAT + ROPE))
    cl = torch.tensor(ctxs, dtype=torch.int32, device=dev)
    scale = (192 ** -0.5) * 1.3
    out = C.mla_decode(q, pool, bt, cl, scale, max_ctx, nsplit)
    torch.cuda.synchronize()
    ref = _ref_attention(q, pool, bt, cl, scale)
    err = (out.float() - ref).abs().max().item()
    assert err < 2e-2, err                     # bf16 P and bf16 output: ~3 significant digits on values of O(1)
    rel = ((out.float() - ref).norm() / ref.norm()).item()
    assert rel < 6e-3, rel


def test_mla_prologue_matches_reference():
    from mlx_sharding_b200.ops import b200

    C = b200.load_extension()
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(3)
    T, W = 5, NH * 576 + 576
    qkv = (torch.randn(T, W, device=dev, generator=g)).to(torch.bfloat16)
    q = qkv[:, : NH * 576].unflatten(1, (NH, 576))
    ckv, kpe = qkv[:, NH * 576: NH * 576 + 512], qkv[:, NH * 576 + 512:]
    w = (1 + 0.1 * torch.randn(512, device=dev, generator=g)).to(torch.bfloat16)
    pool = torch.zeros(8, 1, PAGE, 576, dtype=torch.bfloat16, device=dev)
    slots = torch.tensor([70, 3, 129, 200, 64], dtype=torch.int32, device=dev)
    pos = torch.tensor([6, 3, 1, 300, 0], dtype=torch.int32, device=dev)
    inv = (1.0 / (10000 ** (torch.arange(0, 64, 2, device=dev).float() / 64))).contiguous()
    q0, ckv0, kpe0 = q.float().clone(), ckv.float().clone(), kpe.float().clone()
    C.mla_absorbed_prologue(q, ckv, kpe, w, 1e-6, pool, slots, pos, inv, 1.0)
    torch.cuda.synchronize()

    def rope(x, p):          # interleaved pairs
        ang = p.float()[:, None] * inv[None]
        a, b = x[..., 0::2], x[..., 1::2]
        cs, sn = ang.cos(), ang.sin()
        while cs.dim() < a.dim():
            cs, sn = cs.unsqueeze(1), sn.unsqueeze(1)
        return torch.stack([a * cs - b * sn, a * sn + b * cs], -1).flatten(-2)

    lat = ckv0 * torch.rsqrt(ckv0.pow(2).mean(-1, keepdim=True) + 1e-6) * w.float()
    rows = pool.view(-1, 576)[slots.long()].float()
    assert torch.allclose(rows[:, :512], lat, atol=2e-2, rtol=2e-2)
    assert torch.allclose(rows[:, 512:], rope(kpe0, pos), atol=2e-2, rtol=2e-2)
    assert torch.allclose(q.float()[..., 512:], rope(q0[..., 512:], pos), atol=2e-2, rtol=2e-2)
    assert torch.equal(q.float()[..., :512], q0[..., :512])


MLA_CFG = dict(model_type="deepseek_v2", vocab_size=512, hidden_size=512, intermediate_size=1024, moe_intermediate_size=128,
               num_hidden_layers=3, num_attention_heads=16, num_key_value_heads=16, n_shared_experts=2, n_routed_experts=8,
               routed_scaling_factor=1.0, kv_lora_rank=512, q_lora_rank=None, qk_rope_head_dim=64, v_head_dim=128,
               qk_nope_head_dim=128, topk_method="greedy", n_group=1, topk_group=1, num_experts_per_tok=3, moe_layer_freq=1,
               first_k_dense_replace=1, norm_topk_prob=False, rms_norm_eps=1e-6, rope_theta=10000.0, max_position_embeddings=4096,
               tie_word_embeddings=False,
               rope_scaling=dict(beta_fast=32, beta_slow=1, factor=40, mscale=0.707, mscale_all_dim=0.707,
                                 original_max_position_embeddings=4096, type="yarn"))


def test_stage_on_absorbed_weights_matches_decompressed_cache():
    """Whole DeepSeek stage: latent cache + folded weights + wgmma latent attention (decode) / decompressing prefill (chunked, so
    the second chunk attends to cached latents) vs the default decompressed K/V cache — same weights, bf16 tolerances."""
    from helpers import run_sequence
    from mlx_sharding_b200.models.deepseek_v2 import DeepseekV2Stage
    from mlx_sharding_b200.utils.loader import random_model

    base = random_model(MLA_CFG, device="cuda", backend="b200", seed=5)

    class Absorbed(DeepseekV2Stage):
        absorbed_mla = True

    m = Absorbed(base.cfg, base.spec, base.dtype, base.device, "b200")
    # share the loaded tensors, then fold
    m.embed_tokens, m.norm_w, m.lm_head, m.rope = base.embed_tokens, base.norm_w, base.lm_head, base.rope
    m.layer_weights = {i: dict(w) for i, w in base.layer_weights.items()}
    m._post_load()
    L, hk, dk, dv = m.kv_geometry()
    assert (hk, dk, dv) == (1, 576, 0)
    toks = torch.randint(3, 500, (150,), generator=torch.Generator().manual_seed(1)).tolist()
    ref = run_sequence([base], toks, 6, page_size=64, chunk=100)
    got = run_sequence([m], toks, 6, page_size=64, chunk=100)
    for a, b in zip(ref, got):
        assert (a - b).abs().max() < 0.08 * max(1.0, a.abs().max().item()), (a - b).abs().max()
        assert int(a.argmax()) == int(b.argmax()) or (a.max() - a[int(b.argmax())]) < 0.05
