"""Sharded Llama (also Mistral).

Reference: ``shard/server/model/llama.py`` (layer-range wrapper) + upstream ``TransformerBlock``
(SURVEY U1): pre-norm block, GQA, half-split RoPE with optional linear / llama3 scaling, SwiGLU MLP.

Design: Q/K/V projections are concatenated at load into one ``[Nq+2Nkv, H]`` weight (one GEMM
launch, SURVEY K3/K4); gate/up run as one dual-accumulator wgmma GEMM with the SiLU·mul epilogue;
residual adds ride the O-proj / down-proj GEMM epilogues; the last down-proj of a stage is the kernel
that stores straight into the next stage's input buffer (``parallel/p2p_fused.py``).
"""
from __future__ import annotations

import torch

from ..ops import BatchMeta, LinearWeight
from .base import StageModel, llama_rope_spec


class LlamaStage(StageModel):
    arch = "llama"
    act = "silu"
    gemma = False
    PRE_MLP_NORM = "post_attention_layernorm"   # checkpoint name of the norm in front of the MLP block

    def _make_rope(self):
        return llama_rope_spec(self.cfg)

    def _load_layer(self, sd, i, attn=True, mlp=True) -> dict:
        p = f"model.layers.{i}"
        a = p + ".self_attn"
        w = {}
        if attn:
            q, k, v = (self._lin(sd, f"{a}.{n}_proj") for n in ("q", "k", "v"))
            w.update(in_ln=self._vec(sd, p + ".input_layernorm.weight"), qkv=LinearWeight.concat([q, k, v]),
                     o=self._lin(sd, a + ".o_proj"))
        if mlp:
            w.update(mlp_ln=self._vec(sd, f"{p}.{self.PRE_MLP_NORM}.weight"),
                     gate=self._lin(sd, p + ".mlp.gate_proj"), up=self._lin(sd, p + ".mlp.up_proj"),
                     down=self._lin(sd, p + ".mlp.down_proj"))
        return w

    def _attention(self, w, normed: torch.Tensor, meta: BatchMeta, kpool, vpool) -> torch.Tensor:
        O, c = self.ops, self.cfg
        T = normed.shape[0]
        nh, nkv, hd = c.num_attention_heads, c.num_key_value_heads, c.head_dim
        qkv = O.linear(normed, w["qkv"])
        q = qkv[:, : nh * hd].view(T, nh, hd)
        k = qkv[:, nh * hd:(nh + nkv) * hd].view(T, nkv, hd)
        v = qkv[:, (nh + nkv) * hd:].view(T, nkv, hd)
        O.rope_(q, meta.positions, self.rope)
        O.rope_(k, meta.positions, self.rope)
        O.kv_write(k, v, kpool, vpool, meta.slot_mapping)
        attn = O.paged_attention(q, kpool, vpool, meta, c.attn_scale,
                                 float(c.attn_logit_softcapping or 0.0) if self.gemma else 0.0)
        return attn.reshape(T, nh * hd)

    def attn_block(self, i, h, meta, kpool, vpool):
        O, c, w = self.ops, self.cfg, self.layer_weights[i]
        normed = O.rmsnorm(h, w["in_ln"], c.rms_norm_eps)
        attn = self._attention(w, normed, meta, kpool, vpool)
        return O.linear(attn, w["o"], residual=h, **self._final_kwargs(i, h.shape[0], "attn"))

    def mlp_block(self, i, h, meta):
        O, c, w = self.ops, self.cfg, self.layer_weights[i]
        normed = O.rmsnorm(h, w["mlp_ln"], c.rms_norm_eps)
        act = O.gated_up(normed, w["gate"], w["up"], self.act)
        return O.linear(act, w["down"], residual=h, **self._final_kwargs(i, h.shape[0], "mlp"))


Model = LlamaStage
