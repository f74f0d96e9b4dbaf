"""Pure-PyTorch implementation of the op API (device-agnostic, fp32 internal math).

Three roles:
  1. the CPU execution path (tests, gloo plumbing config, machines without a GPU);
  2. the numerical oracle every sm_90a kernel in ``ops/csrc`` is tested against;
  3. on CUDA tensors it *is* the "straight PyTorch + cuBLAS" same-box baseline (``baseline/``).

Each function documents which upstream behaviour (SURVEY §2.2 U1–U12, §2.6 K1–K17) it reproduces.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from .meta import BatchMeta
from .weights import LinearWeight, RopeSpec

NAME = "reference"

# Oracle mode (default): every matmul accumulates and returns true fp32.  ``FAST_BASELINE = True`` turns
# this module into the "straight PyTorch + cuBLAS" baseline: bf16 tensor-core GEMMs via F.linear with bf16
# outputs, the way a plain PyTorch re-implementation of the reference pipeline would run on an H100.
FAST_BASELINE = False


# ------------------------------------------------------------------------------------------ K1
def embed(ids: torch.Tensor, emb: LinearWeight, scale: float = 1.0,
          dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """Embedding gather with optional in-line affine dequant and Gemma ``sqrt(H)`` scale."""
    ids = ids.long()
    if emb.is_quantized:
        rows = LinearWeight(wq=emb.wq[ids], scales=emb.scales[ids], biases=emb.biases[ids],
                            group_size=emb.group_size, bits=emb.bits).dense(torch.float32)
    else:
        rows = emb.weight[ids].float()
    if scale != 1.0:
        # Gemma multiplies in the model dtype (reference gemma2.py:42-43)
        rows = rows.to(dtype).float() * torch.tensor(scale, dtype=dtype).float()
    return rows.to(dtype)


# ------------------------------------------------------------------------------------------ K2
def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float, gemma: bool = False,
            residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``x * rsqrt(mean(x^2)+eps) * g`` (Gemma: ``g = 1 + w``); optional post-norm residual add
    ``residual + norm(x)`` (Gemma-2's post-attention / post-FFN norms)."""
    xf = x.float()
    y = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    g = (1.0 + w.float()) if gemma else w.float()
    y = (y * g).to(x.dtype)
    if residual is not None:
        y = (y.float() + residual.float()).to(x.dtype)
    return y


def add_rmsnorm(x: torch.Tensor, residual: torch.Tensor, w: torch.Tensor, eps: float,
                gemma: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """``h = x + residual`` (rounded to the activation dtype, like the unfused graph) then norm(h)."""
    h = (x.float() + residual.float()).to(x.dtype)
    return rmsnorm(h, w, eps, gemma), h


# ------------------------------------------------------------------------------------------ K3-K5, K8, K9, K12
def linear(x: torch.Tensor, W: LinearWeight, residual: Optional[torch.Tensor] = None,
           out_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    """``y = x @ W^T (+ bias) (+ residual)``; fp32 accumulate, single rounding at the end."""
    if FAST_BASELINE and x.is_cuda and x.dtype != torch.float32:
        y = F.linear(x, W.dense_cached(x.dtype)).float()  # cuBLAS bf16 path (baseline role)
    else:
        y = x.float() @ W.dense(torch.float32).t()
    if W.bias is not None:
        y = y + W.bias.float()
    if residual is not None:
        y = y + residual.float()
    return y.to(out_dtype or x.dtype)


def act_fn(name: str, x: torch.Tensor) -> torch.Tensor:
    if name == "silu":
        return F.silu(x)
    if name in ("gelu_tanh", "gelu_pytorch_tanh", "gelu_approx"):
        return F.gelu(x, approximate="tanh")
    raise ValueError(f"unknown activation {name}")


def gated_up(x: torch.Tensor, Wg: LinearWeight, Wu: LinearWeight, act: str = "silu") -> torch.Tensor:
    """``act(x Wg^T) * (x Wu^T)`` — SwiGLU / GeGLU first half, one rounding (K9)."""
    g = linear(x, Wg, out_dtype=torch.float32)
    u = linear(x, Wu, out_dtype=torch.float32)
    return (act_fn(act, g) * u).to(x.dtype)


# ------------------------------------------------------------------------------------------ K6
def rope_(x: torch.Tensor, positions: torch.Tensor, spec: RopeSpec, rot_offset: int = 0) -> torch.Tensor:
    """In-place rotary embedding on ``x[T, heads, D][..., rot_offset : rot_offset + rot_dim]``.

    ``interleaved=False``: half-split pairs ``(i, i + rot/2)`` (Llama / Gemma, MLX ``traditional=False``).
    ``interleaved=True`` : adjacent pairs ``(2i, 2i+1)`` (DeepSeek-V2, MLX ``traditional=True``)."""
    rd = spec.rot_dim
    ang = positions.float()[:, None] * spec.inv_freq.float().to(x.device)[None, :]  # [T, rd/2]
    cos, sin = ang.cos()[:, None, :], ang.sin()[:, None, :]
    xs = x[..., rot_offset:rot_offset + rd].float() * spec.mscale
    if spec.interleaved:
        x1, x2 = xs[..., 0::2], xs[..., 1::2]
        o = torch.stack((x1 * cos - x2 * sin, x1 * sin + x2 * cos), dim=-1).flatten(-2)
    else:
        x1, x2 = xs[..., : rd // 2], xs[..., rd // 2:]
        o = torch.cat((x1 * cos - x2 * sin, x2 * cos + x1 * sin), dim=-1)
    x[..., rot_offset:rot_offset + rd] = o.to(x.dtype)
    return x


# ------------------------------------------------------------------------------------------ K7
def kv_write(k: torch.Tensor, v: torch.Tensor, kpool: torch.Tensor, vpool: torch.Tensor,
             slot_mapping: torch.Tensor):
    """Append ``k[T,Hk,Dk]`` / ``v[T,Hk,Dv]`` into the paged pools ``[P, Hk, page, D]``."""
    page = kpool.shape[2]
    slots = slot_mapping.long()
    p, o = slots // page, slots % page
    kpool[p, :, o, :] = k.to(kpool.dtype)
    vpool[p, :, o, :] = v.to(vpool.dtype)


def kv_write_mla(kv: torch.Tensor, k_pe: torch.Tensor, kpool: torch.Tensor, vpool: torch.Tensor,
                 slot_mapping: torch.Tensor, nope: int, vdim: int):
    """MLA cache append in the reference's decompressed layout (deepseek_v2.py:120-125):
    ``K = [k_nope | k_pe broadcast over heads]`` (192), ``V`` (128); ``kv[T, heads, nope + vdim]``."""
    T, nh, _ = kv.shape
    k = torch.cat((kv[..., :nope], k_pe[:, None, :].expand(T, nh, k_pe.shape[-1])), dim=-1)
    kv_write(k, kv[..., nope:nope + vdim], kpool, vpool, slot_mapping)


def paged_attention(q: torch.Tensor, kpool: torch.Tensor, vpool: torch.Tensor, meta: BatchMeta,
                    scale: float, softcap: float = 0.0) -> torch.Tensor:
    """Causal attention of ``q[T,Hq,Dk]`` against the paged cache (which already contains this
    step's keys).  Token at absolute position ``p`` sees cache positions ``0..p``.  GQA by head
    grouping; ``softcap>0`` applies Gemma-2's ``tanh(s/cap)*cap`` to the scaled scores."""
    T, Hq, Dk = q.shape
    Hk, page, Dv = kpool.shape[1], kpool.shape[2], vpool.shape[3]
    G = Hq // Hk
    out = torch.empty(T, Hq, Dv, dtype=q.dtype, device=q.device)
    cu = meta.cu_seqlens.tolist()
    ctx = meta.context_lens.tolist()
    for b in range(meta.num_seqs):
        s, e, L = cu[b], cu[b + 1], ctx[b]
        if e == s:
            continue
        nblk = (L + page - 1) // page
        pages = meta.block_tables[b, :nblk].long()
        K = kpool[pages].permute(1, 0, 2, 3).reshape(Hk, nblk * page, Dk)[:, :L].float()
        V = vpool[pages].permute(1, 0, 2, 3).reshape(Hk, nblk * page, Dv)[:, :L].float()
        qb = q[s:e].float().permute(1, 0, 2).reshape(Hk, G, e - s, Dk)
        sc = torch.einsum("hgqd,hkd->hgqk", qb, K) * scale
        if softcap and softcap > 0:
            sc = torch.tanh(sc / softcap) * softcap
        qpos = meta.positions[s:e].long()
        kpos = torch.arange(L, device=q.device)
        mask = kpos[None, :] > qpos[:, None]
        sc = sc.masked_fill(mask[None, None], float("-inf"))
        p = torch.softmax(sc, dim=-1)
        o = torch.einsum("hgqk,hkd->hgqd", p, V).reshape(Hq, e - s, Dv).permute(1, 0, 2)
        out[s:e] = o.to(q.dtype)
    return out


# ------------------------------------------------------------------------------------------ K10
def moe_route(x: torch.Tensor, gate_w: torch.Tensor, top_k: int, method: str = "greedy",
              n_group: int = 1, topk_group: int = 1, scaling: float = 1.0,
              norm_topk: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp32 softmax router + top-k (greedy / group_limited_greedy) -> ``(idx int32 [T,k], w fp32 [T,k])``.
    Ties resolve to the lowest expert id; indices are returned in descending-score order."""
    scores = torch.softmax(x.float() @ gate_w.float().t(), dim=-1)
    T, E = scores.shape
    sel = scores
    if method == "group_limited_greedy" and n_group > 1:
        gs = scores.view(T, n_group, E // n_group).amax(-1)
        gidx = torch.topk(gs, topk_group, dim=-1).indices
        gmask = torch.zeros_like(gs).scatter_(1, gidx, 1.0)
        smask = gmask[:, :, None].expand(T, n_group, E // n_group).reshape(T, E)
        sel = scores.masked_fill(smask == 0, 0.0)
    # stable descending sort => deterministic tie-break on the lowest index
    order = torch.sort(sel, dim=-1, descending=True, stable=True).indices[:, :top_k]
    w = torch.gather(scores, 1, order)
    if norm_topk and top_k > 1:
        w = w / (w.sum(-1, keepdim=True) + 1e-20)
    else:
        w = w * scaling
    return order.to(torch.int32), w


# ------------------------------------------------------------------------------------------ K11
def run_aside(fn):
    """Backend hook: independent work that the CUDA backend forks onto a side stream runs inline here."""
    fn()
    return None


def moe_experts(x: torch.Tensor, idx: torch.Tensor, w: torch.Tensor, Wg: LinearWeight, Wu: LinearWeight,
                Wd: LinearWeight, act: str = "silu", extra: Optional[torch.Tensor] = None,
                residual: Optional[torch.Tensor] = None, join=None) -> torch.Tensor:
    """``y[t] = sum_k w[t,k] * down_e(act(gate_e x) * up_e x) (+ extra[t]) (+ residual[t])``.
    Intermediate activations are rounded to the activation dtype exactly where the kernels round."""
    T, H = x.shape
    E = (Wg.wq if Wg.is_quantized else Wg.weight).shape[0]
    y = torch.zeros(T, H, dtype=torch.float32, device=x.device)
    idx_l = idx.long()
    for e in range(E):
        tok, slot = torch.where(idx_l == e)
        if tok.numel() == 0:
            continue
        xe = x[tok]
        h = gated_up(xe, Wg.select_expert(e), Wu.select_expert(e), act)
        o = linear(h, Wd.select_expert(e), out_dtype=torch.float32)
        y.index_add_(0, tok, o * w[tok, slot].float()[:, None])
    if extra is not None:
        y = y + extra.float()
    if residual is not None:
        y = y + residual.float()
    return y.to(x.dtype)


# ------------------------------------------------------------------------------------------ K12 epilogue
def softcap_(logits: torch.Tensor, cap: float) -> torch.Tensor:
    return torch.tanh(logits / cap) * cap


# ------------------------------------------------------------------------------------------ K13
def apply_repetition_penalty_(logits: torch.Tensor, ctx_tokens: torch.Tensor, penalty: float) -> torch.Tensor:
    """U7: for ids in ctx: ``l<0 ? l*p : l/p`` (in place, 1-D logits)."""
    if ctx_tokens.numel() == 0 or penalty == 1.0:
        return logits
    ids = ctx_tokens.long().unique()
    sel = logits[ids]
    logits[ids] = torch.where(sel < 0, sel * penalty, sel / penalty)
    return logits


def apply_penalties_(logits: torch.Tensor, rep_ctx: torch.Tensor, penalty: torch.Tensor,
                     bias_idx: torch.Tensor, bias_val: torch.Tensor) -> torch.Tensor:
    """Batched in-place repetition penalty (reference utils.py:167-170) then logit_bias add
    (utils.py:127-130, inside ``sample``).  ``rep_ctx int32 [B, C]`` / ``bias_idx int32 [B, Nb]`` are
    padded with ``-1``."""
    B = logits.shape[0]
    for b in range(B):
        c = rep_ctx[b]
        c = c[c >= 0]
        apply_repetition_penalty_(logits[b], c, float(penalty[b]))
        bi = bias_idx[b]
        m = bi >= 0
        if m.any():
            logits[b].index_add_(0, bi[m].long(), bias_val[b][m].to(logits.dtype))
    return logits


def sample(logits: torch.Tensor, temperature: torch.Tensor, top_p: torch.Tensor,
           generator: Optional[torch.Generator] = None, top_logprobs: int = 0):
    """Batched sampler (reference shard/utils.py:126-139 + mlx_lm ``top_p_sampling``).

    ``logits`` fp32 ``[B, V]`` *after* bias / repetition penalty.  Per row: ``temp == 0`` -> argmax;
    ``0 < top_p < 1`` -> nucleus; else categorical(softmax(logits / temp)).
    Returns ``(tokens int64 [B], token_logprob fp32 [B], topk_ids, topk_logprobs)`` where logprobs are
    ``logits - logsumexp(logits)`` (temperature **not** applied — reference utils.py:131)."""
    B, V = logits.shape
    lf = logits.float()
    logprobs = lf - torch.logsumexp(lf, dim=-1, keepdim=True)
    tokens = torch.empty(B, dtype=torch.int64, device=logits.device)
    t_cpu, p_cpu = temperature.tolist(), top_p.tolist()
    for b in range(B):
        t, p = t_cpu[b], p_cpu[b]
        if t == 0:
            tokens[b] = torch.argmax(lf[b])
            continue
        probs = torch.softmax(lf[b] / t, dim=-1)
        if 0 < p < 1.0:
            sp, si = torch.sort(probs, descending=False, stable=True)
            cum = torch.cumsum(sp, dim=0)
            keep = cum > (1 - p)
            sp = torch.where(keep, sp, torch.zeros_like(sp))
            j = torch.multinomial(sp / sp.sum(), 1, generator=generator)
            tokens[b] = si[j].squeeze()
        else:
            tokens[b] = torch.multinomial(probs, 1, generator=generator).squeeze()
    tok_lp = logprobs.gather(1, tokens[:, None]).squeeze(1)
    if top_logprobs > 0:
        tk = torch.topk(logprobs, top_logprobs, dim=-1)
        return tokens, tok_lp, tk.indices, tk.values
    return tokens, tok_lp, None, None


def sample_block(logits: torch.Tensor, sv, tag_out, toks_out, lp_out, top_ids_out, top_lp_out):
    """Sampling driven by a step block (``parallel/graph_decode.py``): penalties, then per-sequence temperature / top-p with a
    per-request random stream — row ``b`` draws from a generator seeded with its ``(seed, tokens sampled so far)`` pair, so a
    request's tokens do not depend on which batch it decodes in.  Results go into the result-message views."""
    lf = logits.float().clone()
    if sv.has_pen:
        apply_penalties_(lf, sv.rep, sv.penalty, sv.bidx, sv.bval)
    B = lf.shape[0]
    rng = sv.rng.view(B, 2).tolist()
    k = 0 if top_ids_out is None else top_ids_out.shape[1]
    for b in range(B):
        g = torch.Generator(device=lf.device)
        g.manual_seed((rng[b][0] * 1000003 + rng[b][1] * 7919 + 12345) & 0x7FFFFFFFFFFFFFFF)
        t, lp, ti, tl = sample(lf[b:b + 1], sv.temps[b:b + 1], sv.top_p[b:b + 1], generator=g, top_logprobs=k)
        toks_out[b], lp_out[b] = t[0], lp[0]
        if k:
            top_ids_out[b], top_lp_out[b] = ti[0], tl[0]
    tag_out.copy_(sv.tag)


def mla_rope_kv_write(q: torch.Tensor, k_pe: torch.Tensor, kv: torch.Tensor, kpool: torch.Tensor, vpool: torch.Tensor,
                      meta: BatchMeta, spec: RopeSpec, nope: int, vdim: int):
    """DeepSeek-V2 attention prologue: rope the ``*_pe`` slices (q in place) and append
    ``K = [k_nope | rope(k_pe)]``, ``V`` to the paged cache (one fused kernel on the b200 backend)."""
    rope_(q, meta.positions, spec, nope)
    kp = k_pe.clone().unsqueeze(1)
    rope_(kp, meta.positions, spec, 0)
    kv_write_mla(kv, kp.squeeze(1), kpool, vpool, meta.slot_mapping, nope, vdim)
