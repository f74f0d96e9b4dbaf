"""Same-box baseline arm: the reference pipeline re-implemented as plain PyTorch (BASELINE.md §1).

What the reference does (shard/utils.py:156-186, server/server.py:27-48, generate.py:52-88): layer-range pipeline stages, one
hidden-state hand-off per stage per token, sampling after the last stage.  MLX-Metal cannot run on an H100, so this module is the
"straight re-implementation" BASELINE.md names — and it is deliberately a *strong* one, not a strawman:

* every GEMM is cuBLAS (``F.linear`` / ``torch.bmm`` on bf16), attention is ``F.scaled_dot_product_attention`` over a contiguous
  KV cache, the MoE experts run as ONE padded batched GEMM over the stacked ``switch_mlp`` banks (each expert weight is read once
  per step, no Python loop over experts or sequences, no host sync);
* a decode step of a micro-batch group is ONE CUDA graph per stage; positions advance on the device;
* stage hand-off = NCCL ``send/recv`` (stream ordered), the last stage samples (argmax) and returns token ids to stage 0;
* the same micro-batching as the product (``world`` groups of ``batch`` sequences in flight), the same cost-balanced whole-layer
  split, the same model / shapes / dtype / synthetic data.

Nothing of the product's kernels, engine or pipeline runtime is on this path (only ``config.py`` for the architecture constants
and the whole-layer partitioner, so both arms split the model the same way).  ``bench.py --impl baseline`` drives it.
"""
from __future__ import annotations

import math
import os
import statistics
import sys
import time
from typing import List, Optional

import torch
import torch.distributed as dist
import torch.nn.functional as F


def _yarn_inv_freq(cfg) -> tuple:
    """(inv_freq [rd/2], mscale) of DeepSeek-V2's YaRN rotary (same formulae as HF modeling_deepseek_v2)."""
    dim, base = cfg.qk_rope_head_dim, cfg.rope_theta
    rs = cfg.rope_scaling
    plain = 1.0 / (base ** (torch.arange(0, dim, 2, dtype=torch.float32) / dim))
    if not rs or rs.get("type", rs.get("rope_type")) != "yarn":
        return plain, 1.0
    factor, orig = float(rs["factor"]), float(rs.get("original_max_position_embeddings", 4096))
    bf, bs = float(rs.get("beta_fast", 32)), float(rs.get("beta_slow", 1))
    corr = lambda n: (dim * math.log(orig / (n * 2 * math.pi))) / (2 * math.log(base))
    low, high = max(math.floor(corr(bf)), 0), min(math.ceil(corr(bs)), dim - 1)
    if low == high:
        high += 0.001
    ramp = ((torch.arange(dim // 2, dtype=torch.float32) - low) / (high - low)).clamp(0, 1)
    inv = plain / factor * ramp + plain * (1 - ramp)
    ms = lambda m: 1.0 if factor <= 1 else 0.1 * m * math.log(factor) + 1.0
    return inv, ms(rs.get("mscale", 1)) / ms(rs.get("mscale_all_dim", 0))


def _rmsnorm(x, w, eps):
    xf = x.float()
    return (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(x.dtype) * w


class TorchStage:
    """Layers ``[start, end)`` of DeepSeek-V2(-Lite) or Llama in bf16 PyTorch, random-init weights, contiguous KV cache."""

    def __init__(self, cfg, start: int, end: int, device, groups: int, batch: int, max_len: int, seed: int = 1):
        self.cfg, self.start, self.end, self.dev = cfg, start, end, device
        self.first, self.last = start == 0, end == cfg.num_hidden_layers
        self.G, self.B, self.S = groups, batch, max_len
        self.moe_arch = cfg.model_type == "deepseek_v2"
        g = torch.Generator(device=device).manual_seed(seed + 7919 * start)
        bf = torch.bfloat16

        def W(*shape, std=0.02):
            return (torch.randn(*shape, generator=g, device=device, dtype=torch.float32) * std).to(bf)

        H = cfg.hidden_size
        self.layers = []
        for i in range(start, end):
            w = dict(in_ln=torch.ones(H, device=device, dtype=bf), post_ln=torch.ones(H, device=device, dtype=bf))
            if self.moe_arch:
                nh, qd = cfg.num_attention_heads, cfg.qk_nope_head_dim + cfg.qk_rope_head_dim
                lr, rd = cfg.kv_lora_rank, cfg.qk_rope_head_dim
                w["qkv_a"] = W(nh * qd + lr + rd, H)                               # q_proj | kv_a_proj_with_mqa (one GEMM)
                w["kv_a_ln"] = torch.ones(lr, device=device, dtype=bf)
                w["kv_b"] = W(nh * (cfg.qk_nope_head_dim + cfg.v_head_dim), lr)
                w["o"] = W(H, nh * cfg.v_head_dim)
                if cfg.is_moe_layer(i):
                    E, I = cfg.n_routed_experts, cfg.moe_intermediate_size
                    w["router"] = W(E, H)
                    w["e_gu"] = W(E, 2 * I, H)                                      # gate | up stacked: one bmm
                    w["e_down"] = W(E, H, I)
                    if cfg.n_shared_experts:
                        Is = I * cfg.n_shared_experts
                        w["s_gu"], w["s_down"] = W(2 * Is, H), W(H, Is)
                else:
                    w["gu"], w["down"] = W(2 * cfg.intermediate_size, H), W(H, cfg.intermediate_size)
            else:
                hd, nh, nkv = cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads
                w["qkv"] = W((nh + 2 * nkv) * hd, H)
                w["o"] = W(H, nh * hd)
                w["gu"], w["down"] = W(2 * cfg.intermediate_size, H), W(H, cfg.intermediate_size)
            self.layers.append(w)
        if self.first:
            self.embed = W(cfg.vocab_size, H)
        if self.last:
            self.norm = torch.ones(H, device=device, dtype=bf)
            self.lm_head = W(cfg.vocab_size, H)
        if self.moe_arch:
            inv, self.mscale = _yarn_inv_freq(cfg)
            self.kdim, self.vdim, self.kvh = cfg.qk_nope_head_dim + cfg.qk_rope_head_dim, cfg.v_head_dim, cfg.num_attention_heads
        else:
            inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, cfg.head_dim, 2, dtype=torch.float32) / cfg.head_dim))
            self.mscale = 1.0
            self.kdim = self.vdim = cfg.head_dim
            self.kvh = cfg.num_key_value_heads
        self.inv_freq = inv.to(device)
        n = end - start
        # contiguous per-group KV cache [layer][B, heads, S, d] (the reference's KVCache layout, grown to max_len up front)
        self.k = [[torch.zeros(batch, self.kvh, max_len, self.kdim, device=device, dtype=bf) for _ in range(n)] for _ in range(groups)]
        self.v = [[torch.zeros(batch, self.kvh, max_len, self.vdim, device=device, dtype=bf) for _ in range(n)] for _ in range(groups)]
        self.ar_s = torch.arange(max_len, device=device)
        self.ar_b = torch.arange(batch, device=device)

    def weight_bytes(self) -> int:
        t = sum(v.numel() * v.element_size() for w in self.layers for v in w.values())
        for n in ("embed", "lm_head"):
            if hasattr(self, n):
                t += getattr(self, n).numel() * 2
        return t

    # ------------------------------------------------------------------------------------------ pieces
    def _rope(self, x, pos, interleaved: bool):
        """x [..., T, heads, rd] rotated at positions pos [T] (fp32 math)."""
        ang = pos.float()[:, None] * self.inv_freq[None, :]                          # [T, rd/2]
        cos, sin = (ang.cos() * self.mscale)[:, None, :], (ang.sin() * self.mscale)[:, None, :]
        xf = x.float()
        if interleaved:
            a, b = xf[..., 0::2], xf[..., 1::2]
            return torch.stack([a * cos - b * sin, a * sin + b * cos], -1).flatten(-2).to(x.dtype)
        h = xf.shape[-1] // 2
        a, b = xf[..., :h], xf[..., h:]
        return torch.cat([a * cos - b * sin, b * cos + a * sin], -1).to(x.dtype)

    def _moe(self, w, x, cap: Optional[int]):
        """Routed experts as one padded batched GEMM: [E, C, H] x [E, H, 2I] -> act -> [E, C, I] x [E, I, H]; C = capacity.
        ``cap=None`` (eager prefill) sizes C from the actual maximum expert load (one host sync)."""
        cfg = self.cfg
        T, H = x.shape
        E, k = cfg.n_routed_experts, cfg.num_experts_per_tok
        scores = torch.softmax(F.linear(x.float(), w["router"].float()), -1)
        wts, idx = torch.topk(scores, k, dim=-1)
        if cfg.norm_topk_prob:
            wts = wts / wts.sum(-1, keepdim=True)
        wts = wts * cfg.routed_scaling_factor
        flat = idx.reshape(-1)
        order = torch.argsort(flat, stable=True)
        e_sorted = flat[order]
        tok_sorted = order // k
        counts = torch.zeros(E, dtype=torch.int64, device=x.device).scatter_add_(0, flat, torch.ones_like(flat))   # no host sync
        starts = torch.cumsum(counts, 0) - counts
        slot = torch.arange(T * k, device=x.device) - starts[e_sorted]
        C = int(counts.max()) if cap is None else cap
        xp = torch.zeros(E, C, H, device=x.device, dtype=x.dtype)
        xp[e_sorted, slot] = x[tok_sorted]
        gu = torch.bmm(xp, w["e_gu"].transpose(1, 2))
        I = gu.shape[-1] // 2
        y = torch.bmm(F.silu(gu[..., :I]) * gu[..., I:], w["e_down"].transpose(1, 2))          # [E, C, H]
        contrib = y[e_sorted, slot].float() * wts.reshape(-1)[order][:, None]
        out = torch.zeros(T, H, device=x.device, dtype=torch.float32).index_add_(0, tok_sorted, contrib)
        return out.to(x.dtype)

    def _mlp(self, w, x, cap):
        if "router" in w:
            y = self._moe(w, x, cap)
            if "s_gu" in w:
                gu = F.linear(x, w["s_gu"])
                I = gu.shape[-1] // 2
                y = y + F.linear(F.silu(gu[..., :I]) * gu[..., I:], w["s_down"])
            return y
        gu = F.linear(x, w["gu"])
        I = gu.shape[-1] // 2
        return F.linear(F.silu(gu[..., :I]) * gu[..., I:], w["down"])

    def _qkv(self, w, x, pos):
        """-> q [T, nh, dk], k [T, kvh, dk], v [T, kvh, dv] (rope applied)."""
        cfg, T = self.cfg, x.shape[0]
        if self.moe_arch:
            nh, nope, rd, vd, lr = cfg.num_attention_heads, cfg.qk_nope_head_dim, cfg.qk_rope_head_dim, cfg.v_head_dim, cfg.kv_lora_rank
            qkv = F.linear(x, w["qkv_a"])
            q = qkv[:, : nh * (nope + rd)].view(T, nh, nope + rd)
            ckv, k_pe = qkv[:, nh * (nope + rd): nh * (nope + rd) + lr], qkv[:, nh * (nope + rd) + lr:]
            kv = F.linear(_rmsnorm(ckv, w["kv_a_ln"], cfg.rms_norm_eps), w["kv_b"]).view(T, nh, nope + vd)
            q = torch.cat([q[..., :nope], self._rope(q[..., nope:], pos, True)], -1)
            k_pe = self._rope(k_pe.view(T, 1, rd), pos, True).expand(T, nh, rd)
            return q, torch.cat([kv[..., :nope], k_pe], -1), kv[..., nope:]
        hd, nh, nkv = cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads
        qkv = F.linear(x, w["qkv"]).view(T, nh + 2 * nkv, hd)
        return self._rope(qkv[:, :nh], pos, False), self._rope(qkv[:, nh:nh + nkv], pos, False), qkv[:, nh + nkv:]

    @property
    def _scale(self) -> float:
        return self.cfg.attn_scale

    # ------------------------------------------------------------------------------------------ steps
    @torch.inference_mode()
    def decode(self, g: int, x: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
        """One token per sequence of group ``g``.  x: ids [B] (first stage) or hidden [B, H]; pos [B] int64 = position of this token.
        Static shapes only (graph-capturable).  Returns hidden [B, H] or sampled ids [B]."""
        cfg = self.cfg
        h = self.embed[x] if self.first else x
        B = h.shape[0]
        mask = (self.ar_s[None, :] <= pos[:, None])[:, None, None, :]                # [B, 1, 1, S]
        for li, w in enumerate(self.layers):
            n = _rmsnorm(h, w["in_ln"], cfg.rms_norm_eps)
            q, k, v = self._qkv(w, n, pos)
            K, V = self.k[g][li], self.v[g][li]
            K[self.ar_b[:B], :, pos] = k
            V[self.ar_b[:B], :, pos] = v
            a = F.scaled_dot_product_attention(q.unsqueeze(2), K[:B], V[:B], attn_mask=mask, scale=self._scale,
                                               enable_gqa=self.kvh != q.shape[1])
            h = h + F.linear(a.reshape(B, -1), w["o"])
            h = h + self._mlp(w, _rmsnorm(h, w["post_ln"], cfg.rms_norm_eps), cap=B)
        if self.last:
            return F.linear(_rmsnorm(h, self.norm, cfg.rms_norm_eps), self.lm_head).float().argmax(-1)
        return h

    @torch.inference_mode()
    def prefill(self, g: int, b0: int, x: torch.Tensor, nseq: int, S: int) -> torch.Tensor:
        """Prompts of sequences [b0, b0+nseq) of group g, S tokens each (eager).  x: ids [nseq*S] or hidden [nseq*S, H]."""
        cfg = self.cfg
        h = self.embed[x] if self.first else x
        pos = torch.arange(S, device=self.dev).repeat(nseq)
        for li, w in enumerate(self.layers):
            n = _rmsnorm(h, w["in_ln"], cfg.rms_norm_eps)
            q, k, v = self._qkv(w, n, pos)
            q, k, v = (t.reshape(nseq, S, t.shape[1], t.shape[2]).transpose(1, 2) for t in (q, k, v))
            self.k[g][li][b0:b0 + nseq, :, :S] = k
            self.v[g][li][b0:b0 + nseq, :, :S] = v
            a = F.scaled_dot_product_attention(q, k, v, is_causal=True, scale=self._scale, enable_gqa=self.kvh != q.shape[1])
            h = h + F.linear(a.transpose(1, 2).reshape(nseq * S, -1), w["o"])
            h = h + self._mlp(w, _rmsnorm(h, w["post_ln"], cfg.rms_norm_eps), cap=None)
        if self.last:
            last = h.view(nseq, S, -1)[:, -1]
            return F.linear(_rmsnorm(last, self.norm, cfg.rms_norm_eps), self.lm_head).float().argmax(-1)
        return h


class BaselinePipeline:
    """``world`` stages x ``G`` micro-batch groups; CUDA-graphed decode steps, NCCL p2p between stages."""

    def __init__(self, stage: TorchStage, rank: int, world: int, use_graphs: bool = True):
        self.st, self.rank, self.world = stage, rank, world
        self.G, self.B, dev = stage.G, stage.B, stage.dev
        H = stage.cfg.hidden_size
        self.first, self.last = rank == 0, rank == world - 1
        self.pos = [torch.zeros(self.B, dtype=torch.int64, device=dev) for _ in range(self.G)]
        self.tok = [torch.zeros(self.B, dtype=torch.int64, device=dev) for _ in range(self.G)]      # stage-0 input / last-stage output
        self.hid = [torch.zeros(self.B, H, dtype=torch.bfloat16, device=dev) for _ in range(self.G)]  # inbox of non-first stages
        self.out = [None] * self.G
        self.graphs = [None] * self.G
        self.use_graphs = use_graphs
        self.steps_done = [0] * self.G

    def _body(self, g: int):
        x = self.tok[g] if self.first else self.hid[g]
        out = self.st.decode(g, x, self.pos[g])
        if self.last:
            self.tok[g].copy_(out)
            out = self.tok[g]
        self.pos[g] += 1
        return out

    def capture(self):
        if not self.use_graphs:
            return
        for g in range(self.G):
            snap = (self.pos[g].clone(), self.tok[g].clone())
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(2):                       # cuBLAS workspace / autotune outside the capture
                    self._body(g)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            self.pos[g].copy_(snap[0]); self.tok[g].copy_(snap[1])
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                self.out[g] = self._body(g)
            self.graphs[g] = gr
        torch.cuda.synchronize()

    def run_body(self, g: int):
        if self.use_graphs:
            self.graphs[g].replay()
            return self.out[g]
        return self._body(g)

    def step_group(self, g: int):
        """recv -> (graph) compute -> send, for one group on this stage."""
        w = self.world
        if w > 1:
            if self.first:
                if self.steps_done[g] > 0:
                    dist.recv(self.tok[g], w - 1)
            else:
                dist.recv(self.hid[g], self.rank - 1)
        out = self.run_body(g)
        if w > 1:
            dist.send(out, 0 if self.last else self.rank + 1)
        self.steps_done[g] += 1

    def step_all(self):
        for g in range(self.G):
            self.step_group(g)

    def drain(self):
        if self.world > 1 and self.first:
            for g in range(self.G):
                if self.steps_done[g] > 0:
                    dist.recv(self.tok[g], self.world - 1)


def _max_over_ranks(v: float, dev) -> float:
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return v
    t = torch.tensor([v], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def run(args, world: int, rank: int, local: int, dev, steps: Optional[int] = None, warmup: Optional[int] = None,
        quiet: bool = False, e2e: bool = True) -> Optional[dict]:
    """Measure the baseline pipeline with the bench.py contract (device-timed decode, TTFT, e2e).  Returns the result dict on
    rank 0.  ``steps`` / ``warmup`` override the CLI values (``bench.py`` uses a short run to fill ``vs_baseline``)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    from bench import model_config
    from mlx_sharding_b200.config import ModelConfig
    from mlx_sharding_b200.parallel.partition import balanced_split
    from mlx_sharding_b200.utils.timing import ClockSampler

    steps = args.steps if steps is None else steps
    warmup = args.warmup if warmup is None else warmup
    log = (lambda *a: None) if quiet else (lambda *a: print(f"[baseline rank {rank}]", *a, file=sys.stderr, flush=True))
    cfg = ModelConfig.from_dict(model_config(args.model, args.layers))
    spec = balanced_split(cfg, world, half_layers=False)[rank]
    G, B, S = (args.groups or world), args.batch, args.prompt_len
    e2e_steps = (warmup + steps + 2) if e2e else 0
    max_len = (S + warmup + steps + e2e_steps + 8 + 63) // 64 * 64
    t0 = time.time()
    stage = TorchStage(cfg, spec.start_layer, spec.end_layer, dev, G, B, max_len, seed=1)
    torch.cuda.synchronize()
    log(f"layers [{spec.start_layer}, {spec.end_layer}) weights {stage.weight_bytes() / 1e9:.2f} GB built in {time.time() - t0:.1f}s")
    H = cfg.hidden_size
    gen = torch.Generator().manual_seed(1234)
    prompts = torch.randint(3, cfg.vocab_size - 1, (G, B, S), generator=gen)

    def chain_prefill(g, b0, nseq, pinned):
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        tt = time.perf_counter()
        if rank == 0:
            x = pinned.to(dev, non_blocking=True)
        else:
            x = torch.empty(nseq * S, H, dtype=torch.bfloat16, device=dev)
            dist.recv(x, rank - 1)
        out = stage.prefill(g, b0, x, nseq, S)
        if rank < world - 1:
            dist.send(out, rank + 1)
            toks = torch.empty(nseq, dtype=torch.int64, device=dev)
        else:
            toks = out
        if world > 1:
            dist.broadcast(toks, world - 1)
        torch.cuda.synchronize()
        return toks, time.perf_counter() - tt

    chunk = max(1, 2048 // S)          # prefill <= 2048 tokens per eager step
    first, batch_ttfts, ttfts = [], [], []
    for g in range(G):
        for rep in range(2):
            tt, parts = 0.0, []
            for b0 in range(0, B, chunk):
                n = min(chunk, B - b0)
                toks, dt = chain_prefill(g, b0, n, prompts[g, b0:b0 + n].reshape(-1).pin_memory())
                parts.append(toks)
                tt += dt
            if rep:
                batch_ttfts.append(tt)
        first.append(torch.cat(parts))
    p1 = prompts[0, 0].pin_memory()
    for rep in range(8):
        _, dt = chain_prefill(0, 0, 1, p1)
        if rep > 1:
            ttfts.append(dt)
    ttft_p50 = _max_over_ranks(statistics.median(ttfts), dev)
    ttft_batch = _max_over_ranks(statistics.median(batch_ttfts), dev)
    log(f"prefill done: TTFT p50 {ttft_p50 * 1e3:.2f} ms (1x{S}), {ttft_batch * 1e3:.1f} ms for {B}x{S}")

    pipe = BaselinePipeline(stage, rank, world, use_graphs=not getattr(args, "no_graphs", False))
    for g in range(G):
        pipe.pos[g].fill_(S)
        pipe.tok[g].copy_(first[g])
    pipe.capture()
    if world > 1:
        dist.barrier()
    for _ in range(warmup):
        pipe.step_all()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler(local) as clocks:
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            pipe.step_all()
        e1.record()
        torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    ms = _max_over_ranks(e0.elapsed_time(e1), dev) / steps
    pipe.drain()
    tok_s = G * B * 1000.0 / ms
    log(f"decode: {ms:.3f} ms/step -> {tok_s:.0f} tok/s")

    # ---- end to end: every step of every group, stage 0 copies the group's token ids host->device from pinned memory and the
    # sampled ids come back device->host (rank 0 holds the host side, as the reference's primary does)
    e2e_res = None
    if e2e:
        host = [torch.empty(B, dtype=torch.int64).pin_memory() for _ in range(G)]
        for g in range(G):
            host[g].copy_(pipe.tok[g].cpu() if rank == 0 else torch.zeros(B, dtype=torch.int64))
        pipe.steps_done = [0] * G

        def e2e_step():
            for g in range(G):
                if rank == 0:
                    if pipe.steps_done[g] > 0 and world > 1:
                        dist.recv(pipe.tok[g], world - 1)
                    if pipe.steps_done[g] > 0:
                        host[g].copy_(pipe.tok[g], non_blocking=True)       # D2H of the sampled ids
                        torch.cuda.current_stream().synchronize()
                    pipe.tok[g].copy_(host[g], non_blocking=True)           # H2D of this step's inputs
                    out = pipe.run_body(g)
                    if world > 1:
                        dist.send(out, 1)
                    pipe.steps_done[g] += 1
                else:
                    dist.recv(pipe.hid[g], rank - 1)
                    out = pipe.run_body(g)
                    dist.send(out, 0 if pipe.last else rank + 1)
                    pipe.steps_done[g] += 1

        for _ in range(warmup):
            e2e_step()
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        tt = time.perf_counter()
        for _ in range(steps):
            e2e_step()
        torch.cuda.synchronize()
        dt = _max_over_ranks(time.perf_counter() - tt, dev)
        if rank == 0 and world > 1:
            for g in range(G):
                dist.recv(pipe.tok[g], world - 1)
        e2e_res = {"value": round(G * B * steps / dt, 1), "unit": "tokens/s", "steps": steps, "ms_per_step": round(dt * 1e3 / steps, 4),
                   "h2d_bytes_per_step": G * B * 8, "d2h_bytes_per_step": G * B * 8,
                   "path": "BaselinePipeline: pinned H2D of token ids -> CUDA-graph stage step -> NCCL send/recv -> D2H of sampled ids"}
    if world > 1:
        dist.barrier()
    if rank != 0:
        return None
    return {
        "metric": "decode tokens/sec, DeepSeek-Coder-V2-Lite @N H100, + p50 TTFT",
        "value": round(tok_s, 1), "unit": "tokens/s", "n_gpus": world, "steps": steps, "warmup": warmup,
        "ms_per_step": round(ms, 4), "higher_is_better": True, "scaling": "weak", "vs_baseline": 1.0, "dtype": "bf16",
        "data": "synthetic prompts, random-init weights", "impl": "baseline",
        "config": {"model": "DeepSeek-Coder-V2-Lite-Instruct" if args.model == "deepseek-v2-lite" else args.model,
                   "global_batch": G * B, "seq_len": S, "parallelism": f"pp{world}", "micro_batches_in_flight": G,
                   "tokens_per_step": G * B, "transport": "nccl send/recv" if world > 1 else "local",
                   "cuda_graphs": pipe.use_graphs, "weights": "bf16",
                   "kernels": "cuBLAS (F.linear, torch.bmm padded expert batches), F.scaled_dot_product_attention, eager elementwise",
                   "l2": "weights streamed per step far exceed the 50 MB L2; no explicit flush",
                   "layers": "cost-balanced whole layers"},
        "ttft_p50_ms": round(ttft_p50 * 1e3, 3), "ttft_microbatch_ms": round(ttft_batch * 1e3, 2),
        "clocks": clocks.summary(), "gpu_launches": 0, "e2e": e2e_res,
    }
