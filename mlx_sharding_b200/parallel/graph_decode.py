"""Step blocks + the CUDA-graph cache for *engine-driven* decode steps (the public serving path).

``decode_loop.py`` is the fully device-resident loop of the benchmark's device-timed phase.  The serving engine
(``LLMEngine`` -> ``LocalPipeline`` / ``FusedChainPipeline``) owns scheduling on the host — sequences join and leave, so the
step metadata comes from the host every step — but the *device work* of a decode step is the same kernel sequence every time
for a given (group, batch size, block-table width, context bucket, sampling variant).  This module

* defines the **step block** (``StepLayout``): ONE int32 vector that carries everything a stage needs for a step — a 16-byte
  step tag, the sampling block (per-sequence temperature / top-p / RNG state and, when any request uses them, repetition-penalty
  contexts, bias tables — logit_bias folded with presence / frequency penalties — top-k / min-p filters and the token masks of
  structured-output requests), the packed ``BatchMeta`` and the token ids.  Stage 0 builds it once per step; every stage
  copies it host->device with one pinned ``cudaMemcpyAsync``; in a multi-GPU pipeline it travels through the shared-memory
  launch ring (``shm_ring.py``);
* defines the **result message** (``ResultLayout``): tag + sampled ids + their log-probs (+ top-k) in one buffer the last stage
  sends back to stage 0 (the reference ships full ``[1, T, V]`` logits instead, server/server.py:36-48);
* captures the kernel sequence once per key into a CUDA graph with static buffers.  Because *sampling parameters live in the
  step block* (device memory) — temperatures, nucleus thresholds, the per-request (seed, step) RNG state, penalties — sampled
  requests (the reference's default ``temperature=1.0``, shard/openai_api.py:209) replay the same graph as greedy ones:

      host step = one pinned H2D copy (step block) -> one graph replay -> one D2H of the result message

The reference has no equivalent (``mx.async_eval`` one-token look-ahead, shard/utils.py:180-186).
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ..engine.sampler import bias_table
from ..ops.meta import BatchMeta


def _ctx_bucket(n: int) -> int:
    b = 512
    while b < n:
        b *= 2
    return b


def _pow2_at_least(n: int, lo: int) -> int:
    b = lo
    while b < n:
        b *= 2
    return b


# ------------------------------------------------------------------------------------------------- layouts
class StepLayout:
    """int32 word offsets of a step block for ``T`` tokens of ``B`` sequences.

    ``C`` / ``NB`` > 0: the block carries repetition-penalty contexts ``[B, C]`` and additive bias tables ``[B, NB]`` (logit_bias
    merged with the presence / frequency penalties; only when a request of the batch uses them); ``F`` = 1: it carries the
    top-k / min-p filter section ``keep_k`` int32 ``[B]`` + ``min_p`` f32 ``[B]`` (only when a request of the batch filters its
    draw); ``W`` > 0: it carries the token-mask section ``allow`` int32 ``[B, W]``, ``W = ceil(V/32)`` (only when a request of
    the batch has a ``response_format``); ``k`` = number of top log-probs the sampler returns (0 or 10)."""

    __slots__ = ("T", "B", "mb", "C", "NB", "k", "F", "W", "tag", "temps", "top_p", "rng", "penalty", "rep", "bidx", "bval",
                 "keep_k", "min_p", "allow", "meta", "tokens", "size")

    def __init__(self, T: int, B: int, mb: int, C: int = 0, NB: int = 0, k: int = 0, F: int = 0, W: int = 0):
        self.T, self.B, self.mb, self.C, self.NB, self.k, self.F, self.W = T, B, mb, C, NB, k, F, W
        o = 0
        self.tag = o; o += 4                       # [seq_lo, seq_hi, k, flags] — 16 bytes, copied into the result message
        self.temps = o; o += B
        self.top_p = o; o += B
        o = (o + 1) // 2 * 2
        self.rng = o; o += 4 * B                   # int64 [B, 2] = (seed, tokens sampled so far) per sequence
        self.penalty = self.rep = self.bidx = self.bval = self.keep_k = self.min_p = self.allow = -1
        if C or NB:
            self.penalty = o; o += B
            self.rep = o; o += B * C
            self.bidx = o; o += B * NB
            self.bval = o; o += B * NB
        if F:
            self.keep_k = o; o += B
            self.min_p = o; o += B
        if W:
            o = (o + 3) // 4 * 4               # 16-byte aligned
            self.allow = o; o += B * W
        o = (o + 3) // 4 * 4
        self.meta = o; o += BatchMeta.packed_size(T, B, mb)
        o = (o + 1) // 2 * 2
        self.tokens = o; o += 2 * T                # int64 [T] (used by the first stage only)
        self.size = (o + 3) // 4 * 4

    @property
    def key(self) -> Tuple[int, int, int, int, int, int, int, int]:
        return (self.T, self.B, self.mb, self.C, self.NB, self.k, self.W, self.F)

    @property
    def flags(self) -> int:
        """Header word 7: bit 0 = filter section present, bits 1-31 = ``W`` of the token-mask section (0 = absent)."""
        return self.F | (self.W << 1)


HEADER_WORDS = 8      # prepended to the block on the wire: T, B, mb, C, NB, k, is_prefill, flags (``StepLayout.flags``)


class ResultLayout:
    """Byte offsets of the result message of ``B`` sequences with ``k`` top log-probs."""

    __slots__ = ("B", "k", "tokens", "logprobs", "top_ids", "top_lp", "nbytes")

    def __init__(self, B: int, k: int):
        self.B, self.k = B, k
        o = 16                                       # tag
        self.tokens = o; o += 8 * B
        self.logprobs = o; o += 4 * B
        o = (o + 7) // 8 * 8
        self.top_ids = o; o += 8 * B * k
        self.top_lp = o; o += 4 * B * k
        self.nbytes = (o + 15) // 16 * 16

    @staticmethod
    def max_bytes(max_seqs: int, k: int = 10) -> int:
        return ResultLayout(max_seqs, k).nbytes

    def views(self, buf: torch.Tensor):
        """(tag int32[4], tokens int64[B], logprobs f32[B], top_ids int64[B,k] | None, top_lp f32[B,k] | None) into a uint8 buffer."""
        B, k = self.B, self.k
        tag = buf[:16].view(torch.int32)
        toks = buf[self.tokens:self.tokens + 8 * B].view(torch.int64)
        lp = buf[self.logprobs:self.logprobs + 4 * B].view(torch.float32)
        if not k:
            return tag, toks, lp, None, None
        ti = buf[self.top_ids:self.top_ids + 8 * B * k].view(torch.int64).view(B, k)
        tl = buf[self.top_lp:self.top_lp + 4 * B * k].view(torch.float32).view(B, k)
        return tag, toks, lp, ti, tl


def sampling_variant(params, counts=None) -> Tuple[int, int, int]:
    """(C, NB, k) table sizes a batch needs: 0/0 when no request uses a repetition penalty, logit bias or (once it has generated
    a token) a presence / frequency penalty.  ``counts[b]``: the ``OutputCounts`` of requests with such a penalty."""
    C = NB = k = 0
    for b, p in enumerate(params):
        if p.repetition_penalty not in (0, 1.0) and p.repetition_context_size > 0:
            C = max(C, int(p.repetition_context_size))
        nb = len(p.logit_bias) if p.logit_bias else 0
        if counts is not None and counts[b]:
            nb += len(counts[b])        # upper bound of the merged table (entries for the same id are folded into one)
        NB = max(NB, nb)
        if p.logprobs:
            k = 10
    if C or NB:
        C, NB = _pow2_at_least(max(C, 1), 32), _pow2_at_least(max(NB, 1), 16)
    return C, NB, k


def decode_bucket(B: int) -> int:
    """Batch sizes of captured decode graphs: 1, 2, 4, 8, then multiples of 8 up to 64, then multiples of 16."""
    if B <= 8:
        return _pow2_at_least(B, 1)
    return (B + 7) // 8 * 8 if B <= 64 else (B + 15) // 16 * 16


def _pad_decode(meta: BatchMeta, tokens: torch.Tensor, params, contexts, rng, counts, allow, Bp: int):
    """Pad a pure-decode step to ``Bp`` sequences with dummy rows that read / write the reserved null page (page 0, position 0)."""
    B, n = meta.num_seqs, Bp - meta.num_seqs
    z = lambda k: torch.zeros(k, dtype=torch.int32)
    mb = meta.block_tables.shape[1]
    meta = BatchMeta(torch.cat([meta.positions, z(n)]), torch.cat([meta.slot_mapping, z(n)]), torch.arange(Bp + 1, dtype=torch.int32),
                     torch.cat([meta.context_lens, torch.ones(n, dtype=torch.int32)]),
                     torch.cat([meta.block_tables, torch.zeros(n, mb, dtype=torch.int32)]), torch.arange(Bp, dtype=torch.int32),
                     Bp, Bp, 1, meta.max_ctx_len, meta.page_size)
    tokens = torch.cat([tokens, torch.zeros(n, dtype=tokens.dtype)])
    params = list(params) + [_PAD_PARAMS] * n
    contexts = (list(contexts) + [[]] * n) if contexts is not None else None
    rng = (list(rng) + [(0, 0)] * n) if rng is not None else None
    counts = (list(counts) + [None] * n) if counts is not None else None
    if allow is not None:   # dummy rows may draw anything
        allow = np.concatenate([allow, np.full((n, allow.shape[1]), -1, dtype=np.int32)])
    return meta, tokens, params, contexts, rng, counts, allow


_PAD_PARAMS = None


def pack_step(seq: int, meta: BatchMeta, tokens: torch.Tensor, params, contexts, rng, is_prefill: bool,
              pad_decode: bool = False, counts=None, allow: Optional[np.ndarray] = None) -> Tuple[np.ndarray, StepLayout]:
    """Host side (stage 0): one int32 vector ``[header | step block]`` for this step.  ``rng[b]`` = (seed, sampled so far);
    ``counts[b]`` = ``OutputCounts`` of a request with a presence / frequency penalty (else ``None``), folded with
    its ``logit_bias`` into one bias entry per token id; ``allow`` = token masks int32 ``[B, ceil(V/32)]`` of a batch with a
    structured-output request (rows of the other requests all ones), else ``None``.

    ``pad_decode``: a pure decode step is padded to the next batch-size bucket (``decode_bucket``) with dummy rows on the null
    page, so that continuous batching — sequences joining and leaving every few steps — keeps replaying a handful of captured
    graphs instead of capturing one per distinct batch size (the caller drops the dummy rows of the result)."""
    global _PAD_PARAMS
    if pad_decode and meta.max_q_len == 1 and meta.num_tokens == meta.num_seqs:
        Bp = decode_bucket(meta.num_seqs)
        if Bp != meta.num_seqs:
            if _PAD_PARAMS is None:
                from ..engine.sampler import SamplingParams

                _PAD_PARAMS = SamplingParams()
            meta, tokens, params, contexts, rng, counts, allow = _pad_decode(meta, tokens, params, contexts, rng, counts, allow, Bp)
    T, B = meta.num_tokens, meta.num_seqs
    mb = meta.block_tables.shape[1]
    C, NB, k = sampling_variant(params, counts)
    F = int(any(p.uses_filter for p in params))
    W = 0 if allow is None else int(allow.shape[1])
    lay = StepLayout(T, B, mb, C, NB, k, F, W)
    buf = np.zeros(HEADER_WORDS + lay.size, dtype=np.int32)
    buf[:HEADER_WORDS] = (T, B, mb, C, NB, k, int(is_prefill), lay.flags)
    blk = buf[HEADER_WORDS:]
    blk[lay.tag] = seq & 0x7FFFFFFF
    blk[lay.tag + 1] = (seq >> 31) & 0x7FFFFFFF
    blk[lay.tag + 2] = k
    f32 = blk.view(np.float32)
    f32[lay.temps:lay.temps + B] = [p.temperature for p in params]
    f32[lay.top_p:lay.top_p + B] = [p.top_p for p in params]
    r64 = blk[lay.rng:lay.rng + 4 * B].view(np.int64)
    r64[:] = np.asarray(rng, dtype=np.int64).reshape(-1) if rng is not None else 0
    if C or NB:
        pen = f32[lay.penalty:lay.penalty + B]
        pen[:] = 1.0
        rep = blk[lay.rep:lay.rep + B * C].reshape(B, C)
        rep[:] = -1
        bidx = blk[lay.bidx:lay.bidx + B * NB].reshape(B, NB)
        bidx[:] = -1
        bval = f32[lay.bval:lay.bval + B * NB].reshape(B, NB)
        for b, p in enumerate(params):
            if p.repetition_penalty not in (0, 1.0) and p.repetition_context_size > 0 and contexts is not None:
                c = contexts[b][-min(p.repetition_context_size, C):]
                if c:
                    rep[b, :len(c)] = c
                pen[b] = p.repetition_penalty
            ids, vals = bias_table(p, counts[b] if counts is not None else None)
            bidx[b, :len(ids)] = ids
            bval[b, :len(ids)] = vals
    if F:
        blk[lay.keep_k:lay.keep_k + B] = [max(p.top_k, 0) if p.uses_filter else 0 for p in params]
        f32[lay.min_p:lay.min_p + B] = [p.min_p if p.uses_filter else 0.0 for p in params]
    if W:
        blk[lay.allow:lay.allow + B * W].reshape(B, W)[:] = allow
    blk[lay.meta:lay.meta + BatchMeta.packed_size(T, B, mb)] = meta.pack().numpy()
    blk[lay.tokens:lay.tokens + 2 * T].view(np.int64)[:] = tokens.numpy()
    return buf, lay


def unpack_header(buf: np.ndarray) -> Tuple[StepLayout, bool]:
    T, B, mb, C, NB, k, pre, flags = (int(v) for v in buf[:HEADER_WORDS])
    return StepLayout(T, B, mb, C, NB, k, flags & 1, flags >> 1), bool(pre)


class StepViews:
    """Typed views into a step block that lives in one int32 tensor (host or device)."""

    def __init__(self, flat: torch.Tensor, lay: StepLayout, page_size: int, max_ctx: int, max_q: int = 1):
        B, T, mb = lay.B, lay.T, lay.mb
        f32 = flat.view(torch.float32)
        self.flat, self.lay = flat, lay
        self.tag = flat[lay.tag:lay.tag + 4]
        self.temps = f32[lay.temps:lay.temps + B]
        self.top_p = f32[lay.top_p:lay.top_p + B]
        self.rng = flat[lay.rng:lay.rng + 4 * B].view(torch.int64)
        self.has_pen = bool(lay.C or lay.NB)
        if self.has_pen:
            self.penalty = f32[lay.penalty:lay.penalty + B]
            self.rep = flat[lay.rep:lay.rep + B * lay.C].view(B, lay.C)
            self.bidx = flat[lay.bidx:lay.bidx + B * lay.NB].view(B, lay.NB)
            self.bval = f32[lay.bval:lay.bval + B * lay.NB].view(B, lay.NB)
        self.has_filter = bool(lay.F)
        self.keep_k = flat[lay.keep_k:lay.keep_k + B] if lay.F else None
        self.min_p = f32[lay.min_p:lay.min_p + B] if lay.F else None
        self.allow = flat[lay.allow:lay.allow + B * lay.W].view(B, lay.W) if lay.W else None
        o = lay.meta + 6
        take = lambda n: (flat[o:o + n], o + n)
        pos, o = take(T)
        slots, o = take(T)
        cu, o = take(B + 1)
        ctx, o = take(B)
        last_idx, o = take(B)
        bt, o = take(B * mb)
        self.meta = BatchMeta(pos, slots, cu, ctx, bt.view(B, mb), last_idx, T, B, max_q, max_ctx, page_size)
        self.tokens = flat[lay.tokens:lay.tokens + 2 * T].view(torch.int64)


def device_sample(ops, logits: torch.Tensor, sv: StepViews, res: torch.Tensor, rl: ResultLayout):
    """Last stage: penalties + sampling from the step block, results written straight into the result message ``res``."""
    tag, toks, lp, ti, tl = rl.views(res)
    if hasattr(ops, "sample_block"):
        ops.sample_block(logits, sv, tag, toks, lp, ti, tl)
        return
    raise NotImplementedError(f"backend {getattr(ops, 'NAME', ops)} has no sample_block")


def parse_result(host: torch.Tensor, rl: ResultLayout, expect_seq: Optional[int] = None):
    """Host side: result message (uint8 tensor) -> ``(tokens, logprobs, top_ids, top_logprobs)`` python lists."""
    tag, toks, lp, ti, tl = rl.views(host)
    if expect_seq is not None:
        t = tag.tolist()
        got = t[0] | (t[1] << 31)
        if got != expect_seq:
            raise RuntimeError(f"pipeline result out of order: expected step {expect_seq}, got {got}")
    return toks.tolist(), lp.tolist(), None if ti is None else ti.tolist(), None if tl is None else tl.tolist()


# ------------------------------------------------------------------------------------------------- graph cache
class _Entry:
    def __init__(self, stage, lay: StepLayout, ctx_bucket: int, group: int):
        dev = stage.device
        self.lay, self.group = lay, group
        self.flat = torch.zeros(lay.size, dtype=torch.int32, device=dev)
        self.sv = StepViews(self.flat, lay, stage.kv.page_size, ctx_bucket)
        self.meta = self.sv.meta
        spec = stage.model.spec
        H = stage.model.cfg.hidden_size
        # input of the stage: token ids (a view of the step block) on the first stage; a static hidden buffer otherwise (pipelines
        # with a resident inbox read the inbox instead and never touch ``x``)
        self.x = self.sv.tokens if spec.is_first else torch.zeros(lay.B, H, dtype=stage.model.dtype, device=dev)
        self.rl = ResultLayout(lay.B, lay.k)
        self.res = torch.zeros(self.rl.nbytes, dtype=torch.uint8, device=dev) if spec.is_last else None
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.out = None       # hidden [B, H] (non-last) or the result message (last)
        self.uses = 0
        self.launches = 0     # kernels in the captured body


class DecodeGraphCache:
    """Per-stage cache of captured decode graphs keyed by (group, B, block-table width, context bucket, sampling variant).

    ``body(entry) -> output`` is the device work of one step; the default runs the stage on ``entry.x`` and samples on the last
    stage.  Pipelines with a fused hand-off pass their own body (flag wait -> layers with the boundary armed -> result send)."""

    WARM_USES = 2   # run eagerly this many times before paying for a capture

    def __init__(self, stage, body: Optional[Callable] = None, per_group: bool = False):
        self.stage = stage
        self.entries: Dict[tuple, _Entry] = {}
        self.enabled = stage.device.type == "cuda" and stage.model.backend_name == "b200"
        self.body = body or self._default_body
        self.per_group = per_group
        self.replays = 0
        self.captures = 0

    def eligible(self, meta: BatchMeta, params=None) -> bool:
        """Pure decode micro-batches replay a graph — whatever their sampling parameters (they live in the step block)."""
        return self.enabled and meta.max_q_len == 1 and meta.num_tokens == meta.num_seqs

    def entry(self, lay: StepLayout, max_ctx: int, group: int = 0) -> _Entry:
        key = (group if self.per_group else 0, lay.key, _ctx_bucket(max_ctx))
        e = self.entries.get(key)
        if e is None:
            e = _Entry(self.stage, lay, key[2], group)
            self.entries[key] = e
            if len(self.entries) > 48:  # bound memory: drop the least used graph
                k = min((k for k in self.entries if k != key), key=lambda k: self.entries[k].uses)
                del self.entries[k]
        return e

    def _default_body(self, e: _Entry):
        st = self.stage
        out = st.model.forward(e.x, e.meta, st.kv)
        if st.model.spec.is_last:
            device_sample(st.model.ops, out, e.sv, e.res, e.rl)
            return e.res
        return out

    @torch.inference_mode()
    def run(self, e: _Entry):
        """The step block is already in ``e.flat``.  Returns the static output tensor."""
        e.uses += 1
        if e.graph is None:
            if e.uses <= self.WARM_USES:
                return self.body(e)       # eager (also warms allocator / scratch before capture)
            from ..ops import b200 as _b

            g = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            n0 = _b.C().launch_count()
            with torch.cuda.graph(g):
                e.out = self.body(e)
            e.launches = _b.C().launch_count() - n0
            e.graph = g
            self.captures += 1
        e.graph.replay()
        self.replays += 1
        return e.out
