"""Per-request sampling parameters + the batched sampler front-end.

Reference: the ``sample()`` closure and repetition-penalty bookkeeping inside
``create_generate_step_with_grpc`` (shard/utils.py:126-139,152-177):
logit_bias add -> repetition penalty over the last ``repetition_context_size`` tokens ->
``logprobs = logits - logsumexp`` -> argmax | nucleus | categorical.

In this engine sampling runs on the *last* stage, on device, for the whole micro-batch at once; only
token ids (+ optional top-k logprobs, k <= 10) travel back to stage 0 (SURVEY X3).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch


@dataclass
class SamplingParams:
    temperature: float = 0.0
    top_p: float = 1.0
    repetition_penalty: float = 1.0
    repetition_context_size: int = 20
    logit_bias: Optional[Dict[int, float]] = None
    logprobs: int = 0               # number of top logprobs to return (0 = none, <= 10)
    seed: Optional[int] = None
    # filters of the temperature draw, in the order top-k -> top-p -> min-p (temperature 0 stays argmax and ignores them)
    top_k: int = 0                  # keep logits >= the k-th largest (ties kept); 0 or -1 = off
    min_p: float = 0.0              # keep p >= min_p * p_max at the request's temperature; 0 = off
    # OpenAI penalties over the tokens this request has generated (prompt excluded):
    # logit[j] -= frequency_penalty * count[j] + presence_penalty * (count[j] > 0)
    presence_penalty: float = 0.0
    frequency_penalty: float = 0.0
    # structured output: canonical JSON text of the request's OpenAI ``response_format`` (``engine/grammar.py::canonical_format``);
    # None = unconstrained
    response_format: Optional[str] = None

    def validate(self):
        if self.temperature < 0:
            raise ValueError("temperature must be a non-negative float")
        if not (0 <= self.top_p <= 1):
            raise ValueError("top_p must be a float between 0 and 1")
        if self.repetition_penalty < 0:
            raise ValueError("repetition_penalty must be a non-negative float")
        if self.repetition_context_size < 0:
            raise ValueError("repetition_context_size must be a non-negative integer")
        if not (0 <= self.logprobs <= 10):
            raise ValueError("logprobs must be between 1 and 10")
        if not isinstance(self.top_k, int) or isinstance(self.top_k, bool) or self.top_k < -1:
            raise ValueError("top_k must be an integer >= -1 (0 or -1 disables it)")
        if not (0 <= self.min_p <= 1):
            raise ValueError("min_p must be a float between 0 and 1")
        if not (-2 <= self.presence_penalty <= 2):
            raise ValueError("presence_penalty must be a float between -2 and 2")
        if not (-2 <= self.frequency_penalty <= 2):
            raise ValueError("frequency_penalty must be a float between -2 and 2")
        if self.response_format is not None:
            from .grammar import check_format_text

            check_format_text(self.response_format)

    @property
    def uses_filter(self) -> bool:
        """True when top-k or min-p narrows this request's draw (greedy requests ignore both)."""
        return self.temperature > 0 and (self.top_k > 0 or self.min_p > 0)

    @property
    def uses_output_penalty(self) -> bool:
        return self.presence_penalty != 0 or self.frequency_penalty != 0


# Largest additive bias table of a request with a presence / frequency penalty: its logit_bias entries plus one entry per distinct
# generated token, bounded by len(logit_bias) + max_tokens.  Requests that could exceed it are refused at submission, so a step
# block always fits the multi-process control ring (``parallel/pipeline.py::control_slot_bytes``).
MAX_PENALTY_TABLE = 1024


def check_penalty_table(p: SamplingParams, max_tokens: int):
    """Refuse a penalised request whose bias table could outgrow ``MAX_PENALTY_TABLE``."""
    if p.uses_output_penalty and len(p.logit_bias or {}) + max_tokens > MAX_PENALTY_TABLE:
        raise ValueError(f"with presence_penalty or frequency_penalty, max_tokens plus the number of logit_bias entries must be "
                         f"at most {MAX_PENALTY_TABLE}")


class OutputCounts:
    """How often each token id occurs in a request's output, kept as growing arrays (first-seen order) so that folding them
    into the bias table is a vectorised expression instead of a Python loop over every distinct token."""

    __slots__ = ("pos", "ids", "cnt", "n")

    def __init__(self):
        self.pos: Dict[int, int] = {}              # token id -> index into ids / cnt
        self.ids = np.empty(64, np.int64)
        self.cnt = np.empty(64, np.float64)
        self.n = 0

    @classmethod
    def of(cls, tokens) -> "OutputCounts":
        c = cls()
        for t in tokens:
            c.add(int(t))
        return c

    def add(self, tok: int):
        i = self.pos.get(tok)
        if i is None:
            if self.n == len(self.ids):
                self.ids = np.concatenate([self.ids, np.empty_like(self.ids)])
                self.cnt = np.concatenate([self.cnt, np.empty_like(self.cnt)])
            i = self.pos[tok] = self.n
            self.ids[i], self.cnt[i] = tok, 0.0
            self.n += 1
        self.cnt[i] += 1.0

    def __len__(self) -> int:
        return self.n


def folded_bias(p: SamplingParams, counts: OutputCounts) -> Tuple[np.ndarray, np.ndarray]:
    """``logit_bias`` merged with the presence / frequency penalty of ``counts``, as ``(ids int32 [n], values float32 [n])``
    with one additive entry per token id, so the device's bias add does not depend on the order in which entries for the same
    id would land."""
    ids = counts.ids[:counts.n]
    f, pr = float(p.frequency_penalty), float(p.presence_penalty)
    vals = 0.0 - (f * counts.cnt[:counts.n] + pr)
    extra_ids, extra_vals = [], []
    for t, v in {int(t): float(v) for t, v in (p.logit_bias or {}).items()}.items():
        i = counts.pos.get(t)
        if i is not None:
            vals[i] = v - (f * counts.cnt[i] + pr)
        else:
            extra_ids.append(t)
            extra_vals.append(v)
    if extra_ids:
        ids, vals = np.concatenate([ids, extra_ids]), np.concatenate([vals, extra_vals])
    return ids.astype(np.int32), vals.astype(np.float32)


def bias_table(p: SamplingParams, counts: Optional[OutputCounts]) -> Tuple[np.ndarray, np.ndarray]:
    """One row of the device's additive bias table: ``folded_bias`` once a penalised request has generated tokens, else its
    ``logit_bias`` entries as given."""
    if counts and p.uses_output_penalty:
        return folded_bias(p, counts)
    lb = p.logit_bias or {}
    return (np.fromiter((int(t) for t in lb), np.int32, len(lb)),
            np.fromiter((float(v) for v in lb.values()), np.float64, len(lb)).astype(np.float32))


@dataclass
class SampleOutput:
    tokens: torch.Tensor                      # int64 [B]
    logprobs: torch.Tensor                    # fp32 [B] logprob of the chosen token
    top_ids: Optional[torch.Tensor] = None    # int64 [B, k]
    top_logprobs: Optional[torch.Tensor] = None


class Sampler:
    """Batched sampler; ``ops`` is the backend module (reference or b200)."""

    MAX_CTX = 64    # static width of the repetition-context / bias tables on device
    MAX_BIAS = 64

    def __init__(self, ops, device="cpu", seed: int = 0):
        self.ops = ops
        self.device = torch.device(device)
        self.gen = torch.Generator(device=self.device)
        self.gen.manual_seed(seed)

    def __call__(self, logits: torch.Tensor, params: List[SamplingParams],
                 contexts: Optional[List[List[int]]] = None,
                 counts: Optional[List[Optional[OutputCounts]]] = None, allow=None) -> SampleOutput:
        """``logits`` fp32 ``[B, V]``; ``contexts[b]`` = recent token ids for the repetition penalty; ``counts[b]`` = how often
        each token id has been generated by that request (presence / frequency penalties); ``allow`` = token masks int32
        ``[B, ceil(V/32)]`` of structured-output requests (rows of the others all ones), or ``None``."""
        B = logits.shape[0]
        assert len(params) == B
        logits = logits.float()
        counts = counts if counts is not None else [None] * B
        need_pen = any((p.repetition_penalty not in (0, 1.0) and p.repetition_context_size > 0) or p.logit_bias
                       or (counts[b] and p.uses_output_penalty) for b, p in enumerate(params))
        if need_pen:
            logits = logits.clone()
            C = max(1, min(self.MAX_CTX, max(p.repetition_context_size for p in params)))
            ctx = torch.full((B, C), -1, dtype=torch.int32)
            pen = torch.ones(B, dtype=torch.float32)
            biases = [bias_table(p, counts[b]) for b, p in enumerate(params)]
            nb = max(1, max(len(ids) for ids, _ in biases))
            bidx = torch.full((B, nb), -1, dtype=torch.int32)
            bval = torch.zeros(B, nb, dtype=torch.float32)
            for b, p in enumerate(params):
                if p.repetition_penalty not in (0, 1.0) and contexts is not None and p.repetition_context_size > 0:
                    c = contexts[b][-min(p.repetition_context_size, C):]
                    if c:
                        ctx[b, : len(c)] = torch.tensor(c, dtype=torch.int32)
                    pen[b] = p.repetition_penalty
                ids, vals = biases[b]
                bidx[b, :len(ids)] = torch.from_numpy(ids)
                bval[b, :len(ids)] = torch.from_numpy(vals)
            self.ops.apply_penalties_(logits, ctx.to(self.device), pen.to(self.device),
                                      bidx.to(self.device), bval.to(self.device))
        temps = torch.tensor([p.temperature for p in params], dtype=torch.float32, device=self.device)
        top_p = torch.tensor([p.top_p for p in params], dtype=torch.float32, device=self.device)
        k = max(p.logprobs for p in params)
        filt = {}
        if any(p.uses_filter for p in params):
            filt = dict(top_k=torch.tensor([max(p.top_k, 0) for p in params], dtype=torch.int32, device=self.device),
                        min_p=torch.tensor([p.min_p for p in params], dtype=torch.float32, device=self.device))
        if allow is not None:
            filt["allow"] = torch.as_tensor(allow, dtype=torch.int32).to(self.device)
        toks, lp, ti, tl = self.ops.sample(logits, temps, top_p, generator=self.gen, top_logprobs=k, **filt)
        return SampleOutput(toks, lp, ti, tl)
