"""Generation engine: request queue, sequence slots, micro-batch scheduler, stop logic.

Reference: the per-token relay loop ``create_generate_step_with_grpc`` (shard/utils.py:111-188) and
``generate.generate_step`` (generate.py:52-88) — strictly one sequence at a time, one global cache,
sequential stage execution.  This engine keeps ``num_groups`` micro-batches in flight (one per
pipeline stage) so every stage stays busy (SURVEY §2.4 "micro-batching", BASELINE config 3), supports
many concurrent requests (continuous batching at group granularity) and chunked prefill.

The engine talks to a *pipeline* object (``parallel/pipeline.py``) through two calls:
``submit(StepInput) -> handle`` and ``wait(handle) -> StepOutput``; how stages are connected
(in-process, gloo, NCCL, fused P2P, gRPC) is invisible here.
"""
from __future__ import annotations

import itertools
import queue
import threading
import time
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from ..ops.meta import BatchMeta
from .kv_cache import PageAllocator, PrefixCache, SequenceTable
from .sampler import OutputCounts, SamplingParams, check_penalty_table


# ---------------------------------------------------------------------------------------------
@dataclass
class StepInput:
    """One micro-batch step, built on stage 0 and executed by every stage."""

    group: int
    seq_ids: List[int]
    tokens: torch.Tensor            # int64 [T] (host)
    meta: BatchMeta                 # host-side tensors
    params: List[SamplingParams]
    contexts: List[List[int]]       # repetition-penalty context per sequence
    sample_mask: List[bool]         # False for non-final prefill chunks
    is_prefill: bool
    rng: Optional[List[tuple]] = None   # per sequence: (seed, tokens sampled so far) — the sampler's random stream of that request
    # per sequence: output token counts of requests with a presence / frequency penalty (else None); None when no
    # request of the engine uses one
    counts: Optional[List[Optional[OutputCounts]]] = None
    # token masks int32 [B, ceil(V/32)] when a sampled row of this step belongs to a request with a response_format (the other
    # rows all ones), else None
    allow: Optional[np.ndarray] = None


@dataclass
class StepOutput:
    tokens: List[int]
    logprobs: List[float]
    top_ids: Optional[List[List[int]]] = None
    top_logprobs: Optional[List[List[float]]] = None


@dataclass(slots=True)
class TokenEvent:
    token: int
    logprob: float
    top: Optional[Dict[int, float]]
    finished: bool
    finish_reason: Optional[str]


class Request:
    _ids = itertools.count()

    def __init__(self, prompt: Sequence[int], params: SamplingParams, max_tokens: int,
                 eos_token_id: Optional[int] = None, stop_id_sequences: Optional[List[List[int]]] = None):
        self.id = next(Request._ids)
        self.prompt = [int(t) for t in prompt]
        self.params = params
        self.max_tokens = int(max_tokens)
        self.eos_token_id = eos_token_id
        self.stop_id_sequences = stop_id_sequences or []
        self.output: List[int] = []
        # times each token id occurs in ``output``: kept only for the presence / frequency penalties
        self.counts: Optional[OutputCounts] = OutputCounts() if params.uses_output_penalty else None
        self.matcher = None           # grammar matcher of a request with a response_format (engine/grammar.py)
        self.events: "queue.SimpleQueue[TokenEvent]" = queue.SimpleQueue()   # C implementation: one put per generated token
        self.finished = False
        self.finish_reason: Optional[str] = None
        self.error: Optional[BaseException] = None
        self.cancelled = False
        self.t_submit = time.perf_counter()
        self.t_first: Optional[float] = None
        self.t_done: Optional[float] = None
        # random stream of this request: its own seed if given, else derived from the request id (reproducible per request,
        # independent of the batch it decodes in)
        self.seed = (int(params.seed) if params.seed is not None else (0x9E3779B1 * (self.id + 1))) & 0x7FFFFFFFFFFFFFFF
        self.prefilled = 0            # prompt tokens already in the KV cache
        self.cached_pages = 0         # leading pages of this request that are registered in the prefix cache

    def cancel(self):
        self.cancelled = True

    def __iter__(self):
        """Blocking iterator over ``TokenEvent``s (the generator the reference's handlers consume)."""
        while True:
            ev = self.events.get()
            if ev is None:
                if self.error is not None:
                    raise self.error
                return
            yield ev
            if ev.finished:
                return

    @property
    def ttft(self) -> Optional[float]:
        return None if self.t_first is None else self.t_first - self.t_submit


def stopping_criteria(tokens: List[int], stop_id_sequences: List[List[int]], eos_token_id: Optional[int]):
    """Reference ``stopping_criteria`` (shard/openai_api.py:30-43): returns (stop_met, trim_length)."""
    if tokens and tokens[-1] == eos_token_id:
        return True, 1
    for stop_ids in stop_id_sequences:
        if len(stop_ids) and len(tokens) >= len(stop_ids) and tokens[-len(stop_ids):] == list(stop_ids):
            return True, len(stop_ids)
    return False, 0


# ---------------------------------------------------------------------------------------------
class LLMEngine:
    def __init__(self, pipeline, num_pages: int, page_size: int = 64, num_groups: Optional[int] = None,
                 max_seqs_per_group: int = 64, max_prefill_tokens: int = 2048, max_model_len: int = 32768,
                 prefix_cache: bool = False, mixed_batches: bool = False):
        self.pipe = pipeline
        self.page_size = page_size
        self.num_groups = num_groups or max(1, getattr(pipeline, "num_stages", 1))
        self.max_seqs = max_seqs_per_group
        self.max_prefill_tokens = max_prefill_tokens
        self.max_model_len = max_model_len
        # mixed_batches: a prefill step also carries the next decode token of every running sequence of the group (one ragged
        # batch), so streams in flight keep their inter-token latency while new prompts are being prefilled
        self.mixed_batches = mixed_batches
        self.table = SequenceTable(PageAllocator(num_pages), page_size)
        # automatic prefix caching (engine/kv_cache.py::PrefixCache): full prompt pages are shared between requests
        self.table.prefix = PrefixCache(self.table.alloc, page_size) if prefix_cache else None
        self.waiting: "queue.Queue[Request]" = queue.Queue()
        self.groups: List[List[Request]] = [[] for _ in range(self.num_groups)]
        self.inflight: List[Optional[tuple]] = [None] * self.num_groups
        self._lock = threading.Lock()
        self._thread: Optional[threading.Thread] = None
        self._stop = threading.Event()
        self._wake = threading.Event()
        self.stats = dict(steps=0, prefill_tokens=0, decode_tokens=0, finished=0, prefix_cached_tokens=0)
        self.sinks: list = []      # event sinks of the API worker processes (server/frontend.py): flushed once per scheduler iteration
        self._penalised = 0        # running requests with a presence / frequency penalty (their steps carry output counts)
        # structured output (engine/grammar.py::GrammarBackend, set by the server next to the tokenizer); None = response_format
        # is refused
        self.grammar = None
        self._constrained = 0      # running requests with a response_format (their steps carry token masks)

    # -------------------------------------------------------------------------- public API
    def submit(self, prompt: Sequence[int], params: Optional[SamplingParams] = None, max_tokens: int = 100,
               eos_token_id: Optional[int] = None, stop_id_sequences=None, events=None) -> Request:
        """``events``: optional replacement of the request's event queue (anything with ``put``) — the multi-process API front end
        (server/frontend.py) passes a per-worker sink so a step's tokens leave the engine process as one message."""
        params = params or SamplingParams()
        params.validate()
        check_penalty_table(params, max_tokens)
        if len(prompt) == 0:
            raise ValueError("empty prompt")
        if len(prompt) + max_tokens > self.max_model_len:
            raise ValueError(f"prompt ({len(prompt)}) + max_tokens ({max_tokens}) exceeds max_model_len "
                             f"({self.max_model_len})")
        matcher = None
        if params.response_format is not None:
            if self.grammar is None:
                raise ValueError("response_format is not available on this server (structured output needs the xgrammar "
                                 "package and a tokenizer on the engine)")
            matcher = self.grammar.matcher(params.response_format)   # ValueError: the schema does not compile
        r = Request(prompt, params, max_tokens, eos_token_id, stop_id_sequences)
        r.matcher = matcher
        if events is not None:
            r.events = events
            events.req = r
        if r.max_tokens <= 0:
            # the reference's ``zip(generate_step(...), range(max_tokens))`` yields nothing (openai_api.py:370-381): no forward pass
            r.finished, r.finish_reason = True, "length"
            r.t_done = time.perf_counter()
            r.events.put(None)
            return r
        self.waiting.put(r)
        self._wake.set()
        return r

    def generate(self, prompt, params=None, max_tokens=100, **kw) -> List[int]:
        """Synchronous helper: run one request to completion (drives the loop inline if no thread)."""
        r = self.submit(prompt, params, max_tokens, **kw)
        if self._thread is None:
            while not r.finished:
                self.step()
        else:
            for _ in r:
                pass
        if r.error:
            raise r.error
        return r.output

    def start(self):
        if self._thread is None:
            self._stop.clear()
            self._thread = threading.Thread(target=self._loop, name="engine-loop", daemon=True)
            self._thread.start()
        return self

    def shutdown(self):
        """Stop the loop and fail every request that is still queued or running, so no caller stays blocked in
        ``for ev in request`` (the reference has no such path: its handlers own the generation loop, openai_api.py:370-381)."""
        self._stop.set()
        self._wake.set()
        if self._thread is not None:
            self._thread.join(timeout=10)
            self._thread = None
        err = RuntimeError("engine shut down")
        while True:
            try:
                r = self.waiting.get_nowait()
            except queue.Empty:
                break
            r.error, r.finished = err, True
            r.events.put(None)
        if any(self.groups) or any(h is not None for h in self.inflight):
            self._fail_all(err)
        for s in self.sinks:
            s.flush()

    def busy(self) -> bool:
        return self.has_work()

    # -------------------------------------------------------------------------- scheduling
    def has_work(self) -> bool:
        return (not self.waiting.empty()) or any(self.groups) or any(h is not None for h in self.inflight)

    def _loop(self):
        while not self._stop.is_set():
            if not self.has_work():
                self._wake.wait(timeout=0.05)
                self._wake.clear()
                continue
            try:
                self.step()
            except BaseException as e:  # fail every active request, keep serving
                self._fail_all(e)

    def _fail_all(self, e: BaseException):
        # first let the pipeline drain every step that is still in flight (other groups' steps keep writing KV on the downstream
        # stages until they complete) and drop their results — only then may the pages go back to the allocator
        for g in range(self.num_groups):
            self.inflight[g] = None
        try:
            self.pipe.reset()
        except Exception:
            pass
        for g in range(self.num_groups):
            for r in self.groups[g]:
                r.error, r.finished = e, True
                self.table.release(r.id)
                r.events.put(None)
            self.groups[g] = []
        self._penalised = 0
        self._constrained = 0
        for s in self.sinks:
            s.flush()

    def _admit(self):
        while True:
            g = min(range(self.num_groups), key=lambda i: len(self.groups[i]))
            if len(self.groups[g]) >= self.max_seqs:
                return
            try:
                r = self.waiting.get_nowait()
            except queue.Empty:
                return
            cache = self.table.prefix
            shared = cache.match(r.prompt) if cache is not None else []
            need = (len(r.prompt) + r.max_tokens + self.page_size - 1) // self.page_size - len(shared)
            if need > self.table.alloc.num_free:
                if shared:
                    cache.release(shared)   # give the references back; the request is retried later
                if not any(self.groups):
                    r.error = MemoryError("request does not fit in the KV pool")
                    r.finished = True
                    r.events.put(None)
                    continue
                # put it back and wait for running sequences to finish
                self.waiting.queue.appendleft(r)
                return
            self.table.add(r.id)
            if shared:
                # the matched prefix is already in the KV pool (on every stage): start the prefill behind it
                n = len(shared) * self.page_size
                self.table.pages[r.id] = list(shared)
                self.table.length[r.id] = n
                r.prefilled = n
                r.cached_pages = len(shared)
                self.stats["prefix_cached_tokens"] += n
            self.table.reserve(r.id, len(r.prompt) - r.prefilled + r.max_tokens)
            self.groups[g].append(r)
            if r.counts is not None:
                self._penalised += 1
            if r.matcher is not None:
                self._constrained += 1

    def _build_step(self, g: int) -> Optional[StepInput]:
        reqs = [r for r in self.groups[g] if not r.finished]
        if not reqs:
            return None
        pre = [r for r in reqs if r.prefilled < len(r.prompt)]
        seqs, q_lens, ctx0, toks, mask = [], [], [], [], []
        if pre:
            budget = self.max_prefill_tokens
            for r in pre:
                if budget <= 0:
                    break
                n = min(len(r.prompt) - r.prefilled, budget)
                seqs.append(r)
                q_lens.append(n)
                ctx0.append(r.prefilled)
                toks.extend(r.prompt[r.prefilled:r.prefilled + n])
                mask.append(r.prefilled + n == len(r.prompt))
                budget -= n
            if self.mixed_batches:
                for r in reqs:
                    if r.prefilled >= len(r.prompt) and r.output:
                        seqs.append(r)
                        q_lens.append(1)
                        ctx0.append(self.table.length[r.id])
                        toks.append(r.output[-1])
                        mask.append(True)
            is_prefill = True
        else:
            # pure decode step (the hot host path: runs once per generated token of the whole group)
            length = self.table.length
            seqs = reqs
            q_lens = [1] * len(reqs)
            ctx0 = [length[r.id] for r in reqs]
            toks = [r.output[-1] for r in reqs]
            mask = [True] * len(reqs)
            is_prefill = False
        bts = [self.table.pages[r.id] for r in seqs]
        # block-table width rounded up to a multiple of 8 so captured decode graphs (graph_decode.py) are reused
        width = (max(len(p) for p in bts) + 7) // 8 * 8
        meta = BatchMeta.build(q_lens, ctx0, bts, self.page_size, pad_blocks_to=width)
        ctxs = [(r.prompt + r.output)[-max(1, r.params.repetition_context_size):]
                if r.params.repetition_penalty not in (0, 1.0) else [] for r in seqs]
        counts = [r.counts for r in seqs] if self._penalised else None
        allow = self._token_masks(seqs, mask) if self._constrained else None
        return StepInput(g, [r.id for r in seqs], torch.tensor(toks, dtype=torch.int64), meta,
                         [r.params for r in seqs], ctxs, mask, is_prefill, [(r.seed, len(r.output)) for r in seqs],
                         counts, allow), seqs, q_lens

    def _token_masks(self, seqs: List[Request], mask: List[bool]) -> Optional[np.ndarray]:
        """Token masks of a step: the grammar's next-token masks of the constrained requests that sample in it (one batched
        fill), all ones for every other row; ``None`` when no constrained request samples."""
        rows = [b for b, r in enumerate(seqs) if mask[b] and r.matcher is not None]
        if not rows:
            return None
        allow = np.full((len(seqs), self.grammar.words), -1, dtype=np.int32)
        self.grammar.fill([seqs[b].matcher for b in rows], allow, rows)
        return allow

    def _accept_tokens(self, seqs: List[Request], inp: StepInput, out: StepOutput) -> Dict[int, bool]:
        """Feed the sampled tokens of the constrained requests to their matchers (one batched call): row -> accepted."""
        rows = [b for b, r in enumerate(seqs) if r.matcher is not None and inp.sample_mask[b] and not r.cancelled]
        if not rows:
            return {}
        return dict(zip(rows, self.grammar.accept([seqs[b].matcher for b in rows], [int(out.tokens[b]) for b in rows])))

    def _finish(self, r: Request, reason: str):
        r.finished, r.finish_reason = True, reason
        r.t_done = time.perf_counter()
        self.table.release(r.id)
        self.stats["finished"] += 1
        if r.counts is not None:
            self._penalised -= 1
        if r.matcher is not None:
            self._constrained -= 1

    def _fail(self, r: Request, e: BaseException):
        """Fail one running request (its handler raises ``e``: HTTP 500 or an SSE error); the rest of the batch carries on."""
        self._finish(r, "error")
        r.error = e
        r.events.put(None)

    def _process(self, g: int, seqs: List[Request], q_lens: List[int], inp: StepInput, out: StepOutput):
        length, n_decode = self.table.length, 0
        fits = self._accept_tokens(seqs, inp, out) if self._constrained else None
        for b, r in enumerate(seqs):
            if inp.is_prefill and r.prefilled < len(r.prompt):
                r.prefilled += q_lens[b]
                self.stats["prefill_tokens"] += q_lens[b]
            else:
                n_decode += 1
            length[r.id] += q_lens[b]                      # == self.table.advance(r.id, q_lens[b])
            if inp.is_prefill and self.table.prefix is not None and r.cached_pages * self.page_size < len(r.prompt):
                r.cached_pages = self.table.prefix.insert(r.prompt, self.table.pages[r.id], r.prefilled, r.cached_pages)
            if r.cancelled and not r.finished:
                self._finish(r, "cancelled")
                r.events.put(TokenEvent(-1, 0.0, None, True, "cancelled"))
                continue
            if not inp.sample_mask[b]:
                continue
            tok = int(out.tokens[b])
            if r.matcher is not None and not fits[b]:
                # the sampler draws only allowed ids, so this is a row without any allowed id of finite logit: the token never
                # reaches the client
                self._fail(r, RuntimeError(f"sampled token {tok} does not fit the request's response_format"))
                continue
            if r.t_first is None:
                r.t_first = time.perf_counter()
            r.output.append(tok)
            if r.counts is not None:
                r.counts.add(tok)
            top = None
            if r.params.logprobs > 0 and out.top_ids is not None:
                k = r.params.logprobs
                top = {int(i): float(l) for i, l in zip(out.top_ids[b][:k], out.top_logprobs[b][:k])}
            # (inlined fast path of stopping_criteria for the common no-stop-sequence case)
            stop = tok == r.eos_token_id if not r.stop_id_sequences else stopping_criteria(r.output, r.stop_id_sequences, r.eos_token_id)[0]
            reason = "stop" if stop else ("length" if len(r.output) >= r.max_tokens else None)
            if reason:
                self._finish(r, reason)
            r.events.put(TokenEvent(tok, float(out.logprobs[b]), top, reason is not None, reason))
        self.stats["decode_tokens"] += n_decode
        self.groups[g] = [r for r in self.groups[g] if not r.finished]

    def step(self):
        """One scheduler iteration: for every group collect its in-flight step (if any), then launch
        the next one.  With ``num_groups == num_stages`` all stages have work at all times."""
        self._admit()
        progressed = False
        for g in range(self.num_groups):
            if self.inflight[g] is not None:
                handle, inp, seqs, q_lens = self.inflight[g]
                out = self.pipe.wait(handle)
                self.inflight[g] = None
                self._process(g, seqs, q_lens, inp, out)
                progressed = True
            built = self._build_step(g)
            if built is not None:
                inp, seqs, q_lens = built
                self.inflight[g] = (self.pipe.submit(inp), inp, seqs, q_lens)
                self.stats["steps"] += 1
                progressed = True
        for s in self.sinks:
            s.flush()
        return progressed

    def metrics_snapshot(self):
        """(engine counters, free KV pages) — what ``/metrics`` reports; also served to API worker processes."""
        return dict(self.stats), self.table.alloc.num_free

    def drain(self):
        while self.has_work():
            self.step()
