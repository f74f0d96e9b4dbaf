"""Serving on top of expert parallelism: a lockstep group of data-parallel engines.

With ``enable_expert_parallel`` every rank runs the whole layer stack on *its own* sequences and the routed experts of every
MoE layer are exchanged between the ranks.  That exchange is a collective: every rank must execute the same number of model
forwards, in the same order, even when requests arrive unevenly (or not at all) at some ranks.  ``LockstepGroup`` provides
exactly that:

* rank 0 is the front end — it offers the ``LLMEngine`` surface (``submit / start / shutdown / stats``) to the HTTP server,
  assigns every new request to the least-loaded rank and broadcasts the assignments;
* every rank owns a ``LockstepEngine`` (its KV cache, its scheduler, continuous batching, chunked prefill).  Each iteration the
  ranks tell each other whether they have a step to run; if anybody has, *everybody* runs one forward — ranks without work run
  a one-token dummy step on a scratch page so the expert all-to-all stays aligned;
* token events flow back to rank 0 after every iteration and are pushed into the caller's ``Request`` object, so streaming,
  stop sequences, log-probs and cancellation behave exactly as with a local engine.

The control plane (assignments, need-flags, events) uses a gloo group with pickled Python objects: ONE small
``all_gather_object`` per iteration.  The data plane is whatever ``parallel/ep.py`` uses for the backend (fused NVLink kernels on
``b200``, ``all_to_all`` on the reference backend — which is how this module is tested on CPU, ``tests/test_ep_cpu.py``).

No reference counterpart: the reference serves one request at a time on one pipeline (shard/openai_api.py:552).
"""
from __future__ import annotations

import queue
import threading
import time
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from ..engine.core import LLMEngine, Request, StepInput
from ..engine.sampler import SamplingParams, check_penalty_table
from ..ops.meta import BatchMeta

_SCRATCH_SEQ = -1


class LockstepEngine(LLMEngine):
    """``LLMEngine`` (one group) whose forwards are aligned with the other ranks of the expert-parallel group."""

    def __init__(self, pipeline, num_pages: int, page_size: int = 64, ctrl_group=None, **kw):
        kw["num_groups"] = 1
        super().__init__(pipeline, num_pages, page_size, **kw)
        self.ctrl = ctrl_group
        self.table.add(_SCRATCH_SEQ)            # one page that the dummy steps write their single KV row into
        self.table.reserve(_SCRATCH_SEQ, 1)
        self.dummy_steps = 0

    def _dummy_input(self) -> StepInput:
        pages = [self.table.pages[_SCRATCH_SEQ]]
        meta = BatchMeta.build([1], [0], pages, self.page_size, pad_blocks_to=8)
        return StepInput(0, [_SCRATCH_SEQ], torch.zeros(1, dtype=torch.int64), meta, [SamplingParams(temperature=0.0)], [[]],
                         [True], False)

    def prepare(self):
        """Admit waiting requests and build my next step (``None`` if I have nothing to run)."""
        self._admit()
        return self._build_step(0)

    def run(self, built) -> None:
        """The group decided that a forward happens this iteration: run my step, or a dummy one to stay aligned."""
        if built is None:
            self.pipe.wait(self.pipe.submit(self._dummy_input()))   # keep the expert all-to-all aligned
            self.dummy_steps += 1
            return
        inp, seqs, q_lens = built
        out = self.pipe.wait(self.pipe.submit(inp))
        self.stats["steps"] += 1
        self._process(0, seqs, q_lens, inp, out)

    def step(self) -> bool:
        """Stand-alone lockstep iteration (one extra collective); ``LockstepGroup`` folds this exchange into its own."""
        built = self.prepare()
        need = [None] * dist.get_world_size(self.ctrl)
        dist.all_gather_object(need, built is not None, group=self.ctrl)
        if any(need):
            self.run(built)
        return any(need)


class _Proxy(Request):
    """Front-end handle of a request that executes on some rank of the group."""


class LockstepGroup:
    """See module docstring.  Construct on every rank (collective), then ``start()`` on rank 0 / ``serve_forever()`` elsewhere."""

    def __init__(self, engine: LockstepEngine, ctrl_group=None, idle_wait_s: float = 0.02):
        self.engine = engine
        self.ctrl = ctrl_group
        self.rank, self.world = dist.get_rank(ctrl_group), dist.get_world_size(ctrl_group)
        self.idle_wait_s = idle_wait_s
        self._pending: "queue.Queue[_Proxy]" = queue.Queue()   # rank 0: submitted, not yet assigned
        self._proxies: Dict[int, _Proxy] = {}                   # rank 0: gid -> front-end handle
        self._local: Dict[int, Request] = {}                    # every rank: gid -> request running in my engine
        self._load = [0] * self.world                           # rank 0: unfinished requests per rank
        self._thread: Optional[threading.Thread] = None
        self._stop = threading.Event()
        self._iterations = 0
        self._assigned = [0] * self.world
        self._next_msg: Optional[dict] = None                   # control message received in the previous exchange

    # -------------------------------------------------------------------------- LLMEngine surface (rank 0)
    @property
    def table(self):
        return self.engine.table

    @property
    def stats(self) -> dict:
        """Flat counters for ``/metrics``: this rank's engine counters + the group's."""
        d = dict(self.engine.stats, lockstep_iterations=self._iterations, lockstep_dummy_steps=self.engine.dummy_steps)
        d.update({f"lockstep_assigned_rank{r}": n for r, n in enumerate(self._assigned)})
        return d

    def metrics_snapshot(self):
        """(counters, free KV pages of this rank) — the ``/metrics`` surface shared with ``LLMEngine``."""
        return self.stats, self.engine.table.alloc.num_free

    def submit(self, prompt, params: Optional[SamplingParams] = None, max_tokens: int = 100, eos_token_id: Optional[int] = None,
               stop_id_sequences=None) -> Request:
        assert self.rank == 0, "requests enter the group on rank 0"
        params = params or SamplingParams()
        params.validate()
        check_penalty_table(params, max_tokens)
        if params.response_format is not None:
            raise ValueError("response_format is not available with --expert-parallel serving (its ranks have no tokenizer to "
                             "build token masks from)")
        if len(prompt) == 0:
            raise ValueError("empty prompt")
        if len(prompt) + max_tokens > self.engine.max_model_len:
            raise ValueError(f"prompt ({len(prompt)}) + max_tokens ({max_tokens}) exceeds max_model_len ({self.engine.max_model_len})")
        r = _Proxy(prompt, params, max_tokens, eos_token_id, stop_id_sequences)
        self._pending.put(r)
        return r

    def start(self):
        if self._thread is None:
            self._thread = threading.Thread(target=self.serve_forever, name="ep-lockstep", daemon=True)
            self._thread.start()
        return self

    def shutdown(self):
        """Rank 0: stop the whole group (the other ranks leave ``serve_forever``)."""
        self._stop.set()
        if self._thread is not None:
            self._thread.join(timeout=30)
            self._thread = None

    # -------------------------------------------------------------------------- the loop (every rank)
    def _plan(self) -> dict:
        """Rank 0: turn pending submissions / cancellations into this iteration's control message."""
        assign, cancel, batch = [], [], []
        if not any(self._load):
            # nothing running anywhere: block briefly for a submission instead of spinning the collectives
            try:
                batch.append(self._pending.get(timeout=self.idle_wait_s))
            except queue.Empty:
                pass
        while True:
            try:
                batch.append(self._pending.get_nowait())
            except queue.Empty:
                break
        for r in batch:
            dst = min(range(self.world), key=lambda i: self._load[i])
            self._load[dst] += 1
            self._assigned[dst] += 1
            self._proxies[r.id] = r
            assign.append(dict(rank=dst, gid=r.id, prompt=r.prompt, params=r.params, max_tokens=r.max_tokens, eos=r.eos_token_id,
                               stops=r.stop_id_sequences))
        for gid, r in self._proxies.items():
            if r.cancelled and not getattr(r, "_cancel_sent", False):
                r._cancel_sent = True
                cancel.append(gid)
        return dict(assign=assign, cancel=cancel, stop=self._stop.is_set())

    def _apply(self, msg: dict):
        for a in msg["assign"]:
            if a["rank"] == self.rank:
                self._local[a["gid"]] = self.engine.submit(a["prompt"], a["params"], a["max_tokens"], a["eos"], a["stops"])
        for gid in msg["cancel"]:
            if gid in self._local:
                self._local[gid].cancel()

    def _drain_events(self) -> List[tuple]:
        out = []
        for gid, r in list(self._local.items()):
            while True:
                try:
                    ev = r.events.get_nowait()
                except queue.Empty:
                    break
                if ev is None:   # engine-side failure
                    out.append((gid, None, repr(r.error)))
                    continue
                out.append((gid, ev, None))
            if r.finished:
                del self._local[gid]
        return out

    def _route(self, gathered: List[List[tuple]]):
        for src, events in enumerate(gathered):
            for gid, ev, err in events:
                p = self._proxies.get(gid)
                if p is None:
                    continue
                if ev is None:
                    p.error, p.finished = RuntimeError(f"rank {src}: {err}"), True
                    p.events.put(None)
                else:
                    if ev.token >= 0:
                        if p.t_first is None:
                            p.t_first = time.perf_counter()
                        p.output.append(ev.token)
                    if ev.finished:
                        p.finished, p.finish_reason, p.t_done = True, ev.finish_reason, time.perf_counter()
                    p.events.put(ev)
                if p.finished:
                    self._load[src] -= 1
                    del self._proxies[gid]

    def iterate(self) -> bool:
        """One group iteration = ONE control-plane collective (``all_gather_object``) + at most one forward per rank.

        Every rank contributes ``(I have a step, token events of my last forward, [rank 0] control message)``.  The control
        message (assignments / cancellations / stop) travels with the exchange of iteration *i* and is applied at the start
        of iteration *i + 1* on all ranks, so everybody applies it at the same point of the sequence."""
        msg, self._next_msg = self._next_msg, None
        if msg is not None:
            if msg["stop"]:
                return False
            self._apply(msg)
        try:
            built = self.engine.prepare()
        except BaseException as e:  # noqa: BLE001 — fail my requests, stay in the collective
            self.engine._fail_all(e)
            built = None
        item = (built is not None, self._drain_events(), self._plan() if self.rank == 0 else None)
        gathered = [None] * self.world
        dist.all_gather_object(gathered, item, group=self.ctrl)
        self._next_msg = gathered[0][2]
        if self.rank == 0:
            self._route([g[1] for g in gathered])
        if any(g[0] for g in gathered):
            try:
                self.engine.run(built)
            except BaseException as e:  # noqa: BLE001
                self.engine._fail_all(e)
        self._iterations += 1
        return True

    def serve_forever(self):
        while self.iterate():
            pass


def build_lockstep_group(model, num_pages: int, page_size: int = 64, max_seqs: int = 64, max_prefill_tokens: int = 2048,
                         ep_max_tokens: Optional[int] = None, prefix_cache: bool = False) -> LockstepGroup:
    """Collective helper: expert-parallel ``model`` (loaded with ``expert_shard``) -> a started-able ``LockstepGroup``."""
    from .ep import enable_expert_parallel
    from .pipeline import LocalPipeline, StageExecutor

    ctrl = dist.new_group(backend="gloo")                       # control plane: pickled objects, CPU
    bound = ep_max_tokens or max(max_prefill_tokens, max_seqs)
    enable_expert_parallel(model, max_tokens=bound)
    for layer in model.ep_layers.values():
        layer.peer_tokens_default = bound                       # ranks run different batch sizes: size temporaries for the bound
    pipe = LocalPipeline([StageExecutor(model, num_pages, page_size)])
    if pipe.gcache is not None:
        # No CUDA-graph replay in the lockstep group: a rank *capturing* a decode graph launches nothing for real while its peers
        # execute the same iteration eagerly and wait for its expert dispatch — the ranks' batches (hence their capture points)
        # differ, so captures cannot be aligned without making every rank capture every other rank's bucket.  The graph-resident
        # expert-parallel loop is the symmetric one (parallel/decode_loop.py: bench.py --parallelism ep, generate.py --expert_parallel).
        pipe.gcache.enabled = False
    engine = LockstepEngine(pipe, num_pages, page_size, ctrl_group=ctrl,
                            max_seqs_per_group=max_seqs, max_prefill_tokens=max_prefill_tokens, prefix_cache=prefix_cache)
    return LockstepGroup(engine, ctrl)
