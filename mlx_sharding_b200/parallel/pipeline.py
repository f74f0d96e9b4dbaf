"""Pipeline runtimes: how one scheduler step (``StepInput``) travels through the stages.

* ``LocalPipeline``  – all stages in this process (1 GPU, or CPU tests).
* ``ChainPipeline``  – **direct chain** ``stage i -> i+1`` across processes; the last stage samples on device and only a small
  result message (token ids + log-probs) returns to stage 0.  Replaces the reference's hub-and-spoke relay that bounces every
  hidden state through the primary and ships full ``[1,T,V]`` logits back (shard/utils.py:162-166, server/server.py:36-48;
  SURVEY X1-X3).
* ``worker_loop``    – what a non-first stage process runs.

A step is described by ONE int32 **step block** (``graph_decode.pack_step``: step tag, sampling block, packed metadata, token
ids) that stage 0 builds and every stage copies host->device from pinned memory.  How the block reaches the other stages is the
*control plane*; how hidden states and results move is the *data plane*:

=================  ==========================================================================================================
control plane      ``ShmControl`` (default, one node): launch ring in shared memory — publishing a step is a memcpy, picking
                   it up is a poll; no pickle, no gloo, no system call per step.  ``DistControl``: gloo broadcast fallback for
                   ranks that do not share a host.
data plane         ``FusedPlane`` (CUDA, default): resident inboxes mapped over CUDA IPC; the *last kernel of a stage* (down-proj
                   GEMM epilogue / MoE combine) stores its rows straight into the next stage's inbox over NVLink and bumps its
                   flag; the consumer's step starts with a flag-wait kernel.  A decode step of a group is ONE CUDA-graph replay
                   per stage: no NCCL call, no host hop, no control message on the hand-off.  ``DistPlane``: ``send/recv`` over
                   gloo (CPU plumbing, BASELINE config 1) or NCCL (baseline transport).
=================  ==========================================================================================================

Failure handling (reference: ``success=False`` strings, server/server.py:55-57): a stage that fails a step records the error on
the control plane's status page and still forwards a placeholder, so every stage keeps executing the same launch sequence
(lock-step is what keeps the flag protocol deadlock-free); stage 0 raises on the next ``wait``; ``reset()`` drains every step
that is still in flight *before* the engine releases KV pages; results carry their step id and are checked on receipt.
"""
from __future__ import annotations

import logging
import os
from collections import deque
from typing import List, Optional

import numpy as np
import torch

from ..engine.core import StepInput, StepOutput
from ..engine.kv_cache import PagedKVCache
from ..engine.sampler import MAX_PENALTY_TABLE, Sampler
from ..ops.meta import BatchMeta
from .graph_decode import (HEADER_WORDS, DecodeGraphCache, ResultLayout, StepViews, device_sample, pack_step, parse_result,
                           unpack_header)
from .shm_ring import KIND_SHUTDOWN, KIND_STEP

log = logging.getLogger(__name__)


class StageExecutor:
    """A stage model + its paged KV pool (+ the host-parameter sampler used by the gRPC-compat relay)."""

    def __init__(self, model, num_pages: int, page_size: int = 64, seed: int = 0):
        self.model = model
        self.device = model.device
        self.kv = PagedKVCache.for_model(model, num_pages, page_size)
        self.sampler = Sampler(model.ops, self.device, seed) if model.spec.is_last else None
        from ..utils.tracing import StageTimer

        self.timer = StageTimer(enabled=os.environ.get("MLXB200_STAGE_TIMING", "0") == "1")

    @torch.inference_mode()
    def forward(self, x: torch.Tensor, meta: BatchMeta, all_logits: bool = False) -> torch.Tensor:
        from ..utils.tracing import nvtx_range

        with self.timer.measure(), nvtx_range(f"stage[{self.model.spec.start_layer},{self.model.spec.end_layer}) T={meta.num_tokens}"):
            return self.model.forward(x, meta, self.kv, all_logits)

    @torch.inference_mode()
    def sample(self, logits: torch.Tensor, inp_params, contexts) -> StepOutput:
        so = self.sampler(logits, inp_params, contexts)
        return StepOutput(so.tokens.tolist(), so.logprobs.tolist(),
                          None if so.top_ids is None else so.top_ids.tolist(),
                          None if so.top_logprobs is None else so.top_logprobs.tolist())


# -------------------------------------------------------------------------------------------------
# One stage, one step
# -------------------------------------------------------------------------------------------------
class StepRunner:
    """Executes step blocks on one stage: pinned H2D of the block, then the device work — a CUDA-graph replay for decode
    micro-batches, eager kernels for prefill chunks / mixed batches — with the data plane's hand-off hooks around the layers."""

    def __init__(self, stage: StageExecutor, plane=None):
        self.stage, self.plane = stage, plane
        self.model = stage.model
        self.dev = stage.device
        self.cuda = self.dev.type == "cuda"
        self.first, self.last = self.model.spec.is_first, self.model.spec.is_last
        capturable = plane is None or plane.capturable
        self.gcache = DecodeGraphCache(stage, body=self._graph_body, per_group=plane is not None)
        if not capturable:
            self.gcache.enabled = False
        self.h2d_bytes = 0
        self._phase = 0          # 0: nothing done for the current step, 1: input consumed, 2: output handed on
        self._x_local = None     # input hidden of an in-process (LocalPipeline) non-first stage

    # ---- host -> device ------------------------------------------------------------------------
    def _h2d(self, dst: torch.Tensor, blk: np.ndarray):
        src = torch.from_numpy(blk)
        if self.cuda:
            dst.copy_(src.pin_memory(), non_blocking=True)
            self.h2d_bytes += blk.nbytes
        else:
            dst.copy_(src)

    # ---- device work of one step ---------------------------------------------------------------
    def _graph_body(self, e):
        return self._device_step(e.sv, e.group, e.res, e.rl, e.x)

    def _device_step(self, sv: StepViews, g: int, res, rl: ResultLayout, x_static=None):
        model, plane, T = self.model, self.plane, sv.lay.T
        if self.first:
            x = sv.tokens
        elif plane is not None:
            x = plane.begin(g, T, out=None if plane.capturable else x_static)
        else:
            x = self._x_local
        self._phase = 1
        if plane is not None and not self.last:
            plane.arm(model, g, T)
        out = model.forward(x, sv.meta, self.stage.kv)
        if self.last:
            device_sample(model.ops, out, sv, res, rl)
            if plane is not None:
                plane.send_result(res, g)
            self._phase = 2
            return res
        if plane is not None:
            plane.finish(model, out, g)
        self._phase = 2
        return out

    @torch.inference_mode()
    def run(self, wire: np.ndarray, group: int, x_local: Optional[torch.Tensor] = None):
        """``wire`` = ``[header | step block]`` (int32).  Returns the stage output: hidden ``[T, H]`` or, on the last stage, the
        result message (device uint8 tensor)."""
        lay, _ = unpack_header(wire)
        blk = wire[HEADER_WORDS:HEADER_WORDS + lay.size]
        mq, mctx = int(blk[lay.meta + 2]), int(blk[lay.meta + 3])
        self._phase, self._x_local = 0, x_local
        with self.stage.timer.measure():
            if self.gcache.enabled and mq == 1 and lay.T == lay.B and x_local is None:
                e = self.gcache.entry(lay, mctx, group)
                self._h2d(e.flat, blk)
                return self.gcache.run(e)
            flat = torch.empty(lay.size, dtype=torch.int32, device=self.dev)
            self._h2d(flat, blk)
            sv = StepViews(flat, lay, self.stage.kv.page_size, mctx, mq)
            # host-side hint for the models (the block is still in host memory here): every sequence of this step starts at position
            # 0, i.e. context length == query length — prefill of fresh prompts can skip gathering cached context
            o = lay.meta + 6 + 2 * lay.T
            cu, ctx = blk[o:o + lay.B + 1], blk[o + lay.B + 1:o + 2 * lay.B + 1]
            sv.meta.fresh = bool(lay.B > 0 and np.array_equal(ctx, cu[1:] - cu[:-1]))
            rl = ResultLayout(lay.B, lay.k)
            res = torch.zeros(rl.nbytes, dtype=torch.uint8, device=self.dev) if self.last else None
            return self._device_step(sv, group, res, rl)

    def poison(self, wire: np.ndarray, group: int):
        """After a failed step: consume the input and forward a placeholder so the chain stays in lock-step."""
        if self.plane is None:
            return
        lay, _ = unpack_header(wire)
        try:
            if self._phase < 1 and not self.first:
                self.plane.begin(group, lay.T)
            if self._phase < 2:
                self.model.boundary = None
                if self.last:
                    self.plane.send_result(torch.zeros(ResultLayout(lay.B, lay.k).nbytes, dtype=torch.uint8, device=self.dev), group)
                else:
                    self.plane.send_hidden(torch.zeros(lay.T, self.model.cfg.hidden_size, dtype=self.model.dtype, device=self.dev), group)
        except Exception:  # noqa: BLE001 — nothing more can be done; the status page already carries the first error
            log.exception("could not forward a placeholder after a failed step")


def _fetch(res: torch.Tensor) -> torch.Tensor:
    """Result message device -> host (pinned when on CUDA)."""
    if res.device.type != "cuda":
        return res
    host = torch.empty(res.shape, dtype=res.dtype).pin_memory()
    host.copy_(res, non_blocking=True)
    torch.cuda.current_stream(res.device).synchronize()
    return host


def _step_output(parsed, n_real: int) -> StepOutput:
    """Result lists -> ``StepOutput`` of the ``n_real`` real sequences (decode steps may carry padding rows, see ``pack_step``)."""
    toks, lp, ti, tl = parsed
    if len(toks) != n_real:
        toks, lp = toks[:n_real], lp[:n_real]
        ti, tl = (None if ti is None else ti[:n_real]), (None if tl is None else tl[:n_real])
    return StepOutput(toks, lp, ti, tl)


class LocalPipeline:
    """All stages in-process, executed back to back."""

    def __init__(self, stages: List[StageExecutor]):
        assert stages[0].model.spec.is_first and stages[-1].model.spec.is_last
        self.stages = stages
        self.runners = [StepRunner(s) for s in stages]
        self.num_stages = 1  # one executor thread: a single micro-batch group keeps it busy
        self.d2h_bytes = 0
        self._seq = 0
        self.gcache = self.runners[0].gcache if len(stages) == 1 else None

    @property
    def h2d_bytes(self) -> int:
        return sum(r.h2d_bytes for r in self.runners)

    @classmethod
    def from_models(cls, models, num_pages: int, page_size: int = 64, seed: int = 0):
        return cls([StageExecutor(m, num_pages, page_size, seed) for m in models])

    def submit(self, inp: StepInput) -> StepOutput:
        self._seq += 1
        wire, lay = pack_step(self._seq, inp.meta, inp.tokens, inp.params, inp.contexts, inp.rng, inp.is_prefill,
                              pad_decode=self.gcache is not None and self.gcache.enabled, counts=inp.counts, allow=inp.allow)
        x = None
        for r in self.runners:
            x = r.run(wire, inp.group, x_local=None if x is None else x.to(r.dev))
        rl = ResultLayout(lay.B, lay.k)
        host = _fetch(x)
        self.d2h_bytes += rl.nbytes
        return _step_output(parse_result(host, rl, self._seq), inp.meta.num_seqs)

    def wait(self, handle) -> StepOutput:
        return handle

    def reset(self):
        pass


# -------------------------------------------------------------------------------------------------
# Data planes
# -------------------------------------------------------------------------------------------------
class _Pending:
    """A result message on its way to stage 0."""

    def __init__(self, host: torch.Tensor, event=None, work=None, dev_buf=None):
        self.host, self.event, self.work, self.dev_buf = host, event, work, dev_buf

    def done(self) -> bool:
        if self.event is not None:
            return self.event.query()
        return self.work.is_completed()

    def get(self) -> torch.Tensor:
        if self.event is not None:
            self.event.synchronize()
        else:
            self.work.wait()
            if self.dev_buf is not None:
                self.host.copy_(self.dev_buf)
        return self.host


class FusedPlane:
    """T0: resident inboxes + flags over CUDA IPC (``p2p_fused.py``); every operation is a stream-ordered kernel, so a whole stage
    step — flag wait, layers, epilogue store into the peer, flag bump — is capturable in one CUDA graph."""

    capturable = True
    name = "fused"

    def __init__(self, stage: StageExecutor, num_groups: int, max_tokens: int, max_seqs: int, group=None):
        from .p2p_fused import FusedP2PBoundary

        self.p2p = FusedP2PBoundary(stage.model.cfg.hidden_size, num_groups, max_tokens, max_seqs, group=group,
                                    dtype=stage.model.dtype, result_bytes=ResultLayout.max_bytes(max_seqs))
        self.max_tokens = max_tokens
        self.dev = stage.device
        self.side = torch.cuda.Stream(device=self.dev) if self.p2p.rank == 0 else None
        self.d2h_bytes = 0

    def begin(self, g: int, T: int, out=None) -> torch.Tensor:
        if T > self.max_tokens:
            raise ValueError(f"step of {T} tokens exceeds the hand-off inbox ({self.max_tokens} tokens)")
        self.p2p.wait_hidden(g)
        return self.p2p.hidden_inbox(g, T)

    def arm(self, model, g: int, T: int):
        if T > self.max_tokens:
            raise ValueError(f"step of {T} tokens exceeds the hand-off inbox ({self.max_tokens} tokens)")
        model.boundary = (self.p2p.next_hidden(g, T), self.p2p.next_hidden_flag(g))

    def finish(self, model, out: torch.Tensor, g: int):
        fused = model.boundary_fused
        model.boundary = None
        if not fused:   # the stage's last kernel has no fused epilogue (Gemma-2 ends in a norm): copy + signal
            self.p2p.send_hidden(out, g)

    def send_hidden(self, x: torch.Tensor, g: int):
        self.p2p.send_hidden(x, g)

    def send_result(self, res: torch.Tensor, g: int):
        self.p2p.send_result(res, g)

    def recv_result(self, g: int, nbytes: int) -> _Pending:
        """Stage 0: flag wait + D2H of the result inbox on a side stream (the main stream never blocks on a flag)."""
        host = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
        with torch.cuda.stream(self.side):
            self.p2p.C.pdl_skip_next()
            self.p2p.wait_result(g)
            host.copy_(self.p2p.result_inbox(g, nbytes), non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.side)
        self.d2h_bytes += nbytes
        return _Pending(host, event=ev)

    def failed(self) -> bool:
        return self.p2p.error()


class DistPlane:
    """T1 / T2: two-sided ``send/recv`` through ``TorchDistTransport`` (gloo on CPU, NCCL on GPUs)."""

    name = "dist"

    def __init__(self, stage: StageExecutor, transport):
        self.tp = transport
        self.rank, self.world = transport.rank, transport.world_size
        self.H, self.dtype, self.dev = stage.model.cfg.hidden_size, stage.model.dtype, stage.device
        self.capturable = False
        self.d2h_bytes = 0

    def begin(self, g: int, T: int, out=None) -> torch.Tensor:
        return self.tp.recv_tensor((T, self.H), self.dtype, self.rank - 1, slot=g)

    def arm(self, model, g: int, T: int):
        pass

    def finish(self, model, out: torch.Tensor, g: int):
        self.tp.send_tensor(out, self.rank + 1, slot=g)

    def send_hidden(self, x: torch.Tensor, g: int):
        self.tp.send_tensor(x, self.rank + 1, slot=g)

    def send_result(self, res: torch.Tensor, g: int):
        self.tp.send_tensor(res.clone(), 0, slot=g)

    def recv_result(self, g: int, nbytes: int) -> _Pending:
        import torch.distributed as dist

        host = torch.empty(nbytes, dtype=torch.uint8)
        if self.tp.data_backend == "gloo":
            return _Pending(host, work=dist.irecv(host, self.world - 1, group=self.tp.data_group))
        buf = torch.empty(nbytes, dtype=torch.uint8, device=self.dev)
        self.d2h_bytes += nbytes
        return _Pending(host, work=dist.irecv(buf, self.world - 1, group=self.tp.data_group), dev_buf=buf)

    def failed(self) -> bool:
        return False


# -------------------------------------------------------------------------------------------------
# Control plane fallback (ranks on different hosts)
# -------------------------------------------------------------------------------------------------
class DistControl:
    """``ShmControl``'s interface over a gloo broadcast + the rendezvous store (for ranks that do not share ``/dev/shm``)."""

    def __init__(self, group=None):
        import torch.distributed as dist

        self.dist, self.group = dist, group
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self.store = dist.distributed_c10d._get_default_store()
        self._seq = 0
        self.max_payload_words = 1 << 26

    def publish(self, kind: int, group: int, payload: Optional[np.ndarray] = None, timeout_s: float = 60.0) -> int:
        self._seq += 1
        n = 0 if payload is None else int(payload.size)
        self.dist.broadcast(torch.tensor([self._seq, kind, group, n], dtype=torch.int64), 0, group=self.group)
        if n:
            self.dist.broadcast(torch.from_numpy(np.ascontiguousarray(payload)), 0, group=self.group)
        return self._seq

    def next(self, timeout_s: Optional[float] = None):
        hdr = torch.zeros(4, dtype=torch.int64)
        self.dist.broadcast(hdr, 0, group=self.group)
        seq, kind, group, n = hdr.tolist()
        payload = torch.zeros(n, dtype=torch.int32)
        if n:
            self.dist.broadcast(payload, 0, group=self.group)
        return seq, kind, group, payload.numpy()

    def set_error(self, seq: int, msg: str):
        self.store.set(f"mlxb200/err/{self.rank}", f"{seq}:{msg}")
        self.store.add("mlxb200/nerr", 1)

    def first_error(self):
        if self.store.add("mlxb200/nerr", 0) == 0:
            return None
        for r in range(self.world):
            if self.store.check([f"mlxb200/err/{r}"]):
                seq, _, msg = self.store.get(f"mlxb200/err/{r}").decode().partition(":")
                return r, int(seq or 0), msg
        return None

    def clear_errors(self):
        n = self.store.add("mlxb200/nerr", 0)
        if n:
            self.store.add("mlxb200/nerr", -n)
            for r in range(self.world):
                self.store.delete_key(f"mlxb200/err/{r}")

    def request_shutdown(self):
        pass

    def unlink(self):
        pass


def control_slot_bytes(max_tokens: int, max_seqs: int, vocab_size: int = 0) -> int:
    """Bytes of a control-ring slot: it holds the largest step block — a prefill chunk of ``max_tokens`` tokens (+ block tables
    of ``max_seqs`` sequences) — plus the sampling tables of ``max_seqs`` rows at their largest: a 32-token repetition context,
    a bias table of ``MAX_PENALTY_TABLE`` entries (penalised requests are refused beyond it), the top-k / min-p section and a
    token mask of ``ceil(vocab_size / 32)`` words (structured output).  The ring file is sparse, so slot bytes a step does not
    write take no memory."""
    base = max(256 << 10, 16 * max_tokens + 1024 * max_seqs + 4096)
    sampling = 4 * max_seqs * (1 + 32 + 2 * MAX_PENALTY_TABLE + 2) + 4 * max_seqs * ((vocab_size + 31) // 32) + 16
    return (base + sampling + 4095) // 4096 * 4096


def build_chain(stage: StageExecutor, num_groups: Optional[int] = None, max_tokens: int = 2048, max_seqs: int = 64,
                transport: str = "auto", control: str = "auto"):
    """Collective over all ranks: set up the control plane and the data plane of a chain.  Returns ``(ctl, plane)``.

    transport: ``fused`` (native kernels + CUDA IPC inboxes), ``nccl`` / ``gloo`` (two-sided), ``auto`` = fused on CUDA with the
    b200 backend when every rank is on this host, else nccl on CUDA, gloo on CPU.
    control: ``shm`` / ``dist`` / ``auto`` (shm when every rank is on this host)."""
    import socket

    import torch.distributed as dist

    from .shm_ring import ShmControl

    rank, world = dist.get_rank(), dist.get_world_size()
    G = num_groups or world
    ctrl_group = dist.new_group(backend="gloo")
    hosts = [None] * world
    dist.all_gather_object(hosts, socket.gethostname(), group=ctrl_group)
    one_node = len(set(hosts)) == 1
    if control == "auto":
        control = "shm" if one_node else "dist"
    if control == "shm":
        box = [None]
        ctl = None
        if rank == 0:
            ctl = ShmControl.create(world, slots=128, slot_bytes=control_slot_bytes(max_tokens, max_seqs, stage.model.cfg.vocab_size))
            box[0] = ctl.path
        dist.broadcast_object_list(box, 0, group=ctrl_group)
        if rank != 0:
            ctl = ShmControl.attach(box[0], rank, world)
        dist.barrier(group=ctrl_group)
        if rank == 0:
            ctl.unlink()          # every rank holds a mapping now; nothing is left behind if a process dies
    else:
        ctl = DistControl(ctrl_group)
    cuda = stage.device.type == "cuda"
    if transport == "auto":
        transport = "fused" if (cuda and one_node and stage.model.backend_name == "b200") else ("nccl" if cuda else "gloo")
    if transport == "fused":
        plane = FusedPlane(stage, G, max_tokens, max_seqs, group=ctrl_group)
    else:
        from .transport import TorchDistTransport

        plane = DistPlane(stage, TorchDistTransport(stage.device, data_backend=transport, ctrl_group=ctrl_group))
    return ctl, plane


# -------------------------------------------------------------------------------------------------
# Cross-process chain
# -------------------------------------------------------------------------------------------------
class ChainPipeline:
    """Stage-0 side of the cross-process chain."""

    def __init__(self, stage: StageExecutor, ctl, plane):
        self.stage, self.ctl, self.plane = stage, ctl, plane
        self.num_stages = ctl.world
        assert ctl.rank == 0 and stage.model.spec.is_first and self.num_stages > 1
        self.runner = StepRunner(stage, plane)
        self.gcache = self.runner.gcache
        self._seq = 0
        self._outstanding = deque()
        self._dead: Optional[str] = None

    @classmethod
    def build(cls, stage: StageExecutor, **kw) -> "ChainPipeline":
        return cls(stage, *build_chain(stage, **kw))

    @property
    def h2d_bytes(self) -> int:
        return self.runner.h2d_bytes

    @property
    def d2h_bytes(self) -> int:
        return self.plane.d2h_bytes

    def submit(self, inp: StepInput):
        if self._dead:
            raise RuntimeError(self._dead)
        self._seq += 1
        seq = self._seq
        wire, lay = pack_step(seq, inp.meta, inp.tokens, inp.params, inp.contexts, inp.rng, inp.is_prefill,
                              pad_decode=self.gcache.enabled, counts=inp.counts, allow=inp.allow)
        self.ctl.publish(KIND_STEP, inp.group, wire)
        try:
            self.runner.run(wire, inp.group)
        except Exception as e:  # noqa: BLE001 — report, keep the chain in lock-step, fail the requests on wait()
            log.exception("stage 0 failed step %d", seq)
            self.ctl.set_error(seq, f"{type(e).__name__}: {e}")
            self.runner.poison(wire, inp.group)
        rl = ResultLayout(lay.B, lay.k)
        h = (seq, rl, self.plane.recv_result(inp.group, rl.nbytes), inp.meta.num_seqs)
        self._outstanding.append(h)
        return h

    def _raise_if_failed(self):
        err = self.ctl.first_error()
        if err is not None:
            raise RuntimeError(f"stage {err[0]} failed (step {err[1]}): {err[2]}")

    def wait(self, handle) -> StepOutput:
        seq, rl, pending, n_real = handle
        host = pending.get()
        try:
            self._outstanding.remove(handle)
        except ValueError:
            pass
        self._raise_if_failed()
        if self.plane.failed():
            self._dead = "P2P flag wait timed out: a pipeline stage is not responding"
            raise RuntimeError(self._dead)
        return _step_output(parse_result(host, rl, seq), n_real)

    def reset(self):
        """Called by the engine after a failure, *before* it releases KV pages: wait for every step still in flight (their
        results are discarded — downstream stages may still be writing KV for them), then clear the error state."""
        while self._outstanding:
            _, _, pending, _ = self._outstanding.popleft()
            try:
                pending.get()
            except Exception:  # noqa: BLE001
                log.exception("draining an in-flight step failed")
        self.ctl.clear_errors()

    def shutdown(self):
        try:
            self.reset()
        finally:
            self.ctl.publish(KIND_SHUTDOWN, 0, None)
            self.ctl.request_shutdown()
            tp = getattr(self.plane, "tp", None)
            if tp is not None and hasattr(tp, "flush"):
                tp.flush()


def worker_loop(stage: StageExecutor, ctl, plane):
    """Non-first stage: execute the launch records of the control plane in order until shutdown."""
    runner = StepRunner(stage, plane)
    timed_out = False
    while True:
        rec = ctl.next()
        if rec is None:
            break
        seq, kind, group, wire = rec
        if kind == KIND_SHUTDOWN:
            break
        if kind != KIND_STEP:
            continue
        try:
            runner.run(wire, group)
        except Exception as e:  # noqa: BLE001
            log.exception("stage %d failed", ctl.rank)
            ctl.set_error(seq, f"{type(e).__name__}: {e}")
            runner.poison(wire, group)
        if not timed_out and plane.failed():
            timed_out = True
            ctl.set_error(seq, "P2P flag wait timed out: the previous stage is not responding")
    if stage.device.type == "cuda":
        torch.cuda.synchronize(stage.device)
    tp = getattr(plane, "tp", None)
    if tp is not None and hasattr(tp, "flush"):
        tp.flush()
