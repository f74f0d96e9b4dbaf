"""Multi-process API front end: HTTP / SSE / tokenizer work in worker processes, the engine core alone in its own.

The reference serves HTTP from the process that runs the model (``shard/openai_api.py:487-517``: one ``HTTPServer``, the handler owns
the generation loop).  With continuous batching that design puts every stream's per-token work — incremental detokenisation, the
JSON chunk, the socket write — on threads that share the interpreter lock with the engine loop: at a few hundred streams the
handlers hold the lock most of the time, the engine thread queues behind them, and the GPUs idle.

``--api-workers N`` moves the front end out:

    clients --TCP--> worker 1..N  (ThreadingHTTPServer + tokenizer; all bound to the port with SO_REUSEPORT, the kernel spreads
                        |           the connections)
                        |  one duplex pipe per worker: submit / cancel  -->      <-- per engine step ONE message with every token
                        v                                                            that step produced for this worker's requests
                    engine process (LLMEngine loop + the pipeline; no per-token Python besides the scheduler's own)

so the engine's cost per step is O(workers), not O(streams), and detokenisation / JSON / SSE run in parallel across processes.
The handler code is the same ``APIHandler``: a worker gives it a :class:`RemoteEngine` whose ``submit`` returns an object with the
``Request`` interface (iteration over ``TokenEvent``s, ``cancel``, ``error``, ``ttft``)."""
from __future__ import annotations

import logging
import multiprocessing as mp
import os
import queue
import threading
import time
from typing import Dict, List, Optional

log = logging.getLogger("mlx_sharding_b200.frontend")


# ---------------------------------------------------------------------------------------------- engine side
class _WorkerSink:
    """Engine-side end of one worker: collects the token events of the current step, ships them as one message."""

    def __init__(self, conn, engine):
        self.conn, self.engine = conn, engine
        self.buf: list = []
        self.lock = threading.Lock()
        self.out: "queue.SimpleQueue" = queue.SimpleQueue()
        self.requests: Dict[int, object] = {}          # worker's request id -> engine Request (for cancel)
        self.alive = True
        threading.Thread(target=self._send_loop, name="frontend-send", daemon=True).start()
        threading.Thread(target=self._recv_loop, name="frontend-recv", daemon=True).start()

    # called by the engine loop after every scheduler iteration (and by whoever puts events outside the loop)
    def flush(self):
        if not self.buf:
            return
        with self.lock:
            buf, self.buf = self.buf, []
        if self.alive:      # a dead worker's requests were cancelled; their last events have nowhere to go
            self.out.put(("events", buf))

    def _send_loop(self):
        while True:
            msg = self.out.get()
            if msg is None:
                return
            try:
                self.conn.send(msg)
            except (OSError, ValueError, BrokenPipeError):
                self.alive = False
                return

    def _recv_loop(self):
        while True:
            try:
                msg = self.conn.recv()
            except (EOFError, OSError):
                break
            kind = msg[0]
            if kind == "submit":
                _, rid, prompt, params, max_tokens, eos, stops = msg
                try:
                    ev = _SinkEvents(self, rid)
                    r = self.engine.submit(prompt, params, max_tokens=max_tokens, eos_token_id=eos, stop_id_sequences=stops, events=ev)
                    self.requests[rid] = r
                    self.out.put(("ack", rid, None))
                except Exception as e:  # noqa: BLE001 — validation errors travel back to the handler (HTTP 400)
                    self.out.put(("ack", rid, f"{type(e).__name__}: {e}"))
                self.flush()        # a request that finished inside submit() (max_tokens == 0) has its event buffered already
            elif kind == "cancel":
                r = self.requests.get(msg[1])
                if r is not None:
                    r.cancel()
            elif kind == "stats":
                snap = self.engine.metrics_snapshot()
                self.out.put(("stats", msg[1], snap))
        # worker went away: cancel what it still had in flight so the sequence slots are released
        self.alive = False
        for r in list(self.requests.values()):
            r.cancel()
        self.out.put(None)


class _SinkEvents:
    """Stands in for ``Request.events`` (a queue): ``put`` appends to the worker's step buffer instead of waking a thread."""
    __slots__ = ("sink", "rid", "req")

    def __init__(self, sink: _WorkerSink, rid: int):
        self.sink, self.rid, self.req = sink, rid, None

    def put(self, ev):
        s = self.sink
        if ev is None:      # end of stream without a final event: failure (engine shut down, step error) or already finished
            err = getattr(self.req, "error", None)
            item = (self.rid, None, None if err is None else f"{type(err).__name__}: {err}")
        else:
            ttft = None
            if self.req is not None and len(self.req.output) <= 1 and self.req.ttft is not None:
                ttft = self.req.ttft
            item = (self.rid, (ev.token, ev.logprob, ev.top, ev.finished, ev.finish_reason), ttft)
        with s.lock:
            s.buf.append(item)
        if ev is None or ev.finished:
            s.requests.pop(self.rid, None)


class FrontEnd:
    """Owns the worker processes of one engine.  ``start`` returns once every worker is accepting connections."""

    def __init__(self, engine, num_workers: int, host: str, port: int, static_dir: str, model_path: str, model_key: str,
                 tokenizer_config: Optional[dict] = None, log_level: str = "INFO"):
        self.engine, self.n = engine, int(num_workers)
        self.args = (host, port, static_dir, model_path, model_key, tokenizer_config or {}, log_level)
        self.procs: List[mp.Process] = []
        self.sinks: List[_WorkerSink] = []

    def start(self, timeout: float = 300.0):
        ctx = mp.get_context("spawn")       # never fork a process that holds a CUDA context
        ready = ctx.Queue()
        for i in range(self.n):
            parent, child = ctx.Pipe(duplex=True)
            p = ctx.Process(target=worker_main, args=(child, i, ready) + self.args, name=f"api-worker-{i}", daemon=True)
            p.start()
            child.close()
            self.procs.append(p)
            sink = _WorkerSink(parent, self.engine)
            self.sinks.append(sink)
        self.engine.sinks.extend(self.sinks)
        t0 = time.time()
        for _ in range(self.n):
            try:
                msg = ready.get(timeout=max(1.0, timeout - (time.time() - t0)))
            except queue.Empty:
                raise RuntimeError("API workers did not come up") from None
            if msg[1] is not None:
                raise RuntimeError(f"API worker {msg[0]} failed to start: {msg[1]}")
        return self

    def stop(self):
        for s in self.sinks:
            if s in self.engine.sinks:
                self.engine.sinks.remove(s)
        for p in self.procs:
            if p.is_alive():
                p.terminate()       # the exact processes this object started
        for p in self.procs:
            p.join(timeout=5)


# ---------------------------------------------------------------------------------------------- worker side
class RemoteRequest:
    """Worker-side handle of a request that runs in the engine process (same interface as ``engine.core.Request``)."""

    def __init__(self, rid: int, eng: "RemoteEngine", eos_token_id, stop_id_sequences):
        self.id, self._eng = rid, eng
        self.eos_token_id = eos_token_id
        self.stop_id_sequences = stop_id_sequences or []
        self.events: "queue.SimpleQueue" = queue.SimpleQueue()
        self.error: Optional[BaseException] = None
        self.ttft: Optional[float] = None
        self._ack = threading.Event()
        self._ack_err: Optional[str] = None

    def cancel(self):
        self._eng._send(("cancel", self.id))

    def __iter__(self):
        while True:
            ev = self.events.get()
            if ev is None:
                if self.error is not None:
                    raise self.error
                return
            yield ev
            if ev.finished:
                return


class RemoteEngine:
    """The engine as seen from an API worker: ``submit`` / iteration / ``cancel`` over the worker's pipe."""

    def __init__(self, conn, on_lost=None):
        from ..engine.core import TokenEvent

        self._TokenEvent = TokenEvent
        self.conn = conn
        self.on_lost = on_lost          # called when the engine process closes the pipe (after failing the open requests)
        self._slock = threading.Lock()
        self._ids = 0
        self.reqs: Dict[int, RemoteRequest] = {}
        self._stats_wait: Dict[int, list] = {}
        threading.Thread(target=self._recv_loop, name="engine-recv", daemon=True).start()

    def _send(self, msg):
        with self._slock:
            try:
                self.conn.send(msg)
            except (OSError, ValueError, BrokenPipeError):
                pass

    def _recv_loop(self):
        TE = self._TokenEvent
        while True:
            try:
                msg = self.conn.recv()
            except (EOFError, OSError):
                break
            kind = msg[0]
            if kind == "events":
                for rid, ev, extra in msg[1]:
                    r = self.reqs.get(rid)
                    if r is None:
                        continue
                    if ev is None:
                        if extra is not None:
                            r.error = RuntimeError(extra)
                        self.reqs.pop(rid, None)
                        r.events.put(None)
                        continue
                    if extra is not None:
                        r.ttft = extra
                    if ev[3]:
                        self.reqs.pop(rid, None)
                    r.events.put(TE(*ev))
            elif kind == "ack":
                r = self.reqs.get(msg[1])
                if r is not None:
                    r._ack_err = msg[2]
                    r._ack.set()
            elif kind == "stats":
                w = self._stats_wait.pop(msg[1], None)
                if w is not None:
                    w[1] = msg[2]
                    w[0].set()
        # engine gone: fail everything that is still waiting
        err = RuntimeError("engine process went away")
        for r in list(self.reqs.values()):
            r.error = err
            r._ack_err = r._ack_err or str(err)
            r._ack.set()
            r.events.put(None)
        self.reqs.clear()
        if self.on_lost is not None:
            self.on_lost()

    def submit(self, prompt, params=None, max_tokens: int = 100, eos_token_id=None, stop_id_sequences=None) -> RemoteRequest:
        with self._slock:
            self._ids += 1
            rid = self._ids
        r = RemoteRequest(rid, self, eos_token_id, stop_id_sequences)
        self.reqs[rid] = r
        self._send(("submit", rid, [int(t) for t in prompt], params, int(max_tokens), eos_token_id, stop_id_sequences))
        if not r._ack.wait(timeout=120):
            self.reqs.pop(rid, None)
            raise RuntimeError("engine did not acknowledge the request")
        if r._ack_err is not None:
            self.reqs.pop(rid, None)
            raise ValueError(r._ack_err)     # the handler answers 400 (engine-side validation: empty prompt, too long, bad params)
        return r

    def metrics_snapshot(self, timeout: float = 5.0):
        with self._slock:
            self._ids += 1
            key = self._ids
        w = [threading.Event(), None]
        self._stats_wait[key] = w
        self._send(("stats", key))
        w[0].wait(timeout)
        return w[1] or ({}, 0)

    def busy(self) -> bool:
        return bool(self.reqs)


class RemoteProvider:
    """``ModelProvider`` of a worker: one tokenizer, one remote engine, no hot-swapping (the model lives in another process)."""

    def __init__(self, tokenizer, engine: RemoteEngine, model_key: str):
        self.tokenizer, self.engine, self.model_key, self.model = tokenizer, engine, model_key, None

    def load(self, model_path: str):
        if model_path not in ("default_model", self.model_key):
            raise ValueError("this server runs its engine in a separate process (--api-workers): the model cannot be switched per request")
        return None, self.tokenizer, self.engine


def worker_main(conn, index: int, ready, host: str, port: int, static_dir: str, model_path: str, model_key: str, tok_cfg: dict,
                log_level: str):
    os.environ["CUDA_VISIBLE_DEVICES"] = ""          # a front-end worker never touches a GPU
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):   # ... and is not a rank of the model-parallel group
        os.environ.pop(k, None)
    try:
        logging.basicConfig(level=getattr(logging, log_level.upper(), None), format=f"%(asctime)s - api-worker-{index} - %(levelname)s - %(message)s")
        from ..engine.tokenizer import load_tokenizer
        from ..utils.checkpoint import get_model_path
        from . import openai_api as api

        tok_cfg = dict(tok_cfg)
        use_default = tok_cfg.pop("use_default_chat_template", False)
        tokenizer = load_tokenizer(get_model_path(model_path), tok_cfg)
        if use_default and tokenizer.chat_template is None:
            tokenizer.chat_template = getattr(tokenizer, "default_chat_template", None)
        def engine_lost():      # the engine process ended (or crashed): a front end without an engine must not keep the port
            time.sleep(0.2)     # let handlers that are mid-response report the failure to their clients
            os._exit(0)

        provider = RemoteProvider(tokenizer, RemoteEngine(conn, on_lost=engine_lost), model_key)
        httpd = api.make_server(host, port, provider, static_dir, reuse_port=True)
    except Exception as e:  # noqa: BLE001
        ready.put((index, f"{type(e).__name__}: {e}"))
        raise
    ready.put((index, None))
    try:
        httpd.serve_forever()
    except KeyboardInterrupt:
        pass
