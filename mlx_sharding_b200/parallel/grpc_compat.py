"""gRPC compatibility plane (tier T3): the reference's ``mlxtensor.MLXTensorService`` protocol.

Reference pieces covered here:
* wire protocol ``shard/protos/mlx_tensor.proto`` + generated stubs ``shard/grpc/*`` (C3/C4) — we build
  the protobuf descriptors at runtime instead of shipping generated code;
* tensor (de)serialisation ``shard/utils.py:71-109`` (C5) — raw host bytes + shape + dtype string.  The
  reference only understands ``mlx.core.{float32,int32,int64,float16}``; we also speak bf16 and accept
  the plain torch/numpy spellings, and never silently return ``None`` on a bad reply;
* the stage servicer ``shard/server/server.py:27-71`` (C2): ``SendTensor`` = run this stage on the hidden
  states (token ids on a first stage), ``ResetCache`` = drop the sequence's KV.  Like the reference the
  compat servicer is **single-sequence**: positions are tracked server-side (the reference reads
  ``cache.offset``) and a last stage returns logits for *all* T positions ``[1, T, V]``;
* the hub-and-spoke relay loop of ``create_generate_step_with_grpc`` (utils.py:156-166) — exposed as
  ``GrpcRelayPipeline`` so the engine can drive reference-style peers.

Limits mirror the reference: 32 MiB metadata, 1280 MiB messages (server.py:78-82).
"""
from __future__ import annotations

import logging
import threading
from concurrent import futures
from typing import List, Optional

import numpy as np
import torch

log = logging.getLogger(__name__)

SERVICE = "mlxtensor.MLXTensorService"
GRPC_OPTIONS = [
    ("grpc.max_metadata_size", 32 * 1024 * 1024),
    ("grpc.max_send_message_length", 1280 * 1024 * 1024),
    ("grpc.max_receive_message_length", 1280 * 1024 * 1024),
]

# --------------------------------------------------------------------------------------------- protobuf
_MSG = None


def messages():
    """Runtime-built message classes (Tensor, TensorResponse, ResetCacheRequest, ResetCacheResponse)."""
    global _MSG
    if _MSG is not None:
        return _MSG
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

    fd = descriptor_pb2.FileDescriptorProto()
    fd.name = "b200_mlx_tensor.proto"
    fd.package = "mlxtensor"
    fd.syntax = "proto3"
    F = descriptor_pb2.FieldDescriptorProto

    def msg(name, fields):
        m = fd.message_type.add()
        m.name = name
        for num, (fname, ftype, label, tname) in enumerate(fields, start=1):
            f = m.field.add()
            f.name, f.number, f.type, f.label = fname, num, ftype, label
            if tname:
                f.type_name = tname

    OPT, REP = F.LABEL_OPTIONAL, F.LABEL_REPEATED
    msg("Tensor", [("tensor_data", F.TYPE_BYTES, OPT, None), ("shape", F.TYPE_INT32, REP, None),
                   ("dtype", F.TYPE_STRING, OPT, None)])
    msg("TensorResponse", [("success", F.TYPE_BOOL, OPT, None), ("message", F.TYPE_STRING, OPT, None),
                           ("tensor", F.TYPE_MESSAGE, OPT, ".mlxtensor.Tensor")])
    msg("ResetCacheRequest", [])
    msg("ResetCacheResponse", [("success", F.TYPE_BOOL, OPT, None), ("message", F.TYPE_STRING, OPT, None)])
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)

    class _NS:
        pass

    ns = _NS()
    for n in ("Tensor", "TensorResponse", "ResetCacheRequest", "ResetCacheResponse"):
        setattr(ns, n, message_factory.GetMessageClass(pool.FindMessageTypeByName(f"mlxtensor.{n}")))
    _MSG = ns
    return ns


# --------------------------------------------------------------------------------------------- tensors
DTYPES = {
    "float32": torch.float32, "float16": torch.float16, "bfloat16": torch.bfloat16,
    "int32": torch.int32, "int64": torch.int64,
}


def _parse_dtype(s: str) -> torch.dtype:
    key = s.split(".")[-1]  # "mlx.core.float16" / "torch.float16" / "float16"
    if key not in DTYPES:
        raise ValueError(f"Unsupported dtype: {s}")
    return DTYPES[key]


def tensor_to_message(t: torch.Tensor, mlx_names: bool = True):
    """torch tensor -> ``Tensor`` message.  With ``mlx_names`` the dtype string uses the reference's
    ``mlx.core.*`` spelling so its ``bytes_to_tensor`` (utils.py:93-109) accepts it."""
    M = messages()
    t = t.detach().cpu().contiguous()
    name = str(t.dtype).split(".")[-1]
    raw = t.view(torch.int16).numpy().tobytes() if t.dtype == torch.bfloat16 else t.numpy().tobytes()
    return M.Tensor(tensor_data=raw, shape=list(t.shape), dtype=("mlx.core." + name) if mlx_names else name)


def message_to_tensor(msg, device="cpu") -> torch.Tensor:
    dt = _parse_dtype(msg.dtype)
    if dt == torch.bfloat16:
        arr = np.frombuffer(msg.tensor_data, dtype=np.int16)
        t = torch.from_numpy(arr.copy()).view(torch.bfloat16)
    else:
        npdt = {torch.float32: np.float32, torch.float16: np.float16, torch.int32: np.int32, torch.int64: np.int64}[dt]
        t = torch.from_numpy(np.frombuffer(msg.tensor_data, dtype=npdt).copy())
    shape = list(msg.shape)
    if int(np.prod(shape)) != t.numel():
        raise ValueError(f"tensor payload has {t.numel()} elements but shape {shape}")
    return t.reshape(shape).to(device)


# --------------------------------------------------------------------------------------------- servicer
class StageServicer:
    """``SendTensor`` / ``ResetCache`` for one stage, single compat sequence slot.

    ``wire_dtype``: the reference casts hidden states to fp16 before sending (utils.py:159-160); we reply
    in fp16 by default for compatibility, or bf16 when both ends are ours (``--wire-dtype bfloat16``).
    """

    def __init__(self, model, num_pages: int = 512, page_size: int = 64, wire_dtype: torch.dtype = torch.float16):
        from ..engine.kv_cache import PagedKVCache

        self.model = model
        self.page_size = page_size
        self.kv = PagedKVCache.for_model(model, num_pages, page_size)
        self.pages = list(range(1, num_pages))
        self.offset = 0
        self.wire_dtype = wire_dtype
        self.lock = threading.Lock()  # the reference shares MODEL/CACHE across 10 threads unlocked (SURVEY §5.2)
        self.requests = 0

    def reset(self):
        with self.lock:
            self.offset = 0

    @torch.inference_mode()
    def run(self, x: torch.Tensor) -> torch.Tensor:
        from ..ops.meta import BatchMeta

        with self.lock:
            m = self.model
            if x.dim() == 3:       # [1, T, H]
                x = x[0]
            elif x.dim() == 2 and not x.is_floating_point():  # [1, T] ids
                x = x[0]
            T = x.shape[0]
            cap = len(self.pages) * self.page_size
            if self.offset + T > cap:
                raise MemoryError(f"sequence length {self.offset + T} exceeds the KV pool ({cap} positions)")
            meta = BatchMeta.build([T], [self.offset], [self.pages], self.page_size, device=m.device)
            x = x.to(m.device)
            if x.is_floating_point():
                x = x.to(m.dtype)
            out = m.forward(x, meta, self.kv, all_logits=True)
            self.offset += T
            self.requests += 1
            return out.unsqueeze(0)

    # gRPC handlers ---------------------------------------------------------------------------
    def SendTensor(self, request, context):
        M = messages()
        try:
            x = message_to_tensor(request)
            log.debug("SendTensor: shape=%s dtype=%s", list(x.shape), x.dtype)
            out = self.run(x)
            if out.is_floating_point():
                out = out.to(self.wire_dtype)
            return M.TensorResponse(success=True, message="Tensor processed successfully",
                                    tensor=tensor_to_message(out))
        except Exception as e:  # noqa: BLE001 — mirror server.py:55-57: report, do not crash the server
            log.exception("SendTensor failed")
            return M.TensorResponse(success=False, message=f"{type(e).__name__}: {e}")

    def ResetCache(self, request, context):
        M = messages()
        try:
            self.reset()
            return M.ResetCacheResponse(success=True, message="Cache reset successfully")
        except Exception as e:  # noqa: BLE001
            return M.ResetCacheResponse(success=False, message=str(e))


def add_servicer_to_server(servicer: StageServicer, server):
    import grpc

    M = messages()
    handlers = {
        "SendTensor": grpc.unary_unary_rpc_method_handler(
            servicer.SendTensor, request_deserializer=M.Tensor.FromString,
            response_serializer=M.TensorResponse.SerializeToString),
        "ResetCache": grpc.unary_unary_rpc_method_handler(
            servicer.ResetCache, request_deserializer=M.ResetCacheRequest.FromString,
            response_serializer=M.ResetCacheResponse.SerializeToString),
    }
    server.add_generic_rpc_handlers((grpc.method_handlers_generic_handler(SERVICE, handlers),))


def start_server(servicer: StageServicer, port: int = 0, host: str = "[::]", max_workers: int = 10):
    """Start the gRPC server; ``port=0`` binds an ephemeral port like the reference (server.py:88-90).
    Returns ``(server, bound_port)``."""
    import grpc

    server = grpc.server(futures.ThreadPoolExecutor(max_workers=max_workers), options=GRPC_OPTIONS)
    add_servicer_to_server(servicer, server)
    bound = server.add_insecure_port(f"{host}:{port}")
    if bound == 0:
        raise RuntimeError(f"could not bind {host}:{port}")
    server.start()
    return server, bound


# --------------------------------------------------------------------------------------------- client
class StageStub:
    """Client stub (equivalent of the generated ``MLXTensorServiceStub``)."""

    def __init__(self, address: str, timeout_s: Optional[float] = 120.0):
        import grpc

        M = messages()
        self.address = address
        self.timeout = timeout_s
        self.channel = grpc.insecure_channel(address, options=GRPC_OPTIONS)
        self._send = self.channel.unary_unary(f"/{SERVICE}/SendTensor", request_serializer=M.Tensor.SerializeToString,
                                              response_deserializer=M.TensorResponse.FromString)
        self._reset = self.channel.unary_unary(f"/{SERVICE}/ResetCache",
                                               request_serializer=M.ResetCacheRequest.SerializeToString,
                                               response_deserializer=M.ResetCacheResponse.FromString)

    def send_tensor(self, t: torch.Tensor, device="cpu") -> torch.Tensor:
        resp = self._send(tensor_to_message(t), timeout=self.timeout)
        if not resp.success:
            raise RuntimeError(f"shard {self.address}: {resp.message}")
        return message_to_tensor(resp.tensor, device)

    def reset_cache(self):
        resp = self._reset(messages().ResetCacheRequest(), timeout=self.timeout)
        if not resp.success:
            raise RuntimeError(f"shard {self.address}: ResetCache failed: {resp.message}")

    def close(self):
        self.channel.close()


def connect_stubs(addresses: str, timeout_s: Optional[float] = 120.0) -> List[StageStub]:
    """Comma-separated ``host:port`` list; list order is pipeline order (reference openai_api.py:665-672)."""
    return [StageStub(a.strip(), timeout_s) for a in addresses.split(",") if a.strip()]


class GrpcRelayPipeline:
    """Engine pipeline that drives reference-protocol shards: run the local (first) stage, then relay the
    hidden states through every stub in order (hub-and-spoke, utils.py:162-164), take the last position's
    logits from the final reply and sample locally.  One sequence at a time (a property of the protocol:
    shards hold a single cache) — the engine is configured with one group / one sequence for this path."""

    num_stages = 1

    def __init__(self, stage, stubs: List[StageStub], wire_dtype: torch.dtype = torch.float16, seed: int = 0):
        from ..engine.sampler import Sampler

        self.stage = stage
        self.stubs = stubs
        self.wire_dtype = wire_dtype
        self.sampler = Sampler(stage.model.ops, stage.device, seed)
        self._active_seq = None

    def submit(self, inp):
        from ..engine.core import StepOutput

        if len(inp.seq_ids) != 1:
            raise RuntimeError("the gRPC compat relay serves one sequence at a time")
        if inp.meta.positions[0].item() == 0:  # new request: reset every shard (utils.py:122-124)
            for s in self.stubs:
                s.reset_cache()
        dev = self.stage.device
        x = self.stage.forward(inp.tokens.to(dev), inp.meta.to(dev), all_logits=True)
        if self.stubs:
            x = x.unsqueeze(0)
            for s in self.stubs:
                if x.is_floating_point():
                    x = x.to(self.wire_dtype)
                x = s.send_tensor(x, dev)
            x = x[0]
        logits = x[-1:].float()
        so = self.sampler(logits, inp.params, inp.contexts, inp.counts, allow=inp.allow)
        return StepOutput(so.tokens.tolist(), so.logprobs.tolist(),
                          None if so.top_ids is None else so.top_ids.tolist(),
                          None if so.top_logprobs is None else so.top_logprobs.tolist())

    def wait(self, h):
        return h

    def reset(self):
        for s in self.stubs:
            try:
                s.reset_cache()
            except Exception:  # noqa: BLE001
                pass
