"""``mlx-sharding-api`` — OpenAI-compatible HTTP server + primary pipeline stage.

Reference: ``shard/openai_api.py`` (C14).  Same routes, request fields, response envelope, SSE framing,
CORS behaviour, static UI serving and CLI flags; what changed underneath:

* requests go through the micro-batching ``LLMEngine`` (many concurrent requests, one engine thread)
  instead of a single-threaded ``HTTPServer`` that runs the model inside the handler;
* the stage topology is chosen at start-up: all layers local (1 GPU), native chain over
  NCCL / fused-P2P (torchrun), or the reference's gRPC hub-and-spoke relay when
  ``--llm-shard-addresses`` points at ``mlx-sharding-server`` peers;
* parameter validation errors are reported as HTTP 400 JSON instead of tearing down the connection;
  ``logit_bias`` is honoured in streaming mode too (the reference drops it, openai_api.py:455-462);
* extra read-only routes: ``GET /v1/models``, ``GET /health``, ``GET /metrics``.

Kept quirks (for drop-in compatibility): ``object`` is ``chat.completions`` / ``chat.completions.chunk``
(plural, openai_api.py:513-515); ``usage`` only on non-streaming replies; streaming chunks carry
``finish_reason: null`` until the final chunk.
"""
from __future__ import annotations

import argparse
import json
import logging
import mimetypes
import os
import threading
import time
import uuid
import warnings
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer
from pathlib import Path
from typing import Dict, List, Optional

import torch

from ..engine.core import LLMEngine, stopping_criteria
from ..engine.grammar import canonical_format
from ..engine.sampler import SamplingParams

log = logging.getLogger("mlx_sharding_b200.api")


# ------------------------------------------------------------------------------------------------ helpers
def convert_chat(messages: List[dict], role_mapping: Optional[dict] = None) -> str:
    """Fallback prompt formatter for tokenizers without a chat template (reference openai_api.py:46-67)."""
    mapping = role_mapping if role_mapping is not None else {
        "system_prompt": ("A chat between a curious user and an artificial intelligence assistant. "
                          "The assistant follows the given rules no matter what."),
        "system": "ASSISTANT's RULE: ",
        "user": "USER: ",
        "assistant": "ASSISTANT: ",
        "stop": "\n",
    }
    stop = mapping.get("stop", "")
    parts = [f"{mapping.get(m['role'], '')}{m.get('content', '')}{stop}" for m in messages]
    return ("".join(parts) + mapping.get("assistant", "")).rstrip()


class RequestError(ValueError):
    pass


def parse_request_params(body: dict) -> dict:
    """Extract + validate generation parameters (reference openai_api.py:206-215, 252-294)."""
    p = dict(
        stream=body.get("stream", False),
        model=body.get("model", "default_model"),
        max_tokens=body.get("max_tokens", 100),
        temperature=body.get("temperature", 1.0),
        top_p=body.get("top_p", 1.0),
        repetition_penalty=body.get("repetition_penalty", 1.0),
        repetition_context_size=body.get("repetition_context_size", 20),
        logit_bias=body.get("logit_bias", None),
        logprobs=body.get("logprobs", -1),
        seed=body.get("seed", None),      # OpenAI's `seed`: the request's own random stream (the reference has no such field)
    )
    if not isinstance(p["stream"], bool):
        raise RequestError("stream must be a boolean")
    if not isinstance(p["max_tokens"], int) or isinstance(p["max_tokens"], bool) or p["max_tokens"] < 0:
        raise RequestError("max_tokens must be a non-negative integer")
    if not isinstance(p["temperature"], (float, int)) or p["temperature"] < 0:
        raise RequestError("temperature must be a non-negative float")
    if not isinstance(p["top_p"], (float, int)) or p["top_p"] < 0 or p["top_p"] > 1:
        raise RequestError("top_p must be a float between 0 and 1")
    if not isinstance(p["repetition_penalty"], (float, int)) or p["repetition_penalty"] < 0:
        raise RequestError("repetition_penalty must be a non-negative float")
    lp = p["logprobs"]
    if lp is None or lp is False:
        lp = -1
    if lp is True:
        lp = int(body.get("top_logprobs", 1) or 1)
    if lp != -1 and not (isinstance(lp, int) and 0 < lp <= 10):
        raise RequestError(f"logprobs must be between 1 and 10 but got {lp}")
    p["logprobs"] = lp
    if not isinstance(p["repetition_context_size"], int) or p["repetition_context_size"] < 0:
        raise RequestError("repetition_context_size must be a non-negative integer")
    if p["logit_bias"] is not None:
        if not isinstance(p["logit_bias"], dict):
            raise RequestError("logit_bias must be a dict of int to float")
        try:
            p["logit_bias"] = {int(k): float(v) for k, v in p["logit_bias"].items()}
        except (ValueError, TypeError):
            raise RequestError("logit_bias must be a dict of int to float")
    if not isinstance(p["model"], str):
        raise RequestError("model must be a string")
    if p["seed"] is not None and (not isinstance(p["seed"], int) or isinstance(p["seed"], bool)):
        raise RequestError("seed must be an integer")
    # OpenAI's presence / frequency penalties and the top_k / min_p filters of vLLM, llama.cpp and mlx_lm (null = default)
    num = lambda v: isinstance(v, (float, int)) and not isinstance(v, bool)
    for name, default in (("top_k", 0), ("min_p", 0.0), ("presence_penalty", 0.0), ("frequency_penalty", 0.0)):
        v = body.get(name)
        p[name] = default if v is None else v
    if not isinstance(p["top_k"], int) or isinstance(p["top_k"], bool) or p["top_k"] < -1:
        raise RequestError("top_k must be an integer >= -1 (0 or -1 disables it)")
    if not num(p["min_p"]) or not 0 <= p["min_p"] <= 1:
        raise RequestError("min_p must be a float between 0 and 1")
    for name in ("presence_penalty", "frequency_penalty"):
        if not num(p[name]) or not -2 <= p[name] <= 2:
            raise RequestError(f"{name} must be a float between -2 and 2")
    # structured output: {"type": "text" | "json_object" | "json_schema", "json_schema": {...}} (engine/grammar.py)
    try:
        p["response_format"] = canonical_format(body.get("response_format"))
    except ValueError as e:
        raise RequestError(str(e)) from None
    return p


# ------------------------------------------------------------------------------------------------ model provider
def _ep_device(args) -> str:
    """Device of this rank in an expert-parallel group: its own GPU under NCCL, the CPU under gloo."""
    import torch.distributed as dist

    return f"cuda:{torch.cuda.current_device()}" if dist.get_backend() == "nccl" else "cpu"


def serve_expert_parallel_worker(args):
    """Rank r > 0 of ``mlx-sharding-api --expert-parallel``: load my expert shard, join the lockstep group, serve until rank 0
    shuts the group down."""
    from ..parallel.ep_serving import build_lockstep_group
    from ..utils.loader import load_model

    model = load_model(args.model, device=_ep_device(args), expert_shard=(int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])),
                       adapter_path=args.adapter_path)
    group = build_lockstep_group(model, args.kv_pages or 2048, args.page_size, max_seqs=args.max_batch)
    logging.info("expert-parallel worker rank %s ready", os.environ["RANK"])
    group.serve_forever()


class ModelProvider:
    """Loads models on demand and keeps (model, tokenizer, engine) alive across requests
    (reference ``ModelProvider``, openai_api.py:70-127; hot-swap by the request's ``model`` field)."""

    def __init__(self, cli_args: argparse.Namespace, stubs=None):
        self.cli_args = cli_args
        self.stubs = stubs or []
        self.model_key = None
        self.model = None
        self.tokenizer = None
        self.engine: Optional[LLMEngine] = None
        self._lock = threading.Lock()
        if getattr(cli_args, "model", None) is not None:
            self.load("default_model")

    @staticmethod
    def _validate_model_path(model_path: str):
        p = Path(model_path)
        if p.exists() and not p.resolve().is_relative_to(Path.cwd()):
            raise RuntimeError("Local models must be relative to the current working dir.")

    def _build_engine(self, model):
        from ..parallel.grpc_compat import GrpcRelayPipeline
        from ..parallel.pipeline import ChainPipeline, LocalPipeline, StageExecutor

        a = self.cli_args
        page_size = getattr(a, "page_size", 64)
        num_pages = getattr(a, "kv_pages", None)
        if num_pages is None:
            # every stage of a chain must use the same pool geometry (block ids are global): fixed default there
            num_pages = 2048 if int(os.environ.get("WORLD_SIZE", "1")) > 1 else self._default_pages(model, page_size)
        world = int(os.environ.get("WORLD_SIZE", "1"))
        if world > 1 and getattr(a, "expert_parallel", False):
            from ..parallel.ep_serving import build_lockstep_group

            return build_lockstep_group(model, num_pages, page_size, max_seqs=getattr(a, "max_batch", 64),
                                        prefix_cache=getattr(a, "prefix_cache", False))
        stage = StageExecutor(model, num_pages, page_size)
        if world > 1:
            # native chain: launch records through the shared-memory ring, hidden states through the fused P2P hand-off (one CUDA
            # graph replay per stage per decode step; no NCCL / gloo / pickle on that path) — parallel/pipeline.py
            mb, mp = getattr(a, "max_batch", 64), getattr(a, "max_prefill_tokens", 2048)
            pipe = ChainPipeline.build(stage, num_groups=world, max_tokens=mp, max_seqs=mb,
                                       transport=getattr(a, "transport", "auto"))
            return LLMEngine(pipe, num_pages, page_size, num_groups=world, max_seqs_per_group=mb, max_prefill_tokens=mp,
                             prefix_cache=getattr(a, "prefix_cache", False), mixed_batches=getattr(a, "mixed_batches", False))
        if not model.spec.is_last:
            if not self.stubs:
                raise RuntimeError("this process only holds layers "
                                   f"[{model.spec.start_layer},{model.spec.end_layer}) and no --llm-shard-addresses "
                                   "were given")
            pipe = GrpcRelayPipeline(stage, self.stubs)
            return LLMEngine(pipe, num_pages, page_size, num_groups=1, max_seqs_per_group=1)
        return LLMEngine(LocalPipeline([stage]), num_pages, page_size, num_groups=1,
                         max_seqs_per_group=getattr(a, "max_batch", 64), prefix_cache=getattr(a, "prefix_cache", False),
                         mixed_batches=getattr(a, "mixed_batches", False))

    def _default_pages(self, model, page_size) -> int:
        """Size the KV pool: ``--cache-limit-gb`` (the reference's Metal cache limit flag) caps it."""
        from ..engine.kv_cache import PagedKVCache

        L, hk, dk, dv = model.kv_geometry()
        per_page = PagedKVCache.bytes_per_page(L, page_size, hk, dk, dv, 2 if model.dtype != torch.float32 else 4)
        limit = getattr(self.cli_args, "cache_limit_gb", None)
        if limit is not None:
            budget = limit * (1 << 30)
        elif model.device.type == "cuda":
            free, _ = torch.cuda.mem_get_info(model.device)
            budget = int(free * 0.6)
        else:
            budget = 256 << 20
        return max(16, min(int(budget // max(per_page, 1)), 1 << 16))

    def load(self, model_path: str):
        with self._lock:
            if self.model_key == model_path:
                return self.model, self.tokenizer, self.engine
            from ..engine.tokenizer import load_tokenizer
            from ..utils.checkpoint import get_model_path
            from ..utils.loader import load_model

            if self.engine is not None:
                # Hot-swapping (reference ModelProvider.load, openai_api.py:87-127) is only safe on an idle single-process engine:
                # under torchrun the other ranks keep their layer range (a swap on rank 0 alone would also dead-lock in the
                # collective set-up), and requests in flight would lose their engine.
                if int(os.environ.get("WORLD_SIZE", "1")) > 1:
                    raise ValueError("this server is one stage of a multi-process pipeline: the model cannot be switched per request")
                busy = getattr(self.engine, "busy", None)
                if busy is not None and busy():
                    raise ValueError("requests are in flight: the model cannot be switched now")
                self.engine.shutdown()
            self.model = self.tokenizer = self.engine = self.model_key = None
            a = self.cli_args
            tok_cfg = {"trust_remote_code": True if getattr(a, "trust_remote_code", False) else None}
            if getattr(a, "chat_template", ""):
                tok_cfg["chat_template"] = a.chat_template
            if model_path == "default_model" and a.model is not None:
                path = a.model
            else:
                self._validate_model_path(model_path)
                path = model_path
            ep = int(os.environ.get("WORLD_SIZE", "1")) > 1 and getattr(a, "expert_parallel", False)
            if ep and self.model_key is not None:
                raise RuntimeError("model hot-swapping is not available in --expert-parallel mode")
            # the LoRA adapter belongs to the --model checkpoint; a model picked per request is served as it is
            adapter = getattr(a, "adapter_path", None) if path == a.model else None
            model = load_model(path, start_layer=None if ep else a.start_layer, end_layer=None if ep else a.end_layer,
                               device=_ep_device(a) if ep else getattr(a, "device", None),
                               expert_shard=(int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])) if ep else None,
                               adapter_path=adapter)
            tokenizer = load_tokenizer(get_model_path(path), tok_cfg)
            if getattr(a, "use_default_chat_template", False) and tokenizer.chat_template is None:
                tokenizer.chat_template = getattr(tokenizer, "default_chat_template", None)
            engine = self._build_engine(model)
            if isinstance(engine, LLMEngine):
                # structured output: token masks from the tokenizer's vocabulary at the model's vocab_size (None without xgrammar)
                from ..engine.grammar import GrammarBackend

                engine.grammar = GrammarBackend.create(tokenizer, model.cfg.vocab_size)
            engine.start()
            self.model_key, self.model, self.tokenizer, self.engine = model_path, model, tokenizer, engine
            return model, tokenizer, engine


# ------------------------------------------------------------------------------------------------ handler
METRICS = dict(requests=0, completion_tokens=0, prompt_tokens=0, errors=0, ttft_sum=0.0, ttft_n=0)
_METRICS_LOCK = threading.Lock()


class APIHandler(BaseHTTPRequestHandler):
    protocol_version = "HTTP/1.1"
    server_version = "mlx-sharding-b200"

    def __init__(self, model_provider: ModelProvider, static_dir: str, *args, **kwargs):
        self.created = int(time.time())
        self.model_provider = model_provider
        self.static_dir = static_dir
        super().__init__(*args, **kwargs)

    def log_message(self, fmt, *args):  # route through logging
        log.debug("%s - %s", self.address_string(), fmt % args)

    # -- headers ---------------------------------------------------------------------------------
    def _cors(self):
        self.send_header("Access-Control-Allow-Origin", "*")
        self.send_header("Access-Control-Allow-Methods", "*")
        self.send_header("Access-Control-Allow-Headers", "*")

    def _send_json(self, status: int, obj, extra_headers=()):
        data = json.dumps(obj).encode()
        self.send_response(status)
        self.send_header("Content-type", "application/json")
        self._cors()
        self.send_header("Content-Length", str(len(data)))
        for k, v in extra_headers:
            self.send_header(k, v)
        self.end_headers()
        self.wfile.write(data)
        self.wfile.flush()

    def _send_plain(self, status: int, text: bytes):
        self.send_response(status)
        self.send_header("Content-type", "application/json")
        self._cors()
        self.send_header("Content-Length", str(len(text)))
        self.end_headers()
        self.wfile.write(text)

    # -- verbs -----------------------------------------------------------------------------------
    def do_OPTIONS(self):
        self.send_response(204)
        self.send_header("Content-type", "application/json")
        self._cors()
        self.send_header("Content-Length", "0")
        self.end_headers()

    def do_GET(self):
        path = self.path.split("?", 1)[0]
        if path == "/health":
            return self._send_json(200, {"status": "ok"})
        if path == "/v1/models":
            key = self.model_provider.model_key or "default_model"
            return self._send_json(200, {"object": "list", "data": [{"id": key, "object": "model", "created": self.created}]})
        if path == "/metrics":
            with _METRICS_LOCK:
                m = dict(METRICS)
            eng = self.model_provider.engine
            lines = [f"mlx_sharding_{k} {v}" for k, v in m.items()]
            if eng is not None:
                stats, free_pages = eng.metrics_snapshot()      # RPC to the engine process when this is an API worker
                lines += [f"mlx_sharding_engine_{k} {v}" for k, v in stats.items()]
                lines.append(f"mlx_sharding_kv_pages_free {free_pages}")
            data = ("\n".join(lines) + "\n").encode()
            self.send_response(200)
            self.send_header("Content-type", "text/plain; version=0.0.4")
            self.send_header("Content-Length", str(len(data)))
            self.end_headers()
            self.wfile.write(data)
            return
        # static files (reference do_GET, openai_api.py:157-176); path traversal is refused
        root = os.path.realpath(self.static_dir)
        full = os.path.realpath(os.path.join(root, path.lstrip("/")))
        if not (full == root or full.startswith(root + os.sep)):
            return self.send_error(404, "File not found")
        if os.path.isdir(full):
            full = os.path.join(full, "index.html")
        if not os.path.exists(full):
            return self.send_error(404, "File not found")
        ctype = mimetypes.types_map.get(os.path.splitext(full)[1], "application/octet-stream")
        with open(full, "rb") as f:
            data = f.read()
        self.send_response(200)
        self.send_header("Content-type", ctype)
        self._cors()
        self.send_header("Content-Length", str(len(data)))
        self.end_headers()
        self.wfile.write(data)

    def do_POST(self):
        path = self.path.split("?", 1)[0]
        endpoints = {
            "/v1/completions": self._prompt_text,
            "/v1/chat/completions": self._prompt_chat,
            "/chat/completions": self._prompt_chat,
        }
        if path not in endpoints:
            return self._send_plain(404, b"Not Found")
        try:
            n = int(self.headers.get("Content-Length", "0"))
            body = json.loads(self.rfile.read(n).decode())
            if not isinstance(body, dict):
                raise RequestError(f"Request should be dict, but got {type(body).__name__}")
            log.debug("Incoming Request Body: %s", json.dumps(body, indent="\t"))
            self.body = body
            prm = parse_request_params(body)
        except (RequestError, json.JSONDecodeError, UnicodeDecodeError) as e:
            self._count(errors=1)
            return self._send_json(400, {"error": {"message": str(e), "type": "invalid_request_error"}})
        self.stream = prm["stream"]
        self.requested_model = prm["model"]
        try:
            self.model, self.tokenizer, self.engine = self.model_provider.load(self.requested_model)
        except ValueError as e:   # a switch that cannot be honoured right now (multi-process pipeline / requests in flight)
            self._count(errors=1)
            return self._send_json(400, {"error": {"message": str(e), "type": "invalid_request_error"}})
        except Exception as e:  # noqa: BLE001 — reference answers 404 on any load failure (openai_api.py:219-226)
            log.warning("model load failed: %s", e)
            self._count(errors=1)
            return self._send_plain(404, b"Not Found")
        try:
            stop_words = body.get("stop") or []
            stop_words = [stop_words] if isinstance(stop_words, str) else stop_words
            stop_ids = [self.tokenizer.encode(w, add_special_tokens=False) for w in stop_words]
            prompt = endpoints[path]()
            params = SamplingParams(temperature=float(prm["temperature"]), top_p=float(prm["top_p"]),
                                    repetition_penalty=float(prm["repetition_penalty"]),
                                    repetition_context_size=prm["repetition_context_size"],
                                    logit_bias=prm["logit_bias"], logprobs=max(prm["logprobs"], 0), seed=prm["seed"],
                                    top_k=prm["top_k"], min_p=float(prm["min_p"]),
                                    presence_penalty=float(prm["presence_penalty"]),
                                    frequency_penalty=float(prm["frequency_penalty"]),
                                    response_format=prm["response_format"])
            req = self.engine.submit(prompt, params, max_tokens=prm["max_tokens"],
                                     eos_token_id=self.tokenizer.eos_token_id, stop_id_sequences=stop_ids)
        except (RequestError, ValueError, AssertionError, KeyError) as e:
            self._count(errors=1)
            return self._send_json(400, {"error": {"message": str(e), "type": "invalid_request_error"}})
        self._count(requests=1, prompt_tokens=len(prompt))
        try:
            if self.stream:
                self._handle_stream(req, prompt, prm)
            else:
                self._handle_completion(req, prompt, prm)
        except (BrokenPipeError, ConnectionResetError):
            req.cancel()  # client went away: release the sequence slot (SURVEY §5.3)
        except Exception as e:  # noqa: BLE001
            log.exception("generation failed")
            req.cancel()
            self._count(errors=1)
            if not self.stream:
                self._send_json(500, {"error": {"message": f"{type(e).__name__}: {e}", "type": "server_error"}})

    # -- prompts ---------------------------------------------------------------------------------
    def _prompt_chat(self) -> List[int]:
        body = self.body
        if "messages" not in body:
            raise RequestError("Request did not contain messages")
        self.request_id = f"chatcmpl-{uuid.uuid4()}"
        self.object_type = "chat.completions.chunk" if self.stream else "chat.completions"
        tok = self.tokenizer
        if hasattr(tok, "apply_chat_template") and tok.chat_template:
            out = tok.apply_chat_template(body["messages"], tokenize=True, add_generation_prompt=True)
            if hasattr(out, "keys") and "input_ids" in out:  # transformers >= 5 returns a BatchEncoding
                out = out["input_ids"]
            return list(out)
        return list(tok.encode(convert_chat(body["messages"], body.get("role_mapping"))))

    def _prompt_text(self) -> List[int]:
        self.request_id = f"cmpl-{uuid.uuid4()}"
        self.object_type = "text_completion"
        if "prompt" not in self.body:
            raise RequestError("Request did not contain a prompt")
        return list(self.tokenizer.encode(self.body["prompt"]))

    # -- responses -------------------------------------------------------------------------------
    def _response(self, text: str, finish_reason, prompt_tokens=None, completion_tokens=None,
                  token_logprobs=None, top_logprobs=None, tokens=None) -> dict:
        choice = {
            "index": 0,
            "logprobs": {"token_logprobs": token_logprobs or [], "top_logprobs": top_logprobs or [], "tokens": tokens},
            "finish_reason": finish_reason,
        }
        resp = {
            "id": self.request_id,
            "system_fingerprint": f"fp_{uuid.uuid4()}",
            "object": self.object_type,
            "model": self.requested_model,
            "created": self.created,
            "choices": [choice],
        }
        if not self.stream:
            resp["usage"] = {"prompt_tokens": prompt_tokens, "completion_tokens": completion_tokens,
                             "total_tokens": prompt_tokens + completion_tokens}
        if self.object_type.startswith("chat.completion"):
            choice["delta" if self.stream else "message"] = {"role": "assistant", "content": text}
        else:
            choice["text"] = text
        return resp

    def _count(self, **kw):
        with _METRICS_LOCK:
            for k, v in kw.items():
                METRICS[k] += v

    def _handle_completion(self, req, prompt, prm):
        detok = self.tokenizer.new_detokenizer()
        tokens, token_logprobs, top_tokens = [], [], []
        finish_reason, trim = "length", 0
        for ev in req:
            if ev.token < 0:
                break
            detok.add_token(ev.token)
            tokens.append(ev.token)
            token_logprobs.append(ev.logprob)
            if prm["logprobs"] > 0 and ev.top is not None:
                top_tokens.append({str(k): v for k, v in ev.top.items()})
            if ev.finished:
                finish_reason = ev.finish_reason
                if finish_reason == "stop":
                    _, trim = stopping_criteria(tokens, req.stop_id_sequences, req.eos_token_id)
        if req.error is not None:
            raise req.error
        detok.finalize()
        text = detok.text
        if trim:
            suffix = self.tokenizer.decode(tokens[-trim:])
            if suffix and text.endswith(suffix):
                text = text[: -len(suffix)]
        if req.ttft is not None:
            self._count(ttft_sum=req.ttft, ttft_n=1)
        self._count(completion_tokens=len(tokens))
        resp = self._response(text, finish_reason, len(prompt), len(tokens), token_logprobs, top_tokens, tokens)
        log.debug("Outgoing Response: %s", json.dumps(resp, indent="\t"))
        self._send_json(200, resp)

    def _sse(self, obj):
        self.wfile.write(f"data: {json.dumps(obj)}\n\n".encode())
        self.wfile.flush()

    def _handle_stream(self, req, prompt, prm):
        self.send_response(200)
        self.send_header("Content-type", "text/event-stream")
        self.send_header("Cache-Control", "no-cache")
        self._cors()
        self.send_header("Connection", "close")
        self.end_headers()
        self.close_connection = True
        detok = self.tokenizer.new_detokenizer()
        tokens: List[int] = []
        hold = max((len(s) for s in req.stop_id_sequences), default=0)
        buffered = 0
        finish_reason, trim = "length", 0
        for ev in req:
            if ev.token < 0:
                break
            detok.add_token(ev.token)
            tokens.append(ev.token)
            buffered += 1
            if ev.finished:
                finish_reason = ev.finish_reason
                if finish_reason == "stop":
                    _, trim = stopping_criteria(tokens, req.stop_id_sequences, req.eos_token_id)
                break
            # hold text back while the tail could still turn into a stop sequence (openai_api.py:448-472)
            if buffered < hold:
                continue
            seg = detok.last_segment
            if seg:
                self._sse(self._response(seg, None))
            buffered = 0
        if req.error is not None:
            self._sse({"error": {"message": str(req.error), "type": "server_error"}})
        detok.finalize()
        seg = detok.last_segment
        if trim:
            suffix = self.tokenizer.decode(tokens[-trim:])
            if suffix and seg.endswith(suffix):
                seg = seg[: -len(suffix)]
        self._sse(self._response(seg, finish_reason))
        self.wfile.write(b"data: [DONE]\n\n")
        self.wfile.flush()
        if req.ttft is not None:
            self._count(ttft_sum=req.ttft, ttft_n=1)
        self._count(completion_tokens=len(tokens))


# ------------------------------------------------------------------------------------------------ entry
def make_server(host: str, port: int, model_provider, static_dir: str, reuse_port: bool = False) -> ThreadingHTTPServer:
    class _Server(ThreadingHTTPServer):
        daemon_threads = True
        request_queue_size = 1024     # listen backlog: hundreds of clients may connect at once (the stdlib default is 5)
        allow_reuse_port = reuse_port  # API worker processes all bind the port; the kernel spreads the connections (frontend.py)

    return _Server((host, port), lambda *a, **k: APIHandler(model_provider, static_dir, *a, **k))


def run(host: str, port: int, model_provider: ModelProvider, static_dir: str, api_workers: int = 0):
    """Serve until interrupted.  ``api_workers > 0``: the HTTP / SSE / tokenizer work runs in that many worker processes and this
    process keeps only the engine loop (server/frontend.py); 0: the reference's layout, HTTP threads next to the engine."""
    warnings.warn("this server implements only basic security checks; do not expose it to untrusted networks")
    front = httpd = None
    if api_workers > 0:
        from .frontend import FrontEnd

        a = model_provider.cli_args
        if model_provider.engine is None:
            raise SystemExit("--api-workers needs --model (the engine is built at start-up; per-request model loading is off)")
        if not hasattr(model_provider.engine, "sinks"):
            raise SystemExit("--api-workers is not available with --expert-parallel (the lockstep group owns the request routing)")
        tok_cfg = {"trust_remote_code": True if getattr(a, "trust_remote_code", False) else None,
                   "chat_template": getattr(a, "chat_template", "") or None,
                   "use_default_chat_template": bool(getattr(a, "use_default_chat_template", False))}
        front = FrontEnd(model_provider.engine, api_workers, host, port, static_dir, a.model, model_provider.model_key or "default_model",
                         tok_cfg, getattr(a, "log_level", "INFO")).start()
        log.info("%d API worker processes accepting on %s:%d", api_workers, host, port)
    else:
        httpd = make_server(host, port, model_provider, static_dir)
        log.info("Starting httpd at %s on port %d...", host, port)
    print(f"A web-based UI is available at http://{host}:{port}")
    print("Press Ctrl+C to stop the server.")
    try:
        if httpd is not None:
            httpd.serve_forever()
        else:
            while all(p.is_alive() for p in front.procs):
                time.sleep(0.5)
            log.error("an API worker exited; shutting down")
    except KeyboardInterrupt:
        pass
    finally:
        if front is not None:
            front.stop()
        if model_provider.engine is not None:
            model_provider.engine.shutdown()


def build_arg_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description="H100-native OpenAI-compatible HTTP server (mlx-sharding-api).")
    p.add_argument("--model", type=str, help="The path to the model weights, tokenizer, and config")
    p.add_argument("--adapter-path", type=str,
                   help="mlx_lm LoRA adapter directory (adapter_config.json + adapters.safetensors) applied to --model at load; "
                        "every process of a pipeline applies it to the layers it holds (docs/SERVING.md)")
    p.add_argument("--host", type=str, default="127.0.0.1", help="Host for the HTTP server (default: 127.0.0.1)")
    p.add_argument("--port", type=int, default=8080, help="Port for the HTTP server (default: 8080)")
    p.add_argument("--trust-remote-code", action="store_true", help="Enable trusting remote code for tokenizer")
    p.add_argument("--log-level", type=str, default="INFO", choices=["DEBUG", "INFO", "WARNING", "ERROR", "CRITICAL"],
                   help="Set the logging level (default: INFO)")
    p.add_argument("--cache-limit-gb", type=int, default=None,
                   help="Cap of the KV-cache pool in GB (the reference's MLX cache limit flag)")
    p.add_argument("--chat-template", type=str, default="", help="Specify a chat template for the tokenizer")
    p.add_argument("--use-default-chat-template", action="store_true", help="Use the default chat template")
    p.add_argument("-s", "--llm-shard-addresses", type=str, default="localhost:50051",
                   help="Comma-separated gRPC addresses of the remaining stages, in pipeline order "
                        "(ignored when this process holds the last layer)")
    p.add_argument("-sl", "--start-layer", type=int, default=None, help="Start layer index for model sharding")
    p.add_argument("-el", "--end-layer", type=int, default=None, help="End layer index for model sharding")
    p.add_argument("--static-dir", type=str, default=None, help="Directory for static files (default: packaged UI)")
    # extensions
    p.add_argument("--device", type=str, default=None)
    p.add_argument("--kv-pages", type=int, default=None, help="number of KV pages (default: sized from free memory)")
    p.add_argument("--page-size", type=int, default=64)
    p.add_argument("--max-batch", type=int, default=64, help="max concurrent sequences per micro-batch group")
    p.add_argument("--max-prefill-tokens", type=int, default=2048, help="prompt tokens per prefill step (chunked prefill)")
    p.add_argument("--transport", type=str, default="auto", choices=["auto", "fused", "nccl", "gloo"],
                   help="stage hand-off of the native chain (torchrun): fused = GEMM-epilogue P2P store over NVLink (default on "
                        "CUDA), nccl / gloo = send/recv")
    p.add_argument("--prefix-cache", action="store_true",
                   help="automatic prefix caching: full KV pages of prompt prefixes are shared between requests (chat system "
                        "prompts are prefilled once); not available with gRPC reference shards")
    p.add_argument("--api-workers", type=int, default=0,
                   help="run the HTTP / SSE / tokenizer front end in this many worker processes (SO_REUSEPORT on --port) and keep only "
                        "the engine loop in this process — needed to stream to hundreds of clients at GPU speed; 0 = in-process "
                        "HTTP threads like the reference")
    p.add_argument("--mixed-batches", action="store_true",
                   help="scheduler: prefill chunks and the decode tokens of running sequences share one ragged step, so streams in "
                        "flight keep their inter-token latency while new prompts are prefilled")
    p.add_argument("--expert-parallel", action="store_true",
                   help="under torchrun, MoE models: instead of a layer pipeline every rank serves its own share of the requests "
                        "through all layers and holds E/world routed experts per MoE layer (parallel/ep.py, lockstep group of "
                        "engines: parallel/ep_serving.py); rank 0 is the HTTP front end")
    return p


def main(argv=None):
    args = build_arg_parser().parse_args(argv)
    logging.basicConfig(level=getattr(logging, args.log_level.upper(), None),
                        format="%(asctime)s - %(levelname)s - %(message)s")
    stubs = []
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1 and args.expert_parallel:
        # expert-parallel group (torchrun): every rank is a full data-parallel engine, rank 0 additionally serves HTTP
        from ..parallel.transport import init_distributed

        rank, _ = init_distributed(device=args.device)
        if args.model is None:
            raise SystemExit("--expert-parallel needs --model (all ranks load their expert shard at start-up)")
        if rank != 0:
            return serve_expert_parallel_worker(args)
    elif world > 1:
        # native chain (torchrun): rank 0 serves HTTP + the first stage, every other rank is a stage worker.
        # Layer ranges default to a cost-balanced split when neither --start-layer/--end-layer nor the config give them.
        from ..parallel.transport import init_distributed

        rank, _ = init_distributed(device=args.device)
        if args.start_layer is None and args.end_layer is None and args.model is not None:
            from ..config import ModelConfig
            from ..parallel.partition import balanced_split
            from ..utils.checkpoint import get_model_path

            cfg = ModelConfig.from_path(get_model_path(args.model))
            if cfg.start_layer is None:
                spec = balanced_split(cfg, world)[rank]  # cost-balanced whole layers (LM head / dense layers weighted)
                args.start_layer, args.end_layer = spec.start_layer, spec.end_layer
        if rank != 0:
            from .shard_server import serve_chain

            return serve_chain(args.model, args.start_layer, args.end_layer, args.device, None,
                               args.kv_pages or 2048, args.page_size, num_groups=world, max_tokens=args.max_prefill_tokens,
                               max_seqs=args.max_batch, transport=args.transport, adapter_path=args.adapter_path)
    needs_remote = args.end_layer is not None and world == 1 and not args.expert_parallel
    if args.model is not None and not needs_remote:
        try:
            from ..config import ModelConfig
            from ..utils.checkpoint import get_model_path

            cfg = ModelConfig.from_path(get_model_path(args.model))
            needs_remote = not cfg.shard(args.start_layer, args.end_layer).is_last
        except Exception:  # noqa: BLE001
            needs_remote = False
    if needs_remote and world == 1:
        from ..parallel.grpc_compat import connect_stubs

        stubs = connect_stubs(args.llm_shard_addresses)
        log.info("Connected to %d LLM shard(s)", len(stubs))
    if args.start_layer is not None or args.end_layer is not None:
        log.info("Loading model with layers %s to %s", args.start_layer or 0, args.end_layer or "end")
    if args.static_dir is None:
        args.static_dir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "static")
    provider = ModelProvider(args, stubs)
    run(args.host, args.port, provider, args.static_dir, api_workers=args.api_workers)


if __name__ == "__main__":
    main()
