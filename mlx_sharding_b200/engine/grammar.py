"""Structured output: OpenAI ``response_format`` (JSON mode / JSON Schema) as per-step token masks.

A constrained request owns a grammar matcher.  Before each step that samples it, the engine fills the request's row of the
step's token mask (int32 ``[B, ceil(V/32)]``, bit ``j & 31`` of word ``j >> 5`` = "id ``j`` allowed") from the matcher; the
sampler draws only allowed ids (``ops/csrc/sampler.cu``); the sampled token is then fed back to the matcher.  EOS is allowed
exactly where the grammar can end.

The grammar engine is xgrammar, an optional dependency: it is imported only when a ``GrammarBackend`` is built, and a server
without it refuses ``response_format`` with a client error.  Grammars are compiled with ``any_whitespace=False`` — the only
whitespace allowed is the single space after ``:`` and ``,`` of xgrammar's default separators — so a model cannot spend its
tokens on unbounded whitespace.
"""
from __future__ import annotations

import json
import re
import threading
from collections import OrderedDict
from typing import List, Optional, Sequence

import numpy as np


def mask_words(vocab_size: int) -> int:
    """Words of one token-mask row."""
    return (int(vocab_size) + 31) // 32


def canonical_format(value) -> Optional[str]:
    """OpenAI ``response_format`` value -> the canonical JSON text the engine compiles (``None`` = unconstrained).

    ``None`` / ``{"type": "text"}`` -> ``None``; ``{"type": "json_object"}``; ``{"type": "json_schema", "json_schema":
    {"name": str, "schema": object, "strict": bool?}}`` -> ``{"schema": ..., "type": "json_schema"}`` (``name`` and ``strict`` do
    not change what is compiled).  A malformed value raises ``ValueError``."""
    if value is None:
        return None
    if not isinstance(value, dict):
        raise ValueError("response_format must be an object")
    kind = value.get("type")
    if kind == "text":
        return None
    if kind == "json_object":
        return json.dumps({"type": "json_object"}, sort_keys=True, separators=(",", ":"))
    if kind != "json_schema":
        raise ValueError("response_format.type must be one of 'text', 'json_object', 'json_schema'")
    js = value.get("json_schema")
    if not isinstance(js, dict):
        raise ValueError("response_format.json_schema must be an object")
    if "name" in js and not isinstance(js["name"], str):
        raise ValueError("response_format.json_schema.name must be a string")
    if "strict" in js and js["strict"] is not None and not isinstance(js["strict"], bool):
        raise ValueError("response_format.json_schema.strict must be a boolean")
    schema = js.get("schema")
    if not isinstance(schema, dict):
        raise ValueError("response_format.json_schema.schema must be an object")
    return json.dumps({"type": "json_schema", "schema": schema}, sort_keys=True, separators=(",", ":"))


def check_format_text(text: str):
    """Shape check of a canonical format text (``SamplingParams.validate``)."""
    try:
        spec = json.loads(text)
    except (TypeError, ValueError):
        raise ValueError("response_format must be JSON text") from None
    if not isinstance(spec, dict) or spec.get("type") not in ("json_object", "json_schema"):
        raise ValueError("response_format.type must be 'json_object' or 'json_schema'")
    if spec["type"] == "json_schema" and not isinstance(spec.get("schema"), dict):
        raise ValueError("response_format.json_schema.schema must be an object")


_XGR_PREFIX = re.compile(r"^\[[^\]]*\]\s*\S+:\d+:\s*")   # "[hh:mm:ss] /path/file.cc:123: " of xgrammar's C++ errors


class GrammarBackend:
    """xgrammar state of one model: the tokenizer's vocabulary at the model's ``vocab_size`` (ids past the tokenizer are never
    allowed), a compiler, a bounded cache of compiled grammars keyed by the canonical format text, and a batched mask fill."""

    CACHE_SIZE = 256

    def __init__(self, tokenizer, vocab_size: int, eos_token_id: Optional[int] = None):
        import xgrammar as xgr

        self._xgr = xgr
        hf = getattr(tokenizer, "_tokenizer", tokenizer)     # the HF tokenizer inside ``engine.tokenizer.TokenizerWrapper``
        eos = tokenizer.eos_token_id if eos_token_id is None else eos_token_id
        self.vocab_size = int(vocab_size)
        self.words = mask_words(vocab_size)
        self.info = xgr.TokenizerInfo.from_huggingface(hf, vocab_size=self.vocab_size,
                                                       stop_token_ids=None if eos is None else [int(eos)])
        self.compiler = xgr.GrammarCompiler(self.info, cache_enabled=False)
        self._batch = xgr.BatchGrammarMatcher()
        self._cache: "OrderedDict[str, object]" = OrderedDict()
        self._lock = threading.Lock()

    @classmethod
    def create(cls, tokenizer, vocab_size: int) -> Optional["GrammarBackend"]:
        """The backend, or ``None`` when xgrammar is not installed (the engine then refuses ``response_format``)."""
        try:
            import xgrammar  # noqa: F401
        except ImportError:
            return None
        return cls(tokenizer, vocab_size)

    def compile(self, fmt: str):
        with self._lock:
            hit = self._cache.get(fmt)
            if hit is not None:
                self._cache.move_to_end(fmt)
                return hit
        check_format_text(fmt)
        spec = json.loads(fmt)
        schema = {"type": "object"} if spec["type"] == "json_object" else spec["schema"]
        try:
            cg = self.compiler.compile_json_schema(json.dumps(schema), any_whitespace=False)
        except Exception as e:  # noqa: BLE001 — xgrammar reports schema errors as RuntimeError from C++
            raise ValueError(f"response_format: invalid JSON schema: {_XGR_PREFIX.sub('', str(e)).strip()}") from None
        with self._lock:
            self._cache[fmt] = cg
            while len(self._cache) > self.CACHE_SIZE:
                self._cache.popitem(last=False)
        return cg

    def matcher(self, fmt: str):
        """A fresh matcher of ``fmt`` (canonical format text); ``ValueError`` if the schema does not compile."""
        return self._xgr.GrammarMatcher(self.compile(fmt))

    def fill(self, matchers: List, allow: np.ndarray, rows: Sequence[int]):
        """Write the next-token masks of ``matchers`` into rows ``rows`` of ``allow`` (int32 ``[B, words]``) in one call."""
        self._batch.batch_fill_next_token_bitmask(matchers, allow, list(rows))

    def accept(self, matchers: List, tokens: List[int]) -> List[bool]:
        """Advance every matcher by its sampled token in one call; ``False`` where the grammar rejects the token."""
        return self._xgr.BatchGrammarMatcher.batch_accept_token(matchers, tokens)
