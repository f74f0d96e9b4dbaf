#!/usr/bin/env python
"""Host-side cost of the serving loop, with the GPUs taken out: ``LLMEngine`` drives a stub pipeline that packs the step block exactly like
``ChainPipeline.submit`` (``pack_step``: tag | sampling block | BatchMeta | tokens) and answers with random tokens immediately.

    python bench/engine_host_bench.py [--groups 4 --batch 64 --requests 512 --max-tokens 64]

The printed ``us_per_step`` is the Python time the scheduler + step packing + result handling need per micro-batch step, i.e. the
floor of the inter-step interval one engine process can sustain; ``tokens_per_s_ceiling`` = batch / that.  (Runs on CPU; no GPU.)

``--constrained N``: N requests of every batch carry a JSON Schema ``response_format``, so each step also fills their token masks
(xgrammar, the synthetic byte tokenizer at ``--vocab`` ids) and feeds the sampled tokens back to their matchers; the stub answers
those rows with a random allowed id (time excluded from ``us_per_step``)."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=4)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--requests", type=int, default=512)
    ap.add_argument("--prompt", type=int, default=24)
    ap.add_argument("--max-tokens", type=int, default=64)
    ap.add_argument("--temperature", type=float, default=1.0)
    ap.add_argument("--constrained", type=int, default=0, help="requests per batch under a JSON Schema response_format")
    ap.add_argument("--vocab", type=int, default=102400, help="model vocabulary size of the token masks (--constrained)")
    a = ap.parse_args()

    import torch

    from mlx_sharding_b200.engine.core import LLMEngine, StepOutput
    from mlx_sharding_b200.engine.sampler import SamplingParams
    from mlx_sharding_b200.parallel.graph_decode import pack_step

    import numpy as np

    rs = np.random.default_rng(0)

    class StubPipeline:
        num_stages = a.groups

        def __init__(self):
            self.seq, self.pack_s, self.answer_s = 0, 0.0, 0.0

        def submit(self, inp):
            self.seq += 1
            t0 = time.perf_counter()
            pack_step(self.seq, inp.meta, inp.tokens, inp.params, inp.contexts, inp.rng, inp.is_prefill, pad_decode=True,
                      allow=inp.allow)
            self.pack_s += time.perf_counter() - t0
            n = inp.meta.num_seqs
            toks = torch.randint(3, 1000, (n,)).tolist()
            if inp.allow is not None:      # a grammar-valid answer for the constrained rows
                t0 = time.perf_counter()
                for b, prm in enumerate(inp.params):
                    if prm.response_format is not None and inp.sample_mask[b]:
                        ok = np.flatnonzero(np.unpackbits(inp.allow[b].view(np.uint8), bitorder="little"))
                        toks[b] = int(rs.choice(ok))
                self.answer_s += time.perf_counter() - t0
            return StepOutput(tokens=toks, logprobs=[0.0] * n)

        def wait(self, h):
            return h

        def reset(self):
            pass

    pipe = StubPipeline()
    eng = LLMEngine(pipe, 1 << 15, 64, num_groups=a.groups, max_seqs_per_group=a.batch, max_prefill_tokens=2048)
    prm = SamplingParams(temperature=a.temperature)
    extra, eos = {}, None
    if a.constrained:
        import tempfile

        from mlx_sharding_b200.engine.grammar import GrammarBackend, canonical_format
        from mlx_sharding_b200.engine.tokenizer import load_tokenizer, write_byte_tokenizer

        tok_dir = write_byte_tokenizer(tempfile.mkdtemp(prefix="engine_host_bench_tok_"), vocab_size=min(a.vocab, 4096))
        tok = load_tokenizer(tok_dir)
        eng.grammar = GrammarBackend(tok, a.vocab)
        eos = tok.eos_token_id
        schema = {"type": "object", "properties": {"name": {"type": "string"}, "colour": {"enum": ["red", "green", "blue"]},
                                                   "count": {"type": "integer"}, "ok": {"type": "boolean"}},
                  "required": ["name", "colour", "count", "ok"], "additionalProperties": False}
        fmt = canonical_format({"type": "json_schema", "json_schema": {"name": "item", "schema": schema}})
        extra = {"vocab": a.vocab, "tokenizer": f"synthetic byte tokenizer ({len(tok._tokenizer)} tokens)"}
    # requests are admitted round-robin into the groups' batches: every a.batch consecutive requests share a group's batch
    reqs = [eng.submit(list(range(3, 3 + a.prompt)),
                       SamplingParams(temperature=a.temperature, response_format=fmt) if (i // a.groups) % a.batch < a.constrained
                       else prm, max_tokens=a.max_tokens, eos_token_id=eos) for i in range(a.requests)]
    t0 = time.perf_counter()
    eng.drain()
    dt = time.perf_counter() - t0 - pipe.answer_s
    steps, toks = eng.stats["steps"], eng.stats["decode_tokens"]
    print(json.dumps({"bench": "engine host loop, stub pipeline", "groups": a.groups, "batch": a.batch, "requests": a.requests,
                      "constrained": a.constrained, **extra,
                      "steps": steps, "decode_tokens": toks, "wall_s": round(dt, 3), "us_per_step": round(dt / steps * 1e6, 1),
                      "ms_per_step": round(dt / steps * 1e3, 3), "us_per_step_pack": round(pipe.pack_s / steps * 1e6, 1),
                      "tokens_per_s_ceiling": round(toks / dt, 0)}))
    assert all(r.finished and r.error is None for r in reqs)
    assert all(r.finished for r in reqs)


if __name__ == "__main__":
    main()
