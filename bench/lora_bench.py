#!/usr/bin/env python
"""LoRA adapter overhead on the decode step: a synthetic 4-bit ``llama3-8b`` (random weights, mlx-community layout, packed int4
GEMMs) with and without a rank-16 adapter on q/k/v/o/gate/up/down of every layer.  The adapter stays unfused on the packed
weights: one ``lora_shrink`` launch per adapted GEMM plus the adapter term in its epilogue.

One decode step of ``--batch`` sequences at context ``--ctx`` is captured as a CUDA graph per model and replayed; the two models
alternate for ``--rounds`` rounds of ``--iters`` replays, each timed with CUDA events.  Prints ms per step (median over rounds)
and the overhead, with the card name and power limit, as one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mlx_sharding_b200.config import llama3_8b_config  # noqa: E402
from mlx_sharding_b200.engine.kv_cache import PagedKVCache  # noqa: E402
from mlx_sharding_b200.ops import b200  # noqa: E402
from mlx_sharding_b200.ops.meta import BatchMeta  # noqa: E402
from mlx_sharding_b200.utils.adapters import load_adapter  # noqa: E402
from mlx_sharding_b200.utils.checkpoint import write_synthetic_adapter  # noqa: E402
from mlx_sharding_b200.utils.loader import random_model  # noqa: E402

MODULES = ["self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj", "mlp.up_proj",
           "mlp.down_proj"]


def card() -> dict:
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        power = f"{float(out.splitlines()[0]):.0f} W"
    except Exception:  # noqa: BLE001
        power = "unknown"
    return {"gpu": name, "power_limit": power}


def decode_graph(model, B, ctx, page):
    """A captured decode step of B sequences (one token each, ``ctx`` tokens of context) and its input ids."""
    per_seq = (ctx + 1 + page - 1) // page
    kv = PagedKVCache.for_model(model, B * per_seq + 1, page)
    pages = [list(range(1 + b * per_seq, 1 + (b + 1) * per_seq)) for b in range(B)]
    meta = BatchMeta.build([1] * B, [ctx] * B, pages, page, device=model.device)
    ids = torch.randint(0, model.cfg.vocab_size, (B,), device=model.device)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            model(ids, meta, kv)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = model(ids, meta, kv)
    return g, out


def time_graph(g, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--ctx", type=int, default=512)
    ap.add_argument("--rank", type=int, default=16)
    ap.add_argument("--layers", type=int, default=None, help="fewer layers (default: all 32)")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    b200.load_extension()
    cfg = llama3_8b_config()
    if a.layers:
        cfg["num_hidden_layers"] = a.layers
    q4 = {"group_size": 64, "bits": 4}
    with tempfile.TemporaryDirectory() as tmp:
        write_synthetic_adapter(tmp, cfg, rank=a.rank, scale=20.0, modules=MODULES, seed=1)
        adapter = load_adapter(tmp)
    models = {"base": random_model(cfg, dtype=torch.bfloat16, device="cuda", backend="b200", seed=0, quantization=q4),
              "lora": random_model(cfg, dtype=torch.bfloat16, device="cuda", backend="b200", seed=0, quantization=q4,
                                   adapter=adapter)}
    graphs = {k: decode_graph(m, a.batch, a.ctx, 64) for k, m in models.items()}
    for g, _ in graphs.values():
        time_graph(g, 5)
    times = {k: [] for k in graphs}
    for _ in range(a.rounds):
        for k, (g, _) in graphs.items():
            times[k].append(time_graph(g, a.iters))
    ms = {k: statistics.median(v) for k, v in times.items()}
    res = dict(card(), model="llama3-8b 4-bit (synthetic)", layers=cfg["num_hidden_layers"], batch=a.batch, ctx=a.ctx,
               rank=a.rank, adapted_modules=MODULES, ms_per_step_base=round(ms["base"], 4), ms_per_step_lora=round(ms["lora"], 4),
               overhead_pct=round(100.0 * (ms["lora"] / ms["base"] - 1.0), 2),
               rounds={k: [round(t, 4) for t in v] for k, v in times.items()})
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
