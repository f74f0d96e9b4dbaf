#!/usr/bin/env python
"""Sampler microbenchmark: ``sample_into`` (ops/csrc/sampler.cu) on B rows (default 64) of V = 102400 seeded fp32 logits, CUDA-event
timed, for the default path, the top-p / top-k / min-p filters and token masks (structured output) with about 1 % and 50 % of
the ids allowed.  Prints microseconds per call with the card name and power limit, one JSON line at the end.

``--dump DIR`` writes the default-path tokens and log-probs at T = 0, T = 1 and T = 1 with top-p 0.9 (``default_*.npy``).  That
part passes only the arguments every build's ``sample_into`` has, so the dumps of two builds can be compared byte for byte."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mlx_sharding_b200.ops import b200  # noqa: E402

V = 102400


def card() -> dict:
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        power = f"{float(out.splitlines()[0]):.0f} W"
    except Exception:  # noqa: BLE001
        power = "unknown"
    return {"gpu": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64, help="rows B (one CTA each)")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--dump", default=None, help="directory for the default-path tokens / log-probs")
    a = ap.parse_args()
    B = a.batch
    C = b200.load_extension()
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    logits = (torch.randn(B, V, device=dev, generator=g) * 3.0).contiguous()
    rng = torch.stack([torch.arange(B) + 1000, torch.full((B,), 5)], 1).to(torch.int64).to(dev).contiguous()
    toks = torch.empty(B, dtype=torch.int64, device=dev)
    lp = torch.empty(B, dtype=torch.float32, device=dev)
    full = lambda v, dt=torch.float32: torch.full((B,), v, dtype=dt, device=dev)

    if a.dump:
        os.makedirs(a.dump, exist_ok=True)
        for name, t, p in (("t0", 0.0, 1.0), ("t1", 1.0, 1.0), ("t1_top_p0.9", 1.0, 0.9)):
            C.sample_into(logits, full(t), full(p), rng, 0, toks, lp)
            torch.cuda.synchronize()
            np.save(os.path.join(a.dump, f"default_{name}_tokens.npy"), toks.cpu().numpy())
            np.save(os.path.join(a.dump, f"default_{name}_logprobs.npy"), lp.cpu().numpy())

    # token masks: each bit set with probability ~1 % / ~50 % (seeded), int32 [B, ceil(V/32)]
    gm = torch.Generator(device=dev).manual_seed(1)
    words = (V + 31) // 32
    bits = lambda frac: (torch.rand(B, words * 32, device=dev, generator=gm) < frac).view(B, words, 32).to(torch.int64)
    pack = lambda b: (b << torch.arange(32, device=dev)).sum(-1).to(torch.int32).contiguous()   # wraps bit 31 into the sign
    masks = {"1%": pack(bits(0.01)), "50%": pack(bits(0.5))}
    cases = [("greedy", 0.0, 1.0, 0, 0.0, None), ("T=1", 1.0, 1.0, 0, 0.0, None), ("top-p 0.9", 1.0, 0.9, 0, 0.0, None),
             ("top-k 50", 1.0, 1.0, 50, 0.0, None), ("top-k 50 + top-p 0.9", 1.0, 0.9, 50, 0.0, None),
             ("min-p 0.05", 1.0, 1.0, 0, 0.05, None)]
    for m in ("1%", "50%"):
        cases += [(f"mask {m}, greedy", 0.0, 1.0, 0, 0.0, m), (f"mask {m}, T=1", 1.0, 1.0, 0, 0.0, m),
                  (f"mask {m}, top-p 0.9", 1.0, 0.9, 0, 0.0, m)]
    info = card()
    print(f"sample_into, B={B}, V={V}, fp32 logits; {info['gpu']}, power limit {info['power_limit']}")
    rows = []
    for name, t, p, k, mp, m in cases:
        args = (logits, full(t), full(p), rng, 0, toks, lp)
        kw = dict(keep_k=full(k, torch.int32), min_p=full(mp)) if (k or mp) else {}
        if m is not None:
            kw["allow"] = masks[m]
        try:
            C.sample_into(*args, **kw)
        except TypeError:          # a build without the filter / mask arguments
            print(f"  {name:<24} not supported by this build")
            rows.append({"case": name, "us": None})
            continue
        for _ in range(a.warmup):
            C.sample_into(*args, **kw)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(a.iters):
            C.sample_into(*args, **kw)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / a.iters
        print(f"  {name:<24} {us:9.1f} us/call")
        rows.append({"case": name, "us": round(us, 2)})
    print(json.dumps({"bench": "sampler", "B": B, "V": V, **info, "rows": rows}))


if __name__ == "__main__":
    main()
