#!/usr/bin/env python
"""One eager decode step of the flagship model between cudaProfilerStart/Stop, for a per-launch device-time list:

    ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off --csv --log-file gpurun_out/launches.csv \
        python scripts/launch_profile.py [--ep (under torchrun: not with ncu)] [--ctx 128] [--batch 64]
    python scripts/launch_profile.py --summarise gpurun_out/launches.csv profiles/launches_decode_v3.md

Kernels are serialised by ncu (no PDL overlap, no CUDA graph): use the list for *shares*, not for the step time."""
import argparse
import csv
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def summarise(path, out, title):
    rows = [r for r in csv.reader(open(path, errors="replace")) if len(r) > 5]
    hdr = next(r for r in rows if "Kernel Name" in r)
    i_name, i_val, i_grid = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Grid Size") if "Grid Size" in hdr else None
    data = [r for r in rows if r is not hdr and len(r) > i_val and r[hdr.index("Metric Name")] == "gpu__time_duration.sum"]
    unit = data[0][hdr.index("Metric Unit")]
    scale = {"ns": 1e-3, "us": 1.0, "usecond": 1.0, "nsecond": 1e-3, "ms": 1e3, "msecond": 1e3}.get(unit, 1.0)
    short = lambda n: re.sub(r"\(.*$", "", n).replace("void ", "").replace("b200::", "").replace("<unnamed>::", "").replace("(anonymous namespace)::", "")[:64]
    agg, order = {}, []
    for r in data:
        n, v = short(r[i_name]), float(r[i_val].replace(",", "")) * scale
        order.append((n, v, r[i_grid] if i_grid is not None else ""))
        a = agg.setdefault(n, [0, 0.0])
        a[0] += 1
        a[1] += v
    tot = sum(a[1] for a in agg.values())
    with open(out, "w") as f:
        f.write(f"# {title}\n\n{len(order)} launches, {tot:.0f} us summed (serialised by ncu: shares, not the step time)\n\n")
        f.write("| kernel | launches | total us | avg us | share |\n|---|---:|---:|---:|---:|\n")
        for n, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"| `{n}` | {c} | {t:.0f} | {t / c:.1f} | {100 * t / tot:.1f}% |\n")
        # one MoE layer in launch order: the last occurrence of the router back to the previous one
        idx = [i for i, (n, _, _) in enumerate(order) if n.startswith("moe_route")]
        if len(idx) >= 2:
            f.write("\n## one MoE layer in launch order\n\n| us | grid | kernel |\n|---:|---|---|\n")
            a, b = idx[-2], idx[-1]
            for n, v, g in order[a:b]:
                f.write(f"| {v:.1f} | {g} | `{n}` |\n")
    print(open(out).read())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--summarise", nargs=2)
    ap.add_argument("--title", default="Launch list of one decode step (DeepSeek-Coder-V2-Lite bf16, 1 GPU, 64 sequences, context 128)")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--ctx", type=int, default=128)
    a = ap.parse_args()
    if a.summarise:
        return summarise(a.summarise[0], a.summarise[1], a.title)
    import torch

    from mlx_sharding_b200.config import deepseek_v2_lite_config
    from mlx_sharding_b200.ops.meta import BatchMeta
    from mlx_sharding_b200.parallel.pipeline import StageExecutor
    from mlx_sharding_b200.utils.loader import random_model

    dev = torch.device("cuda", 0)
    cfgd = deepseek_v2_lite_config()
    model = random_model(cfgd, dtype=torch.bfloat16, device=dev, backend="b200", seed=1)
    B, S, PS = a.batch, a.ctx, 64
    pps = (S + 8 + PS - 1) // PS
    stage = StageExecutor(model, B * pps + 1, PS)
    bts = [[1 + b * pps + i for i in range(pps)] for b in range(B)]
    gen = torch.Generator().manual_seed(1)
    prompts = torch.randint(3, 100000, (B, S), generator=gen)
    for b0 in range(0, B, 16):
        meta = BatchMeta.build([S] * 16, [0] * 16, bts[b0:b0 + 16], PS, device=dev)
        toks = stage.forward(prompts[b0:b0 + 16].reshape(-1).to(dev), meta).argmax(-1)
    toks = torch.randint(3, 100000, (B,), device=dev)
    for step in range(3):
        meta = BatchMeta.build([1] * B, [S + step] * B, bts, PS, device=dev)
        torch.cuda.synchronize()
        if step == 2:
            torch.cuda.cudart().cudaProfilerStart()
        out = stage.forward(toks, meta)
        toks = out.argmax(-1)
        torch.cuda.synchronize()
        if step == 2:
            torch.cuda.cudart().cudaProfilerStop()
    print("done")


if __name__ == "__main__":
    main()
