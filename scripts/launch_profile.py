#!/usr/bin/env python
"""Per-kernel device time of the flagship decode step (DeepSeek-Coder-V2-Lite bf16, 1 GPU, 64 sequences, context 128, 64-token
pages), from torch.profiler with CUDA activities:

    python scripts/launch_profile.py --out OUT_DIR [--steps 4] [--batch 64] [--ctx 128]
    python scripts/launch_profile.py --summarise OUT_DIR/launches.csv OUT_DIR/summary.md

The profiled steps are eager (no CUDA graph) and follow warm-up steps; take step times from bench.py, not from this run (tracing
slows the host).  With programmatic dependent launch a kernel becomes resident, and its trace interval starts, while its predecessor
still runs, so each launch also gets an *exclusive* time: the part of its interval after every earlier kernel has ended.  Exclusive
times add up to the busy time of the device and are what the shares use.

Every GEMM binding call is wrapped in a profiler range that carries its weight bytes (from the weight shapes: whole expert banks
for grouped launches), so GEMM launches also get GB/s over their exclusive time.  Writes launches.csv (one row per launch), summary.md
and the chrome trace decode.pt.trace.json under --out."""
import argparse
import csv
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

GEMM_CALLS = ("linear", "grouped_linear", "linear_q", "grouped_linear_q", "linear_fp8")
DATASHEET_HBM = 3350e9   # H100 SXM data-sheet HBM3 bandwidth, used when MEASURED_PEAKS.json is absent


def short(n):
    n = n.replace("void ", "").replace("b200::", "").replace("<unnamed>::", "").replace("(anonymous namespace)::", "")
    return re.sub(r"\(.*$", "", n).replace("__nv_bfloat16", "bf16")[:72]


def hbm_peak(root):
    try:
        return json.load(open(os.path.join(root, "MEASURED_PEAKS.json")))["hbm_gbs"] * 1e9, "MEASURED_PEAKS.json"
    except Exception:  # noqa: BLE001
        return DATASHEET_HBM, "data sheet (MEASURED_PEAKS.json absent)"


def summarise(path, out, title, hbm=None, hbm_src=""):
    rows = list(csv.DictReader(open(path)))
    steps = max(int(r["step"]) for r in rows) + 1
    if hbm is None:
        hbm, hbm_src = hbm_peak(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    agg, gemm = {}, {}
    for r in rows:
        a = agg.setdefault(r["kernel"], [0, 0.0, 0.0])
        a[0] += 1
        a[1] += float(r["us"])
        a[2] += float(r["excl_us"])
        if r["gemm_call"]:
            key = (r["gemm_call"], r["kernel"])
            g = gemm.setdefault(key, [0, 0.0, 0.0, 0])
            g[0] += 1
            g[1] += float(r["us"])
            g[2] += float(r["excl_us"])
            g[3] += int(r["weight_bytes"])
    busy = sum(a[2] for a in agg.values()) / steps
    with open(out, "w") as f:
        f.write(f"# {title}\n\n{len(rows) // steps} launches per step, {busy:.0f} us of device busy time per step "
                f"(sum of exclusive times, mean of {steps} profiled eager steps)\n\n")
        f.write("| kernel | launches | total us | excl us | avg excl us | share |\n|---|---:|---:|---:|---:|---:|\n")
        for n, (c, t, x) in sorted(agg.items(), key=lambda kv: -kv[1][2]):
            f.write(f"| `{n}` | {c // steps} | {t / steps:.0f} | {x / steps:.0f} | {x / c:.1f} | {100 * x / steps / busy:.1f}% |\n")
        f.write(f"\n## GEMM launches: weight bytes from shapes over exclusive time\n\nHBM reference: {hbm / 1e9:.0f} GB/s, {hbm_src}\n\n"
                "| call | kernel | launches | excl us | weight MB | GB/s | of HBM | share of step |\n|---|---|---:|---:|---:|---:|---:|---:|\n")
        for (call, n), (c, t, x, b) in sorted(gemm.items(), key=lambda kv: -kv[1][2]):
            gbs = b / (x * 1e-6) if x > 0 else 0.0
            f.write(f"| {call} | `{n}` | {c // steps} | {x / steps:.0f} | {b / steps / 1e6:.0f} | {gbs / 1e9:.0f} | {100 * gbs / hbm:.0f}% | "
                    f"{100 * x / steps / busy:.1f}% |\n")
        # one MoE layer in launch order: the last occurrence of the router back to the previous one
        step0 = [r for r in rows if r["step"] == "0"]
        idx = [i for i, r in enumerate(step0) if r["kernel"].startswith("moe_route")]
        if len(idx) >= 2:
            f.write("\n## one MoE layer in launch order\n\n| us | excl us | gap before us | kernel |\n|---:|---:|---:|---|\n")
            for r in step0[idx[-2]:idx[-1]]:
                f.write(f"| {float(r['us']):.1f} | {float(r['excl_us']):.1f} | {float(r['gap_us']):.1f} | `{r['kernel']}` |\n")
    print(open(out).read())


def wrap_gemm_calls(C, torch):
    """Each GEMM binding call runs inside a profiler range named gemm:<call>:<weight bytes>."""
    def nbytes(*ts):
        return sum(t.numel() * t.element_size() for t in ts if isinstance(t, torch.Tensor))

    weights = {
        "linear": lambda a: nbytes(a[1], a[2] if len(a) > 2 else None),
        "grouped_linear": lambda a: nbytes(a[1], a[2] if len(a) > 2 else None),
        "linear_q": lambda a: nbytes(*a[1:7]),
        "grouped_linear_q": lambda a: nbytes(*a[1:7]),
        "linear_fp8": lambda a: nbytes(*a[2:6]),
    }
    for name in GEMM_CALLS:
        fn = getattr(C, name, None)
        if fn is None:
            continue

        def wrapped(*args, _fn=fn, _name=name, **kw):
            with torch.profiler.record_function(f"gemm:{_name}:{weights[_name](args)}"):
                return _fn(*args, **kw)

        setattr(C, name, wrapped)


def launches_from_trace(trace_path, steps_ts):
    """One dict per kernel launch, in device start order, tagged with its step and the GEMM range it was launched from."""
    ev = json.load(open(trace_path))["traceEvents"]
    kernels = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    launch_ts = {e["args"]["correlation"]: e["ts"] for e in ev if e.get("cat") == "cuda_runtime" and "correlation" in e.get("args", {})}
    ranges = sorted(((e["ts"], e["ts"] + e["dur"], e["name"]) for e in ev
                     if e.get("cat") == "user_annotation" and e.get("name", "").startswith("gemm:")))
    out, last_end = [], None
    for k in kernels:
        t0, t1 = k["ts"], k["ts"] + k["dur"]
        step = next((i for i, (a, b) in enumerate(steps_ts) if a <= t0 <= b), None)
        host = launch_ts.get(k["args"].get("correlation"))
        call, wbytes = "", 0
        if host is not None:
            inner = [r for r in ranges if r[0] <= host <= r[1]]
            if inner:
                _, c, b = inner[-1][2].split(":")
                call, wbytes = c, int(b)
        excl = max(0.0, t1 - max(t0, last_end)) if last_end is not None else k["dur"]
        gap = max(0.0, t0 - last_end) if last_end is not None else 0.0
        last_end = t1 if last_end is None else max(last_end, t1)
        if step is None:
            continue
        out.append({"step": step, "kernel": short(k["name"]), "us": k["dur"], "excl_us": excl, "gap_us": gap,
                    "grid": "x".join(str(g) for g in k["args"].get("grid", [])), "gemm_call": call, "weight_bytes": wbytes})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--summarise", nargs=2, metavar=("CSV", "OUT_MD"))
    ap.add_argument("--title", default="Kernels of one decode step (DeepSeek-Coder-V2-Lite bf16, 1 GPU, 64 sequences, context 128)")
    ap.add_argument("--out", metavar="OUT_DIR", help="directory for launches.csv, summary.md and the trace (required to profile)")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--ctx", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=4)
    a = ap.parse_args()
    if a.summarise:
        return summarise(a.summarise[0], a.summarise[1], a.title)
    if not a.out:
        ap.error("--out OUT_DIR is required")
    import torch
    from torch.profiler import ProfilerActivity, profile

    from mlx_sharding_b200.config import deepseek_v2_lite_config
    from mlx_sharding_b200.ops import b200
    from mlx_sharding_b200.ops.meta import BatchMeta
    from mlx_sharding_b200.parallel.pipeline import StageExecutor
    from mlx_sharding_b200.utils.loader import random_model

    if not torch.cuda.is_available():
        raise SystemExit("launch_profile.py needs a CUDA device")
    os.makedirs(a.out, exist_ok=True)
    dev = torch.device("cuda", 0)
    wrap_gemm_calls(b200.load_extension(), torch)
    cfgd = deepseek_v2_lite_config()
    model = random_model(cfgd, dtype=torch.bfloat16, device=dev, backend="b200", seed=1)
    B, S, PS = a.batch, a.ctx, 64
    pps = (S + a.warmup + a.steps + PS - 1) // PS
    stage = StageExecutor(model, B * pps + 1, PS)
    bts = [[1 + b * pps + i for i in range(pps)] for b in range(B)]
    gen = torch.Generator().manual_seed(1)
    prompts = torch.randint(3, 100000, (B, S), generator=gen)
    for b0 in range(0, B, 16):
        meta = BatchMeta.build([S] * 16, [0] * 16, bts[b0:b0 + 16], PS, device=dev)
        stage.forward(prompts[b0:b0 + 16].reshape(-1).to(dev), meta)
    toks = torch.randint(3, 100000, (B,), device=dev)

    def step(i):
        meta = BatchMeta.build([1] * B, [S + i] * B, bts, PS, device=dev)
        return stage.forward(toks, meta).argmax(-1)

    for i in range(a.warmup):
        toks = step(i)
    torch.cuda.synchronize()
    marks = []
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(a.steps):
            with torch.profiler.record_function(f"decode_step_{i}"):
                toks = step(a.warmup + i)
            torch.cuda.synchronize()
    trace = os.path.join(a.out, "decode.pt.trace.json")
    prof.export_chrome_trace(trace)
    # device-side step windows: from the first to the last kernel launched inside each decode_step range
    ev = json.load(open(trace))["traceEvents"]
    launch_ts = {e["args"]["correlation"]: e["ts"] for e in ev if e.get("cat") == "cuda_runtime" and "correlation" in e.get("args", {})}
    spans = sorted((e["ts"], e["ts"] + e["dur"]) for e in ev if e.get("cat") == "user_annotation" and e["name"].startswith("decode_step_"))
    for lo, hi in spans:
        ks = [k for k in ev if k.get("cat") == "kernel" and lo <= launch_ts.get(k["args"].get("correlation"), -1) <= hi]
        marks.append((min(k["ts"] for k in ks), max(k["ts"] + k["dur"] for k in ks)))
    rows = launches_from_trace(trace, marks)
    path = os.path.join(a.out, "launches.csv")
    with open(path, "w", newline="") as f:
        w = csv.DictWriter(f, fieldnames=list(rows[0].keys()))
        w.writeheader()
        w.writerows(rows)
    name = torch.cuda.get_device_name(0)
    summarise(path, os.path.join(a.out, "summary.md"), f"{a.title}, {name}")


if __name__ == "__main__":
    main()
