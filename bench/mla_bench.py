#!/usr/bin/env python
"""Decode-attention microbenchmark: absorbed-latent MLA on wgmma (ops/csrc/mla_decode.cu, 576-dim latent cache) vs the
decompressed-cache split-KV kernel (ops/csrc/attention.cu, 16 heads x (192 + 128) per token) on DeepSeek-V2-Lite shapes.
CUDA-event timed, L2 flushed between iterations, reports microseconds and achieved KV bytes/s against MEASURED_PEAKS.json."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mlx_sharding_b200.ops import b200  # noqa: E402
from mlx_sharding_b200.utils.timing import flush_l2  # noqa: E402


def timed(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush_l2()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    C = b200.load_extension()
    dev = torch.device("cuda")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    try:
        hbm = json.load(open(os.path.join(root, "MEASURED_PEAKS.json")))["hbm_gbs"] * 1e9
        basis = "measured"
    except Exception:  # noqa: BLE001
        hbm, basis = 3350e9, "fallback"
    out = {"bench": "decode attention, DeepSeek-V2-Lite shapes (16 heads), B sequences x ctx tokens", "hbm_basis": f"{basis} {hbm / 1e9:.0f} GB/s",
           "rows": []}
    scale = 192 ** -0.5
    only = os.environ.get("MLA_BENCH_ONLY")          # "B,ctx": a single configuration (ncu captures)
    cfgs = ((64, 128), (64, 1024), (64, 4096), (8, 16384), (1, 32768))
    if only:
        cfgs = (tuple(int(v) for v in only.split(",")),)
    for B, ctx in cfgs:
        mb = (ctx + 63) // 64
        npages = B * mb + 1
        g = torch.Generator(device=dev).manual_seed(1)
        bt = (torch.randperm(npages - 1, device=dev, generator=g)[: B * mb] + 1).view(B, mb).to(torch.int32).contiguous()
        cl = torch.full((B,), ctx, dtype=torch.int32, device=dev)
        pos = cl - 1
        # latent path
        pool = (torch.randn(npages, 1, 64, 576, device=dev, generator=g) * 0.5).to(torch.bfloat16)
        q = (torch.randn(B, 16, 576, device=dev, generator=g) * 0.3).to(torch.bfloat16)
        t_lat = timed(lambda: C.mla_decode(q, pool, bt, cl, scale, ctx, 0))
        lat_bytes = B * ctx * 576 * 2
        if os.environ.get("MLA_BENCH_TRACE"):
            # per-tile pipeline timeline of CTA (0,0): clock64 stamps of load issue / QK issue / PV issue / S ready / P ready / O consumed
            tr = torch.zeros(6, 16, dtype=torch.int64, device=dev)
            C.mla_decode(q, pool, bt, cl, scale, ctx, 1, tr)
            torch.cuda.synchronize()
            t = tr.cpu()
            t0 = int(t[0, 0])
            names = ["load_issue", "qk_issue", "pv_issue", "s_ready", "p_ready", "o_done"]
            print(f"trace B={B} ctx={ctx} (cycles since first load issue)", file=sys.stderr)
            for e in range(6):
                print(f"  {names[e]:>10}: " + " ".join(f"{int(v) - t0:7d}" if int(v) else "      -" for v in t[e, :12]), file=sys.stderr)
        sweep = {}
        if os.environ.get("MLA_BENCH_SWEEP"):
            for ns in (1, 2, 3, 4, 6, 8, 16):
                if ns <= mb:
                    sweep[ns] = round(timed(lambda: C.mla_decode(q, pool, bt, cl, scale, ctx, ns), iters=8), 2)
        # decompressed path
        kpool = (torch.randn(npages, 16, 64, 192, device=dev, generator=g) * 0.5).to(torch.bfloat16)
        vpool = (torch.randn(npages, 16, 64, 128, device=dev, generator=g) * 0.5).to(torch.bfloat16)
        q2 = (torch.randn(B, 16, 192, device=dev, generator=g) * 0.3).to(torch.bfloat16)
        ts = torch.arange(B, dtype=torch.int32, device=dev)
        t_dec = timed(lambda: C.paged_attention(q2, kpool, vpool, bt, pos, ts, scale, 0.0, ctx))
        dec_bytes = B * ctx * 16 * 320 * 2
        del kpool, vpool
        out["rows"].append({"B": B, "ctx": ctx, "latent_tcgen05_us": round(t_lat, 2), "latent_kv_bytes": lat_bytes,
                            "latent_frac_of_hbm": round(lat_bytes / (t_lat * 1e-6) / hbm, 3),
                            "decompressed_cudacore_us": round(t_dec, 2), "decompressed_kv_bytes": dec_bytes,
                            "decompressed_frac_of_hbm": round(dec_bytes / (t_dec * 1e-6) / hbm, 3), "speedup": round(t_dec / t_lat, 2), **({"nsplit_sweep_us": sweep} if sweep else {})})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
