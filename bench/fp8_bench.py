#!/usr/bin/env python
"""Expert-bank GEMM microbenchmark: block-scaled FP8 (wgmma e4m3 + block scales, ops/csrc/gemm_fp8.cu) vs bf16 (gemm_persistent.cu) on
the DeepSeek-V2-Lite MoE block of a decode step (66 experts incl. the appended shared ones, 64 tokens x 8 pairs, scatter layout).
CUDA-event timed, L2 flushed between iterations; GB/s = weight bytes / time against MEASURED_PEAKS.json."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mlx_sharding_b200.ops import b200  # noqa: E402
from mlx_sharding_b200.utils.quant import to_mxfp8  # noqa: E402
from mlx_sharding_b200.utils.timing import flush_l2  # noqa: E402


def timed(fn, iters=12, warm=3):
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
    except Exception:  # noqa: BLE001
        hbm = 3350e9
    E, H, I, T, k, stride = 66, 2048, 1408, 64, 8, 64
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s, sc=0.03: (torch.randn(*s, device=dev, generator=g) * sc).to(torch.bfloat16)
    wg, wu, wd = rnd(E, I, H), rnd(E, I, H), rnd(E, H, I)
    x = rnd(E * stride, H, sc=1.0)
    counts = torch.full((E,), 6, dtype=torch.int32, device=dev)
    counts[-2:] = T
    hb = C.grouped_linear(x, wg, wu, counts, stride, 1, False, None, None, None, T * k, stride)
    t_dual_bf16 = timed(lambda: C.grouped_linear(x, wg, wu, counts, stride, 1, False, None, None, None, T * k, stride))
    t_down_bf16 = timed(lambda: C.grouped_linear(hb, wd, None, counts, stride, 0, True, None, None, None, T * k, stride))
    (gq, gs), (uq, us), (dq, ds) = to_mxfp8(wg), to_mxfp8(wu), to_mxfp8(wd)
    xq, xsf = C.quant_mxfp8(x)
    hq, hsf = C.quant_mxfp8(hb)
    t_dual_fp8 = timed(lambda: C.linear_fp8(xq, xsf, gq, gs, uq, us, counts, stride, None, 1, False, T * k, stride))
    t_down_fp8 = timed(lambda: C.linear_fp8(hq, hsf, dq, ds, None, None, counts, stride, None, 0, True, T * k, stride))
    t_qx = timed(lambda: C.quant_mxfp8(x))
    t_qh = timed(lambda: C.quant_mxfp8(hb))
    nb = lambda *ts: sum(t.numel() * t.element_size() for t in ts)
    row = lambda name, us_, by: {"kernel": name, "us": round(us_, 2), "weight_MB": round(by / 1e6, 1), "GB_s": round(by / us_ / 1e3, 0),
                                 "frac_of_hbm": round(by / (us_ * 1e-6) / hbm, 3)}
    out = {"bench": "MoE expert bank of one decode step: 66 experts (64 routed + 2 shared), 64 tokens x 8 pairs, scatter layout",
           "rows": [row("gate/up DUAL bf16 (gemm_persistent)", t_dual_bf16, nb(wg, wu)), row("down bf16", t_down_bf16, nb(wd)),
                    row("gate/up DUAL mxfp8 (gemm_fp8)", t_dual_fp8, nb(gq, gs, uq, us)), row("down mxfp8", t_down_fp8, nb(dq, ds)),
                    {"kernel": "quant_mxfp8 x [4224, 2048]", "us": round(t_qx, 2)}, {"kernel": "quant_mxfp8 h [4224, 1408]", "us": round(t_qh, 2)}],
           "block_us": {"bf16": round(t_dual_bf16 + t_down_bf16, 1), "mxfp8_incl_quant": round(t_dual_fp8 + t_down_fp8 + t_qx + t_qh, 1)}}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
