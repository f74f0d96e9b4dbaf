"""Hash the output of every wgmma GEMM launch route, so two builds of the extension can be compared bit for bit.

    python scripts/gemm_routes.py --so mlx_sharding_b200/ops/_b200_C.so --out new.json
    python scripts/gemm_routes.py --compare old.json new.json

Each case is seeded and runs through the raw bindings of the ``.so`` given (loaded with importlib, so two builds can run in two
processes).  Routes are forced with ``splits`` and the route ``gemm_plan`` reports is recorded next to the SHA-256 of the valid
output rows.  Cases that raise the fused stage-boundary flag (counting mode, zeroed device counter) or the EP-return peer flag
record its value after the launch, which must be 1.  ``--compare`` prints the cases that differ and exits non-zero if any do.
"""
from __future__ import annotations

import argparse
import hashlib
import importlib.util
import itertools
import json
import sys

import torch

DEV = "cuda"
SILU, GELU = 1, 2


def load(path):
    spec = importlib.util.spec_from_file_location("_b200_C", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.init_scratch(torch.cuda.current_device(), 32 << 20)
    return mod


def rnd(*shape, seed, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


def rnd_i32(*shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-2**31, 2**31 - 1, shape, generator=g, dtype=torch.int64).to(torch.int32).to(DEV)


def digest(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def scatter_rows(counts, stride):
    return torch.cat([torch.arange(e * stride, e * stride + c) for e, c in enumerate(counts)]).to(DEV)


def run_cases(C):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    res = {}

    def record(name, out, kind, max_rows, n, k, pair, splits=0, experts=0, expected=0, rows=None, flag=None):
        torch.cuda.synchronize()
        plan = C.gemm_plan(kind, max_rows, n, k, pair, splits, experts, expected, sms)
        res[name] = {"route": plan["route"], "sha256": digest(out if rows is None else out[rows])}
        if flag is not None:
            res[name]["flag"] = int(flag.item())

    def flag_args(signal):
        if not signal:
            return None, 0
        flag = torch.zeros(1, dtype=torch.int32, device=DEV)
        return flag, flag.data_ptr()

    # ---- bf16 linear: persistent at several T, cluster and workspace split-K
    K, N = 2048, 1408
    w, w2 = rnd(N, K, seed=1, scale=0.03), rnd(N, K, seed=2, scale=0.03)
    bias = rnd(N, seed=3, scale=0.5)
    for T in (1, 17, 64, 200):
        x = rnd(T, K, seed=10 + T)
        res_t = rnd(T, N, seed=20 + T)
        xs = rnd(T, 2 * K, seed=30 + T)[:, :K]   # row stride 2K
        variants = {
            "single": dict(x=x),
            "silu_pair": dict(x=x, w2=w2, act=SILU),
            "gelu_pair": dict(x=x, w2=w2, act=GELU),
            "bias_residual": dict(x=x, bias=bias, residual=res_t),
            "fp32_softcap": dict(x=x, out_fp32=True, softcap=30.0),
            "strided_x": dict(x=xs, bias=bias),
        }
        for vname, kw in variants.items():
            for signal in (False, True):
                flag, ptr = flag_args(signal)
                out = C.linear(kw["x"], w, kw.get("w2"), kw.get("residual"), kw.get("bias"), kw.get("act", 0), kw.get("softcap", 0.0),
                               kw.get("out_fp32", False), None, 1, ptr, 0)
                record(f"linear/persistent/T{T}/{vname}" + ("/signal" if signal else ""), out, "bf16", T, N, K, "w2" in kw, 1, flag=flag)
    for T in (1, 16, 64):
        x = rnd(T, K, seed=40 + T)
        res_t = rnd(T, N, seed=50 + T)
        for splits in (2, 4, 8, 16):
            for vname, kw in {"single": {}, "silu_pair": dict(w2=w2, act=SILU), "bias_residual": dict(bias=bias, residual=res_t),
                              "fp32_softcap": dict(out_fp32=True, softcap=30.0)}.items():
                for signal in (False, True):
                    flag, ptr = flag_args(signal)
                    out = C.linear(x, w, kw.get("w2"), kw.get("residual"), kw.get("bias"), kw.get("act", 0), kw.get("softcap", 0.0),
                                   kw.get("out_fp32", False), None, splits, ptr, 0)
                    record(f"linear/splits{splits}/T{T}/{vname}" + ("/signal" if signal else ""), out, "bf16", T, N, K, "w2" in kw,
                           splits, flag=flag)

    # ---- bf16 grouped_linear: offsets layout, scatter layout (return path included)
    E, Kg, Ng = 8, 1024, 768
    wg, wg2 = rnd(E, Ng, Kg, seed=60, scale=0.03), rnd(E, Ng, Kg, seed=61, scale=0.03)
    counts = [5, 0, 37, 1, 64, 0, 12, 90]
    offsets = torch.tensor([0] + list(itertools.accumulate(counts)), dtype=torch.int32, device=DEV)
    R = sum(counts)
    xg = rnd(R, Kg, seed=62)
    for pair in (False, True):
        for out_fp32 in ((False, True) if not pair else (False,)):
            out = C.grouped_linear(xg, wg, wg2 if pair else None, offsets, max(counts), SILU if pair else 0, out_fp32)
            record(f"grouped/offsets/pair{int(pair)}/fp32{int(out_fp32)}", out, "bf16", max(counts), Ng, Kg, pair, 0, E, R)
    for stride in (64, 128):
        cnt = [min(c, stride) for c in counts]
        cnt_t = torch.tensor(cnt, dtype=torch.int32, device=DEV)
        xs = rnd(E * stride, Kg, seed=63 + stride)
        rows = scatter_rows(cnt, stride)
        for pair in (False, True):
            out_fp32 = not pair
            out = C.grouped_linear(xs, wg, wg2 if pair else None, cnt_t, stride, SILU if pair else 0, out_fp32, None, None, None,
                                   sum(cnt), stride)
            record(f"grouped/scatter{stride}/pair{int(pair)}", out, "bf16", stride, Ng, Kg, pair, 0, E, sum(cnt), rows=rows)
            # EP return path on one GPU: row addresses into a local buffer, one local peer flag
            dst = torch.zeros(E * stride, Ng, dtype=torch.float32 if out_fp32 else torch.bfloat16, device=DEV)
            row_dst = dst.data_ptr() + torch.arange(E * stride, dtype=torch.int64, device=DEV) * (Ng * dst.element_size())
            flag = torch.zeros(1, dtype=torch.int32, device=DEV)
            peers = torch.tensor([flag.data_ptr()], dtype=torch.int64, device=DEV)
            done = torch.zeros(1, dtype=torch.int32, device=DEV)
            C.grouped_linear(xs, wg, wg2 if pair else None, cnt_t, stride, SILU if pair else 0, out_fp32, row_dst, peers, done,
                             sum(cnt), stride)
            record(f"grouped/scatter{stride}/pair{int(pair)}/row_dst", dst, "bf16", stride, Ng, Kg, pair, 0, E, sum(cnt), rows=rows,
                   flag=flag)

    # ---- quantised: persistent and workspace split-K routes, grouped offsets
    Kq, Nq = 1024, 768
    for bits in (4, 8):
        for group in (64, 128):
            def qweight(rows, seed):
                return (rnd_i32(rows, Kq * bits // 32, seed=seed), rnd(Kq // group, rows, seed=seed + 1, scale=0.01),
                        rnd(Kq // group, rows, seed=seed + 2, scale=0.01))
            q1, q2 = qweight(Nq, 70), qweight(Nq, 80)
            for T in (1, 17, 64):
                x = rnd(T, Kq, seed=90 + T)
                res_t = rnd(T, Nq, seed=100 + T)
                for splits in (1, 4):
                    for vname, kw in {"single": {}, "silu_pair": dict(pair=True, act=SILU), "gelu_pair_residual": dict(pair=True, act=GELU, residual=res_t),
                                      "bias_residual": dict(bias=rnd(Nq, seed=7, scale=0.5), residual=res_t),
                                      "fp32_softcap": dict(out_fp32=True, softcap=30.0)}.items():
                        for signal in (False, True):
                            flag, ptr = flag_args(signal)
                            pq = q2 if kw.get("pair") else (None, None, None)
                            out = C.linear_q(x, *q1, *pq, bits, group, Nq, kw.get("residual"), kw.get("bias"), kw.get("act", 0),
                                             kw.get("softcap", 0.0), kw.get("out_fp32", False), None, splits, ptr, 0)
                            record(f"linear_q/b{bits}g{group}/splits{splits}/T{T}/{vname}" + ("/signal" if signal else ""), out, "q", T,
                                   Nq, Kq, bool(kw.get("pair")), splits, flag=flag)
            gq1, gq2 = qweight(E * Nq, 110), qweight(E * Nq, 120)
            xq = rnd(R, Kq, seed=130)
            for pair in (False, True):
                pq = gq2 if pair else (None, None, None)
                out = C.grouped_linear_q(xq, *gq1, *pq, bits, group, E, Nq, offsets, max(counts), SILU if pair else 0, not pair)
                record(f"grouped_q/b{bits}g{group}/pair{int(pair)}", out, "q", max(counts), Nq, Kq, pair, 0, E, R)

    # ---- MXFP8: dense, grouped offsets, scatter
    def fp8(t):
        q, sf = C.quant_mxfp8(t.reshape(-1, t.shape[-1]))
        return q.reshape(t.shape), sf.reshape(*t.shape[:-1], -1)
    Kf, Nf = 1024, 768
    wf, wf2 = fp8(rnd(Nf, Kf, seed=140, scale=0.03)), fp8(rnd(Nf, Kf, seed=141, scale=0.03))
    for T in (1, 17, 64):
        xf = fp8(rnd(T, Kf, seed=150 + T))
        res_t = rnd(T, Nf, seed=160 + T)
        for vname, kw in {"single": {}, "silu_pair": dict(pair=True), "residual": dict(residual=res_t), "fp32": dict(out_fp32=True)}.items():
            p2 = wf2 if kw.get("pair") else (None, None)
            out = C.linear_fp8(*xf, *wf, *p2, None, 0, kw.get("residual"), SILU if kw.get("pair") else 0, kw.get("out_fp32", False))
            record(f"fp8/dense/T{T}/{vname}", out, "fp8", T, Nf, Kf, bool(kw.get("pair")))
    wfg, wfg2 = fp8(rnd(E, Nf, Kf, seed=170, scale=0.03)), fp8(rnd(E, Nf, Kf, seed=171, scale=0.03))
    xfg = fp8(rnd(R, Kf, seed=172))
    for pair in (False, True):
        p2 = wfg2 if pair else (None, None)
        out = C.linear_fp8(*xfg, *wfg, *p2, offsets, max(counts), None, SILU if pair else 0, False, R, 0)
        record(f"fp8/offsets/pair{int(pair)}", out, "fp8", max(counts), Nf, Kf, pair, 0, E, R)
    for stride in (64, 128):
        cnt = [min(c, stride) for c in counts]
        cnt_t = torch.tensor(cnt, dtype=torch.int32, device=DEV)
        xfs = fp8(rnd(E * stride, Kf, seed=173 + stride))
        for pair in (False, True):
            p2 = wfg2 if pair else (None, None)
            out = C.linear_fp8(*xfs, *wfg, *p2, cnt_t, stride, None, SILU if pair else 0, False, sum(cnt), stride)
            record(f"fp8/scatter{stride}/pair{int(pair)}", out, "fp8", stride, Nf, Kf, pair, 0, E, sum(cnt), rows=scatter_rows(cnt, stride))
    return res


def compare(a_path, b_path):
    a, b = json.load(open(a_path)), json.load(open(b_path))
    bad = 0
    for name in sorted(set(a) | set(b)):
        if a.get(name) != b.get(name):
            bad += 1
            print(f"differs: {name}: {a.get(name)} vs {b.get(name)}")
    for side, d in ((a_path, a), (b_path, b)):
        for name, r in sorted(d.items()):
            if "flag" in r and r["flag"] != 1:
                bad += 1
                print(f"flag != 1: {side}: {name}: {r['flag']}")
    print(f"{len(set(a) | set(b))} cases, {bad} problems")
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--so", help="path of the extension (_b200_C.so) to run")
    ap.add_argument("--out", help="JSON file to write")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"), help="compare two result files")
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    if not (args.so and args.out):
        ap.error("--so and --out are required unless --compare is given")
    if not torch.cuda.is_available():
        sys.exit("gemm_routes.py runs the kernels: it needs a CUDA device")
    res = run_cases(load(args.so))
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
    print(f"{len(res)} cases -> {args.out}")


if __name__ == "__main__":
    main()
