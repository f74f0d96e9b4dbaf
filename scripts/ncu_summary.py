#!/usr/bin/env python
"""Summarise an ``.ncu-rep`` (``ncu --set full``) per kernel: one markdown row per distinct kernel (first captured launch).

    python scripts/ncu_summary.py gpurun_out/ncu_smoke.ncu-rep profiles/ncu_all_kernels.md [profiles/raw/ncu_smoke_raw.csv]
"""
import csv
import io
import re
import subprocess
import sys

COLS = [("gpu__time_duration.sum", "us", 1.0),
        ("launch__grid_size", "grid", 1.0),
        ("launch__block_size", "block", 1.0),
        ("launch__registers_per_thread", "regs", 1.0),
        ("launch__shared_mem_per_block_dynamic", "dyn smem KB", 1.0),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "occupancy %", 1.0),
        ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM %", 1.0),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM %", 1.0),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor %", 1.0),
        ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue %", 1.0)]


def short(name):
    name = re.sub(r"\(.*$", "", name).replace("void ", "").replace("b200::", "").replace("<unnamed>::", "")
    return name.replace("(anonymous namespace)::", "")[:70]


def main():
    rep, out = sys.argv[1], sys.argv[2]
    if rep.endswith(".csv"):      # already exported with `ncu -i x.ncu-rep --page raw --csv`
        raw = open(rep, errors="replace").read()
    else:
        raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    if len(sys.argv) > 3 and not sys.argv[3].startswith("--"):
        open(sys.argv[3], "w").write(raw)
    title = next((a.split("=", 1)[1] for a in sys.argv[3:] if a.startswith("--title=")), None)
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    iname = hdr.index("Kernel Name")
    seen, lines = {}, []
    for r in data:
        n = short(r[iname])
        seen.setdefault(n, []).append(r)
    hdr_lines = [f"# ncu --set full: every kernel launched by `__graft_entry__.smoke()` ({len(data)} launches, {len(seen)} distinct kernels)", "",
          "`ncu --set full --clock-control none --import-source on -c 200` under `gpurun` (1 GPU) over the smoke decode of the tiny DeepSeek-V2 flagship",
          "(prefill + graph-free decode steps through `LLMEngine`).  One row per distinct kernel = its first captured launch; the tiny model makes every",
          "kernel latency-bound, so read this table as *coverage* (each hand-written kernel ran and was captured with source) — the",
          "roofline-relevant captures are `ncu_decode_kernels.md` and `ncu_gemm_persistent.md`.  Durations under ncu are not benchmark numbers.", ""]
    if title is not None:
        hdr_lines = [f"# {title} ({len(data)} launches, {len(seen)} distinct kernels)", "",
                     "One row per distinct kernel = its first captured launch.  Durations under ncu are not benchmark numbers.", ""]
    md = hdr_lines + [
          "| kernel | launches | " + " | ".join(c[1] for c in COLS) + " |", "|---|---:|" + "---:|" * len(COLS)]
    for n, rs in seen.items():
        r = rs[0]
        vals = []
        for key, _, _ in COLS:
            if key in hdr:
                v = r[hdr.index(key)].replace(",", "")
                try:
                    f = float(v)
                    vals.append(f"{f:.1f}" if (f != int(f) or "pct" in key or "duration" in key) else str(int(f)))
                except ValueError:
                    vals.append(v or "-")
            else:
                vals.append("-")
        md.append(f"| `{n}` | {len(rs)} | " + " | ".join(vals) + " |")
    open(out, "w").write("\n".join(md) + "\n")
    print(f"{len(seen)} kernels -> {out}")


if __name__ == "__main__":
    main()
