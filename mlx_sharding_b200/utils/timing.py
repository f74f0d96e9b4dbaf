"""Measurement helpers: CUDA-event timing (max over ranks), clock / throttle sampling, L2 flush.

The reference's only instrumentation is a wall-clock tokens-per-second print (generate.py:114-122,
SURVEY §5.1); these follow a GPU profiling recipe instead: device-timed, warm-up first, clocks sampled
*during* the timed region, multi-GPU numbers reported as the max over ranks.
"""
from __future__ import annotations

import statistics
import subprocess
import threading
import time
from typing import Dict, List, Optional

import torch

_QUERY = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
          "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
          "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")


class ClockSampler:
    """Samples ``nvidia-smi`` clocks / throttle reasons every ``period_ms`` in a background thread."""

    def __init__(self, gpu_index: int = 0, period_ms: int = 100):
        self.idx, self.period = gpu_index, period_ms / 1000.0
        self.samples: List[Dict] = []
        self._stop = threading.Event()
        self._thr: Optional[threading.Thread] = None

    def _poll_nvml(self) -> bool:
        """Fast path: NVML bindings (no process spawn) — ~1 ms per sample."""
        try:
            import pynvml as nv

            nv.nvmlInit()
            try:  # CUDA device index -> physical GPU (CUDA_VISIBLE_DEVICES may reorder / hide devices)
                uuid = "GPU-" + str(torch.cuda.get_device_properties(self.idx).uuid)
                h = nv.nvmlDeviceGetHandleByUUID(uuid.encode() if hasattr(uuid, "encode") else uuid)
            except Exception:  # noqa: BLE001
                h = nv.nvmlDeviceGetHandleByIndex(self.idx)
            sm_max = float(nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM))
            get_reasons = getattr(nv, "nvmlDeviceGetCurrentClocksEventReasons", None) or nv.nvmlDeviceGetCurrentClocksThrottleReasons
            bits = dict(hw_slowdown=0x8, sw_power_cap=0x4, sw_thermal=0x20, hw_thermal=0x40)
        except Exception:  # noqa: BLE001
            return False
        while not self._stop.is_set():
            try:
                r = int(get_reasons(h))
                on = lambda k: "Active" if r & bits[k] else "Not Active"
                self.samples.append(dict(sm=float(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)), sm_max=sm_max,
                                         power=nv.nvmlDeviceGetPowerUsage(h) / 1000.0, active=hex(r), hw_slowdown=on("hw_slowdown"),
                                         hw_thermal=on("hw_thermal"), sw_thermal=on("sw_thermal"), sw_power_cap=on("sw_power_cap")))
            except Exception:  # noqa: BLE001
                pass
            self._stop.wait(min(self.period, 0.02))
        return True

    def _poll(self):
        if self._poll_nvml():
            return
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={_QUERY}", "--format=csv,noheader,nounits", "-i",
                                      str(self.idx)], capture_output=True, text=True, timeout=5).stdout.strip()
                f = [x.strip() for x in out.split(",")]
                if len(f) >= 9:
                    self.samples.append(dict(sm=float(f[1]), sm_max=float(f[2]), power=float(f[3]), active=f[4],
                                             hw_slowdown=f[5], hw_thermal=f[6], sw_thermal=f[7], sw_power_cap=f[8]))
            except Exception:  # noqa: BLE001 — sampling must never break a benchmark
                pass
            self._stop.wait(self.period)

    def __enter__(self):
        self._thr = threading.Thread(target=self._poll, daemon=True)
        self._thr.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        if self._thr:
            self._thr.join(timeout=6)

    def summary(self) -> Dict:
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        reasons = set()
        for s in self.samples:
            for key, name in (("hw_slowdown", "hw_slowdown"), ("hw_thermal", "hw_thermal_slowdown"),
                              ("sw_thermal", "sw_thermal_slowdown"), ("sw_power_cap", "sw_power_cap")):
                if s[key].lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(s["sm"] for s in self.samples), "sm_max_mhz": self.samples[0]["sm_max"],
                "power_w_max": max(s["power"] for s in self.samples), "reasons": sorted(reasons),
                "samples": len(self.samples)}


_flush_buf = None


def flush_l2(nbytes: int = 256 << 20):
    """Write a buffer larger than the 50 MB L2 so the next kernel starts cold."""
    global _flush_buf
    if _flush_buf is None or _flush_buf.numel() < nbytes:
        _flush_buf = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    _flush_buf.fill_(1)


def max_over_ranks(value: float) -> float:
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return value
    t = torch.tensor([value], dtype=torch.float64, device="cuda" if torch.cuda.is_available() else "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


class CudaTimer:
    def __init__(self):
        self.e0 = torch.cuda.Event(enable_timing=True)
        self.e1 = torch.cuda.Event(enable_timing=True)

    def __enter__(self):
        self.e0.record()
        return self

    def __exit__(self, *a):
        self.e1.record()
        self.e1.synchronize()
        self.ms = self.e0.elapsed_time(self.e1)
