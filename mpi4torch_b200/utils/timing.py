"""Measurement hygiene shared by bench.py and the sweep scripts.

Rules: time on the device with CUDA events on the launching
stream, >= 3 warm-ups, flush L2 between timed iterations (or use inputs larger
than L2), take the max over ranks, and sample SM clocks / throttle reasons
DURING the timed region.
"""
from __future__ import annotations

import statistics
import subprocess
import threading
import time
from typing import Callable, Dict, List, Optional

import torch


class L2Flusher:
    """Writes a buffer larger than the 50 MB L2 so the next iteration starts cold."""

    def __init__(self, device, nbytes: int = 256 << 20):
        self.buf = torch.empty(nbytes, dtype=torch.uint8, device=device)

    def flush(self) -> None:
        self.buf.zero_()


def cuda_time_ms(fn: Callable[[], None], steps: int, warmup: int = 3, flusher: Optional[L2Flusher] = None,
                 barrier: Optional[Callable[[], None]] = None) -> List[float]:
    """Per-iteration device times in milliseconds (CUDA events around each call)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        if flusher is not None:
            flusher.flush()
        if barrier is not None:
            barrier()
        a = torch.cuda.Event(enable_timing=True)
        b = torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return times


def max_over_ranks(value: float, comm) -> float:
    """Max over ranks of a host scalar (through the library's own Allreduce)."""
    import mpi4torch_b200 as m4t

    t = torch.tensor([value], dtype=torch.float64)
    return float(comm.Allreduce(t, m4t.MPI_MAX)[0])


class ClockSampler:
    """Samples ``nvidia-smi`` clocks and throttle reasons in a background thread."""

    QUERY = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
             "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int = 0, period_ms: int = 200):
        self.gpu_index = gpu_index
        self.period_ms = period_ms
        self.samples: List[Dict[str, str]] = []
        self._proc: Optional[subprocess.Popen] = None
        self._thread: Optional[threading.Thread] = None

    def start(self) -> "ClockSampler":
        try:
            self._proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={self.QUERY}", "--format=csv,noheader,nounits", "-i", str(self.gpu_index),
                 "-lms", str(self.period_ms)],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except OSError:
            self._proc = None
            return self
        self._thread = threading.Thread(target=self._pump, daemon=True)
        self._thread.start()
        return self

    def _pump(self) -> None:
        assert self._proc is not None and self._proc.stdout is not None
        keys = self.QUERY.split(",")
        for line in self._proc.stdout:
            parts = [p.strip() for p in line.strip().split(",")]
            if len(parts) == len(keys):
                self.samples.append(dict(zip(keys, parts)))

    def stop(self) -> Dict[str, object]:
        if self._proc is not None:
            time.sleep(self.period_ms / 1000.0)
            self._proc.terminate()
            try:
                self._proc.wait(timeout=2)
            except subprocess.TimeoutExpired:  # pragma: no cover
                self._proc.kill()
        if self._thread is not None:
            self._thread.join(timeout=2)
        return self.summary()

    def summary(self) -> Dict[str, object]:
        sm, smax, reasons = [], [], set()
        for s in self.samples:
            try:
                sm.append(float(s["clocks.sm"]))
                smax.append(float(s["clocks.max.sm"]))
            except (KeyError, ValueError):
                continue
            for key in ("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"):
                if s.get(f"clocks_event_reasons.{key}", "").lower().startswith("active"):
                    reasons.add(key)
        return {
            "sm_mhz": statistics.median(sm) if sm else None,
            "sm_max_mhz": max(smax) if smax else None,
            "reasons": sorted(reasons),
            "samples": len(sm),
        }
