"""Measurement helpers: per-kernel CUDA-event timing inside a live step, and nvidia-smi clock sampling."""
from __future__ import annotations

import statistics
import subprocess
import threading
import time
from collections import defaultdict
from typing import Dict, List, Optional, Tuple

import torch


class KernelTimer:
    """Records CUDA events around tagged launches on the current stream. Enabled only while `active` so the
    untimed path pays nothing. Durations are read after a synchronize (never under a profiler)."""

    def __init__(self):
        self.active = False
        self._pairs: Dict[str, List[Tuple[torch.cuda.Event, torch.cuda.Event]]] = defaultdict(list)
        self._open: Dict[str, torch.cuda.Event] = {}

    def begin(self, tag: str) -> None:
        if self.active:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self._open[tag] = ev

    def end(self, tag: str) -> None:
        if self.active:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self._pairs[tag].append((self._open.pop(tag), ev))

    def reset(self) -> None:
        self._pairs.clear()
        self._open.clear()

    def summary(self) -> Dict[str, Dict[str, float]]:
        """tag -> {count, mean_ms, total_ms}; call after torch.cuda.synchronize()."""
        out = {}
        for tag, pairs in self._pairs.items():
            ms = [a.elapsed_time(b) for a, b in pairs]
            out[tag] = dict(count=len(ms), mean_ms=sum(ms) / len(ms), total_ms=sum(ms))
        return out


class ClockSampler:
    """Samples SM clocks and throttle reasons of one GPU in a background thread while a timed region runs: NVML every 20 ms
    when `pynvml` can open the device (a 40 ms multi-GPU step still gets several samples under load), else the `nvidia-smi`
    query line below every 200 ms. Both read the same driver counters."""

    QUERY = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
             "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
    # NVML clocks-event-reason bits (nvml.h: nvmlClocksEventReason*)
    _NVML_BITS = (("hw_slowdown", 0x8), ("hw_thermal_slowdown", 0x40), ("sw_thermal_slowdown", 0x20), ("sw_power_cap", 0x4))

    def __init__(self, gpu_index: int = 0):
        self.gpu_index = gpu_index
        self.samples: List[List[str]] = []
        self.source = "nvidia-smi"
        self._stop = threading.Event()
        self._thread: Optional[threading.Thread] = None
        self._nvml = None

    def _open_nvml(self):
        try:
            import pynvml
            pynvml.nvmlInit()
            handle = None
            try:                                                   # CUDA ordinal -> NVML handle through the UUID
                import torch
                uuid = str(torch.cuda.get_device_properties(self.gpu_index).uuid)
                handle = pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + uuid) if not uuid.startswith("GPU-") else uuid)
            except Exception:
                handle = pynvml.nvmlDeviceGetHandleByIndex(self.gpu_index)
            pynvml.nvmlDeviceGetClockInfo(handle, pynvml.NVML_CLOCK_SM)
            return pynvml, handle
        except Exception:
            return None

    def _run(self):
        if self._nvml is not None:
            nv, h = self._nvml
            mx = nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)
            get_reasons = getattr(nv, "nvmlDeviceGetCurrentClocksEventReasons", None) or nv.nvmlDeviceGetCurrentClocksThrottleReasons
            while not self._stop.is_set():
                try:
                    bits = int(get_reasons(h))
                    self.samples.append([str(self.gpu_index), str(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)), str(mx), "", ""]
                                        + [("Active" if bits & b else "Not Active") for _, b in self._NVML_BITS])
                except Exception:
                    pass
                self._stop.wait(0.02)
            return
        while not self._stop.is_set():
            try:
                r = subprocess.run(["nvidia-smi", f"--query-gpu={self.QUERY}", "--format=csv,noheader,nounits",
                                    "-i", str(self.gpu_index)], capture_output=True, text=True, timeout=5)
                if r.returncode == 0 and r.stdout.strip():
                    self.samples.append([c.strip() for c in r.stdout.strip().splitlines()[0].split(",")])
            except Exception:
                pass
            self._stop.wait(0.2)

    def __enter__(self):
        self._nvml = self._open_nvml()
        self.source = "nvml" if self._nvml is not None else "nvidia-smi"
        self._thread = threading.Thread(target=self._run, daemon=True)
        self._thread.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        if self._thread:
            self._thread.join(timeout=6)

    def summary(self) -> dict:
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for s in self.samples:
            try:
                sm.append(float(s[1]))
                mx.append(float(s[2]))
            except (ValueError, IndexError):
                continue
            for name, val in zip(names, s[5:9]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no_samples"]}
        return {"sm_mhz": statistics.median(sm), "sm_max_mhz": max(mx), "reasons": sorted(reasons),
                "samples": len(sm), "source": self.source}
