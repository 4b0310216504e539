"""Time the attention launch alone at the shapes the engines run, optionally alternating with a second build of the
library in the same process (A B A B ...), so that two kernels are compared on the same card, clocks and inputs.

    python tools/bench_attention.py                              # this tree's library
    python tools/bench_attention.py --other /path/libyume_b200.so --rounds 3 --out result.json

Each timing is CUDA events around back-to-back launches filling a window of --seconds (default 1.5 s). The rate is
4 * Lq * Lk * 128 * heads / time, the algorithmic work of non-causal attention with head dim 128. With --other, the outputs
of the two libraries are also compared bit for bit on the same seeded inputs.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

# (name, Lq, Lk, heads): 5B 720p step (L = 18 480, 24 heads), its cross-attention over the 512-token context, the 14B
# FramePack chunk (L = 21 930, 40 heads), the full 81-frame 14B grid (L = 42 840), and one rank of the 5B step and of the
# 14B grid on 8 GPUs under Ulysses (3 of 24 and 5 of 40 heads, all rows). On a 132-SM H100 the 5B self shape and the 14B
# grid rank take the KV tail split (attention_plan); the 5B rank does not (its last wave is 87 of 132 units).
SHAPES = [
    ("5b_self", 18480, 18480, 24),
    ("5b_cross", 18480, 512, 24),
    ("14b_chunk_self", 21930, 21930, 40),
    ("14b_grid_self", 42840, 42840, 40),
    ("5b_sp8_rank_self", 18480, 18480, 3),
    ("14b_grid_sp8_rank_self", 42840, 42840, 5),
]


def _bind(path: Path):
    lib = C.CDLL(str(path))
    lib.yb_attention_ex.restype = C.c_int
    lib.yb_attention_ex.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong,
                                    C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int,
                                    C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p]
    lib.yb_attention_workspace_bytes.restype = C.c_longlong
    lib.yb_attention_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    return lib


def _card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


class Case:
    def __init__(self, Lq, Lk, heads, libs, seed=0):
        g = torch.Generator(device="cuda").manual_seed(seed)
        cols = heads * 128
        self.q = torch.randn(Lq, cols, device="cuda", dtype=torch.bfloat16, generator=g)
        self.k = torch.randn(Lk, cols, device="cuda", dtype=torch.bfloat16, generator=g)
        self.v = torch.randn(Lk, cols, device="cuda", dtype=torch.bfloat16, generator=g)
        self.Lq, self.Lk, self.heads, self.cols = Lq, Lk, heads, cols
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        ws = max(lib.yb_attention_workspace_bytes(Lq, Lk, heads, sms, 0) for lib in libs)
        self.ws = torch.empty(max(ws, 16), device="cuda", dtype=torch.uint8)
        self.outs = {}

    def launch(self, lib, out):
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        rc = lib.yb_attention_ex(self.q.data_ptr(), self.cols, self.k.data_ptr(), self.cols, self.v.data_ptr(), self.cols,
                                 out.data_ptr(), self.cols, self.Lq, self.Lk, self.heads, 1.0 / math.sqrt(128.0), 0,
                                 self.ws.data_ptr(), self.ws.numel(), None, stream)
        if rc != 0:
            raise RuntimeError(f"yb_attention_ex returned {rc}")

    def out_for(self, label):
        if label not in self.outs:
            self.outs[label] = torch.empty(self.Lq, self.cols, device="cuda", dtype=torch.bfloat16)
        return self.outs[label]

    def time_ms(self, lib, label, seconds):
        out = self.out_for(label)
        for _ in range(3):
            self.launch(lib, out)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        self.launch(lib, out)
        t1.record()
        torch.cuda.synchronize()
        n = max(5, math.ceil(seconds * 1e3 / max(t0.elapsed_time(t1), 1e-3)))
        t0.record()
        for _ in range(n):
            self.launch(lib, out)
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / n, n


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lib", type=Path, default=ROOT / "yume_b200" / "csrc" / "libyume_b200.so", help="library A")
    ap.add_argument("--other", type=Path, help="library B, alternated with A in every round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=1.5, help="timed window per measurement")
    ap.add_argument("--shapes", default=",".join(s[0] for s in SHAPES))
    ap.add_argument("--out", type=Path, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention needs a GPU")

    libs = {"A": _bind(args.lib)}
    if args.other:
        libs["B"] = _bind(args.other)
    wanted = set(args.shapes.split(","))
    result = {"card": _card(), "libs": {k: str(v) for k, v in (("A", args.lib), ("B", args.other)) if v}, "shapes": []}
    for name, Lq, Lk, heads in SHAPES:
        if name not in wanted:
            continue
        case = Case(Lq, Lk, heads, list(libs.values()))
        flop = 4.0 * Lq * Lk * 128 * heads
        runs = {label: [] for label in libs}
        for _ in range(args.rounds):
            for label, lib in libs.items():
                ms, n = case.time_ms(lib, label, args.seconds)
                runs[label].append({"ms": ms, "launches": n, "tflops": flop / (ms * 1e-3) / 1e12})
        entry = {"name": name, "Lq": Lq, "Lk": Lk, "heads": heads, "tflop_per_launch": flop / 1e12, "runs": runs}
        for label in libs:
            ms = [r["ms"] for r in runs[label]]
            entry[label] = {"mean_ms": sum(ms) / len(ms), "min_ms": min(ms), "max_ms": max(ms),
                            "mean_tflops": flop / (sum(ms) / len(ms) * 1e-3) / 1e12}
        if "B" in libs:
            a, b = case.out_for("A").float(), case.out_for("B").float()
            entry["outputs_identical"] = bool(torch.equal(case.out_for("A"), case.out_for("B")))
            entry["max_abs_diff"] = float((a - b).abs().max())
            entry["speedup_B_over_A"] = entry["A"]["mean_ms"] / entry["B"]["mean_ms"]   # > 1: B is faster
        result["shapes"].append(entry)
        line = f"{name:22s} Lq={Lq} Lk={Lk} heads={heads}: " + "  ".join(
            f"{lab} {entry[lab]['mean_ms']:.3f} ms [{entry[lab]['min_ms']:.3f}, {entry[lab]['max_ms']:.3f}] "
            f"{entry[lab]['mean_tflops']:.0f} TFLOP/s" for lab in libs)
        if "B" in libs:
            line += f"  identical={entry['outputs_identical']}"
        print(line, flush=True)
        del case
        torch.cuda.empty_cache()
    print(json.dumps(result))
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(json.dumps(result, indent=1))
    return 0


if __name__ == "__main__":
    sys.exit(main())
