"""Time the bf16 GEMM launch alone at the DiT block shapes, each with its production epilogue, optionally alternating with a
second build of the library in the same process (A B A B ...), so that two kernels are compared on the same card, clocks and
inputs.

    python tools/bench_gemm.py                              # this tree's library
    python tools/bench_gemm.py --other /path/libyume_b200.so --rounds 3 --out result.json

Shapes: q|k|v, o, cross q, cross o, ffn.0 and ffn.2 of the 5B step (L = 18 480, C = 3072, ffn 14 336) and of the 14B FramePack
chunk (L = 21 930, C = 5120, ffn 13 824). o and ffn.2 are gated residual updates (x += (acc + b) * gate[tok]) with one gate row
per latent frame, cross o is the ungated one. Each timing is CUDA events around back-to-back launches filling a window of
--seconds (default 1.5 s); the rate is 2 * M * N * K / time. With --other, the outputs of the two libraries are compared on the
same seeded inputs (one launch each from the same starting residual): bit for bit, and for the gated residual updates also as
the largest difference in fp32 ulps of the residual's magnitude and the relative Frobenius norm of the difference.
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
from yume_b200._lib import GemmArgs  # noqa: E402

EPI_BF16, EPI_GELU_BF16, EPI_GATE_RES = 0, 1, 3


def _shapes(tag, L, C_, F, frames):
    # (name, M, N, K, epilogue, gated, frames of the gate table)
    return [(f"{tag}_qkv", L, 3 * C_, C_, EPI_BF16, False, frames), (f"{tag}_o", L, C_, C_, EPI_GATE_RES, True, frames),
            (f"{tag}_cross_q", L, C_, C_, EPI_BF16, False, frames), (f"{tag}_cross_o", L, C_, C_, EPI_GATE_RES, False, frames),
            (f"{tag}_ffn0", L, F, C_, EPI_GELU_BF16, False, frames), (f"{tag}_ffn2", L, C_, F, EPI_GATE_RES, True, frames)]


SHAPES = _shapes("5b", 18480, 3072, 14336, 21) + _shapes("14b", 21930, 5120, 13824, 13)


def _bind(path: Path):
    lib = C.CDLL(str(path))
    lib.yb_gemm_bf16.restype = C.c_int
    lib.yb_gemm_bf16.argtypes = [C.POINTER(GemmArgs), C.c_void_p]
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
    def __init__(self, M, N, K, epi, gated, frames, seed=0):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.M, self.N, self.K, self.epi = M, N, K, epi
        self.a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
        self.w = (torch.randn(N, K, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
        self.bias = torch.randn(N, device="cuda", generator=g)
        self.gate = self.tok = None
        if gated:   # one gate row per latent frame, tokens frame-major (the engine's per-frame timestep layout)
            self.gate = torch.randn(frames, N, device="cuda", generator=g)
            self.tok = (torch.arange(M, device="cuda") * frames // M).to(torch.int32)
        dtype = torch.float32 if epi == EPI_GATE_RES else torch.bfloat16
        self.x0 = torch.randn(M, N, device="cuda", generator=g) if epi == EPI_GATE_RES else None
        self.out = torch.empty(M, N, device="cuda", dtype=dtype)

    def launch(self, lib, out):
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        args = GemmArgs(struct_bytes=C.sizeof(GemmArgs), cta_pair=0, A=self.a.data_ptr(), B=self.w.data_ptr(),
                        bias=self.bias.data_ptr(), out=out.data_ptr(), gate=ptr(self.gate), tok_idx=ptr(self.tok),
                        lda=self.K, ldb=self.K, ldo=self.N, gate_ld=self.N if self.gate is not None else 0,
                        M=self.M, N=self.N, K=self.K, epilogue=self.epi, block_n=0, split_k=1)
        rc = lib.yb_gemm_bf16(C.byref(args), C.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc != 0:
            raise RuntimeError(f"yb_gemm_bf16 returned {rc}")

    def result(self, lib):
        """One launch from the seeded starting state."""
        out = self.x0.clone() if self.x0 is not None else torch.empty_like(self.out)
        self.launch(lib, out)
        torch.cuda.synchronize()
        return out

    def time_ms(self, lib, seconds):
        if self.x0 is not None:
            self.out.copy_(self.x0)   # the residual grows by one update per launch; start every window from the same state
        for _ in range(3):
            self.launch(lib, self.out)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        self.launch(lib, self.out)
        t1.record()
        torch.cuda.synchronize()
        n = max(5, math.ceil(seconds * 1e3 / max(t0.elapsed_time(t1), 1e-3)))
        t0.record()
        for _ in range(n):
            self.launch(lib, self.out)
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / n, n


def _compare(a: torch.Tensor, b: torch.Tensor, x0=None) -> dict:
    r = {"identical": bool(torch.equal(a, b))}
    af, bf = a.float(), b.float()
    r["max_abs_diff"] = float((af - bf).abs().max())
    r["rel_frobenius"] = float((af - bf).norm() / bf.norm().clamp_min(1e-30))
    if x0 is not None:
        # residual updates: the difference in ulps of the residual's scale, max(|x0|, |a|, |b|) per element (where x and the
        # update cancel, ulps of the small result itself would be no measure of the rounding)
        scale = torch.maximum(torch.maximum(af.abs(), bf.abs()), x0.abs())
        _, ex = torch.frexp(scale)
        ulp = torch.ldexp(torch.ones_like(scale), ex.to(torch.int32) - 24)
        r["max_diff_ulps"] = float(((af - bf).abs() / ulp).max())
    return r


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
        raise SystemExit("bench_gemm needs a GPU")

    libs = {"A": _bind(args.lib)}
    if args.other:
        libs["B"] = _bind(args.other)
    wanted = set(args.shapes.split(","))
    result = {"card": _card(), "libs": {k: str(v) for k, v in (("A", args.lib), ("B", args.other)) if v}, "shapes": []}
    print(json.dumps(result["card"]), flush=True)
    for name, M, N, K, epi, gated, frames in SHAPES:
        if name not in wanted:
            continue
        case = Case(M, N, K, epi, gated, frames)
        flop = 2.0 * M * N * K
        runs = {label: [] for label in libs}
        for _ in range(args.rounds):
            for label, lib in libs.items():
                ms, n = case.time_ms(lib, args.seconds)
                runs[label].append({"ms": ms, "launches": n, "tflops": flop / (ms * 1e-3) / 1e12})
        entry = {"name": name, "M": M, "N": N, "K": K, "epilogue": epi, "gated": gated, "tflop_per_launch": flop / 1e12,
                 "runs": runs}
        for label in libs:
            ms = [r["ms"] for r in runs[label]]
            entry[label] = {"mean_ms": sum(ms) / len(ms), "min_ms": min(ms), "max_ms": max(ms),
                            "mean_tflops": flop / (sum(ms) / len(ms) * 1e-3) / 1e12}
        line = f"{name:14s} {M}x{N}x{K} epi={epi}{' gated' if gated else ''}: " + "  ".join(
            f"{lab} {entry[lab]['mean_ms'] * 1e3:.0f} us [{entry[lab]['min_ms'] * 1e3:.0f}, {entry[lab]['max_ms'] * 1e3:.0f}] "
            f"{entry[lab]['mean_tflops']:.0f} TFLOP/s" for lab in libs)
        if "B" in libs:
            entry["outputs"] = _compare(case.result(libs["A"]), case.result(libs["B"]), case.x0)
            entry["speedup_A_over_B"] = entry["B"]["mean_ms"] / entry["A"]["mean_ms"]   # > 1: A (this tree) is faster
            line += f"  A/B {entry['speedup_A_over_B']:.3f}x  " + " ".join(f"{k}={v}" for k, v in entry["outputs"].items())
        result["shapes"].append(entry)
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
