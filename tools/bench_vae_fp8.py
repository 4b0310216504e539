"""Wan2.2 VAE decode, bf16 against precision="fp8", on one GPU: per-conv-shape TFLOP/s of the converted convs (bf16
yb_conv3d_causal against yb_conv3d_fp8, launch alone, the same shapes), the decode time of 13 latent frames (49 video frames)
and of the sampler's 8-frame tail, both at 704 x 1280, and the fp8-vs-bf16 PSNR of the 13-frame video. bf16 and fp8 alternate
in one process; the card's name and power limit are read in the same run. The weights are seeded random ones
(oracle/wan22vae.make_state_dict), not a checkpoint: the PSNR says how far e4m3 moves this network, not a trained one.

    python tools/bench_vae_fp8.py [--rounds 3] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import math
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle import wan22vae  # noqa: E402
from oracle.fp8 import quantize_act, quantize_weight  # noqa: E402
from yume_b200 import ops  # noqa: E402
from yume_b200.vae22 import Wan22VaeDecoder  # noqa: E402

# the converted convs of a 13-latent-frame decode at 704 x 1280: (name, frames, H, W, Cp, Cout, taps, launches per decode)
SHAPES = [("L0 res 1024", 13, 44, 80, 1024, 1024, (3, 3, 3), 10), ("L0 resample 1024", 25, 88, 160, 1024, 1024, (1, 3, 3), 1),
          ("L1 res 1024", 25, 88, 160, 1024, 1024, (3, 3, 3), 6), ("L1 resample 1024", 49, 176, 320, 1024, 1024, (1, 3, 3), 1),
          ("L2 res 1024->512", 49, 176, 320, 1024, 512, (3, 3, 3), 1), ("L2 res 512", 49, 176, 320, 512, 512, (3, 3, 3), 5),
          ("L2 resample 512", 49, 352, 640, 512, 512, (1, 3, 3), 1), ("L3 res 512->256", 49, 352, 640, 512, 256, (3, 3, 3), 1),
          ("L3 res 256", 49, 352, 640, 256, 256, (3, 3, 3), 5)]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps / 1e3


def conv_shapes(rounds, reps):
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, T, H, W, Cp, Cout, taps, n in SHAPES:
        K = math.prod(taps) * Cp
        x = torch.empty(T * H * W, Cp, dtype=torch.bfloat16, device="cuda")
        q = torch.empty(T * H * W, Cp, dtype=torch.float8_e4m3fn, device="cuda")
        s = torch.empty(Cp // 128, T * H * W, device="cuda")
        for t in range(T):                                   # SiLU-like activations, quantised frame by frame
            sl = slice(t * H * W, (t + 1) * H * W)
            x[sl] = torch.nn.functional.silu(torch.randn(H * W, Cp, device="cuda", generator=g)).to(torch.bfloat16)
            q[sl], s[:, sl] = quantize_act(x[sl].float())
        q = q.view(T, H, W, Cp)
        s = s.view(Cp // 128, T, H, W).transpose(0, 1).contiguous()
        x = x.view(T, H, W, Cp)
        w = torch.randn(Cout, K, device="cuda", generator=g) * K ** -0.5
        wb = w.to(torch.bfloat16)
        wq, sw = quantize_weight(w)
        del w
        bias = torch.zeros(Cout, device="cuda")
        out = torch.empty(T * H * W, Cout, dtype=torch.bfloat16, device="cuda")
        flop = 2.0 * T * H * W * K * Cout
        tb, t8 = [], []
        for _ in range(rounds):
            tb.append(timed(lambda: ops.conv3d_causal(x, wb, bias, out, T, H, W, taps=taps, oob_zero_pad=True), reps))
            t8.append(timed(lambda: ops.conv3d_fp8(q, s, wq, sw, bias, out, T, H, W, 0, taps=taps), reps))
        b, f = min(tb), min(t8)
        rows.append(dict(shape=name, launches=n, bf16_ms=b * 1e3, fp8_ms=f * 1e3, bf16_tflops=flop / b / 1e12,
                         fp8_tflops=flop / f / 1e12, speedup=b / f))
        print(f"{name:18s} x{n:2d}: bf16 {b * 1e3:7.2f} ms {flop / b / 1e12:6.0f} TFLOP/s | fp8 {f * 1e3:7.2f} ms "
              f"{flop / f / 1e12:6.0f} TFLOP/s | {b / f:.2f}x", flush=True)
        del x, q, s, wb, wq, out
        torch.cuda.empty_cache()
    return rows


def psnr(a, b):
    mse = float((a.double() - b.double()).pow(2).mean())
    return math.inf if mse == 0 else 10 * math.log10(4.0 / mse)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", type=str, default=None)
    ap.add_argument("--skip-convs", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_vae_fp8 measures on a GPU"
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    res = dict(gpu=info, weights="seeded random (oracle/wan22vae.make_state_dict(0)), not a checkpoint")
    if not args.skip_convs:
        res["convs"] = conv_shapes(args.rounds, args.reps)
    sd = wan22vae.make_state_dict(0, dec_dim=256, z_dim=48)
    eng = {p: Wan22VaeDecoder(sd, dec_dim=256, z_dim=48, device="cuda", precision=p) for p in ("bf16", "fp8")}
    del sd
    res["decode"] = []
    for T in (13, 8):
        z = torch.randn(48, T, 44, 80, generator=torch.Generator().manual_seed(T)).cuda()
        plans = {p: e.plan_chunks(T, 44, 80) for p, e in eng.items()}
        outs = {p: e.decode(z) for p, e in eng.items()}                      # warm-up
        times = {p: [] for p in eng}
        for _ in range(args.rounds):
            for p, e in eng.items():
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                outs[p] = e.decode(z)
                b.record()
                torch.cuda.synchronize()
                times[p].append(a.elapsed_time(b) / 1e3)
        row = dict(latent_frames=T, video_frames=1 + 4 * (T - 1), size="704x1280", chunks=plans,
                   bf16_s=min(times["bf16"]), fp8_s=min(times["fp8"]), speedup=min(times["bf16"]) / min(times["fp8"]),
                   psnr_fp8_vs_bf16_db=psnr(outs["fp8"], outs["bf16"]))
        res["decode"].append(row)
        print(f"decode {T} latent frames ({row['video_frames']} frames, 704x1280, chunks {plans['fp8']}): bf16 {row['bf16_s']:.3f} s, "
              f"fp8 {row['fp8_s']:.3f} s, {row['speedup']:.2f}x; fp8 vs bf16 PSNR {row['psnr_fp8_vs_bf16_db']:.1f} dB", flush=True)
        del outs, z
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    print(f"GPU after: {res['gpu_after']}")
    if args.json:
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
