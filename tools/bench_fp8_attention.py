"""bf16 vs fp8 self-attention, and the bf16 / fp8 / fp8_attn forwards, on one GPU in one process (DESIGN.md §3).

Attention launches, at the 5B (L = 18 480, 24 heads), 14B-chunk (L = 21 930, 40 heads) and 14B-grid (L = 42 840, 40 heads) self
shapes: yb_attention (bf16), yb_attention_fp8 alone, and yb_attention_fp8 with its two quantiser launches (yb_quant_rows_fp8 over
the [L, 2C] q|k view and yb_quant_vt_fp8), alternated launch by launch, 3 rounds (CUDA events, median per round).

Forwards: the full-depth 5B denoise step and 14B chunk forward (tools/bench_fp8.py's inputs) in "bf16", "fp8" and "fp8_attn",
alternated in one process, with the rel-Frobenius distance between each pair. The 14B engines do not fit three at a time in
80 GB, so bf16 is timed on its own first, then fp8 and fp8_attn alternate. Prints one JSON line at the end.

    python tools/bench_fp8_attention.py [--reps 20] [--skip-forwards]
"""
import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from bench_fp8 import card, full_depth_state_dict, timed  # noqa: E402
from oracle import synth  # noqa: E402
from yume_b200 import ops  # noqa: E402
from yume_b200.dit import WanDiT  # noqa: E402

E4M3 = torch.float8_e4m3fn
SHAPES = [("5b", 18480, 24), ("14b_chunk", 21930, 40), ("14b_grid", 42840, 40)]


def bench_attention(name, L, H, reps, rounds=3):
    W = H * 128
    g = torch.Generator(device="cuda").manual_seed(L)
    qkv = torch.randn(L, 3 * W, device="cuda", generator=g).to(torch.bfloat16)
    qkv[:, :W].mul_(2.0)
    out16 = torch.empty(L, W, device="cuda", dtype=torch.bfloat16)
    out8 = torch.empty_like(out16)
    qk8 = torch.empty(L, 2 * W, device="cuda", dtype=E4M3)
    qk_s = torch.empty(2 * H, ops.fp8_scale_ld(L), device="cuda")
    Lkp = ops.vt8_keys(L)
    vt8 = torch.empty(H, 128, Lkp, device="cuda", dtype=E4M3)
    v_s = torch.empty(H, Lkp // 128, device="cuda")
    q, k, v = qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:]

    def quant():
        ops.quant_rows_fp8(qkv[:, :2 * W], qk8, qk_s)
        ops.quant_vt_fp8(v, vt8, v_s, H)

    def f16():
        ops.attention(q, k, v, out16, H)

    def f8():
        ops.attention_fp8(qk8[:, :W], qk8[:, W:], qk_s, vt8, v_s, out8, H)

    def f8q():
        quant()
        f8()
    quant()
    res = dict(shape=name, L=L, heads=H, rounds=[])
    for _ in range(rounds):
        t16, t8, t8q = timed([f16, f8, f8q], reps)
        res["rounds"].append(dict(bf16_ms=round(t16, 3), fp8_ms=round(t8, 3), fp8_with_quant_ms=round(t8q, 3)))
    fl = 4.0 * L * L * H * 128
    for key in ("bf16_ms", "fp8_ms", "fp8_with_quant_ms"):
        best = min(r[key] for r in res["rounds"])
        res[key.replace("_ms", "_tflops_best")] = round(fl / best / 1e9, 1)
    res["speedup_with_quant"] = round(min(r["bf16_ms"] for r in res["rounds"]) / min(r["fp8_with_quant_ms"] for r in res["rounds"]), 3)
    f16()
    f8q()
    torch.cuda.synchronize()
    res["rel_frobenius_fp8_vs_bf16"] = float((out8.float() - out16.float()).norm() / out16.float().norm())
    print(json.dumps(res), flush=True)
    del qkv, out16, out8, qk8, vt8
    torch.cuda.empty_cache()
    return res


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def bench_forwards(name, reps):
    cfg = getattr(synth, name)
    sd = full_depth_state_dict(cfg, 5)
    kw = synth.oracle_kwargs(cfg)
    variant = kw.pop("variant")
    if variant == "5b":
        inp = synth.make_inputs(cfg, 9, 21, 44, 80, 512)
        args = (inp["x"], torch.tensor([500.0]), inp["context"].cuda(), 18480)
        fkw = dict(packed=False)
    else:
        inp = synth.make_inputs(cfg, 9, 13, 68, 120, 512)
        args = (inp["x"], torch.tensor([500.0]), inp["context"].cuda(), 0)
        fkw = dict(y=inp["y"], clip_fea=inp["clip_fea"], latent_frame_zero=8, packed=True)
    res = dict(model=name, layers=cfg["num_layers"])
    outs = {}
    groups = [("bf16", "fp8", "fp8_attn")] if variant == "5b" else [("bf16",), ("fp8", "fp8_attn")]
    for group in groups:
        engines = {p: WanDiT(sd, variant, device="cuda", precision=p, **kw) for p in group}
        for p in group:
            outs[p] = engines[p].forward(*args, **fkw).float().cpu()
        ts = timed([lambda e=engines[p]: e.forward(*args, **fkw) for p in group], reps)
        for p, t in zip(group, ts):
            res[f"{p}_ms"] = round(t, 2)
        del engines
        torch.cuda.empty_cache()
    res["alternated"] = [list(gr) for gr in groups]
    res["rel_frobenius"] = {"fp8_vs_bf16": _rel(outs["fp8"], outs["bf16"]), "fp8_attn_vs_bf16": _rel(outs["fp8_attn"], outs["bf16"]),
                            "fp8_attn_vs_fp8": _rel(outs["fp8_attn"], outs["fp8"])}
    res["fp8_attn_speedup_vs_fp8"] = round(res["fp8_ms"] / res["fp8_attn_ms"], 3)
    print(json.dumps(res), flush=True)
    del sd
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--skip-forwards", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_attention measures on the GPU: no CUDA device")
    info = card()
    print(json.dumps(info), flush=True)
    att = [bench_attention(n, L, H, args.reps) for n, L, H in SHAPES]
    fwd = [] if args.skip_forwards else [bench_forwards("CFG_5B", max(3, args.reps // 4)),
                                         bench_forwards("CFG_14B", max(3, args.reps // 4))]
    print(json.dumps(dict(card=info, card_after=card(), attention=att, forwards=fwd)))


if __name__ == "__main__":
    main()
