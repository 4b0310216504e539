"""bf16 vs fp8 block GEMMs and forwards on one GPU, in one process (DESIGN.md §3): per production GEMM shape of the 5B (L = 18 480)
and 14B-chunk (L = 21 930) blocks the TFLOP/s of yb_gemm_bf16 and of yb_gemm_fp8 (the fp8 time of o / cross o includes the
quantiser launch the fp8 path adds in front of them; the LayerNorm in front of q|k|v, cross q and ffn.0 is left out of both, the
fp8 one replacing the bf16 one), then the full-depth 5B step and 14B chunk forward in both precisions (alternated, CUDA events),
the weight bytes and memory of both engines and the rel-Frobenius distance of the outputs. Prints one JSON line at the end.

    python tools/bench_fp8.py [--reps 20]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import synth  # noqa: E402
from oracle.fp8 import quantize_act, quantize_weight  # noqa: E402
from yume_b200 import ops  # noqa: E402
from yume_b200.dit import WanDiT  # noqa: E402

E4M3 = torch.float8_e4m3fn


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = (v.strip() for v in q.split(","))
    return dict(name=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)


def timed(fns, reps):
    """Alternate the callables rep by rep; median ms of each (CUDA events)."""
    for f in fns:
        f(), f()
    ts = [[] for _ in fns]
    for _ in range(reps):
        for i, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            ts[i].append(a.elapsed_time(b))
    return [sorted(t)[len(t) // 2] for t in ts]


def gemm_shapes(L, C, F):
    # name, M, N, K, bf16 epilogue, fp8 epilogue, input quantiser in front of the fp8 GEMM
    return [("qkv", L, 3 * C, C, ops.YB_EPI_BF16, ops.YB_EPI_BF16, None), ("o", L, C, C, ops.YB_EPI_GATE_RES, ops.YB_EPI_GATE_RES, "rows"),
            ("cross_q", L, C, C, ops.YB_EPI_BF16, ops.YB_EPI_BF16, None),
            ("cross_o", L, C, C, ops.YB_EPI_GATE_RES, ops.YB_EPI_GATE_RES, "rows"),
            ("ffn0", L, F, C, ops.YB_EPI_GELU_BF16, ops.YB_EPI_GELU_FP8, None), ("ffn2", L, C, F, ops.YB_EPI_GATE_RES, ops.YB_EPI_GATE_RES, None)]


def bench_gemms(tree, L, C, F, reps):
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, M, N, K, e16, e8, quant in gemm_shapes(L, C, F):
        x = torch.randn(M, K, device="cuda", generator=g)
        w = torch.randn(N, K, device="cuda", generator=g) * 0.02
        bias = torch.randn(N, device="cuda", generator=g)
        a16, w16 = x.to(torch.bfloat16), w.to(torch.bfloat16)
        aq, sa = quantize_act(x)
        sa = torch.nn.functional.pad(sa, (0, (-M) % 4)).contiguous()
        wq, sw = quantize_weight(w)
        gate = torch.randn(1, N, device="cuda", generator=g) if e16 == ops.YB_EPI_GATE_RES else None
        o16 = torch.zeros(M, N, device="cuda", dtype=torch.float32 if e16 == ops.YB_EPI_GATE_RES else torch.bfloat16)
        o8 = torch.zeros(M, N, device="cuda", dtype=E4M3 if e8 == ops.YB_EPI_GELU_FP8 else o16.dtype)
        os8 = torch.zeros(N // 128, sa.shape[1], device="cuda") if e8 == ops.YB_EPI_GELU_FP8 else None
        q_in, s_in = torch.empty_like(aq), torch.empty_like(sa)

        def f16():
            ops.gemm(a16, w16, bias, o16, e16, gate=gate)

        def f8():
            if quant == "rows":
                ops.quant_rows_fp8(a16, q_in, s_in)
                ops.gemm_fp8(q_in, s_in, wq, sw, bias, o8, e8, gate=gate, out_scale=os8)
            else:
                ops.gemm_fp8(aq, sa, wq, sw, bias, o8, e8, gate=gate, out_scale=os8)
        t16, t8 = timed([f16, f8], reps)
        fl = 2.0 * M * N * K
        rows.append(dict(tree=tree, gemm=name, M=M, N=N, K=K, bf16_ms=round(t16, 4), fp8_ms=round(t8, 4),
                         bf16_tflops=round(fl / t16 / 1e9, 1), fp8_tflops=round(fl / t8 / 1e9, 1), speedup=round(t16 / t8, 3)))
        print(json.dumps(rows[-1]), flush=True)
        del x, w, a16, w16, aq, wq, o16, o8
        torch.cuda.empty_cache()
    return rows


def full_depth_state_dict(cfg, seed):
    """State dict of the full-depth model whose blocks all hold block 0's (seeded) tensors: the engine still re-packs and stores
    one copy per layer, so launches, weight bytes and times are those of the real model, at the host cost of one block."""
    sd = synth.make_state_dict(cfg, seed, num_layers=1)
    for k in [k for k in sd if k.startswith("blocks.0.")]:
        for i in range(1, cfg["num_layers"]):
            sd[f"blocks.{i}." + k[len("blocks.0."):]] = sd[k]
    return sd


def bench_forward(name, reps):
    """The full-depth forward bench.py times: 5B = the denoise step on the regular grid 21 x 44 x 80 (L = 18 480, t = 500);
    14B = the chunk forward, latent 13 x 68 x 120 through FramePack with latent_frame_zero 8 (L = 21 930), CLIP + text context."""
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
    outs, engines = {}, {}
    for prec in ("bf16", "fp8"):
        base = torch.cuda.memory_allocated()
        eng = WanDiT(sd, variant, device="cuda", precision=prec, **kw)
        res[f"{prec}_weight_GiB"] = round(eng.weight_bytes() / 2 ** 30, 3)
        res[f"{prec}_engine_alloc_GiB"] = round((torch.cuda.memory_allocated() - base) / 2 ** 30, 3)
        engines[prec] = eng
    del sd
    for prec in ("bf16", "fp8"):
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        outs[prec] = engines[prec].forward(*args, **fkw)
        torch.cuda.synchronize()
        res[f"{prec}_forward_peak_above_resident_GiB"] = round((torch.cuda.max_memory_allocated() - before) / 2 ** 30, 3)
    t16, t8 = timed([lambda: engines["bf16"].forward(*args, **fkw), lambda: engines["fp8"].forward(*args, **fkw)], reps)
    res.update(bf16_ms=round(t16, 2), fp8_ms=round(t8, 2), speedup=round(t16 / t8, 3),
               rel_frobenius_fp8_vs_bf16=float((outs["fp8"] - outs["bf16"]).norm() / outs["bf16"].norm()))
    print(json.dumps(res), flush=True)
    del engines, outs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8 measures on the GPU: no CUDA device")
    info = card()
    print(json.dumps(info), flush=True)
    gemms = bench_gemms("5b", 18480, 3072, 14336, args.reps) + bench_gemms("14b_chunk", 21930, 5120, 13824, args.reps)
    fwd = [bench_forward("CFG_5B", max(3, args.reps // 4)), bench_forward("CFG_14B", max(3, args.reps // 4))]
    info2 = card()
    print(json.dumps(dict(card=info, card_after=info2, gemms=gemms, forwards=fwd)))


if __name__ == "__main__":
    main()
