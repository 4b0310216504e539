"""Time the umT5-XXL text encoder (yume_b200/t5.py) on one 512-token call and print one JSON line.

    python tools/bench_t5.py [--steps K] [--warmup W]

Workload: T5Encoder.forward at the real umT5-XXL size (24 layers, dim 4096, 64 heads of 64, ffn 10240, the full 256 384-row
vocabulary), B = 1, L = 512, with prompts of 120 and 512 tokens; seeded bf16 weights generated on the device. Reports, from the
same process: the card name and power limit (nvidia-smi); the engine's time per call (CUDA events, mean over K after W
warm-ups) and its host enqueue time (wall time of the call, which includes the host-side input checks); the reference's regime
(oracle/t5.py in bf16, eager) on the same GPU; the time per launch family from CUDA events around every launch in a separate
pass; the engine's time with every GEMM forced to block_n 256 and to 128 next to the per-launch rule; max_memory_allocated of
the engine's call; and the rel-Frobenius error of the engine and of the reference regime against oracle/t5.py in fp32.
Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from collections import defaultdict
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import t5 as ot5  # noqa: E402


def _card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (r.stdout.strip().splitlines() or [","])[0].split(",")[:2]
    return name.strip(), power.strip()


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def flops(cfg, L):
    """GEMM and attention FLOPs of one call at B = 1 (2 per multiply-add)."""
    C, A, Fd, n = cfg["dim"], cfg["dim_attn"], cfg["dim_ffn"], cfg["num_layers"]
    gemm = 2 * L * (3 * A * C + C * A + 2 * Fd * C + C * Fd)
    return n * gemm, n * 4 * L * L * A


def _family_times(enc, ids, mask, passes=5):
    """ms per launch family of one call, from CUDA events around every launch (separate, instrumented passes; mean over
    `passes` calls)."""
    from yume_b200 import ops
    C, A, Fd = enc.dim, enc.dim_attn, enc.dim_ffn
    names = {(3 * A, C): "gemm_qkv", (C, A): "gemm_o", (2 * Fd, C): "gemm_fc1_gate", (C, Fd): "gemm_fc2"}
    ev = []
    real = {n: getattr(ops, n) for n in ("gemm", "t5_attention", "t5_rmsnorm", "t5_geglu")}

    def wrap(name, fam):
        def f(*a, **k):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            r = real[name](*a, **k)
            e.record()
            ev.append((fam(a), s, e))
            return r
        return f
    ops.gemm = wrap("gemm", lambda a: names.get(tuple(a[1].shape), "gemm_other"))
    ops.t5_attention = wrap("t5_attention", lambda a: "t5_attention")
    ops.t5_rmsnorm = wrap("t5_rmsnorm", lambda a: "t5_rmsnorm")
    ops.t5_geglu = wrap("t5_geglu", lambda a: "t5_geglu")
    try:
        for _ in range(passes):
            enc(ids, mask)
        torch.cuda.synchronize()
    finally:
        for n, f in real.items():
            setattr(ops, n, f)
    out = defaultdict(float)
    for fam, s, e in ev:
        out[fam] += s.elapsed_time(e) / passes
    out["launches"] = len(ev) // passes
    return {k: round(v, 4) if isinstance(v, float) else v for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_t5 needs a CUDA device")
    import yume_b200
    from yume_b200.t5 import T5TextEncoder
    yume_b200.load()
    dev = "cuda"
    cfg = dict(ot5.UMT5_XXL)
    card, power = _card()
    sd = ot5.make_state_dict(4321, **cfg, device=dev, dtype=torch.bfloat16)
    enc = T5TextEncoder(sd, **cfg, device=dev)
    g = torch.Generator().manual_seed(8)
    L = 512
    result = {"workload": "umt5_xxl T5Encoder.forward, B = 1, L = 512, full vocabulary", "device": card, "power_limit": power,
              "steps": args.steps, "warmup": args.warmup}
    gf, af = flops(cfg, L)
    result["tflop_per_call"] = dict(gemm=gf / 1e12, attention=af / 1e12)
    for n_tok in (120, 512):
        ids = torch.randint(0, cfg["vocab"], (1, L), generator=g)
        ids[0, n_tok:] = 0
        mask = torch.zeros(1, L, dtype=torch.long)
        mask[0, :n_tok] = 1
        ids, mask = ids.to(dev), mask.to(dev)
        r = {}
        enc(ids, mask)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = enc(ids, mask)
        torch.cuda.synchronize()
        r["engine_call_peak_extra_gib"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
        r["max_memory_allocated_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
        r["engine_ms"] = round(_time(lambda: enc(ids, mask), args.steps, args.warmup), 3)
        r["engine_tflops"] = round((gf + af) / (r["engine_ms"] * 1e-3) / 1e12, 1)
        enq = []
        for _ in range(args.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            enc(ids, mask)
            enq.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        r["host_enqueue_ms"] = round(1e3 * sorted(enq)[len(enq) // 2], 3)
        r["launch_families_ms"] = _family_times(enc, ids, mask)
        st = enc._state[(1, L)]
        rule = dict(st["bn"])
        for label, bn in (("block_n_256", 0), ("block_n_128", 128)):
            st["bn"] = {k: bn for k in rule}
            r[f"engine_ms_{label}"] = round(_time(lambda: enc(ids, mask), args.steps, args.warmup), 3)
            r[f"launch_families_ms_{label}"] = {k: v for k, v in _family_times(enc, ids, mask).items() if k.startswith("gemm")}
        st["bn"] = rule
        r["block_n_rule"] = rule

        def regime():
            with torch.no_grad():
                return ot5.encode(sd, ids, mask, **cfg, dtype=torch.bfloat16)
        out_reg = regime()
        r["reference_regime_ms"] = round(_time(regime, max(2, args.steps // 2), 1), 3)
        with torch.no_grad():
            ref = ot5.encode(sd, ids, mask, **cfg, dtype=torch.float32)
        rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())  # noqa: E731
        r["rel_fro_engine_vs_fp32"] = rel(out, ref)
        r["rel_fro_reference_regime_vs_fp32"] = rel(out_reg, ref)
        r["rel_fro_engine_vs_fp32_prompt_rows"] = rel(out[:, :n_tok], ref[:, :n_tok])
        r["rel_fro_reference_regime_vs_fp32_prompt_rows"] = rel(out_reg[:, :n_tok], ref[:, :n_tok])
        del ref, out_reg, out
        torch.cuda.empty_cache()
        result[f"prompt_{n_tok}"] = r
    print(json.dumps(result))


if __name__ == "__main__":
    main()
