"""Time the CLIP ViT-H/14 image encoder (yume_b200/clip.py) on one 544x960 image and print one JSON line.

    python tools/bench_clip.py [--steps K] [--warmup W]

Reports, from the same process: the card name and power limit (nvidia-smi), the encode time eagerly and with CUDA-graph
replay (CUDA events after warm-up, mean over K), and the comparator — oracle/clip.py run the way the reference runs
(bf16 weights, fp16 autocast, SDPA attention) — with its time and output dtype. Accuracy: rel-Frobenius of the engine and of
the comparator, each against oracle/clip.py in fp32 on the device. Roofline inputs computed from the shapes: FLOPs per image
and the bytes of useful (and head-padded) block weights. Weights and image are seeded; nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import clip as oclip  # noqa: E402


def flops_per_image(image_size, patch_size, dim, heads, layers, mlp_ratio, eps=1e-5):
    """Algorithmic FLOPs (2 per multiply-add) of the patch conv and the layers-1 blocks that run, head_dim unpadded."""
    L, P, mid = (image_size // patch_size) ** 2 + 1, (image_size // patch_size) ** 2, int(dim * mlp_ratio)
    block = 2 * L * dim * 3 * dim + 4 * L * L * dim + 2 * L * dim * dim + 2 * 2 * L * dim * mid
    return 2 * P * 3 * patch_size ** 2 * dim + (layers - 1) * block


def weight_bytes(dim, heads, layers, mlp_ratio, padded=False, **_):
    """bf16 bytes of the block GEMM weights that run (q|k|v, o, fc1, fc2); padded: heads widened to 128 columns."""
    hw = heads * 128 if padded else dim
    mid = int(dim * mlp_ratio)
    return 2 * (layers - 1) * (3 * hw * dim + dim * hw + 2 * dim * mid)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_clip needs a CUDA device")
    import yume_b200
    from yume_b200.clip import ClipVisionEncoder
    yume_b200.load()
    dev = "cuda"
    cfg = oclip.VIT_H_14
    sd = oclip.make_state_dict(1234, **cfg)
    g = torch.Generator().manual_seed(99)
    img = (torch.rand(3, 1, 544, 960, generator=g) * 2 - 1).to(dev)
    card, power = _card()

    enc = ClipVisionEncoder(sd, mean=oclip.MEAN, std=oclip.STD, device=dev, **cfg)
    out_eager = enc.encode([img])
    t_eager = _time(lambda: enc.encode([img]), args.steps, args.warmup)
    enc.use_cuda_graph = True
    out_graph = enc.encode([img])
    t_graph = _time(lambda: enc.encode([img]), args.steps, args.warmup)
    graph_equal = bool(torch.equal(out_graph, out_eager))
    del enc

    sd32 = {k: v.to(dev) for k, v in sd.items()}
    with torch.no_grad():
        ref = oclip.visual(sd32, [img], **cfg)
    del sd32
    sd16 = {k: v.to(device=dev, dtype=torch.bfloat16) for k, v in sd.items()}

    def comparator():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            return oclip.visual(sd16, [img], **cfg)
    out_cmp = comparator()
    t_cmp = _time(comparator, args.steps, args.warmup)

    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())  # noqa: E731
    fl = flops_per_image(**cfg)
    print(json.dumps({
        "workload": "clip_vit_h_14_visual 1 image 544x960 -> [1, 257, 1280]",
        "device": card, "power_limit": power, "steps": args.steps, "warmup": args.warmup,
        "engine_eager_ms": round(t_eager, 3), "engine_graph_ms": round(t_graph, 3), "graph_equals_eager": graph_equal,
        "comparator_ms": round(t_cmp, 3), "comparator": "oracle, bf16 weights, fp16 autocast, SDPA",
        "comparator_out_dtype": str(out_cmp.dtype), "engine_out_dtype": str(out_graph.dtype),
        "rel_fro_engine_vs_fp32": rel(out_graph, ref), "rel_fro_comparator_vs_fp32": rel(out_cmp, ref),
        "gflop_per_image": fl / 1e9, "engine_graph_tflops": fl / (t_graph * 1e-3) / 1e12,
        "weight_gb_useful": weight_bytes(**cfg) / 1e9, "weight_gb_padded": weight_bytes(**cfg, padded=True) / 1e9,
    }))


if __name__ == "__main__":
    main()
