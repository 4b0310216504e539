"""Time the row-parallel Wan VAE decode (or, with --encode, encode) against the one-GPU one, in the same call, alternating,
after warm-up.

  torchrun --nproc-per-node P tools/bench_vae_rows.py [--which wan22|wan21] [--encode] [--iters 5] [--backend nccl]

Every rank decodes a seeded real-width 13-latent-frame latent (49 frames: Wan2.2 at 704x1280, Wan2.1 at 544x960). The one-GPU
decode runs on rank 0 alone (the others wait at a barrier); the P-rank decode runs on all ranks, one GPU each. Rank 0 prints one
JSON line: the card's name and power limit, both times (median over the iterations, host clock around work that ends in a
device synchronise), the speed-up, and the halo / gather bytes one rank exchanges, computed from shapes. With fewer GPUs than
ranks (several ranks on one card) the parallel time says nothing about P GPUs, so it is reported as "not measured".

--encode: every rank encodes a seeded real-width 49-frame video (Wan2.2 at 704x1280, Wan2.1 at 544x960); the bytes are the halo
rows, the attention gather, the band copy a Resample with C % 64 == 0 makes (read and written) and the padded band of mu."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests" / "helpers"))


def exchanged_bytes(eng, T, H, W, P, rank):
    """Bytes one rank sends in one decode of T latent frames at H x W: two halo rows per conv with kh = 3 per new frame, the
    padded band of the mid attention's input, and the padded band of the video."""
    from yume_b200.vae_rows import band
    hmax = max(band(H, P, r)[1] - band(H, P, r)[0] for r in range(P))
    halo, t, w = 0, T, W                                      # frames and columns at the running level
    for L in eng.layers:
        if L.kind == "in":
            halo += 2 * t * w * 64 * 2                           # conv1's input buffer: 64 channels
        elif L.kind == "res":
            halo += 2 * t * w * (_rup(L.ci, 64) + _rup(L.co, 64)) * 2
        elif L.kind == "up":
            t, w = (2 * t - 1 if L.ft == 2 else t), 2 * w
            halo += 2 * t * w * _rup(L.ci, 64) * 2               # resample.1's input, after the 2x upsample
        elif L.kind == "head":
            halo += 2 * t * w * _rup(L.ci, 64) * 2
    attn = next(L for L in eng.layers if L.kind == "attn")
    gather_attn = T * hmax * W * attn.ci * 2
    F, S = 1 + (T - 1) * eng._t_scale(), eng.SCALE
    gather_video = 3 * F * hmax * S * W * S * 4
    return dict(halo_bytes=halo, attn_gather_bytes=gather_attn, video_gather_bytes=gather_video)


def encode_bytes(eng, T, H, W, P):
    """Bytes one rank moves in one encode of T video frames at H x W beyond the one-GPU encode: two halo rows per unit-stride conv
    with kh = 3 per frame (the input reader reads its halos from the video), one row per Resample conv (the row below), the
    band copy of a Resample input whose channels are a multiple of 64 (the one-GPU encode reads it in place), the padded band of
    the mid attention's input, and the padded band of mu."""
    from yume_b200.vae_rows import band
    S = eng.SCALE
    hmax = max(band(H // S, P, r)[1] - band(H // S, P, r)[0] for r in range(P))
    halo = copy = 0
    for L in eng.layers:
        if L.kind == "in":
            t, w, s = T, W // L.fs, S // L.fs                       # frames, columns and rows per latent row at the level
        elif L.kind == "res":
            halo += 2 * t * w * (_rup(L.ci, 64) + _rup(L.co, 64)) * 2
        elif L.kind == "down":
            halo += t * w * _rup(L.ci, 64) * 2
            if L.ci % 64 == 0:
                copy += 2 * t * hmax * s * w * L.ci * 2
            t, w, s = (1 + (t - 1) // 2 if L.ft == 2 else t), w // 2, s // 2
        elif L.kind == "head":
            halo += 2 * t * w * _rup(L.ci, 64) * 2
    attn = next(L for L in eng.layers if L.kind == "attn")
    return dict(halo_bytes=halo, attn_gather_bytes=t * hmax * w * attn.ci * 2, downsample_copy_bytes=copy,
                mu_gather_bytes=eng.z_dim * t * hmax * w * 4)


def _rup(v, m):
    return (v + m - 1) // m * m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--which", choices=["wan22", "wan21"], default="wan22")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--backend", default="nccl")
    ap.add_argument("--encode", action="store_true", help="time the encode instead of the decode")
    a = ap.parse_args()
    import vae_rows_enc_mp
    import vae_rows_mp
    rank, P = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    shared = torch.cuda.device_count() < P
    dev = torch.device("cuda", 0 if shared else int(os.environ["LOCAL_RANK"]))
    torch.cuda.set_device(dev)
    backend = "gloo" if shared else a.backend
    dist.init_process_group(backend, device_id=dev if backend == "nccl" else None)
    mod = vae_rows_enc_mp if a.encode else vae_rows_mp
    x = (vae_rows_enc_mp.video(a.which) if a.encode else vae_rows_mp.latent(a.which)).to(dev)
    one = mod.engine(a.which, dev) if rank == 0 else None
    par = mod.engine(a.which, dev).enable_row_parallel()
    run = (lambda eng: eng.encode(x)) if a.encode else (lambda eng: eng.decode(x))  # noqa: E731
    if shared:
        free = torch.cuda.mem_get_info(dev)[0]
        par.MEM_MARGIN = (2 << 30) + free - free // P

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    t_one, t_par = [], []
    for i in range(a.warmup + a.iters):
        if rank == 0:
            dt, ref = timed(lambda: run(one))
            if i >= a.warmup:
                t_one.append(dt)
            del ref
        dist.barrier()
        dt, got = timed(lambda: run(par))
        if i >= a.warmup:
            t_par.append(dt)
        del got
        dist.barrier()
    if rank == 0:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True).stdout.strip().splitlines()
        _, T, H, W, _ = mod.CASES[a.which]
        moved = encode_bytes(par, T, H, W, P) if a.encode else exchanged_bytes(par, T, H, W, P, rank)
        res = dict(which=a.which, side="encode" if a.encode else "decode", ranks=P, gpus=torch.cuda.device_count(), backend=backend, card=q[0] if q else "unknown",
                   one_gpu_s=round(statistics.median(t_one), 4),
                   parallel_s="not measured" if shared else round(statistics.median(t_par), 4),
                   **moved)
        if not shared:
            res["speedup"] = round(res["one_gpu_s"] / res["parallel_s"], 3)
        print(json.dumps(res), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
