"""bf16, fp8 and fp8_attn forwards under Ulysses sequence parallelism, per rank (DESIGN.md §6). Launch with torchrun, one process per
GPU:

    torchrun --nproc-per-node=8 tools/bench_fp8_sp.py [--reps 8] [--transport auto|p2p|nccl]

The full-depth 5B denoise step (L = 18 480) and 14B chunk forward (L = 21 930), tools/bench_fp8.py's inputs, in the three
precisions alternated in one process (CUDA events, median per rank). Three 14B engines do not fit in 80 GB, so the 14B bf16 engine
is timed on its own first, then fp8 and fp8_attn alternate (as tools/bench_fp8_attention.py does). Per precision it also reports the
rel-Frobenius distance of the N-GPU output to the same engine's output on one GPU (`sequence_parallel_disabled`). Rank 0 prints one
JSON line with the card name and power limit of every rank.
"""
import argparse
import json
import os
import sys
from pathlib import Path

import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from bench_fp8 import card, full_depth_state_dict, timed  # noqa: E402
from oracle import synth  # noqa: E402
from yume_b200.dit import WanDiT  # noqa: E402


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def bench_model(name, transport, reps, dev):
    cfg = getattr(synth, name)
    sd = full_depth_state_dict(cfg, 5)
    kw = synth.oracle_kwargs(cfg)
    variant = kw.pop("variant")
    if variant == "5b":
        inp = synth.make_inputs(cfg, 9, 21, 44, 80, 512)
        args = (inp["x"], torch.tensor([500.0]), inp["context"].to(dev), 18480)
        fkw = dict(packed=False)
    else:
        inp = synth.make_inputs(cfg, 9, 13, 68, 120, 512)
        args = (inp["x"], torch.tensor([500.0]), inp["context"].to(dev), 0)
        fkw = dict(y=inp["y"], clip_fea=inp["clip_fea"], latent_frame_zero=8, packed=True)
    res = dict(model=name, layers=cfg["num_layers"], world=dist.get_world_size())
    groups = [("bf16", "fp8", "fp8_attn")] if variant == "5b" else [("bf16",), ("fp8", "fp8_attn")]
    for group in groups:
        engines = {p: WanDiT(sd, variant, device=dev, precision=p, **kw) for p in group}
        for p in group:
            engines[p].enable_sequence_parallel(dist.group.WORLD, transport=transport)
            out = engines[p].forward(*args, **fkw).float()
            with engines[p].sequence_parallel_disabled():
                one = engines[p].forward(*args, **fkw).float()
            res[f"{p}_vs_one_gpu"] = _rel(out, one)
            res[f"{p}_transport"] = engines[p].sp_transport + ("/p2p" if engines[p]._sp_p2p else "")
            res[f"{p}_weight_gib"] = round(engines[p].weight_bytes() / 2 ** 30, 2)
            del out, one
        dist.barrier()
        ts = timed([lambda e=engines[p]: e.forward(*args, **fkw) for p in group], reps)
        for p, t in zip(group, ts):
            res[f"{p}_ms"] = round(t, 2)
        del engines
        torch.cuda.empty_cache()
    res["alternated"] = [list(gr) for gr in groups]
    for p in ("fp8", "fp8_attn"):
        res[f"{p}_speedup_vs_bf16"] = round(res["bf16_ms"] / res[f"{p}_ms"], 3)
    del sd
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--transport", default="auto", choices=("auto", "p2p", "nccl"))
    args = ap.parse_args()
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    info = card()
    results = [bench_model(n, args.transport, args.reps, dev) for n in ("CFG_5B", "CFG_14B")]
    per_rank = [None] * dist.get_world_size()
    dist.all_gather_object(per_rank, dict(rank=dist.get_rank(), card=info, results=results))
    if dist.get_rank() == 0:
        print(json.dumps(dict(transport=args.transport, ranks=per_rank)), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
