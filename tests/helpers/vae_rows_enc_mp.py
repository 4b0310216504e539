"""TEST INFRASTRUCTURE: one rank of a row-parallel Wan VAE encode under torchrun (tests/test_gpu_vae_rows_enc_mp.py). Every rank
encodes a seeded real-width 49-frame video with WanVaeEngine.enable_row_parallel and compares its mu with the one-GPU mu in
`--want` (a file the test wrote): one call, a call forced into several chunks, and the 14B loop's resumed pair [history, zeros]
then [history + new frames, zeros], the second call resuming from the first call's fork snapshot. Prints one line per check and
exits non-zero on a mismatch.

  torchrun --nproc-per-node P tests/helpers/vae_rows_enc_mp.py --which wan22 --backend gloo --want mu.pt [--same-device]"""
import argparse
import os
import sys
from pathlib import Path

import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

# (engine config, video frames, rows, columns, video seed)
CASES = {"wan22": (dict(dim=160, z_dim=48), 49, 704, 1280, 21), "wan21": (dict(dim=96, z_dim=16), 49, 544, 960, 22)}
HIST, ZEROS = 17, 32     # the resumed pair: [video[:HIST], zeros(ZEROS)], then [video[:HIST + ZEROS], zeros(ZEROS)]


def engine(which, device, **kw):
    from oracle import wan21vae_enc, wan22vae_enc
    from yume_b200 import vae_enc
    mod, Eng = (wan22vae_enc, vae_enc.Wan22VaeEncoder) if which == "wan22" else (wan21vae_enc, vae_enc.Wan21VaeEncoder)
    cfg = CASES[which][0]
    gen = torch.Generator().manual_seed(4)
    zd = cfg["z_dim"]
    return Eng(mod.make_state_dict(0, **cfg), mean=0.2 * torch.randn(zd, generator=gen), std=0.5 + torch.rand(zd, generator=gen),
               device=device, **cfg, **kw)


def video(which):
    _, T, H, W, seed = CASES[which]
    return torch.randn(3, T, H, W, generator=torch.Generator().manual_seed(seed)).clamp_(-1, 1)


def resumed_pair(v):
    """The two inputs of the 14B loop's resumed pair, built from the video v."""
    z = torch.zeros(3, ZEROS, *v.shape[2:], dtype=v.dtype, device=v.device)
    return torch.cat([v[:, :HIST], z], 1), torch.cat([v[:, :HIST + ZEROS], z], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--which", choices=sorted(CASES), required=True)
    ap.add_argument("--backend", default="gloo")
    ap.add_argument("--want", required=True)
    ap.add_argument("--same-device", action="store_true", help="every rank on cuda:0")
    a = ap.parse_args()
    rank = int(os.environ["RANK"])
    dev = torch.device("cuda", 0 if a.same_device else int(os.environ["LOCAL_RANK"]))
    torch.cuda.set_device(dev)
    dist.init_process_group(a.backend, device_id=dev if a.backend == "nccl" else None)
    want = torch.load(a.want, weights_only=True)
    v = video(a.which).to(dev)
    ok = True

    def check(name, got, ref):
        nonlocal ok
        same = tuple(got.shape) == tuple(ref.shape) and torch.equal(got.cpu(), ref)
        ok &= same
        print(f"rank {rank} {a.which} {name}: {'equal' if same else 'DIFFERS'}", flush=True)

    eng = engine(a.which, dev).enable_row_parallel()
    res = engine(a.which, dev, resume=True).enable_row_parallel()
    if a.same_device:            # the ranks share one card: each plans with its share of the free memory
        P = dist.get_world_size()
        free = torch.cuda.mem_get_info(dev)[0]
        eng.MEM_MARGIN = res.MEM_MARGIN = (2 << 30) + free - free // P
    check("one call", eng.encode(v), want["mu"])
    check("chunks [5, 5, 3]", eng._encode_chunks(v, [5, 5, 3]), want["mu"])
    first, second = resumed_pair(v)
    check("[history, zeros]", res.encode(first), want["first"])
    check("resumed [history + new, zeros]", res.encode(second), want["second"])
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
