"""TEST INFRASTRUCTURE: one rank of a row-parallel Wan VAE decode under torchrun (tests/test_gpu_vae_rows_mp.py). Every rank
decodes a seeded real-width latent with WanVaeDecoder.enable_row_parallel and compares its video with the one-GPU video
`--want` (a file the test wrote): one call, a call forced into several chunks, and a resumed second call whose latent extends the
first. Prints one line per check and exits non-zero on a mismatch.

  torchrun --nproc-per-node P tests/helpers/vae_rows_mp.py --which wan22 --backend gloo --want video.pt [--same-device]"""
import argparse
import os
import sys
from pathlib import Path

import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

# (engine config, latent frames, rows, columns, latent seed)
CASES = {"wan22": (dict(dec_dim=256, z_dim=48), 13, 44, 80, 11), "wan21": (dict(dim=96, z_dim=16), 13, 68, 120, 12)}


def engine(which, device, **kw):
    from oracle import wan21vae, wan22vae
    from yume_b200 import vae21, vae22
    mod, Eng = (wan22vae, vae22.Wan22VaeDecoder) if which == "wan22" else (wan21vae, vae21.Wan21VaeDecoder)
    cfg = CASES[which][0]
    gen = torch.Generator().manual_seed(3)
    zd = cfg["z_dim"]
    return Eng(mod.make_state_dict(0, **cfg), mean=0.2 * torch.randn(zd, generator=gen), std=0.5 + torch.rand(zd, generator=gen),
               device=device, **cfg, **kw)


def latent(which):
    cfg, T, H, W, seed = CASES[which]
    return torch.randn(cfg["z_dim"], T, H, W, generator=torch.Generator().manual_seed(seed))


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
    z = latent(a.which).to(dev)
    ok = True

    def check(name, got):
        nonlocal ok
        same = tuple(got.shape) == tuple(want.shape) and torch.equal(got.cpu(), want)
        ok &= same
        print(f"rank {rank} {a.which} {name}: {'equal' if same else 'DIFFERS'}", flush=True)

    eng = engine(a.which, dev).enable_row_parallel()
    res = engine(a.which, dev, resume=True).enable_row_parallel()
    if a.same_device:            # the ranks share one card: each plans with its share of the free memory
        P = dist.get_world_size()
        free = torch.cuda.mem_get_info(dev)[0]
        eng.MEM_MARGIN = res.MEM_MARGIN = (2 << 30) + free - free // P
    check("one call", eng.decode(z))
    check("chunks [5, 5, 3]", eng._decode_chunks(z, [5, 5, 3]))
    res.decode(z[:, :7].clone())
    check("resumed", res.decode(z))
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
