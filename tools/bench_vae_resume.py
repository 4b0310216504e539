"""Per-chunk VAE cost of the 14B I2V loop with `resume` off and on, printed as JSON lines with the card's name and power limit
read in the same run.

At chunk k the loop's video history has 49 + 32k frames at 544x960. Each chunk decodes the whole latent (13 + 8k latent frames)
with the Wan2.1 decoder and encodes [history, zeros(32)] with the Wan2.1 encoder (fastvideo/sample/sample.py, wan/image2video.py).
Without resume both calls cost time in proportion to the history. With resume the engines keep the previous chunk's state: the
decode runs the 8 new latent frames and the encode the 32 new history frames and the 32 zeros.

For each k the off call and the on call alternate, `--reps` times. Before each timed on call the resuming engines are reset and
run once, untimed, on chunk k - 1's inputs, which is the state a session reaches at chunk k. The line reports the time of both
calls (best of reps), the peak allocation above the weights during the timed call (for on: including the state kept from chunk
k - 1), `retained_bytes()` after it, and whether the on results equal the off results bit for bit.

Random weights at the real widths; every timed call ends in a device synchronise.
usage: python tools/bench_vae_resume.py [--chunks 1 5 10 20] [--reps 2]"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

H, W = 544, 960


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def _engines(resume):
    from yume_b200 import vae21, vae_enc
    g = torch.Generator(device="cuda").manual_seed(0)
    out = []
    for Eng, shapes in ((vae21.Wan21VaeDecoder, vae21.decoder_param_shapes), (vae_enc.Wan21VaeEncoder, vae_enc.encoder_param_shapes_21)):
        sd = {k: torch.randn(*v, device="cuda", generator=g) * (0.5 / (v[1] * (v[2] if len(v) > 2 else 1)) ** 0.5 if len(v) > 1 else 0.05)
              for k, v in shapes(dim=96, z_dim=16).items()}
        out.append(Eng(sd, dim=96, z_dim=16, device="cuda", resume=resume))
    return out


def _inputs(k, z_all, video_all, zeros):
    hist = 49 + 32 * k
    return z_all[:, :13 + 8 * k], torch.cat([video_all[:, :hist], zeros], 1)


def _call(dec, enc, z, v, base):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t = time.perf_counter()
    x, mu = dec.decode(z), enc.encode(v)
    torch.cuda.synchronize()
    return x, mu, time.perf_counter() - t, (torch.cuda.max_memory_allocated() - base) / 2**30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, nargs="+", default=[1, 5, 10, 20])
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    print(json.dumps({"card": _card()}), flush=True)
    off, on = _engines(False), _engines(True)
    kmax = max(args.chunks)
    gen = torch.Generator(device="cuda").manual_seed(1)
    z_all = torch.randn(16, 13 + 8 * kmax, H // 8, W // 8, device="cuda", generator=gen)
    video_all = torch.rand(3, 49 + 32 * kmax, H, W, device="cuda", generator=gen) * 2 - 1
    zeros = torch.zeros(3, 32, H, W, device="cuda")
    _call(*off, *_inputs(0, z_all, video_all, zeros), 0)                 # warm-up of every launch shape
    for e in on:
        e.reset()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()                                  # weights and the inputs above
    for k in args.chunks:
        z, v = _inputs(k, z_all, video_all, zeros)
        best = {"off": (1e9, 0.0), "on": (1e9, 0.0)}
        same = True
        for _ in range(args.reps):
            x_off, mu_off, s, gib = _call(*off, z, v, base)
            best["off"] = min(best["off"], (s, gib))
            for e in on:
                e.reset()
            if k:
                _call(*on, *_inputs(k - 1, z_all, video_all, zeros), base)
            x_on, mu_on, s, gib = _call(*on, z, v, base)
            best["on"] = min(best["on"], (s, gib))
            same = same and torch.equal(x_on, x_off) and torch.equal(mu_on, mu_off)
            retained = sum(e.retained_bytes() for e in on)
            del x_off, mu_off, x_on, mu_on
        print(json.dumps({"chunk": k, "history_frames": 49 + 32 * k, "latent_frames": z.shape[1], "encode_frames": v.shape[1],
                          "off_s": round(best["off"][0], 3), "on_s": round(best["on"][0], 3),
                          "off_peak_gib": round(best["off"][1], 2), "on_peak_gib": round(best["on"][1], 2),
                          "retained_gib": round(retained / 2**30, 2), "bit_identical": bool(same)}), flush=True)
        del z, v
    for e in on:
        e.reset()


if __name__ == "__main__":
    main()
