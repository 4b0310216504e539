"""Time and peak memory of the chunk-streamed Wan VAE decodes on one GPU, printed as JSON lines with the card's name and power
limit read in the same run.

  * 49 frames (13 latent frames) at production size: one pass against forced chunk lengths (the cost of streaming);
  * Wan2.1 decode of 145 frames at 544x960 (the 14B loop's third chunk) and Wan2.2 decode of 81 frames at 704x1280, in the
    chunks the planner picks, with `torch.cuda.max_memory_allocated` on top of the weights and the planner's bound;
  * the same for the encoders: 49 frames one pass against forced chunks, Wan2.1 encode of 177 frames (81 + 32k + 32 zero frames
    of the 14B loop at k = 2) and Wan2.2 encode of 81 frames at 704x1280.

Random weights at the real widths; every timed call is warmed up once and ends in a device synchronise.
usage: python tools/bench_vae_stream.py [--reps 2]  (chunk lengths are in latent frames)"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def _engine(which):
    from yume_b200 import vae21, vae22, vae_enc
    Eng, shapes, cfg = {
        "wan22": (vae22.Wan22VaeDecoder, vae22.decoder_param_shapes, dict(dec_dim=256, z_dim=48)),
        "wan21": (vae21.Wan21VaeDecoder, vae21.decoder_param_shapes, dict(dim=96, z_dim=16)),
        "wan22-encode": (vae_enc.Wan22VaeEncoder, vae_enc.encoder_param_shapes_22, dict(dim=160, z_dim=48)),
        "wan21-encode": (vae_enc.Wan21VaeEncoder, vae_enc.encoder_param_shapes_21, dict(dim=96, z_dim=16))}[which]
    g = torch.Generator(device="cuda").manual_seed(0)
    sd = {k: torch.randn(*v, device="cuda", generator=g) * (0.5 / (v[1] * (v[2] if len(v) > 2 else 1)) ** 0.5 if len(v) > 1 else 0.05)
          for k, v in shapes(**cfg).items()}
    return Eng(sd, device="cuda", **cfg)


def _run(eng, z, lengths, reps):
    enc = hasattr(eng, "encode") and z.shape[0] == 3
    fn = ((lambda: eng.encode(z)) if lengths is None else (lambda: eng._encode_chunks(z, lengths))) if enc else \
        ((lambda: eng.decode(z)) if lengths is None else (lambda: eng._decode_chunks(z, lengths)))
    out = fn()
    del out
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    times = []
    for _ in range(reps):
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t)
        del out
    return min(times), (torch.cuda.max_memory_allocated() - base) / 2**30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    print(json.dumps({"card": _card()}), flush=True)
    for which, T, H, W, forced in (("wan21", 13, 68, 120, [[4, 4, 4, 1], [1] * 13]),
                                   ("wan22", 13, 44, 80, [[4, 4, 4, 1], [1] * 13]),
                                   ("wan21", 37, 68, 120, []), ("wan22", 21, 44, 80, []),
                                   ("wan21-encode", 49, 544, 960, [[4, 4, 4, 1], [1] * 13]),
                                   ("wan22-encode", 49, 704, 1280, [[4, 4, 4, 1], [1] * 13]),
                                   ("wan21-encode", 177, 544, 960, []), ("wan22-encode", 81, 704, 1280, [])):
        eng = _engine(which)
        enc = which.endswith("encode")
        z = torch.rand(3, T, H, W, device="cuda") * 2 - 1 if enc else torch.randn(eng.z_dim, T, H, W, device="cuda")
        plan = eng.plan_chunks(T, H, W)
        for lengths in [None] + forced:
            s, gib = _run(eng, z, lengths, args.reps)
            used = plan if lengths is None else lengths
            print(json.dumps({"engine": which, "input": list(z.shape),
                              "frames": T if enc else eng._out_shape(T, H, W)[1],
                              "chunks": used, "planned": lengths is None, "seconds": round(s, 3), "peak_gib": round(gib, 2),
                              "planner_bound_gib": round(eng.chunk_bytes(max(used), T, H, W) / 2**30, 2)}), flush=True)
        del eng, z
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
