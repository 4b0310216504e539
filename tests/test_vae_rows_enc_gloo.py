"""Row-parallel encode of the REAL Wan VAE encoders (yume_b200/vae_enc.py; WanVaeEngine.enable_row_parallel) over gloo at world
2 and 3, on CPU, over the torch stand-in of the ops extended with the encode's row-band entry points
(tests/helpers/torch_ops_rows_enc.py). World 2 runs the fixtures' videos (2 latent rows); world 3 runs seeded taller videos (3
and 4 latent rows: bands of 1 and 2 rows). On every rank:
  * mu is the full one, within 1e-6 of the one-rank encode over the same stand-in (the CPU convolutions may round differently
    for a band; the GPU twin, tests/test_gpu_vae_rows_enc_mp.py, requires equality), and on the fixtures within the bar of
    tests/test_host_logic_vae_enc.py of the reference's own encode;
  * forced chunk lengths give that mu too, and so does the 14B loop's resumed pair: [h, zeros] then [h + new frames, zeros],
    the second call resuming from the first call's fork snapshot (it reads only the new and the zero frames);
  * ranks that report different free memory plan the same chunks (the smallest budget);
  * the refusals raise on every rank, before any collective (the group is still usable after them)."""
import socket
import sys
from pathlib import Path

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = Path(__file__).resolve().parents[1]
FIXTURE_CASES = ("t1", "t5", "t9", "t17_wide")


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _video(T, H, W, seed):
    return torch.randn(3, T, H, W, generator=torch.Generator().manual_seed(seed)).clamp_(-1, 1)


def _worker(rank, world, port, errs):
    try:
        sys.path.insert(0, str(ROOT))
        sys.path.insert(0, str(ROOT / "tests"))
        from helpers import torch_ops_rows_enc
        from oracle import wan21vae_enc, wan22vae_enc
        from yume_b200 import YumeB200Error, vae_enc, wan_vae
        vae_enc.ops = torch_ops_rows_enc
        torch.set_num_threads(2)
        dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
        solo = [dist.new_group([r]) for r in range(world)]        # every rank takes part in creating every group

        def fail(msg):
            errs.put(f"world {world} rank {rank}: {msg}")

        for which in ("wan22", "wan21"):
            mod, Engine, name = ((wan22vae_enc, vae_enc.Wan22VaeEncoder, "wan22vae_enc_tiny.pt") if which == "wan22" else
                                 (wan21vae_enc, vae_enc.Wan21VaeEncoder, "wan21vae_enc_tiny.pt"))
            S = Engine.SCALE
            g = torch.load(ROOT / "tests" / "golden" / name, weights_only=False)
            sd = mod.make_state_dict(g["seed_w"], **g["cfg"])
            make = lambda **k: Engine(sd, mean=g["mean"], std=g["std"], device="cpu", **g["cfg"], **k)  # noqa: E731
            one, par, res = make(), make().enable_row_parallel(), make(resume=True).enable_row_parallel()
            if make().enable_row_parallel(solo[rank])._rows is not None:
                fail(f"{which}: a group of one rank left the one-GPU path")
            if world == 2:
                cases = [(k, g["cases"][k]) for k in FIXTURE_CASES]
            else:                                                  # 3 and 4 latent rows
                cases = [("h3", dict(T=9, H=3 * S, W=4 * S, seed=31)), ("h4", dict(T=5, H=4 * S, W=2 * S, seed=32))]
            for case, c in cases:
                x = _video(c["T"], c["H"], c["W"], c["seed"])
                want = one.encode(x)
                torch_ops_rows_enc.calls.clear()
                got = par.encode(x)
                for op in ("conv3d_rows", "conv3d_rows_down"):
                    if op not in torch_ops_rows_enc.calls:
                        fail(f"{which} {case}: no {op} launched")
                if got.shape != want.shape or _rel(got, want) > 1e-6:
                    fail(f"{which} {case}: shape {tuple(got.shape)} rel {_rel(got, want):.3e} vs one rank")
                if "mu" in c and _rel(got, c["mu"]) >= 3e-2:
                    fail(f"{which} {case}: rel {_rel(got, c['mu']):.3e} vs the reference fixture")
                n = want.shape[1]
                for parts in ([1] * n, [n - 1, 1] if n > 1 else [1]):
                    r = _rel(par._encode_chunks(x, parts), want)
                    if r > 1e-6:
                        fail(f"{which} {case}: chunks {parts} rel {r:.3e}")
            # the 14B loop: [h, zeros(4)], then [h + 4 new frames, zeros(4)] resumes from the fork snapshot after h
            H, W = 3 * S, 2 * S
            h, new = _video(5, H, W, 41), _video(4, H, W, 42)
            first, second = torch.cat([h, torch.zeros(3, 4, H, W)], 1), torch.cat([h, new, torch.zeros(3, 4, H, W)], 1)
            res.reset()
            r = _rel(res.encode(first), one.encode(first))
            torch_ops_rows_enc.read_frames.clear()
            r2 = _rel(res.encode(second), one.encode(second))
            if r > 1e-6 or r2 > 1e-6:
                fail(f"{which}: resumed pair rel {r:.3e}, {r2:.3e}")
            if sum(torch_ops_rows_enc.read_frames) != 8:
                fail(f"{which}: the resumed call read {torch_ops_rows_enc.read_frames} frames, not the 8 after the fork")
            # ranks that see different free memory agree on the smallest budget
            T, H, W = 17, 3 * S, 4 * S
            nb = lambda n: par.chunk_bytes(n, T, H, W)  # noqa: E731
            budgets = [nb(2) + 1000 * (r + 1) for r in range(world)]
            par._free_bytes = lambda: budgets[rank] + par.MEM_MARGIN
            plan = par.plan_chunks(T, H, W)
            del par._free_bytes
            every = [None] * world
            dist.all_gather_object(every, plan)
            if any(p != plan for p in every) or plan != wan_vae.chunk_lengths(5, nb, budgets[0]) or len(plan) < 2:
                fail(f"{which}: chunk plans {every}")
            # refusals: raised on every rank, before any collective
            for what, bad in (("not a video", torch.zeros(4, 5, 2 * S, S)), ("H % SCALE", torch.zeros(3, 5, 2 * S + 2, S)),
                              ("W % SCALE", torch.zeros(3, 5, 2 * S, S + 2)), ("rows", torch.zeros(3, 5, (world - 1) * S, S))):
                for eng in (par, res):
                    try:
                        eng.encode(bad)
                        fail(f"{which}: no refusal of {what}")
                    except YumeB200Error:
                        pass
            try:
                make(precision="fp8")
                fail(f"{which}: fp8 encoder accepted")
            except YumeB200Error:
                pass
        dist.barrier()                                            # nothing above left a collective half-issued
        dist.destroy_process_group()
    except Exception as e:  # pragma: no cover
        import traceback
        errs.put(f"world {world} rank {rank}: {type(e).__name__}: {e}\n{traceback.format_exc()[-2500:]}")


@pytest.mark.parametrize("world", [2, 3])
def test_row_parallel_encode_over_gloo(world):
    ctx = mp.get_context("spawn")
    errs = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, errs)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(600)
    alive = [p for p in procs if p.is_alive()]
    for p in alive:
        p.kill()
    out = []
    while not errs.empty():
        out.append(errs.get())
    assert not alive, "a rank hung"
    assert not out, "\n".join(out)
    assert all(p.exitcode == 0 for p in procs)


def test_encoder_refused_without_a_process_group(golden_dir):
    from oracle import wan22vae_enc
    from yume_b200 import YumeB200Error, vae_enc
    g = torch.load(golden_dir / "wan22vae_enc_tiny.pt", weights_only=False)
    eng = vae_enc.Wan22VaeEncoder(wan22vae_enc.make_state_dict(g["seed_w"], **g["cfg"]), mean=g["mean"], std=g["std"],
                                  device="cpu", **g["cfg"])
    assert not dist.is_initialized()
    with pytest.raises(YumeB200Error):
        eng.enable_row_parallel()


# ------------------------------------------------------------------------------------------------------------
# C-ABI guards over include/yume_b200_vae_rows_enc.h
# ------------------------------------------------------------------------------------------------------------
ENC_SYMBOLS = {"yb_conv3d_rows_down", "yb_vae_patchify2_bf16_rows", "yb_nchw_to_nhwc_bf16_rows"}


def test_library_exports_the_rows_enc_header_symbols():
    import re

    import yume_b200
    from yume_b200 import _lib
    header = ROOT / "include" / "yume_b200_vae_rows_enc.h"
    declared = set(re.findall(r"^\s*(?:int|long long)\s+(yb_\w+)\s*\(", header.read_text(), flags=re.M))
    assert declared == set(_lib.ROWS_ENC_SIGNATURES) == ENC_SYMBOLS
    lib = yume_b200.load()
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/yume_b200_vae_rows_enc.h but not exported"
    others = (set(_lib.SIGNATURES) | set(_lib.CLIP_SIGNATURES) | set(_lib.T5_SIGNATURES) | set(_lib.STREAM_SIGNATURES)
              | set(_lib.FP8_SIGNATURES) | set(_lib.FP8_ATTN_SIGNATURES) | set(_lib.FP8_VAE_SIGNATURES)
              | set(_lib.RESUME_SIGNATURES) | set(_lib.FP8_SP_SIGNATURES) | set(_lib.ROWS_SIGNATURES))
    assert not declared & others


def _down_args(**kw):
    import ctypes as C

    from yume_b200 import _lib
    a = dict(struct_bytes=C.sizeof(_lib.Conv3dArgs), xpad=1 << 20, w=1 << 20, out=1 << 20, ldo=64, T=2, H=8, W=8, Cp=64,
             Cout=64, epilogue=0, kt=1, kh=3, kw=3, oob_zero_pad=1, stride_t=1, stride_hw=2)
    a.update(kw)
    return _lib.Conv3dArgs(**a)


@pytest.mark.parametrize("bad", [dict(H=7), dict(oob_zero_pad=0), dict(stride_hw=1), dict(kt=3), dict(kh=1), dict(kw=1),
                                 dict(stride_t=2), dict(xpad=0), dict(struct_bytes=8)])
def test_conv3d_rows_down_refuses_bad_arguments(bad):
    """Refused with YB_ERR_ARG (-1) before anything reaches the device, so no GPU is needed."""
    import ctypes as C

    import yume_b200
    assert yume_b200.load().yb_conv3d_rows_down(C.byref(_down_args(**bad)), None) == -1


@pytest.mark.parametrize("fn,args,rc", [
    ("yb_vae_patchify2_bf16_rows", (1 << 20, 2 * 16 * 16, 1 << 20, 64, 2, 15, 16, 0, 7, None), -2),  # odd H
    ("yb_vae_patchify2_bf16_rows", (1 << 20, 2 * 16 * 16, 1 << 20, 8, 2, 16, 16, 0, 8, None), -1),   # ldo < 12
    ("yb_vae_patchify2_bf16_rows", (1 << 20, 2 * 16 * 16, 1 << 20, 64, 2, 16, 16, 4, 5, None), -1),  # band past the image
    ("yb_vae_patchify2_bf16_rows", (1 << 20, 2 * 16 * 16, 1 << 20 | 8, 64, 2, 16, 16, 0, 8, None), -3),  # out misaligned
    ("yb_vae_patchify2_bf16_rows", (1 << 20, 100, 1 << 20, 64, 2, 16, 16, 0, 8, None), -1),        # plane < T*H*W
    ("yb_nchw_to_nhwc_bf16_rows", (1 << 20, 2 * 8 * 8, 1 << 20, 2, 2, 8, 8, 3, 0, 8, None), -1),     # ldo < Cn
    ("yb_nchw_to_nhwc_bf16_rows", (1 << 20, 2 * 8 * 8, 1 << 20, 12, 2, 8, 8, 3, 0, 8, None), -3),    # ldo % 8
    ("yb_nchw_to_nhwc_bf16_rows", (1 << 20, 2 * 8 * 8, 1 << 20, 64, 2, 8, 8, 3, -1, 4, None), -1),   # r0 < 0
    ("yb_nchw_to_nhwc_bf16_rows", (1 << 20, 2 * 8 * 8, 1 << 20, 64, 2, 8, 8, 3, 2, 0, None), -1),    # no rows
    ("yb_nchw_to_nhwc_bf16_rows", (0, 2 * 8 * 8, 1 << 20, 64, 2, 8, 8, 3, 0, 8, None), -1),          # NULL source
])
def test_band_readers_refuse_bad_arguments(fn, args, rc):
    import yume_b200
    assert getattr(yume_b200.load(), fn)(*args) == rc
