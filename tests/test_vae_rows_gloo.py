"""Row-parallel decode of the REAL Wan VAE decoders (yume_b200/vae22.py, vae21.py; WanVaeDecoder.enable_row_parallel) over gloo
at world 2 and 3, on CPU, over the torch stand-in of the ops extended with the row-band entry points
(tests/helpers/torch_ops_rows.py). World 3 on the fixtures' 4 latent rows gives bands of 1, 1 and 2 rows. On every rank:
  * the video is the full one, within the bar of tests/test_host_logic_vae_dec.py of the reference fixtures, and within 1e-6
    of the one-rank decode over the same stand-in (the CPU convolutions may round differently for a band; the GPU twin,
    tests/test_gpu_vae_rows_mp.py, requires equality);
  * forced chunk lengths and a resumed second call whose latent extends the first give that video too;
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
CASES = ("t1", "t2", "t5", "t3_wide")


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _worker(rank, world, port, errs):
    try:
        sys.path.insert(0, str(ROOT))
        sys.path.insert(0, str(ROOT / "tests"))
        from helpers import torch_ops_rows
        from oracle import wan21vae, wan22vae
        from yume_b200 import YumeB200Error, vae21, vae22, wan_vae
        vae22.ops = torch_ops_rows
        vae21.ops = torch_ops_rows
        torch.set_num_threads(2)
        dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)

        def fail(msg):
            errs.put(f"world {world} rank {rank}: {msg}")

        for which in ("wan22", "wan21"):
            mod, Engine, name = ((wan22vae, vae22.Wan22VaeDecoder, "wan22vae_tiny.pt") if which == "wan22" else
                                 (wan21vae, vae21.Wan21VaeDecoder, "wan21vae_tiny.pt"))
            g = torch.load(ROOT / "tests" / "golden" / name, weights_only=False)
            sd = mod.make_state_dict(g["seed_w"], **g["cfg"])
            one = Engine(sd, mean=g["mean"], std=g["std"], device="cpu", **g["cfg"])
            par = Engine(sd, mean=g["mean"], std=g["std"], device="cpu", **g["cfg"]).enable_row_parallel()
            res = Engine(sd, mean=g["mean"], std=g["std"], device="cpu", resume=True, **g["cfg"]).enable_row_parallel()
            for case in CASES:
                c = g["cases"][case]
                z = torch.randn(g["cfg"]["z_dim"], c["T"], c["H"], c["W"], generator=torch.Generator().manual_seed(c["seed"]))
                want = one.decode(z)
                torch_ops_rows.calls.clear()
                got = par.decode(z)
                if "conv3d_rows" not in torch_ops_rows.calls:
                    fail(f"{which} {case}: no row-halo conv launched")
                if tuple(got.shape) != c["shape"] or _rel(got, want) > 1e-6:
                    fail(f"{which} {case}: shape {tuple(got.shape)} rel {_rel(got, want):.3e} vs one rank")
                for key, v in (("sample", got[..., ::3, ::3]), ("rowsum", got.sum(-1)), ("colsum", got.sum(-2))):
                    if _rel(v, c[key]) >= 3e-2:
                        fail(f"{which} {case}: {key} rel {_rel(v, c[key]):.3e} vs the reference fixture")
                T = c["T"]
                for parts in ([1] * T, [T - 1, 1] if T > 1 else [1]):
                    r = _rel(par._decode_chunks(z, parts), want)
                    if r > 1e-6:
                        fail(f"{which} {case}: chunks {parts} rel {r:.3e}")
                if T > 1:
                    res.reset()
                    res.decode(z[:, :T // 2 + 1].clone())
                    r = _rel(res.decode(z), want)
                    if r > 1e-6:
                        fail(f"{which} {case}: resumed call rel {r:.3e}")
            # ranks that see different free memory agree on the smallest budget
            c = g["cases"]["t5"]
            nb = lambda n: par.chunk_bytes(n, c["T"], c["H"], c["W"])  # noqa: E731
            budgets = [nb(2) + 1000 * (r + 1) for r in range(world)]
            par._free_bytes = lambda: budgets[rank] + par.MEM_MARGIN
            plan = par.plan_chunks(c["T"], c["H"], c["W"])
            del par._free_bytes
            every = [None] * world
            dist.all_gather_object(every, plan)
            if any(p != plan for p in every) or plan != wan_vae.chunk_lengths(c["T"], nb, budgets[0]) or len(plan) < 2:
                fail(f"{which}: chunk plans {every}")
            # refusals: raised on every rank, before any collective
            for what, call in (("rows", lambda: par.decode(torch.zeros(g["cfg"]["z_dim"], 2, world - 1, 4))),):
                try:
                    call()
                    fail(f"{which}: no refusal of {what}")
                except YumeB200Error:
                    pass
            if which == "wan22":
                try:
                    Engine(sd, mean=g["mean"], std=g["std"], device="cpu", precision="fp8", **g["cfg"]).enable_row_parallel()
                    fail("fp8 accepted")
                except YumeB200Error:
                    pass
        dist.barrier()                                            # nothing above left a collective half-issued
        dist.destroy_process_group()
    except Exception as e:  # pragma: no cover
        import traceback
        errs.put(f"world {world} rank {rank}: {type(e).__name__}: {e}\n{traceback.format_exc()[-2500:]}")


@pytest.mark.parametrize("world", [2, 3])
def test_row_parallel_decode_over_gloo(world):
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



def test_refused_without_a_process_group(golden_dir):
    from oracle import wan22vae
    from yume_b200 import YumeB200Error, vae22
    g = torch.load(golden_dir / "wan22vae_tiny.pt", weights_only=False)
    eng = vae22.Wan22VaeDecoder(wan22vae.make_state_dict(g["seed_w"], **g["cfg"]), mean=g["mean"], std=g["std"], device="cpu",
                                **g["cfg"])
    assert not dist.is_initialized()
    with pytest.raises(YumeB200Error):
        eng.enable_row_parallel()
