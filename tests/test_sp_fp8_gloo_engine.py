"""World-size-2 `gloo` run (CPU) of the REAL engine with precision="fp8" and "fp8_attn" under Ulysses sequence parallelism:
yume_b200.dit.WanDiT with enable_sequence_parallel(transport="nccl") over the torch stand-ins of the fp8 entry points and of the new
fp8 Ulysses ones (tests/helpers/torch_ops_fp8_sp.py): shard-local fp8 block linears, the q|k|v pack into the send buffer, the two
all-to-alls per block (here over gloo), the fp8 or fp8-attention self-attention on the exchanged heads, the split quantiser in front
of the o projection. Against the fp8-qdq / fp8-attention oracles and the reference's own forwards, with the bars of the one-GPU
CPU tests. Also: the engine's weights do not grow when SP is enabled (no peer-major q|k|v copy), "p2p_gemm" is refused, and a bf16
SP engine still makes exactly the ops calls it made before the fp8 paths existed (pinned in tests/golden/sp_bf16_calls.json).

gloo cannot run symmetric memory, so the p2p host path runs only on two or more GPUs (tools/sp_parity.py); its kernels are checked on
one GPU by tests/test_gpu_kernel_contract_fp8_sp.py."""
import contextlib
import json
import socket
import sys
from pathlib import Path

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = Path(__file__).resolve().parents[1]
QDQ_BAR = 3e-2      # tests/test_fp8_cpu.py, tests/test_fp8_attn_cpu.py
REF_BAR = 5e-2
CASES = {"wan23_h8.pt": ("5b_grid_padded", "5b_pack_h10"), "wan21_h8.pt": ("14b_grid_padded", "14b_pack_lfz8")}


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _desc(x):
    if isinstance(x, torch.Tensor):
        return f"{str(x.dtype).replace('torch.', '')}{list(x.shape)}"
    if isinstance(x, (list, tuple)):
        return "(" + ",".join(_desc(v) for v in x) + ")"
    return repr(x)


class _Recorder:
    """An ops module that logs every entry-point call (name, operand shapes / dtypes, scalars, keyword arguments other than None)
    and forwards it to the wrapped stand-in."""

    def __init__(self, mod, log):
        self._mod, self._log = mod, log

    def __getattr__(self, name):
        v = getattr(self._mod, name)
        if name.startswith("_") or not callable(v) or name in ("fp8_scale_ld", "vt8_keys"):
            return v

        def call(*a, **k):
            kw = ",".join(f"{n}={_desc(u)}" for n, u in sorted(k.items()) if u is not None)
            self._log.append(f"{name}({','.join(_desc(u) for u in a)}{';' + kw if kw else ''})")
            return v(*a, **k)
        return call


def _setup(rank, world, port):
    sys.path.insert(0, str(ROOT))
    sys.path.insert(0, str(ROOT / "tests"))
    torch.cuda.device = lambda *_a, **_k: contextlib.nullcontext()
    torch.cuda.is_current_stream_capturing = lambda: False
    torch.set_num_threads(2)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)


def _forward(eng, variant, c, inp):
    if variant == "5b":
        return eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], latent_frame_zero=c["lfz"], packed=c["flag"])
    return eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], y=inp["y"], clip_fea=inp["clip_fea"],
                       latent_frame_zero=c["lfz"], packed=c["rand_num_img"] >= 0.4)


def _oracle(orc, variant, c, inp):
    if variant == "5b":
        return orc.forward([inp["x"]], torch.tensor(c["t"]), [inp["context"]], seq_len=c["seq_len"], latent_frame_zero=c["lfz"],
                           flag=c["flag"])
    return orc.forward([inp["x"]], torch.tensor(c["t"]), [inp["context"]], seq_len=c["seq_len"], y=[inp["y"]],
                       clip_fea=inp["clip_fea"], latent_frame_zero=c["lfz"], rand_num_img=c["rand_num_img"])


def _worker(rank, world, port, fname, precision, errs, report):
    try:
        _setup(rank, world, port)
        from helpers import torch_ops_fp8_sp
        from oracle import synth
        from oracle.fp8 import WanOracleFp8
        from oracle.fp8_attn import WanOracleFp8Attn
        from yume_b200 import dit
        from yume_b200._lib import YumeB200Error
        dit.ops = torch_ops_fp8_sp
        g = torch.load(ROOT / "tests" / "golden" / fname, weights_only=False)
        cfg = g["cfg"]
        kw = synth.oracle_kwargs(cfg)
        variant = kw.pop("variant")
        sd = synth.make_state_dict(cfg, g["seed_w"])
        eng = dit.WanDiT(sd, variant, device="cpu", precision=precision, **kw)
        wb = eng.weight_bytes()
        try:
            eng.enable_sequence_parallel(dist.group.WORLD, transport="p2p_gemm")
            errs.put(f"rank {rank} {precision}: transport='p2p_gemm' was accepted")
        except YumeB200Error as e:
            if "p2p_gemm" not in str(e) or "e4m3" not in str(e):
                errs.put(f"rank {rank} {precision}: p2p_gemm refused without saying why: {e}")
        eng.enable_sequence_parallel(dist.group.WORLD, transport="nccl")
        if eng.weight_bytes() != wb or "w_qkv_sp" in eng.blocks[0]:
            errs.put(f"rank {rank} {precision}: weights grew from {wb} to {eng.weight_bytes()} bytes under SP")
        orc_cls = WanOracleFp8Attn if precision == "fp8_attn" else WanOracleFp8
        for case in CASES[fname]:
            c = g["cases"][case]
            inp = synth.make_inputs(cfg, c["seed"], c["frames"], c["H"], c["W"], c["ctx_len"])
            out = _forward(eng, variant, c, inp)
            with eng.sequence_parallel_disabled():
                one = _forward(eng, variant, c, inp)
            ref = float((out.float() - c["out"]).norm() / c["out"].norm())
            n1 = float((out - one).norm() / one.norm())
            if tuple(out.shape) != tuple(c["out"].shape) or not ref < REF_BAR:
                errs.put(f"rank {rank} {precision} {case}: shape {tuple(out.shape)} vs reference {ref:.3e}")
            if rank == 0:
                want = _oracle(orc_cls(sd, **synth.oracle_kwargs(cfg)), variant, c, inp)
                qdq = float((out - want).norm() / want.norm())
                report.put(f"{fname}:{case} {precision}: vs oracle {qdq:.2e}, vs reference {ref:.2e}, vs one GPU {n1:.2e}")
                if not qdq < QDQ_BAR:
                    errs.put(f"rank 0 {precision} {case}: vs {orc_cls.__name__} {qdq:.3e}")
        dist.barrier()
        dist.destroy_process_group()
    except Exception as e:  # pragma: no cover
        import traceback
        errs.put(f"rank {rank}: {type(e).__name__}: {e}\n{traceback.format_exc()[-1500:]}")


def _run(target, *args, quiet=False):
    ctx = mp.get_context("spawn")
    errs, report = ctx.Queue(), ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, 2, port, *args, errs, report)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=900)
    msgs, lines = [], []
    while not errs.empty():
        msgs.append(errs.get())
    while not report.empty():
        lines.append(report.get())
    if not quiet:
        print("\n".join(lines))
    assert all(p.exitcode == 0 for p in procs) and not msgs, "\n".join(msgs)
    return lines


@pytest.mark.parametrize("precision", ["fp8", "fp8_attn"])
@pytest.mark.parametrize("fname", list(CASES))
def test_fp8_engine_under_ulysses_world2_gloo(fname, precision):
    _run(_worker, fname, precision)


def _bf16_calls_worker(rank, world, port, errs, report):
    """One 5B padded-grid forward and one 14B FramePack forward of a bf16 SP engine (transport "nccl"), every ops call and
    all-to-all recorded on rank 0."""
    try:
        _setup(rank, world, port)
        from helpers import torch_ops
        from oracle import synth
        from yume_b200 import dit
        log = []
        dit.ops = _Recorder(torch_ops, log)
        a2a = dist.all_to_all_single

        def logged_a2a(out, inp, *a, **k):
            log.append(f"all_to_all_single({_desc(out)},{_desc(inp)})")
            return a2a(out, inp, *a, **k)
        dist.all_to_all_single = logged_a2a
        calls = {}
        for fname, case in (("wan23_h8.pt", "5b_grid_padded"), ("wan21_h8.pt", "14b_pack_lfz8")):
            g = torch.load(ROOT / "tests" / "golden" / fname, weights_only=False)
            cfg = g["cfg"]
            kw = synth.oracle_kwargs(cfg)
            variant = kw.pop("variant")
            eng = dit.WanDiT(synth.make_state_dict(cfg, g["seed_w"]), variant, device="cpu", **kw)
            eng.enable_sequence_parallel(dist.group.WORLD, transport="nccl")
            c = g["cases"][case]
            inp = synth.make_inputs(cfg, c["seed"], c["frames"], c["H"], c["W"], c["ctx_len"])
            log.clear()
            _forward(eng, variant, c, inp)
            calls[f"{fname}:{case}"] = list(log)
        if rank == 0:
            report.put(json.dumps(calls))
        dist.barrier()
        dist.destroy_process_group()
    except Exception as e:  # pragma: no cover
        import traceback
        errs.put(f"rank {rank}: {type(e).__name__}: {e}\n{traceback.format_exc()[-1500:]}")


def test_bf16_sp_engine_makes_the_same_calls_as_before():
    """The bf16 Ulysses paths are untouched by the fp8 ones: the recorded call list of a bf16 SP forward equals the list pinned
    in tests/golden/sp_bf16_calls.json, recorded the same way before the fp8 Ulysses paths were added."""
    got = json.loads(_run(_bf16_calls_worker, quiet=True)[0])
    want = json.loads((ROOT / "tests" / "golden" / "sp_bf16_calls.json").read_text())
    assert sorted(got) == sorted(want)
    for key in want:
        assert got[key] == want[key], f"{key}: first difference at call " \
            f"{next((i for i, (a, b) in enumerate(zip(got[key], want[key])) if a != b), min(len(got[key]), len(want[key])))}"
