"""Ulysses parity on N GPUs (launch with torchrun): every golden forward case of both tiny models, sequence-parallel,
against the reference-generated outputs. Exit code != 0 on any mismatch.

YB_SP_PRECISION (default bf16) builds the engines with that precision. Under "fp8" / "fp8_attn" each output is held to the bars of
the one-GPU CPU tests: within 3e-2 of the fp8-qdq / fp8-attention oracle and within 5e-2 of the reference's forward; the distance
to the same engine on one GPU (`sequence_parallel_disabled`) is printed beside them."""
import os
import sys
from pathlib import Path

import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import synth  # noqa: E402  (test infrastructure)
from yume_b200.dit import WanDiT  # noqa: E402

TOL = 5e-3   # same bar as the single-GPU golden tests (tests/test_gpu_parity.py MODEL_TOL)
QDQ_BAR, REF_BAR = 3e-2, 5e-2   # fp8 precisions: tests/test_fp8_cpu.py, tests/test_fp8_attn_cpu.py


def _forward(ctx, eng, variant, c, inp):
    """The engine's forward of case c inside ctx() (e.g. eng.sequence_parallel_disabled)."""
    with ctx():
        if variant == "5b":
            return eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], latent_frame_zero=c["lfz"],
                               packed=c["flag"])
        return eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], y=inp["y"], clip_fea=inp["clip_fea"],
                           latent_frame_zero=c["lfz"], packed=c["rand_num_img"] >= 0.4)


def _oracle(precision, sd, cfg, variant, c, inp):
    """The fp8-qdq (precision "fp8") or fp8-attention ("fp8_attn") oracle's forward of case c, on the CPU."""
    from oracle.fp8 import WanOracleFp8
    from oracle.fp8_attn import WanOracleFp8Attn
    orc = (WanOracleFp8Attn if precision == "fp8_attn" else WanOracleFp8)(sd, **synth.oracle_kwargs(cfg))
    if variant == "5b":
        return orc.forward([inp["x"]], torch.tensor(c["t"]), [inp["context"]], seq_len=c["seq_len"], latent_frame_zero=c["lfz"],
                           flag=c["flag"])
    return orc.forward([inp["x"]], torch.tensor(c["t"]), [inp["context"]], seq_len=c["seq_len"], y=[inp["y"]],
                       clip_fea=inp["clip_fea"], latent_frame_zero=c["lfz"], rand_num_img=c["rand_num_img"])


def main():
    rank, local = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    if os.environ.get("YB_ATT_FORCE_SPLIT"):          # test hook: drive the KV split + peer-scatter combine path
        from yume_b200 import _lib
        _lib.load().yb_debug_force_split(int(os.environ["YB_ATT_FORCE_SPLIT"]))
    precision = os.environ.get("YB_SP_PRECISION", "bf16")
    bad = ran = 0
    for fname in ("wan23_tiny.pt", "wan21_tiny.pt", "wan23_h8.pt", "wan21_h8.pt"):   # 2-head and 8-head models
        g = torch.load(ROOT / "tests" / "golden" / fname, weights_only=False)
        cfg = g["cfg"]
        if cfg["num_heads"] % dist.get_world_size():
            continue
        sd = synth.make_state_dict(cfg, g["seed_w"])
        kw = synth.oracle_kwargs(cfg)
        variant = kw.pop("variant")
        eng = WanDiT(sd, variant, device=dev, precision=precision, **kw)
        eng.enable_sequence_parallel(dist.group.WORLD, transport=os.environ.get("YB_SP_TRANSPORT", "auto"))
        for name, c in g["cases"].items():
            inp = synth.make_inputs(cfg, c["seed"], c["frames"], c["H"], c["W"], c["ctx_len"])
            if variant == "5b":
                out = eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], latent_frame_zero=c["lfz"],
                                  packed=c["flag"])
            else:
                out = eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], y=inp["y"],
                                  clip_fea=inp["clip_fea"], latent_frame_zero=c["lfz"], packed=c["rand_num_img"] >= 0.4)
            r = float((out.cpu() - c["out"]).norm() / c["out"].norm())
            extra = ""
            if precision == "bf16":
                ok = out.shape == c["out"].shape and bool(torch.isfinite(out).all()) and r < TOL
            else:
                one = _forward(eng.sequence_parallel_disabled, eng, variant, c, inp)
                want = _oracle(precision, sd, cfg, variant, c, inp)
                q = float((out.cpu() - want).norm() / want.norm())
                n1 = float((out - one).norm() / one.norm())
                ok = out.shape == c["out"].shape and bool(torch.isfinite(out).all()) and r < REF_BAR and q < QDQ_BAR
                extra = f" vs {precision} oracle {q:.3e}, vs one GPU {n1:.3e}"
            bad += 0 if ok else 1
            ran += 1
            if rank == 0 or not ok:
                print(f"[rank {rank}] sp{dist.get_world_size()} {precision} ({eng.sp_transport}{'/p2p' if eng._sp_p2p else ''}) "
                      f"{name}: rel {r:.3e}{extra} {'ok' if ok else 'MISMATCH'}", flush=True)
    if ran == 0:
        bad += 1
        print(f"[rank {rank}] no golden model has heads divisible by world={dist.get_world_size()}", flush=True)
    t = torch.tensor([bad], device=dev)
    dist.all_reduce(t)
    dist.destroy_process_group()
    sys.exit(1 if t.item() else 0)


if __name__ == "__main__":
    main()
