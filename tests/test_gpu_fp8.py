"""End to end of WanDiT(precision="fp8") on the H100: against the fp8-qdq oracle (oracle/fp8.py) on the 2-head and 8-head
goldens of both trees, graph replay / context cache / repeat runs bit-identical to eager, and the weight memory it saves."""
import pytest
import torch

from oracle import synth
from oracle.fp8 import WanOracleFp8
from yume_b200.dit import FP8_WEIGHTS, WanDiT

pytestmark = pytest.mark.gpu

# the fp8 engine against the fp8-qdq oracle: the engine rounds q|k|v, the attention output and the cross q to bf16 like the bf16
# engine, and its tensor-core accumulation differs from the oracle's fp64 linear. Measured on the H100: goldens worst 1.55e-2,
# one block at the real 5B / 14B width 2.6e-2 (vs the fp32 oracle 5.3e-2)
QDQ_TOL = 3e-2

# wan21_h8:14b_grid_padded is the one case with k_len < L: seq_len 112 over 105 keys, the zero padding rows masked as keys
CASES = [("wan23_tiny.pt", "5b_pack_h10"), ("wan23_tiny.pt", "5b_grid_padded"), ("wan21_tiny.pt", "14b_pack_h4"),
         ("wan21_tiny.pt", "14b_grid"), ("wan23_h8.pt", "5b_pack_h10"), ("wan21_h8.pt", "14b_pack_lfz8"),
         ("wan21_h8.pt", "14b_grid_padded")]


def _inputs(cfg, c):
    return synth.make_inputs(cfg, c["seed"], c["frames"], c["H"], c["W"], c["ctx_len"])


def _engine_forward(eng, cfg, c, inp):
    if cfg["variant"] == "5b":
        return eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], latent_frame_zero=c["lfz"], packed=c["flag"])
    return eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], y=inp["y"], clip_fea=inp["clip_fea"],
                       latent_frame_zero=c["lfz"], packed=c["rand_num_img"] >= 0.4)


def _oracle_forward(orc, cfg, c, inp):
    if cfg["variant"] == "5b":
        return orc.forward([inp["x"]], torch.tensor(c["t"]), [inp["context"]], seq_len=c["seq_len"], latent_frame_zero=c["lfz"],
                           flag=c["flag"])
    return orc.forward([inp["x"]], torch.tensor(c["t"]), [inp["context"]], seq_len=c["seq_len"], y=[inp["y"]],
                       clip_fea=inp["clip_fea"], latent_frame_zero=c["lfz"], rand_num_img=c["rand_num_img"])


def _engine(cfg, sd, precision):
    kw = synth.oracle_kwargs(cfg)
    variant = kw.pop("variant")
    return WanDiT(sd, variant, device="cuda", precision=precision, **kw)


@pytest.mark.parametrize("fname,case", CASES)
def test_fp8_engine_matches_the_fp8_qdq_oracle(golden_dir, fname, case):
    g = torch.load(golden_dir / fname, weights_only=False)
    cfg, c = g["cfg"], g["cases"][case]
    sd = synth.make_state_dict(cfg, g["seed_w"])
    inp = _inputs(cfg, c)
    got = _engine_forward(_engine(cfg, sd, "fp8"), cfg, c, inp).cpu()
    want = _oracle_forward(WanOracleFp8(sd, **synth.oracle_kwargs(cfg)), cfg, c, inp)
    rel = float((got - want).norm() / want.norm())
    ref = float((got - c["out"]).norm() / c["out"].norm())
    print(f"{fname}:{case} fp8 engine vs fp8-qdq oracle {rel:.3e}, vs the reference's bf16 forward {ref:.3e}")
    assert rel < QDQ_TOL


@pytest.mark.parametrize("name", ["CFG_5B", "CFG_14B"])
def test_one_block_at_real_width(name):
    """Block 0 of a one-layer model at the real 5B / 14B width: the fp8 engine's block seam against the fp8-qdq oracle block
    (tight) and against the fp32 oracle (the cost of fp8)."""
    from oracle.wan_dit import WanOracle, grid_freqs
    cfg = dict(getattr(synth, name), num_layers=1)
    sd = synth.make_state_dict(cfg, 7)
    eng = _engine(cfg, sd, "fp8")
    C, L = cfg["dim"], 2 * 16 * 24
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(L, C, generator=gen)
    e = 0.5 * torch.randn(L, 6, C, generator=gen) if cfg["variant"] == "5b" else 0.5 * torch.randn(6, C, generator=gen)
    ctx = torch.randn(cfg["text_len"] + (257 if cfg["variant"] == "14b" else 0), C, generator=gen)
    got = eng.block_forward(0, x, e, (2, 16, 24), ctx).cpu()
    kw = synth.oracle_kwargs(cfg)
    orc8, orc = WanOracleFp8(sd, **kw), WanOracle(sd, **kw)
    fr = grid_freqs(orc.tables, 2, 16, 24)
    e0 = e[None]
    want8 = orc8.block(0, x[None], e0, fr, ctx.to(torch.bfloat16).float()[None])[0]
    want = orc.block(0, x[None], e0, fr, ctx.to(torch.bfloat16).float()[None])[0]
    d8 = float(((got - x) - (want8 - x)).norm() / (want8 - x).norm())
    d32 = float(((got - x) - (want - x)).norm() / (want - x).norm())
    print(f"{name} block: vs fp8-qdq oracle {d8:.3e}, vs fp32 oracle {d32:.3e}")
    assert d8 < QDQ_TOL
    assert d32 < 0.1


def test_graph_replay_context_cache_and_repeat_runs_are_bit_identical(golden_dir):
    g = torch.load(golden_dir / "wan23_h8.pt", weights_only=False)
    cfg, c = g["cfg"], g["cases"]["5b_pack_h10"]
    sd = synth.make_state_dict(cfg, g["seed_w"])
    inp = _inputs(cfg, c)
    eng = _engine(cfg, sd, "fp8")
    eng.context_cache = False
    a = _engine_forward(eng, cfg, c, inp)
    b = _engine_forward(eng, cfg, c, inp)
    assert torch.equal(a, b), "two eager runs differ"
    eng.context_cache = True
    ctx = inp["context"].cuda()
    inp_c = dict(inp, context=ctx)
    cached = [_engine_forward(eng, cfg, c, inp_c) for _ in range(2)]
    assert torch.equal(a, cached[0]) and torch.equal(a, cached[1])
    eng.use_cuda_graph = True
    graphed = [_engine_forward(eng, cfg, c, inp_c) for _ in range(3)]
    for r in graphed:
        assert torch.equal(a, r)


def test_weight_memory_drops_by_the_converted_bytes():
    cfg = dict(synth.CFG_5B, num_layers=2)
    sd = synth.make_state_dict(cfg, 1)
    bf = _engine(cfg, sd, "bf16")
    f8 = _engine(cfg, sd, "fp8")
    n_conv = sum(bf.blocks[0][k].numel() for k in FP8_WEIGHTS) * cfg["num_layers"]
    n_rows = sum(bf.blocks[0][k].shape[0] for k in FP8_WEIGHTS) * cfg["num_layers"]
    want = n_conv * 2 - (n_conv * 1 + n_rows * 4)          # bf16 -> e4m3 values + one f32 scale per output channel
    saved = bf.weight_bytes() - f8.weight_bytes()
    print(f"weights: bf16 {bf.weight_bytes() / 2**30:.3f} GiB, fp8 {f8.weight_bytes() / 2**30:.3f} GiB, saved {saved / 2**30:.3f} GiB")
    assert abs(saved - want) <= 0.01 * want
