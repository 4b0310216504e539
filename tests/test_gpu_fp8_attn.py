"""End to end of WanDiT(precision="fp8_attn") on the H100: against the fp8-attention oracle (oracle/fp8_attn.py) on the goldens of
tests/test_gpu_fp8.py, one block at the real 5B and 14B width against that oracle and the fp32 oracle, and eager, context-cache
and graph-replay runs bit-identical to each other."""
import pytest
import torch

from oracle import synth
from oracle.fp8_attn import WanOracleFp8Attn
from test_gpu_fp8 import CASES, _engine, _engine_forward, _inputs, _oracle_forward

pytestmark = pytest.mark.gpu

# the engine against the fp8-attention oracle. Besides what tests/test_gpu_fp8.py's QDQ_TOL absorbs, the kernel rounds
# P = 256 p to e4m3 against its running maximum, which the oracle's whole-row fp64 softmax does not model. Measured on the H100:
# goldens worst 1.63e-2, one block at the real 5B / 14B width 2.82e-2 / 3.03e-2 (vs the fp32 oracle 5.3e-2)
QDQ_TOL = 4e-2


@pytest.mark.parametrize("fname,case", CASES)
def test_fp8_attn_engine_matches_the_oracle(golden_dir, fname, case):
    g = torch.load(golden_dir / fname, weights_only=False)
    cfg, c = g["cfg"], g["cases"][case]
    sd = synth.make_state_dict(cfg, g["seed_w"])
    inp = _inputs(cfg, c)
    got = _engine_forward(_engine(cfg, sd, "fp8_attn"), cfg, c, inp).cpu()
    want = _oracle_forward(WanOracleFp8Attn(sd, **synth.oracle_kwargs(cfg)), cfg, c, inp)
    rel = float((got - want).norm() / want.norm())
    ref = float((got - c["out"]).norm() / c["out"].norm())
    print(f"{fname}:{case} fp8_attn engine vs fp8-attention oracle {rel:.3e}, vs the reference's bf16 forward {ref:.3e}")
    assert rel < QDQ_TOL


@pytest.mark.parametrize("name", ["CFG_5B", "CFG_14B"])
def test_one_block_at_real_width(name):
    """Block 0 of a one-layer model at the real 5B / 14B width: the engine's block seam against the fp8-attention oracle block
    and against the fp32 oracle (the cost of fp8), with the bar of precision="fp8"."""
    from oracle.wan_dit import WanOracle, grid_freqs
    cfg = dict(getattr(synth, name), num_layers=1)
    sd = synth.make_state_dict(cfg, 7)
    eng = _engine(cfg, sd, "fp8_attn")
    C, L = cfg["dim"], 2 * 16 * 24
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(L, C, generator=gen)
    e = 0.5 * torch.randn(L, 6, C, generator=gen) if cfg["variant"] == "5b" else 0.5 * torch.randn(6, C, generator=gen)
    ctx = torch.randn(cfg["text_len"] + (257 if cfg["variant"] == "14b" else 0), C, generator=gen)
    got = eng.block_forward(0, x, e, (2, 16, 24), ctx).cpu()
    kw = synth.oracle_kwargs(cfg)
    orc8, orc = WanOracleFp8Attn(sd, **kw), WanOracle(sd, **kw)
    fr = grid_freqs(orc.tables, 2, 16, 24)
    e0 = e[None]
    want8 = orc8.block(0, x[None], e0, fr, ctx.to(torch.bfloat16).float()[None])[0]
    want = orc.block(0, x[None], e0, fr, ctx.to(torch.bfloat16).float()[None])[0]
    d8 = float(((got - x) - (want8 - x)).norm() / (want8 - x).norm())
    d32 = float(((got - x) - (want - x)).norm() / (want - x).norm())
    print(f"{name} block: vs fp8-attention oracle {d8:.3e}, vs fp32 oracle {d32:.3e}")
    assert d8 < QDQ_TOL
    assert d32 < 0.1


def test_eager_context_cache_and_graph_replay_are_bit_identical(golden_dir):
    g = torch.load(golden_dir / "wan23_h8.pt", weights_only=False)
    cfg, c = g["cfg"], g["cases"]["5b_pack_h10"]
    sd = synth.make_state_dict(cfg, g["seed_w"])
    inp = _inputs(cfg, c)
    eng = _engine(cfg, sd, "fp8_attn")
    eng.context_cache = False
    a = _engine_forward(eng, cfg, c, inp)
    b = _engine_forward(eng, cfg, c, inp)
    assert torch.equal(a, b), "two eager runs differ"
    eng.context_cache = True
    inp_c = dict(inp, context=inp["context"].cuda())
    cached = [_engine_forward(eng, cfg, c, inp_c) for _ in range(2)]
    assert torch.equal(a, cached[0]) and torch.equal(a, cached[1])
    eng.use_cuda_graph = True
    graphed = [_engine_forward(eng, cfg, c, inp_c) for _ in range(3)]
    for r in graphed:
        assert torch.equal(a, r)
