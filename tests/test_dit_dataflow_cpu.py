"""The launch-by-launch dataflow check of the WanDiT block (tests/helpers/dit_dataflow.py) over the torch stand-ins at tiny width.

The clean engine must pass every path, precision and seam: each launch of block 1 (of 3) and of the cross K|V GEMMs is the spec's
stage, with the spec's operands, and its output is within the kernel contract's bound. Each wiring defect below, patched into
the engine, must fail with a message that names the stage and the operand; the model-level metric the forward tests use (relative
Frobenius error against the matching oracle) is printed beside it, which shows the defects those tests would miss."""
import contextlib

import pytest
import torch

from helpers import dit_dataflow as DF
from helpers import torch_ops_fp8_attn
from oracle import synth
from oracle.fp8 import WanOracleFp8
from oracle.fp8_attn import WanOracleFp8Attn
from oracle.wan_dit import WanOracle
from yume_b200 import dit

LAYERS, BLOCK = 3, 1
CFGS = {"5b": dict(synth.CFG_5B_TINY, num_layers=LAYERS), "14b": dict(synth.CFG_14B_TINY, num_layers=LAYERS)}
# tiny geometries of the four paths: (frames, H, W, latent_frame_zero, padding rows past the grid)
PATHS = {"5b_grid": (2, 8, 12, None, 16), "5b_framepack": (6, 8, 12, 2, 0), "14b_framepack": (12, 8, 12, 4, 0),
         "14b_grid_padded": (2, 8, 12, None, 16)}
PRECISIONS = ("bf16", "fp8", "fp8_attn")
ORACLES = {"bf16": WanOracle, "fp8": WanOracleFp8, "fp8_attn": WanOracleFp8Attn}
# the end-to-end bars of tests/test_gpu_parity.py, tests/test_gpu_fp8.py and tests/test_gpu_fp8_attn.py
MODEL_BARS = {"bf16": 5e-3, "fp8": 3e-2, "fp8_attn": 4e-2}


@pytest.fixture()
def cpu(monkeypatch):
    monkeypatch.setattr(dit, "ops", torch_ops_fp8_attn)
    monkeypatch.setattr(torch.cuda, "device", lambda *_a, **_k: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    return monkeypatch


def _variant(path):
    return path.split("_")[0]


def _engine(variant, precision, sd):
    kw = synth.oracle_kwargs(CFGS[variant])
    kw.pop("variant")
    return dit.WanDiT(sd, variant, device="cpu", precision=precision, **kw)


def _sd(variant):
    return synth.make_state_dict(CFGS[variant], 11)


def _args(path):
    f, h, w, lfz, pad = PATHS[path]
    return DF.path_inputs(CFGS[_variant(path)], path, f, h, w, lfz, pad, seed=5)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("path", list(PATHS))
def test_clean_engine_meets_the_spec(cpu, path, precision):
    v = _variant(path)
    sd = _sd(v)
    eng = _engine(v, precision, sd)
    ck = DF.run_path(cpu, dit, eng, sd, CFGS[v], precision, _args(path), BLOCK, f"{path}/{precision}")
    assert ck.pos == len(ck.program)
    print(f"{path}/{precision}: worst |err|/bound per stage: {ck.report()}")


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("variant", ["5b", "14b"])
def test_seams_meet_the_spec(cpu, variant, precision):
    """block_forward on the packed-freqs path (with its one-block cross K|V launches) and self_attention_forward."""
    sd = _sd(variant)
    eng = _engine(variant, precision, sd)
    ck = DF.run_block_seam(cpu, dit, eng, sd, CFGS[variant], precision, BLOCK, 96, f"block_forward {variant}/{precision}")
    assert ck.pos == len(ck.program)
    print(f"block_forward {variant}/{precision}: {ck.report()}")
    cpu.undo()
    cpu.setattr(dit, "ops", torch_ops_fp8_attn)
    cpu.setattr(torch.cuda, "device", lambda *_a, **_k: contextlib.nullcontext())
    eng = _engine(variant, precision, sd)
    ck = DF.run_self_attention_seam(cpu, dit, eng, sd, CFGS[variant], precision, BLOCK, 96,
                                    f"self_attention_forward {variant}/{precision}")
    assert ck.pos == len(ck.program)
    print(f"self_attention_forward {variant}/{precision}: {ck.report()}")


# ------------------------------------------------------------------------------------------------------------
# defects
# ------------------------------------------------------------------------------------------------------------
def _padding_keys(mp, eng):
    """14B padded grid: every row a self-attention key (k_len = L, not F*H*W)."""
    mp.setattr(eng, "_block", lambda i, xs, mod, tok, rope, rl, ctx, L_true=None:
               eng._block_body(i, xs, mod[i], tok, rope, rl, ctx[i], xs.shape[0]))


def _tok_boundary(mp, eng):
    """The history / new-frame boundary of the token index one row late: the first new token takes the history timestep."""
    real = eng._block_body

    def body(i, xs, m, tok, *a):
        tok = tok.clone()
        tok[int((tok == 0).sum())] = 0
        return real(i, xs, m, tok, *a)
    mp.setattr(eng, "_block_body", body)


def _ffn_gate(mp, eng):
    """The FFN output gated by the attention gate row."""
    real = eng._cross_and_ffn

    def f(b, xs, qkv, att, m, tok, ctx):
        m = m.clone()
        m[:, 5] = m[:, 2]
        return real(b, xs, qkv, att, m, tok, ctx)
    mp.setattr(eng, "_cross_and_ffn", f)


def _rope_shift(mp, eng):
    """The second FramePack segment's RoPE rows one frame late."""
    real = eng._rope_table

    def table(segments):
        segs = list(segments)
        if len(segs) > 1:
            f, h, w, f0 = segs[1]
            segs[1] = (f, h, w, f0 + 1)
        return real(segs)
    mp.setattr(eng, "_rope_table", table)


def _stale_att8(mp, eng):
    """The cross-attention output quantised into a buffer of its own, the cross o-projection reading the self-attention's att8."""
    real = eng._quant
    n = {"att8": 0}

    def quant(x, key):
        if key != "att8":
            return real(x, key)
        n["att8"] += 1
        if n["att8"] % 2:
            return real(x, key)
        real(x, "att8_cross")
        return eng._act8("att8", *x.shape)
    mp.setattr(eng, "_quant", quant)


def _img_no_accumulate(mp, eng):
    """The image attention overwrites the text attention instead of adding to it."""
    ops = dit.ops

    class Shim:
        def __getattr__(self, name):
            return getattr(ops, name)

        def attention(self, *a, accumulate=False, **k):
            return ops.attention(*a, **k)
    mp.setattr(dit, "ops", Shim())


def _next_block_kv(mp, eng):
    """Block i given block i+1's cross-attention K|V."""
    mp.setattr(eng, "_block", lambda i, xs, mod, tok, rope, rl, ctx, L_true=None:
               eng._block_body(i, xs, mod[i], tok, rope, rl, ctx[(i + 1) % len(ctx)],
                               L_true if L_true is not None else xs.shape[0]))


def _nq_nk_swap(mp, eng):
    """The self-attention's norm_q and norm_k weights swapped in the re-pack."""
    for b in eng.blocks:
        b["nq"], b["nk"] = b["nk"], b["nq"]


# name: (defect, path, precisions, installed after the checker, {precision or None: (stage, operand)})
DEFECTS = {
    "padding_rows_as_keys": (_padding_keys, "14b_grid_padded", PRECISIONS, False,
                             {"bf16": ("self_att", "k"), "fp8": ("self_att", "k"), "fp8_attn": ("v_t8", "v")}),
    "tok_idx_boundary_one_row_late": (_tok_boundary, "5b_framepack", PRECISIONS, False, {None: ("norm1", "tok_idx")}),
    "ffn_gate_is_attention_gate": (_ffn_gate, "5b_framepack", PRECISIONS, False, {None: ("ffn2", "gate")}),
    "framepack_segment_rope_one_frame_late": (_rope_shift, "14b_framepack", PRECISIONS, False, {None: ("qk_rope", "rope")}),
    "stale_att8_in_cross_o": (_stale_att8, "5b_grid", ("fp8", "fp8_attn"), False, {None: ("cross_o", "a")}),
    "image_attention_without_accumulate": (_img_no_accumulate, "14b_framepack", PRECISIONS, True,
                                           {None: ("img_att", "accumulate")}),
    "block_given_next_blocks_cross_kv": (_next_block_kv, "14b_framepack", PRECISIONS, False, {None: ("cross_att", "k")}),
    "nq_nk_swapped": (_nq_nk_swap, "5b_grid", PRECISIONS, False, {None: ("qk_rope", "wq")}),
}
DEFECT_CASES = [(d, p) for d, spec in DEFECTS.items() for p in spec[2]]


def _model_metric(path, precision, defect):
    """Relative Frobenius error of the defective engine's forward against the matching oracle (what the forward tests see)."""
    v = _variant(path)
    sd = _sd(v)
    args = _args(path)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(dit, "ops", torch_ops_fp8_attn)
        mp.setattr(torch.cuda, "device", lambda *_a, **_k: contextlib.nullcontext())
        mp.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
        eng = _engine(v, precision, sd)
        defect(mp, eng)
        got = DF.engine_forward(eng, args)
    want = DF.oracle_forward(ORACLES[precision](sd, **synth.oracle_kwargs(CFGS[v])), CFGS[v], args)
    return float((got - want).norm() / want.norm())


@pytest.mark.parametrize("name,precision", DEFECT_CASES)
def test_defect_is_caught_at_its_stage_and_operand(cpu, name, precision):
    defect, path, _, after, where = DEFECTS[name]
    stage, operand = where.get(precision, where.get(None))
    v = _variant(path)
    sd = _sd(v)
    eng = _engine(v, precision, sd)
    if not after:
        defect(cpu, eng)
    args = _args(path)
    real_install = DF.install

    def install(*a, **k):
        ck = real_install(*a, **k)
        if after:
            defect(cpu, eng)
        return ck
    cpu.setattr(DF, "install", install)
    with pytest.raises(AssertionError) as err:
        DF.run_path(cpu, dit, eng, sd, CFGS[v], precision, args, BLOCK, f"{path}/{precision}")
    msg = str(err.value)
    cpu.undo()
    rel = _model_metric(path, precision, defect)
    bar = MODEL_BARS[precision]
    print(f"{name} [{path}/{precision}]: caught: {msg}\n    model level: {rel:.3e} against the {precision} oracle, bar {bar:.0e}: "
          f"{'missed' if rel < bar else 'caught'} by the forward test")
    assert f"stage '{stage}'" in msg and f"operand '{operand}'" in msg, msg
