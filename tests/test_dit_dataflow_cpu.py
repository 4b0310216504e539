"""The launch-by-launch dataflow check of the WanDiT forward (tests/helpers/dit_dataflow.py) over the torch stand-ins at tiny width.

The clean engine must pass every path, precision and seam: each launch of the forward (the FramePack or grid embedders, the time
tables, the context MLPs, the cross K|V GEMMs, block 1 of 2 and the head) is the spec's stage, with the spec's operands, and its
output is within the kernel contract's bound; the stream the first block receives is the embedders' output in the reference's
token order. Every path runs after an unchecked forward with a longer prompt (and, on a padded grid, a larger grid at the same
seq_len), so a dropped zeroing of a reused workspace shows. Each wiring defect below, patched into the engine, must fail with a
message that names the stage and the operand; the model-level metric the forward tests use (relative Frobenius error against
the matching oracle) is printed beside it, which shows the defects those tests would miss."""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from helpers import dit_dataflow as DF
from helpers import torch_ops_fp8_attn
from oracle import synth
from oracle.fp8 import WanOracleFp8
from oracle.fp8_attn import WanOracleFp8Attn
from oracle.wan_dit import WanOracle
from yume_b200 import dit

LAYERS, BLOCK = 2, 1
CFGS = {"5b": dict(synth.CFG_5B_TINY, num_layers=LAYERS), "14b": dict(synth.CFG_14B_TINY, num_layers=LAYERS)}
PRECISIONS = ("bf16", "fp8", "fp8_attn")
# tiny geometries: (frames, H, W, latent_frame_zero, padding rows past the grid, per-frame t or None)
PATHS = {"5b_grid": (2, 8, 12, None, 16, None), "5b_framepack": (6, 8, 12, 2, 0, None), "14b_framepack": (12, 8, 12, 4, 0, None),
         "14b_grid_padded": (2, 8, 12, None, 16, None),
         # the FramePack ladder at depth 1-5 (history 3, 10, 40, 100, 400), an odd latent where the plain patch_embedding's
         # floor and the convpadd ceil disagree, 20 distinct per-frame timesteps (two 16-row time chunks), 14B at depth 5
         **{f"5b_framepack_d{d}": (h + 2, 8, 12, 2, 0, None) for d, h in enumerate((3, 10, 40, 100, 400), 1)},
         "5b_framepack_odd": (42, 9, 13, 2, 0, None),
         "5b_grid_t20": (20, 8, 12, None, 0, [float(10 + 47 * i) for i in range(20)]),
         "14b_framepack_d5": (404, 8, 12, 4, 0, None)}
CASES = [(p, q) for p in ("5b_grid", "5b_framepack", "14b_framepack", "14b_grid_padded") for q in PRECISIONS] + \
    [(p, "bf16") for p in PATHS if p not in ("5b_grid", "5b_framepack", "14b_framepack", "14b_grid_padded")] + \
    [("5b_framepack_d3", "fp8"), ("5b_framepack_d3", "fp8_attn")]
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
    f, h, w, lfz, pad, t = PATHS[path]
    return DF.path_inputs(CFGS[_variant(path)], path, f, h, w, lfz, pad, seed=5, t=t)


def _warm(path):
    f, h, w, lfz, pad, t = PATHS[path]
    return DF.warm_inputs(CFGS[_variant(path)], path, f, h, w, lfz, pad, seed=5, t=t)


@pytest.mark.parametrize("path,precision", CASES)
def test_clean_engine_meets_the_spec(cpu, path, precision):
    v = _variant(path)
    sd = _sd(v)
    eng = _engine(v, precision, sd)
    ck = DF.run_path(cpu, dit, eng, sd, CFGS[v], precision, _args(path), BLOCK, f"{path}/{precision}", warm=_warm(path))
    assert ck.pos == len(ck.program) and tuple(ck.entered) == DF.PHASES
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


def _shim(mp, **entries):
    """dit.ops with some entries replaced: fn(real entry, *args, **kwargs)."""
    ops = dit.ops

    class Shim:
        def __getattr__(self, name):
            return getattr(ops, name)
    sh = Shim()
    for name, fn in entries.items():
        setattr(sh, name, lambda *a, _f=fn, _r=getattr(ops, name), **k: _f(_r, *a, **k))
    mp.setattr(dit, "ops", sh)


def _window_off_by_one(mp, eng):
    """framepack_plan's third window starting one history frame early (its frames overlap the window before)."""
    real = dit.framepack_plan

    def plan(hist, branch_hist):
        segs = real(hist, branch_hist)
        s = segs[2].frames
        segs[2].frames = slice(s.start - 1, s.stop)
        return segs
    mp.setattr(dit, "framepack_plan", plan)


def _twox_f_view_in_dim(mp, eng):
    """The deepest level's [in_dim, f, h, w] view of the 2x_f GEMM output strided by in_dim instead of its padded row stride."""
    real = torch.as_strided

    def strided(t, size, stride, *a):
        if len(size) == 4 and stride[0] == 1 and stride[3] == t.stride(0) != size[0]:
            ld = size[0]
            stride = (1, size[2] * size[3] * ld, size[3] * ld, ld)
        return real(t, size, stride, *a)
    mp.setattr(torch, "as_strided", strided)


def _patch_embedding_ceil(mp, eng):
    """The plain patch_embedding rounding an odd H / W up (zero fill, as convpadd) instead of dropping the last row / column."""
    real = eng._embed_tokens

    def embed(u, name, patch, *a):
        if name == "patch_embedding":
            u = F.pad(u, (0, u.shape[3] % patch, 0, u.shape[2] % patch))
        return real(u, name, patch, *a)
    mp.setattr(eng, "_embed_tokens", embed)


def _head_scale_shift_swap(mp, eng):
    """The head's LayerNorm modulated with head row 0 as scale and row 1 as shift."""
    def ln(real, x, out, scale, shift, tok_idx=None, weight=None, bias=None, eps=1e-6):
        if out.dtype == torch.float32 and weight is None:
            scale, shift = shift, scale
        return real(x, out, scale, shift, tok_idx, weight, bias, eps=eps)
    _shim(mp, ln_modulate=ln)


def _head_from_e0(mp, eng):
    """The head table built from the first C columns of e0 (the block table's shift_a chunk) instead of e."""
    def tables(t_unique):
        ops = dit.ops
        e = ops.linear_f32_small(ops.sinusoidal(t_unique, eng.freq_dim), *eng.time0)
        e = ops.linear_f32_small(e, *eng.time2, silu_in=True)
        e0 = ops.linear_f32_small(e, *eng.tproj, silu_in=True)
        U, C = e.shape[0], eng.dim
        mod = ops.bcast_add(eng.block_mod, e0).view(eng.layers, U, 6, C)
        return e, mod, ops.bcast_add(e0[:, :C].contiguous(), eng.head_mod).view(U, 2, C)
    mp.setattr(eng, "_time_tables", tables)


def _time_chunk_local(mp, eng):
    """The token index of the second 16-row time chunk counted from that chunk's first row."""
    real = torch.unique

    def unique(t, *a, return_inverse=False, **k):
        out = real(t, *a, return_inverse=return_inverse, **k)
        if not return_inverse:
            return out
        return out[0], torch.where(out[1] >= 16, out[1] - 16, out[1])
    mp.setattr(torch, "unique", unique)


def _ctx_not_zeroed(mp, eng):
    """ctx_in not zeroed: the rows past a shorter prompt keep the previous prompt's."""
    real = eng._buf

    def buf(key, shape, dtype):
        t = real(key, shape, dtype)
        if key == "ctx_in":
            t.zero_ = lambda: t
        return t
    mp.setattr(eng, "_buf", buf)


def _xs_not_zeroed(mp, eng):
    """The padding rows of a reused residual stream not zeroed."""
    mp.setattr(eng, "_token_stream", lambda L, n_real: (eng._buf("xs", (L, eng.dim), torch.float32), (0, L)))


def _text_gelu_erf(mp, eng):
    """The text MLP's GELU evaluated with erf (MLPProj's) instead of tanh."""
    def gemm(real, a, w, bias, out, epilogue, *r, **k):
        if w is eng.text0[0]:
            epilogue = dit.ops.YB_EPI_GELU_ERF_BF16
        return real(a, w, bias, out, epilogue, *r, **k)
    _shim(mp, gemm=gemm)


def _img_ln_eps(mp, eng):
    """The image MLP's LayerNorms at eps 1e-6 (the blocks') instead of nn.LayerNorm's 1e-5."""
    def ln(real, *a, eps=1e-6, **k):
        return real(*a, eps=1e-6 if eps == 1e-5 else eps, **k)
    _shim(mp, ln_modulate=ln)


def _unpatchify_row0(mp, eng):
    """unpatchify reading the head output from row 0 instead of the first new-frame row L_hist."""
    def unpatchify(real, y, *a):
        return real(y._base if y._base is not None else y, *a)
    _shim(mp, unpatchify=unpatchify)


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
    "framepack_window_off_by_one": (_window_off_by_one, "5b_framepack_d2", ("bf16",), False, {None: ("embed[2].patchify", "x")}),
    "2x_f_view_strided_by_in_dim": (_twox_f_view_in_dim, "5b_framepack_d5", ("bf16",), False,
                                    {None: ("embed[1].patchify", "x")}),
    "patch_embedding_ceil_on_odd_latent": (_patch_embedding_ceil, "5b_framepack_odd", ("bf16",), False,
                                           {None: ("embed[0].patchify", "x")}),
    "head_scale_and_shift_swapped": (_head_scale_shift_swap, "5b_framepack", ("bf16",), True, {None: ("head_ln", "scale")}),
    "head_table_from_e0": (_head_from_e0, "5b_framepack", ("bf16",), False, {None: ("time[0].head", "a")}),
    "second_time_chunk_indexed_chunk_locally": (_time_chunk_local, "5b_grid_t20", ("bf16",), False,
                                                {None: ("block 0 input", "tok_idx")}),
    "ctx_in_not_zeroed": (_ctx_not_zeroed, "14b_framepack", ("bf16",), False, {None: ("text0", "a")}),
    "xs_padding_not_zeroed": (_xs_not_zeroed, "5b_grid", ("bf16",), False, {None: ("block 0 input", "xs")}),
    "text_mlp_gelu_erf": (_text_gelu_erf, "5b_grid", ("bf16",), True, {None: ("text0", "epilogue")}),
    "image_layernorm_eps_1e-6": (_img_ln_eps, "14b_framepack", ("bf16",), True, {None: ("img_ln0", "eps")}),
    "unpatchify_from_row_0": (_unpatchify_row0, "5b_framepack", ("bf16",), True, {None: ("unpatchify", "y")}),
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
        DF.engine_forward(eng, _warm(path))
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
    real_install = DF.install_forward

    def install(*a, **k):
        ck = real_install(*a, **k)
        if after:
            defect(cpu, eng)
        return ck
    cpu.setattr(DF, "install_forward", install)
    with pytest.raises(AssertionError) as err:
        DF.run_path(cpu, dit, eng, sd, CFGS[v], precision, args, BLOCK, f"{path}/{precision}", warm=_warm(path))
    msg = str(err.value)
    cpu.undo()
    rel = _model_metric(path, precision, defect)
    bar = MODEL_BARS[precision]
    print(f"{name} [{path}/{precision}]: caught: {msg}\n    model level: {rel:.3e} against the {precision} oracle, bar {bar:.0e}: "
          f"{'missed' if rel < bar else 'caught'} by the forward test")
    assert f"stage '{stage}'" in msg and f"operand '{operand}'" in msg, msg
