"""The WanDiT block launch by launch on the H100 (tests/helpers/dit_dataflow.py): one real-width block (block 1 of a 2-layer 5B / 14B
model) and the cross K|V launches in front of it run inside the engine's own forward, with a checking wrapper around every ops
entry. Each launch must be the spec's next stage, take exactly the operands the spec names (buffer, view, row count, scale table,
gate row, token index, k_len, RoPE rows), and produce an output within its kernel's contract bound, in bf16, fp8 and fp8_attn.

Paths: 5B grid with a scalar t (gate without token index, padding rows as keys), 5B FramePack (token index, per-token RoPE), 14B
FramePack (image branch with accumulate), 14B padded grid (k_len < L), each at a few thousand tokens; the 5B grid at L = 18 480
and the 14B grid at seq_len 43 008 over 42 840 keys; block_forward on the packed-freqs path and self_attention_forward. Each
cell prints its worst |err| / bound per stage and its wall time."""
import ctypes
import time

import pytest
import torch

from helpers import dit_dataflow as DF
from oracle import synth
from yume_b200 import dit

pytestmark = pytest.mark.gpu

LAYERS, BLOCK = 2, 1
CFGS = {"5b": dict(synth.CFG_5B, num_layers=LAYERS), "14b": dict(synth.CFG_14B, num_layers=LAYERS)}
PRECISIONS = ("bf16", "fp8", "fp8_attn")
# (frames, H, W, latent_frame_zero, padding rows past the grid): L = 2 048, 2 496, 3 072, 2 048 (1 920 keys)
PATHS = {"5b_grid": (5, 32, 48, None, 128), "5b_framepack": (8, 32, 48, 4, 0), "14b_framepack": (14, 32, 48, 4, 0),
         "14b_grid_padded": (5, 32, 48, None, 128)}
# production: the 5B 121-frame grid (L = 21 x 22 x 40 = 18 480) and the 14B 81-frame grid at seq_len 43 008 (42 840 keys)
PROD = {"5b_grid": (21, 44, 80, None, 0), "14b_grid_padded": (21, 68, 120, None, 168)}

_SD, _ENG = {}, {}


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()
    yield
    _ENG.clear()
    _SD.clear()


def _sd(variant):
    if variant not in _SD:
        _SD[variant] = synth.make_state_dict(CFGS[variant], 21)
    return _SD[variant]


def _engine(variant, precision):
    if (variant, precision) not in _ENG:
        kw = synth.oracle_kwargs(CFGS[variant])
        kw.pop("variant")
        _ENG[(variant, precision)] = dit.WanDiT(_sd(variant), variant, device="cuda", precision=precision, **kw)
    return _ENG[(variant, precision)]


def _att_plan(Lq, Lk, H, flags):
    """KV segments the library plans for an attention launch (the combine term of attention_bound_prod / attention_fp8_bound)."""
    from yume_b200 import _lib
    out = (ctypes.c_int * 4)()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert _lib.load().yb_attention_plan(Lq, Lk, H, sms, flags, out) == 0
    return out[2]


def _run_path(monkeypatch, path, precision, geom):
    v = path.split("_")[0]
    f, h, w, lfz, pad = geom
    args = DF.path_inputs(CFGS[v], path, f, h, w, lfz, pad, seed=5)
    tag = f"{path} F{f} {h}x{w} seq_len {args['seq_len']} / {precision}"
    t0 = time.time()
    ck = DF.run_path(monkeypatch, dit, _engine(v, precision), _sd(v), CFGS[v], precision, args, BLOCK, tag, att_plan=_att_plan)
    torch.cuda.synchronize()
    assert ck.pos == len(ck.program)
    print(f"\n[dataflow] {tag}: {len(ck.program)} stages, wall {time.time() - t0:.1f} s; worst |err|/bound: {ck.report()}")
    torch.cuda.empty_cache()


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("path", list(PATHS))
def test_block_dataflow(monkeypatch, path, precision):
    _run_path(monkeypatch, path, precision, PATHS[path])


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("path", list(PROD))
def test_block_dataflow_production_length(monkeypatch, path, precision):
    _run_path(monkeypatch, path, precision, PROD[path])


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("variant", ["5b", "14b"])
def test_seams_dataflow(monkeypatch, variant, precision):
    """block_forward (packed freqs, its one-block cross K|V launches) and self_attention_forward of block 1."""
    eng, sd, cfg = _engine(variant, precision), _sd(variant), CFGS[variant]
    t0 = time.time()
    ck = DF.run_block_seam(monkeypatch, dit, eng, sd, cfg, precision, BLOCK, 1536, f"block_forward {variant}/{precision}",
                           att_plan=_att_plan)
    assert ck.pos == len(ck.program)
    print(f"\n[dataflow] block_forward {variant}/{precision}: wall {time.time() - t0:.1f} s; {ck.report()}")
    monkeypatch.undo()
    t0 = time.time()
    ck = DF.run_self_attention_seam(monkeypatch, dit, eng, sd, cfg, precision, BLOCK, 1536,
                                    f"self_attention_forward {variant}/{precision}", att_plan=_att_plan)
    assert ck.pos == len(ck.program)
    print(f"[dataflow] self_attention_forward {variant}/{precision}: wall {time.time() - t0:.1f} s; {ck.report()}")
