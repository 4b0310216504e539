"""The WanDiT forward launch by launch on the H100 (tests/helpers/dit_dataflow.py): a real-width 2-layer 5B / 14B model runs its
own forward with a checking wrapper around every ops entry. Every launch from the token stream to unpatchify is checked (the
FramePack or grid embedders, the time tables, the text and image context MLPs, the cross K|V GEMMs, block 1 and the head; block 0
passes through): each launch must be the spec's next stage, take exactly the operands the spec names (buffer, view, row count,
scale table, gate row, token index, k_len, RoPE rows, the reference's segment frames and pad multiples) and produce an output
within its kernel's contract bound, in bf16, fp8 and fp8_attn. The stream the first block receives must be the embedders' output
row for row in the reference's token order, with zero padding rows.

Every path runs twice on one engine: an unchecked forward with a longer prompt (and on a padded grid a larger grid at the same
seq_len) fills the reused workspaces first, so the checked forward shows any zeroing that was dropped.

Paths: small geometries of the 5B grid (scalar t, padding rows as keys), 5B FramePack, 14B FramePack and 14B padded grid (k_len <
L); the 5B FramePack ladder at 44x80 (704x1280), latent_frame_zero 8, history 3 / 10 / 40 / 100 / 400 (L = 9 020 / 11 240 /
12 230 / 12 344 / 13 854); the 14B FramePack at 68x120 (544x960), history 5 and 400 (L = 23 970 / 33 860); the production grids
(5B L = 18 480; 14B seq_len 43 008 over 42 840 keys); the 5B grid with a per-frame t over 21 frames; an odd 45x79 latent. bf16 on
every path; fp8 and fp8_attn change only the block and run on one FramePack path of each tree and on the production
grids. Each cell prints its worst |err| / bound per stage and its wall time. On an H100 80GB HBM3 (700 W power limit) the whole
file took 80 s: at most 2.6 s per cell after the first of each engine (up to 14 s, which also builds the engine); the worst
|err| / bound of any stage was 0.996, and the bit-exact entries (patchify, bcast_add, unpatchify) matched.

The checker cannot run inside a CUDA-graph capture, so the graph replay of the forward is compared with the eager forward bit for
bit at production geometry (5B FramePack depth 3, 14B FramePack with the context cache on and off), replayed again with new x, t
and context of the same shapes; that replay must make no launch from Python."""
import ctypes
import time

import pytest
import torch

from helpers import dit_dataflow as DF
from oracle import synth
from yume_b200 import dit, ops

pytestmark = pytest.mark.gpu

LAYERS, BLOCK = 2, 1
CFGS = {"5b": dict(synth.CFG_5B, num_layers=LAYERS), "14b": dict(synth.CFG_14B, num_layers=LAYERS)}
PRECISIONS = ("bf16", "fp8", "fp8_attn")
# (frames, H, W, latent_frame_zero, padding rows past the grid, per-frame t or None): L = 2 048, 2 496, 3 072, 2 048 (1 920 keys)
PATHS = {"5b_grid": (5, 32, 48, None, 128, None), "5b_framepack": (8, 32, 48, 4, 0, None),
         "14b_framepack": (14, 32, 48, 4, 0, None), "14b_grid_padded": (5, 32, 48, None, 128, None)}
# production geometry
PROD = {**{f"5b_framepack_h{h}": (h + 8, 44, 80, 8, 0, None) for h in (3, 10, 40, 100, 400)},
        **{f"14b_framepack_h{h}": (h + 9, 68, 120, 9, 0, None) for h in (5, 400)},
        "5b_grid": (21, 44, 80, None, 0, None), "14b_grid_padded": (21, 68, 120, None, 168, None),
        "5b_grid_t21": (21, 44, 80, None, 0, [float(999 - 47 * i) for i in range(21)]),
        "5b_framepack_odd": (18, 45, 79, 8, 0, None)}
PROD_CASES = [(p, "bf16") for p in PROD] + [(p, q) for p in ("5b_framepack_h40", "14b_framepack_h5", "5b_grid", "14b_grid_padded")
                                             for q in ("fp8", "fp8_attn")]

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
    f, h, w, lfz, pad, t = geom
    cfg = CFGS[v]
    args = DF.path_inputs(cfg, path, f, h, w, lfz, pad, seed=5, t=t)
    warm = DF.warm_inputs(cfg, path, f, h, w, lfz, pad, seed=5, t=t)
    tag = f"{path} F{f} {h}x{w} seq_len {args['seq_len']} / {precision}"
    t0 = time.time()
    ck = DF.run_path(monkeypatch, dit, _engine(v, precision), _sd(v), cfg, precision, args, BLOCK, tag, att_plan=_att_plan,
                     warm=warm)
    torch.cuda.synchronize()
    assert ck.pos == len(ck.program) and tuple(ck.entered) == DF.PHASES
    print(f"\n[dataflow] {tag}: L {ck.geo.layout.L}, {len(ck.program)} stages, wall {time.time() - t0:.1f} s; worst |err|/bound: "
          f"{ck.report()}")
    del ck
    torch.cuda.empty_cache()


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("path", list(PATHS))
def test_block_dataflow(monkeypatch, path, precision):
    _run_path(monkeypatch, path, precision, PATHS[path])


@pytest.mark.parametrize("path,precision", PROD_CASES)
def test_block_dataflow_production_length(monkeypatch, path, precision):
    """The whole forward around block 1 at production geometry."""
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


@pytest.mark.parametrize("path,cache", [("5b_framepack_h40", True), ("14b_framepack_h5", True), ("14b_framepack_h5", False)])
def test_graph_replay_matches_eager_at_production_geometry(path, cache):
    """use_cuda_graph=True against the eager forward, bit for bit: the first call captures, the second replays with new x, t and
    context of the same shapes (a new context is a new cache entry, so with the cache on a third call replays with new x and t
    over the second call's context); the static input buffers must be refreshed on every replay."""
    v = path.split("_")[0]
    f, h, w, lfz, pad, _ = PROD[path]
    cfg = CFGS[v]
    eng = _engine(v, "bf16")
    calls = [DF.path_inputs(cfg, path, f, h, w, lfz, pad, seed=s) for s in (7, 8, 9)]
    for k, a in enumerate(calls):
        a["t"] = a["t"] * (1 - 0.25 * k) + 10.0 * k
    calls[2]["context"] = calls[1]["context"]
    if v == "14b":
        calls[2]["clip_fea"] = calls[1]["clip_fea"]
    saved = (eng.use_cuda_graph, eng.context_cache)
    try:
        eng.use_cuda_graph, eng.context_cache = False, cache
        eager = [DF.engine_forward(eng, a) for a in calls]
        eng.use_cuda_graph = True
        t0 = time.time()
        graphed, launches = [], []
        for a in calls:
            n0 = ops.launch_count()
            graphed.append(DF.engine_forward(eng, a))
            launches.append(ops.launch_count() - n0)
        torch.cuda.synchronize()
        n_graphs = len(eng._graphs)
    finally:
        eng.use_cuda_graph, eng.context_cache = saved
        eng._graphs.clear()
        eng._ctx_entries.clear()
    print(f"\n[graph] {path} context_cache={cache}: {n_graphs} graphs, 3 calls in {time.time() - t0:.1f} s, launches {launches}")
    replay = 2 if cache else 1                  # the call that must be a pure replay (no launch from Python)
    assert launches[0] > 0 and launches[replay] == 0, f"{path} context_cache={cache}: launches per call {launches}"
    assert not torch.equal(eager[0], eager[1]) and not torch.equal(eager[1], eager[2])
    for k, (g, e) in enumerate(zip(graphed, eager)):
        assert torch.equal(g, e), f"{path} context_cache={cache}: call {k}: graph replay differs from eager in " \
                                  f"{int((g != e).sum())} of {g.numel()} elements (max {float((g - e).abs().max()):.3g})"
    torch.cuda.empty_cache()
