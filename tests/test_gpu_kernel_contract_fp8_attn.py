"""Per-element contract of the fp8 self-attention entry points (include/yume_b200_fp8_attn.h) on the H100.

- FP8_ATTN_TABLE lists every launch the precision="fp8_attn" self-attention makes at the 5B (L = 18 480), 14B-chunk (L = 21 930)
  and 14B-grid (L = 42 840) configurations, plus the k_lens row (43 008 queries over 42 840 keys), a ragged row
  (Lq % 256 != 0, Lk % 128 != 0) and forced KV splits 2-4. test_fp8_attn_table_covers_the_engines_launches runs the engine's
  block with recording wrappers and fails on a launch without a row.
- yb_attention_fp8, every row: each sampled output element (4 rows of every 128-row query tile plus one whole unit per head,
  test_gpu_kernel_contract_prod.attention_sample) against fp64 attention over the DEQUANTISED operands, within
  `attention_fp8_bound`. Outputs are NaN-poisoned with guard rows.
- yb_quant_vt_fp8 and the [L, 2C] yb_quant_rows_fp8 launch: bit-identical to their twins (oracle/fp8_attn.py, oracle/fp8.py).

`attention_fp8_bound` is plain torch and is also exercised on the CPU (tests/test_fp8_attn_cpu.py) against a tile-by-tile model
of the kernel and realistic defects."""
import ctypes as C
import math

import pytest
import torch

from oracle.fp8 import dequantize_act, quantize_act
from oracle.fp8_attn import dequantize_vt, quantize_vt

U16, U32 = 2.0 ** -8, 2.0 ** -24
ACC_BITS = 13          # mantissa bits the e4m3 tensor-core accumulator keeps (tests/test_gpu_kernel_contract_fp8.py)
P_REL = 2.0 ** -4      # largest relative rounding error of a normal e4m3 value
P_SUB = 2.0 ** -18     # largest absolute rounding error of a subnormal P8 = e4m3(256 p), in units of p
Z_P = 6.0              # standard deviations allowed for the sum of the independent P roundings


def attention_fp8_bound(q, k, v, scale, nkv, ns=1):
    """(ref, bound) in fp64 for q [R, 128] sampled rows, k / v [Lk, 128] of one head, all dequantised (fp64).
    ref = softmax(q k^T scale) v. With p the exact probabilities and l = sum_j exp(s_j - max s):
      logits      e = 4 2^-ACC_BITS scale (|q| |k|^T)  (four truncating k32 steps of the S wgmma) + 4 u32 |s|  (k scale, row
                  factor, exp2 argument); a logit error e moves the output by at most 2 e (p |v|)
      P8          round-to-nearest e4m3 of 256 p against the running max: relative error <= 2^-4 per key, zero-mean and
                  independent between distinct keys, so their sum is bounded by Z_P standard deviations,
                  Z_P 2^-4 / sqrt(3) sqrt(sum_g (p_g |v_g|)^2); keys with identical (k, v) rows round alike (the zero padding
                  rows of a padded 5B grid are keys, and after a block they are all the same row), so each group g of them
                  counts as one key holding their summed p_g; subnormal P8 (and P8 flushed to 0) add at most 2^-18 per key:
                  2^-18 sum_j |v_j| / l
      O_tile      four truncating k32 steps per tile: 4 2^-ACC_BITS (1 + 2^-4) (p |v|)
      fp32        promotion, alpha, l and the combine as attention_bound_prod counts them: (26 nkv + 36 + 3 ns) u32 (p |v|)
      output      bf16 rounding U16 |ref|"""
    s = (q @ k.t()) * scale
    p = torch.softmax(s, dim=-1)
    ref = p @ v
    pv = p @ v.abs()
    e = (4 * 2.0 ** -ACC_BITS * scale * (q.abs() @ k.abs().t()) + 4 * U32 * s.abs()).amax(dim=-1, keepdim=True)
    l = torch.exp(s - s.amax(dim=-1, keepdim=True)).sum(dim=-1, keepdim=True)
    rows, group = torch.unique(torch.cat([k, v], dim=1), dim=0, return_inverse=True)
    pg = torch.zeros(p.shape[0], rows.shape[0], dtype=p.dtype, device=p.device).index_add_(1, group, p)
    vg = rows[:, k.shape[1]:]
    stat = Z_P * P_REL / math.sqrt(3.0) * torch.sqrt((pg * pg) @ (vg * vg))
    sub = P_SUB * v.abs().sum(dim=0, keepdim=True) / l
    extra = (26 * nkv + 36 + (3 * ns if ns > 1 else 0)) * U32 + 4 * 2.0 ** -ACC_BITS * (1 + P_REL)
    return ref, U16 * ref.abs() + (2 * e + extra) * pv + stat + sub


# ------------------------------------------------------------------------------------------------------------
# everything below needs the GPU
# ------------------------------------------------------------------------------------------------------------
gpu = pytest.mark.gpu
E4M3 = torch.float8_e4m3fn

COVERS = {
    "yb_attention_fp8": ["test_attention_fp8_per_element", "test_attention_fp8_rejects_bad_arguments",
                         "test_fp8_attn_table_covers_the_engines_launches"],
    "yb_quant_vt_fp8": ["test_quant_vt_fp8_bit_identical_to_twin"],
}

from test_gpu_kernel_contract_prod import DIT_CFGS  # noqa: E402


def _rows():
    rows = []
    for cfg, d in DIT_CFGS.items():
        L, H = d["L"], d["heads"]
        rows.append(dict(id=f"{cfg}.quant_qk", entry="quant_rows_fp8", cfg=cfg, M=L, K=2 * H * 128))
        rows.append(dict(id=f"{cfg}.quant_vt", entry="quant_vt_fp8", cfg=cfg, Lk=d["Lk"], heads=H))
        rows.append(dict(id=f"{cfg}.self_attention", entry="attention_fp8", cfg=cfg, Lq=L, Lk=d["Lk"], heads=H, split=0))
    # the k_lens form (seq_len > L_grid: padded rows are queries but not keys), with its partial last KV tile
    rows.append(dict(id="14b_grid_seq_len_43008.self_attention", entry="attention_fp8", cfg="k_lens", Lq=43008, Lk=42840,
                     heads=40, split=0))
    rows.append(dict(id="14b_grid_seq_len_43008.quant_vt", entry="quant_vt_fp8", cfg="k_lens", Lk=42840, heads=40))
    # ragged: a partial last query unit and a partial last KV tile
    rows.append(dict(id="ragged.self_attention", entry="attention_fp8", cfg="ragged", Lq=300, Lk=200, heads=2, split=0))
    rows.append(dict(id="ragged.quant_vt", entry="quant_vt_fp8", cfg="ragged", Lk=200, heads=2))
    # forced KV splits: every unit cut into 2..4 segments, the combine on every row
    for ns in (2, 3, 4):
        rows.append(dict(id=f"split{ns}.self_attention", entry="attention_fp8", cfg=f"split{ns}", Lq=1000, Lk=2000, heads=3,
                         split=ns))
    return rows


FP8_ATTN_TABLE = _rows()


def _ids(entry):
    return [r["id"] for r in FP8_ATTN_TABLE if r["entry"] == entry]


def _row(rid):
    return next(r for r in FP8_ATTN_TABLE if r["id"] == rid)


def _lib():
    import yume_b200
    from yume_b200 import _lib as L
    yume_b200.load()
    return L.load()


def _operands(Lq, Lk, H, key):
    """One fused bf16 q|k|v buffer [max(Lq, Lk), 3 H 128] (q doubled so that the softmax is not flat) and its fp8 operands as
    the engine makes them: q|k quantised by one yb_quant_rows_fp8 over the [L, 2C] view, v by yb_quant_vt_fp8."""
    from test_gpu_kernel_contract_prod import _cuda_gen, _rand
    from yume_b200 import ops
    W = H * 128
    L = max(Lq, Lk)
    g = _cuda_gen(("fp8_attn",) + tuple(key))
    buf = _rand(g, L, 3 * W)
    buf[:, :W].mul_(2.0)
    qk8 = torch.empty(L, 2 * W, dtype=E4M3, device="cuda")
    qk_s = torch.empty(2 * H, ops.fp8_scale_ld(L), device="cuda")
    Lkp = ops.vt8_keys(Lk)
    vt8 = torch.empty(H, 128, Lkp, dtype=E4M3, device="cuda")
    v_s = torch.empty(H, Lkp // 128, device="cuda")
    ops.quant_rows_fp8(buf[:, :2 * W], qk8, qk_s)
    ops.quant_vt_fp8(buf[:Lk, 2 * W:], vt8, v_s, H)
    return buf, qk8, qk_s, vt8, v_s


@gpu
@pytest.mark.parametrize("rid", _ids("attention_fp8"))
def test_attention_fp8_per_element(rid):
    import test_gpu_kernel_contract as KC
    from test_gpu_kernel_contract_prod import Lean, attention_sample
    from yume_b200 import ops
    lib = _lib()
    row = _row(rid)
    Lq, Lk, H, split = row["Lq"], row["Lk"], row["heads"], row["split"]
    W = H * 128
    buf, qk8, qk_s, vt8, v_s = _operands(Lq, Lk, H, (rid,))
    del buf
    plan = (C.c_int * 4)()
    assert lib.yb_attention_plan(Lq, Lk, H, torch.cuda.get_device_properties(0).multi_processor_count, (split & 7) << 4, plan) == 0
    nkv, ns = -(-Lk // 128), plan[2]
    if split:
        assert ns == split and plan[1] > 0, f"split {split} was not planned: {tuple(plan)}"
    out = Lean(Lq, W, torch.bfloat16)
    scale = 1 / math.sqrt(128.0)
    ops.attention_fp8(qk8[:Lq, :W], qk8[:Lk, W:], qk_s, vt8, v_s, out.view, H, scale=scale, split=split)
    torch.cuda.synchronize()
    tag = f"attention_fp8 {rid} Lq{Lq} Lk{Lk} h{H} tail{plan[1]} ns{ns}"
    out.check(tag)
    qd = dequantize_act(qk8[:Lq, :W], qk_s[:H])
    kd = dequantize_act(qk8[:Lk, W:], qk_s[H:])
    vd = dequantize_vt(vt8, v_s, Lk)
    samples = attention_sample(Lq, H, ("fp8_attn", rid))
    worst = 0.0
    for h in range(H):
        sl = slice(h * 128, (h + 1) * 128)
        kh, vh = kd[:, sl].double(), vd[:, sl].double()
        r = samples[h].to("cuda")
        for c0 in range(0, len(r), 1024):
            rc = r[c0:c0 + 1024]
            ref, bound = attention_fp8_bound(qd[rc, sl].double(), kh, vh, scale, nkv, ns)
            ratio = float(((out.view[rc, sl].double() - ref).abs() / bound).max())
            worst = max(worst, ratio)
    KC.WORST[f"fp8_attn.{rid}"] = max(KC.WORST.get(f"fp8_attn.{rid}", 0.0), worst)
    print(f"[contract] {tag}: worst |err|/bound {worst:.3f}")
    assert worst <= 1.0, f"{tag}: worst |err|/bound {worst:.3f}"


def _special_v(Lk, W, g):
    v = torch.randn(Lk, W, device="cuda", generator=g) * torch.exp(torch.randn(1, W, device="cuda", generator=g))
    v[:128, :128] = 0.0                                 # zero block (head 0, tile 0)
    if Lk > 128:
        v[128:256, :128] = 1e-38                        # 448 / amax overflows: stored as zeros with scale 0
    v[5, 130] = float("nan")                            # NaN passes through, the block's other values are quantised
    return v.to(torch.bfloat16)


@gpu
@pytest.mark.parametrize("rid", _ids("quant_vt_fp8") + ["special"])
def test_quant_vt_fp8_bit_identical_to_twin(rid):
    from yume_b200 import ops
    Lk, H = (300, 3) if rid == "special" else (_row(rid)["Lk"], _row(rid)["heads"])
    W = H * 128
    g = torch.Generator(device="cuda").manual_seed(Lk + H)
    if rid == "special":
        v = _special_v(Lk, W, g)
    else:
        full = torch.randn(Lk, 3 * W, device="cuda", generator=g).to(torch.bfloat16)   # the engine's v: a [Lk, C] window
        v = full[:, 2 * W:]
    Lkp = ops.vt8_keys(Lk)
    vt8 = torch.full((H, 128, Lkp), float("nan"), device="cuda").to(E4M3)
    v_s = torch.full((H, Lkp // 128), float("nan"), device="cuda")
    ops.quant_vt_fp8(v, vt8, v_s, H)
    torch.cuda.synchronize()
    tq, ts = quantize_vt(v.float(), H)
    nan = torch.isnan(tq.float())
    assert torch.equal(torch.isnan(vt8.float()), nan)
    qb, tb = vt8.view(torch.uint8), tq.view(torch.uint8)
    assert torch.equal(qb[~nan], tb[~nan]), f"{int((qb != tb).sum())} bytes differ from the twin"
    assert torch.equal(v_s, ts)
    if rid == "special":
        assert float(v_s[0, 0]) == 0.0 and float(v_s[0, 1]) == 0.0 and bool((vt8[0, :, :256].float() == 0).all())
        assert bool((vt8.float()[:, :, -(-Lk // 32) * 32:] == 0).all()), "keys >= Lk must be stored as zeros"


@gpu
@pytest.mark.parametrize("rid", _ids("quant_rows_fp8"))
def test_quant_qk_view_bit_identical_to_twin(rid):
    """The [L, 2C] yb_quant_rows_fp8 launch over the fused q|k|v rows (row stride 3C): bit-identical to the 1x128 twin."""
    from yume_b200 import ops
    r = _row(rid)
    M, K = r["M"], r["K"]
    g = torch.Generator(device="cuda").manual_seed(M)
    buf = (torch.randn(M, K // 2 * 3, device="cuda", generator=g) * 3).to(torch.bfloat16)
    x = buf[:, :K]
    q = torch.empty(M, K, dtype=E4M3, device="cuda")
    s = torch.full((K // 128, ops.fp8_scale_ld(M)), float("nan"), device="cuda")
    ops.quant_rows_fp8(x, q, s)
    torch.cuda.synchronize()
    tq, ts = quantize_act(x.float())
    assert torch.equal(q.view(torch.uint8), tq.view(torch.uint8))
    assert torch.equal(s[:, :M], ts)


@gpu
def test_attention_fp8_rejects_bad_arguments():
    lib = _lib()
    H, Lq, Lk = 2, 256, 256
    W = H * 128
    q8 = torch.zeros(Lq, W, dtype=E4M3, device="cuda")
    sc = torch.zeros(2 * H, Lq, device="cuda")
    vt8 = torch.zeros(H, 128, 256, dtype=E4M3, device="cuda")
    vs = torch.zeros(H, 2, device="cuda")
    out = torch.zeros(Lq, W, dtype=torch.bfloat16, device="cuda")
    s = torch.cuda.current_stream().cuda_stream

    def call(**kw):
        a = dict(q8=q8.data_ptr(), ldq=W, k8=q8.data_ptr(), ldk=W, sc=sc.data_ptr(), lds=Lq, vt=vt8.data_ptr(), vs=vs.data_ptr(),
                 out=out.data_ptr(), ldo=W, Lq=Lq, Lk=Lk, H=H, scale=0.088, flags=0)
        a.update(kw)
        return lib.yb_attention_fp8(a["q8"], a["ldq"], a["k8"], a["ldk"], a["sc"], a["lds"], a["vt"], a["vs"], a["out"], a["ldo"],
                                    a["Lq"], a["Lk"], a["H"], a["scale"], a["flags"], None, 0, s)
    assert call() == 0
    assert call(q8=None) == -1
    assert call(lds=Lq - 4) == -1                       # scale table shorter than the queries
    assert call(flags=2) == -1                          # YB_ATT_ACCUMULATE has no fp8 form
    assert call(flags=1) == -1                          # nor the P-in-shared-memory variant
    assert call(flags=5 << 4) == -1                     # split policy out of range
    assert call(ldq=W + 8) == -3                        # e4m3 row stride not a multiple of 16 bytes
    assert call(ldo=W + 4) == -3
    assert call(Lk=0) == -1
    assert lib.yb_quant_vt_fp8(None, W, vt8.data_ptr(), vs.data_ptr(), Lk, H, s) == -1
    v = torch.zeros(Lk, W + 4, dtype=torch.bfloat16, device="cuda")
    assert lib.yb_quant_vt_fp8(v.data_ptr(), W + 4, vt8.data_ptr(), vs.data_ptr(), Lk, H, s) == -3
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------
# the table against the engine's launches
# ------------------------------------------------------------------------------------------------------------
def _record(monkeypatch):
    from yume_b200 import ops
    calls = []
    real = dict(quant_rows_fp8=ops.quant_rows_fp8, quant_vt_fp8=ops.quant_vt_fp8, attention_fp8=ops.attention_fp8,
                attention=ops.attention)

    def quant_rows_fp8(x, out, out_scale):
        calls.append(dict(entry="quant_rows_fp8", M=x.shape[0], K=x.shape[1]))
        return real["quant_rows_fp8"](x, out, out_scale)

    def quant_vt_fp8(v, vt8, v_scale, heads):
        calls.append(dict(entry="quant_vt_fp8", Lk=v.shape[0], heads=heads))
        return real["quant_vt_fp8"](v, vt8, v_scale, heads)

    def attention_fp8(q8, k8, qk_scale, vt8, v_scale, out, heads, scale=None, split=0):
        calls.append(dict(entry="attention_fp8", Lq=q8.shape[0], Lk=k8.shape[0], heads=heads, split=split))
        return real["attention_fp8"](q8, k8, qk_scale, vt8, v_scale, out, heads, scale=scale, split=split)

    def attention(q, k, v, out, heads, **kw):
        calls.append(dict(entry="attention", Lq=q.shape[0], Lk=k.shape[0], heads=heads))
        return real["attention"](q, k, v, out, heads, **kw)
    for name, fn in (("quant_rows_fp8", quant_rows_fp8), ("quant_vt_fp8", quant_vt_fp8), ("attention_fp8", attention_fp8),
                     ("attention", attention)):
        monkeypatch.setattr(ops, name, fn)
    return calls


@gpu
@pytest.mark.parametrize("cfg_name", list(DIT_CFGS))
def test_fp8_attn_table_covers_the_engines_launches(monkeypatch, cfg_name):
    """A real-width, one-layer WanDiT(precision="fp8_attn") block at the production L: every launch of its self-attention must
    have a row, and no bf16 self-attention may remain (cross-attention stays bf16: Lk = 512 / 257)."""
    import test_gpu_kernel_contract_prod as P
    from oracle import synth
    from yume_b200.dit import WanDiT
    _lib()
    d = DIT_CFGS[cfg_name]
    cfg = synth.CFG_5B if cfg_name == "5b" else synth.CFG_14B
    sd = synth.make_state_dict(cfg, 1234, num_layers=1)
    kw = synth.oracle_kwargs(cfg)
    variant = kw.pop("variant")
    kw["num_layers"] = 1
    eng = WanDiT(sd, variant, device="cuda", precision="fp8_attn", **kw)
    del sd
    L, C = P.production_L(cfg_name), d["C"]
    g = torch.Generator(device="cuda").manual_seed(L)
    xs = torch.randn(L, C, generator=g, device="cuda")
    ctx = torch.randn((257 if d["img"] else 0) + 512, C, generator=g, device="cuda").to(torch.bfloat16)
    t_unique = torch.tensor([0.0, 900.0] if cfg_name == "5b" else [500.0], device="cuda")
    _, mod, _ = eng._time_tables(t_unique)
    tok_idx = (torch.arange(L, device="cuda") >= L // 3).to(torch.int32) if cfg_name == "5b" else None
    rope = eng._rope_table([(1, 1, L, 0)])
    kv = eng._cross_kv(ctx)
    calls = _record(monkeypatch)
    eng._block(0, xs, mod, tok_idx, rope, L, kv, L)
    torch.cuda.synchronize()
    monkeypatch.undo()
    att = [c for c in calls if c["entry"] == "attention_fp8"]
    assert len(att) == 1, f"expected one fp8 self-attention launch, got {att}"
    assert all(c["Lk"] in (512, 257) for c in calls if c["entry"] == "attention"), "a bf16 self-attention remains"
    rows = [r for r in FP8_ATTN_TABLE if r["cfg"] == cfg_name]
    bad = []
    for c in calls:
        if c["entry"] == "attention":
            continue
        if c["entry"] == "quant_rows_fp8" and c["K"] == C:       # the attention output in front of o / cross o (fp8 table)
            continue
        keys = [k for k in c if k != "entry"]
        if not any(r["entry"] == c["entry"] and all(r.get(k) == c[k] for k in keys) for r in rows):
            bad.append(c)
    assert not bad, f"{cfg_name}: {len(bad)} launch(es) without a table row: {bad}"
    assert torch.isfinite(xs).all()
