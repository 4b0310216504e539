"""Per-element contract of the fp8 entry points (include/yume_b200_fp8.h) on the H100.

- FP8_TABLE lists every launch of the fp8 engine's block at the 5B (L = 18 480), 14B-chunk (L = 21 930) and 14B-grid
  (L = 42 840) configurations; test_fp8_table_covers_the_engines_launches runs the engine with recording wrappers and fails on a
  launch without a row.
- yb_gemm_fp8, every row: each output element against an fp64 product of the DEQUANTISED operands, within `gemm_bound`.
  Outputs are NaN-poisoned with a guard band of rows and columns that must stay NaN.
- yb_quant_rows_fp8 and yb_ln_modulate_fp8, every row: bit-identical to the torch twin (oracle/fp8.py) of the fp32 values they
  quantise.
- The accumulator probe measures how many mantissa bits the e4m3 wgmma keeps when it adds a small product to a large one; the
  bound below is derived from it (DESIGN.md §3).

`gemm_bound` is plain torch and is also exercised on the CPU (tests/test_fp8_cpu.py) against realistic defects."""
import ctypes as C

import pytest
import torch

from oracle.fp8 import dequantize_act, quantize_act, quantize_weight

# mantissa bits the fp8 tensor-core accumulator keeps (measured by test_fp8_accumulator_probe: a product 2^-p added to 1.0
# survives for every p <= ACC_BITS)
ACC_BITS = 13
# additions inside one 128-wide k-group that can each lose up to 2^-ACC_BITS of the running magnitude: 4 wgmma k-steps of 32,
# with at most one truncation per step on each side of the internal sum
ROUNDS_PER_GROUP = 4


def gemm_bound(a_abs: torch.Tensor, w_abs: torch.Tensor, K: int, out_ulp: float, ref: torch.Tensor) -> torch.Tensor:
    """Per-element error bound of one fp8 GEMM. a_abs [M, K], w_abs [N, K]: |dequantised operands| (fp64). The tensor-core
    accumulator loses at most 2^-ACC_BITS of |partial| per rounding, ROUNDS_PER_GROUP per group, bounded by the group's sum of
    |products|; promotion and the epilogue add fp32 roundings; the output type adds out_ulp * |ref|."""
    s = a_abs @ w_abs.t()
    groups = K // 128
    return (ROUNDS_PER_GROUP * 2.0 ** -ACC_BITS + (groups + 4) * 2.0 ** -23) * s + out_ulp * ref.abs() + 1e-30


def gelu_fp8_bound(ref, bound, sc):
    """(gelu_tanh(ref), bound) of the GELU_FP8 epilogue, from the pre-activation ref and its gemm_bound: |gelu'| <= 1.13 carries the
    accumulation error through, the e4m3 store adds 2^-4 relative and half a subnormal step of the group scale sc (per element),
    tanh.approx.f32 (relative error < 2^-10.99) 1e-3 |ref| up to |ref| = 10."""
    gref = _gelu_tanh64(ref)
    return gref, 1.13 * bound + 2.0 ** -4 * gref.abs() + sc * 2.0 ** -9 + 1e-3 * ref.abs().clamp(max=10.0)


def _worst(err, bound):
    return float((err / bound).max())


# ------------------------------------------------------------------------------------------------------------
# everything below needs the GPU
# ------------------------------------------------------------------------------------------------------------
gpu = pytest.mark.gpu
E4M3 = torch.float8_e4m3fn

COVERS = {
    "yb_gemm_fp8": ["test_gemm_fp8_per_element_at_production_shapes", "test_gemm_fp8_rejects_bad_arguments",
                    "test_fp8_accumulator_probe", "test_fp8_table_covers_the_engines_launches"],
    "yb_ln_modulate_fp8": ["test_ln_modulate_fp8_bit_identical_to_twin"],
    "yb_quant_rows_fp8": ["test_quant_rows_fp8_bit_identical_to_twin"],
}

# ------------------------------------------------------------------------------------------------------------
# the fp8 engine's launch table: every launch WanDiT(precision="fp8") makes in a block, per production configuration of
# test_gpu_kernel_contract_prod.DIT_CFGS (5B L = 18 480, 14B chunk L = 21 930, 14B 81-frame grid L = 42 840), plus a ragged M
# (not an engine shape: a partial last row tile). test_fp8_table_covers_the_engines_launches ties the rows to the engine.
# ------------------------------------------------------------------------------------------------------------
from test_gpu_kernel_contract_prod import DIT_CFGS  # noqa: E402

EPI = dict(BF16=0, F32=2, GATE_RES=3, GELU_FP8=8)


def _fp8_rows():
    rows = []
    cfgs = {k: dict(C=d["C"], F=d["F"], L=d["L"], gated=frozenset(d["gated"])) for k, d in DIT_CFGS.items()}
    cfgs["ragged"] = dict(C=256, F=512, L=300, gated=frozenset(("gate", "tok_idx")))
    for cfg, d in cfgs.items():
        C, L, Fd, g = d["C"], d["L"], d["F"], d["gated"]

        def gemm(name, N, K, epi, flags=frozenset()):
            rows.append(dict(id=f"{cfg}.{name}", entry="gemm_fp8", cfg=cfg, M=L, N=N, K=K, epi=EPI[epi], flags=frozenset(flags)))
        gemm("qkv", 3 * C, C, "BF16")
        gemm("o", C, C, "GATE_RES", g)
        gemm("cross_q", C, C, "BF16", {"out_window"})             # q2 = qkv[:, :C]: ldo = 3C
        gemm("cross_o", C, C, "GATE_RES")
        gemm("ffn0", Fd, C, "GELU_FP8")
        gemm("ffn2", C, Fd, "GATE_RES", g)
        rows.append(dict(id=f"{cfg}.ln_adaln", entry="ln_modulate_fp8", cfg=cfg, L=L, C=C, form="adaln",
                         tok_idx="tok_idx" in g))
        rows.append(dict(id=f"{cfg}.ln_affine", entry="ln_modulate_fp8", cfg=cfg, L=L, C=C, form="affine", tok_idx=False))
        rows.append(dict(id=f"{cfg}.quant_att", entry="quant_rows_fp8", cfg=cfg, M=L, K=C))
    rows.append(dict(id="ragged.f32", entry="gemm_fp8", cfg="ragged", M=300, N=256, K=256, epi=EPI["F32"], flags=frozenset()))
    return rows


FP8_TABLE = _fp8_rows()


def _ids(entry):
    return [r["id"] for r in FP8_TABLE if r["entry"] == entry]


def _row(rid):
    return next(r for r in FP8_TABLE if r["id"] == rid)


def _lib():
    import yume_b200
    from yume_b200 import _lib as L
    yume_b200.load()
    return L


def _gelu_tanh64(x):
    return 0.5 * x * (1.0 + torch.tanh(0.7978845608028654 * (x + 0.044715 * x ** 3)))


@gpu
def test_fp8_accumulator_probe():
    """A = [1, 2^-f, 0...], W = [1, 2^-e, 0...] (scales 1, one k-group): out = 1 + 2^-(e+f) exactly while the accumulator keeps
    e + f bits. Reports the largest p that survives for every (e, f) with e + f = p and asserts it is at least ACC_BITS."""
    from yume_b200 import ops
    dev = "cuda"
    M = N = 128
    K = 128
    f = torch.arange(M) % 10            # 2^-9 is the smallest e4m3 subnormal
    e = torch.arange(N) % 10
    A = torch.zeros(M, K)
    W = torch.zeros(N, K)
    A[:, 0], W[:, 0] = 1.0, 1.0
    A[:, 1], W[:, 1] = 2.0 ** -f.float(), 2.0 ** -e.float()
    aq = A.to(E4M3).to(dev)
    wq = W.to(E4M3).to(dev)
    assert torch.equal(aq.float().cpu(), A) and torch.equal(wq.float().cpu(), W)
    sa = torch.ones(1, M, device=dev)
    sw = torch.ones(N, device=dev)
    out = torch.empty(M, N, device=dev)
    ops.gemm_fp8(aq, sa, wq, sw, None, out, ops.YB_EPI_F32)
    torch.cuda.synchronize()
    p = (f[:, None] + e[None, :])
    exact = out.cpu().double() == (1.0 + 2.0 ** -p.double())
    kept = [q for q in range(0, 19) if bool(exact[p == q].all())]
    best = max(q for q in range(0, 19) if all(r in kept for r in range(0, q + 1)))
    print(f"fp8 wgmma accumulator: 1 + 2^-p exact for every p <= {best}")
    assert best >= ACC_BITS


@gpu
@pytest.mark.parametrize("rid", _ids("gemm_fp8"))
def test_gemm_fp8_per_element_at_production_shapes(rid):
    """Every element against an fp64 product of the dequantised operands (row chunks of 4096), inside a NaN-poisoned buffer
    whose guard rows / columns must stay NaN; GELU_FP8 also: every 1x128 group of the output reaches exactly +-448."""
    from yume_b200 import ops
    r = _row(rid)
    M, N, K, epi, flags = r["M"], r["N"], r["K"], r["epi"], r["flags"]
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(M + N + K + epi)
    x = torch.randn(M, K, device=dev, generator=g) * (1.0 + 3.0 * torch.rand(M, 1, device=dev, generator=g))
    if rid.endswith("ffn2"):
        x = _gelu_tanh64(x.double()).float()          # what ffn.2 reads: mostly positive
    aq, sa = quantize_act(x)
    del x
    lds = (M + 3) // 4 * 4 + 4
    sa_buf = torch.full((K // 128, lds), float("nan"), device=dev)
    sa_buf[:, :M] = sa
    w = torch.randn(N, K, device=dev, generator=g) * 0.02
    wq, sw = quantize_weight(w)
    del w
    bias = torch.randn(N, device=dev, generator=g)
    pad_r = 8
    ldo = 3 * N if "out_window" in flags else N + 32
    gate = tok = osc = None
    if epi == EPI["GELU_FP8"]:
        buf = torch.full((M + pad_r, ldo), 0x7F, dtype=torch.uint8, device=dev)      # 0x7F: e4m3 NaN
        osc = torch.full((N // 128, lds + 8), float("nan"), device=dev)
        out = buf.view(E4M3)[:M, :N]
    else:
        buf = torch.full((M + pad_r, ldo), float("nan"), dtype=torch.bfloat16 if epi == EPI["BF16"] else torch.float32, device=dev)
        out = buf[:M, :N]
        if epi == EPI["GATE_RES"]:
            out.copy_(torch.randn(M, N, device=dev, generator=g))
            if "gate" in flags:
                gate = torch.randn(2 if "tok_idx" in flags else 1, N, device=dev, generator=g)
            if "tok_idx" in flags:
                tok = torch.randint(0, 2, (M,), device=dev, generator=g, dtype=torch.int32)
    x0 = out.clone() if epi == EPI["GATE_RES"] else None
    ops.gemm_fp8(aq, sa_buf, wq, sw, bias, out, epi, gate=gate, tok_idx=tok, out_scale=osc)
    torch.cuda.synchronize()
    full = buf.view(E4M3).float() if epi == EPI["GELU_FP8"] else buf.float()
    assert torch.isnan(full[M:]).all() and torch.isnan(full[:, N:]).all(), "write outside [M, N]"
    del full
    if osc is not None:
        assert torch.isnan(osc[:, M:]).all()
    wd = wq.double() * sw.double()[:, None]
    wabs = wd.abs()
    out_ulp = {EPI["BF16"]: 2.0 ** -8, EPI["F32"]: 2.0 ** -24, EPI["GATE_RES"]: 2.0 ** -24, EPI["GELU_FP8"]: 0.0}[epi]
    worst = 0.0
    for r0 in range(0, M, 4096):
        r1 = min(M, r0 + 4096)
        ad = dequantize_act(aq[r0:r1], sa[:, r0:r1]).double()
        ref = ad @ wd.t() + bias.double()
        bound = gemm_bound(ad.abs(), wabs, K, out_ulp, ref)
        del ad
        if epi == EPI["GELU_FP8"]:
            sc = osc[:, r0:r1]
            deq = dequantize_act(out[r0:r1], sc).double()
            gref, bound = gelu_fp8_bound(ref, bound, sc.t().repeat_interleave(128, dim=1).double())
            worst = max(worst, _worst((deq - gref).abs(), bound))
            gmax = out[r0:r1].float().abs().view(r1 - r0, N // 128, 128).amax(dim=-1)
            assert bool((gmax == 448.0).all()), "every group reaches exactly +-448"
            continue
        if epi == EPI["GATE_RES"]:
            gt = torch.ones(r1 - r0, N, dtype=torch.float64, device=dev)
            if gate is not None:
                gt = gate.double()[tok[r0:r1].long()] if tok is not None else gate.double()[:1].expand(r1 - r0, N)
            ref = x0[r0:r1].double() + ref * gt
            bound = bound * gt.abs() + 2.0 ** -24 * ref.abs()
        got = out[r0:r1].double()
        assert torch.isfinite(got).all()
        worst = max(worst, _worst((got - ref).abs(), bound))
    print(f"{rid} epi={epi} M={M} N={N} K={K}: worst |err|/bound = {worst:.3f}")
    assert worst <= 1.0


@gpu
def test_gemm_fp8_rejects_bad_arguments():
    L = _lib()
    from yume_b200 import ops
    dev = "cuda"
    M, N, K = 64, 128, 256
    aq = torch.zeros(M, K, device=dev).to(E4M3)
    sa = torch.zeros(K // 128, 64, device=dev)
    wq = torch.zeros(N, K, device=dev).to(E4M3)
    sw = torch.zeros(N, device=dev)
    out = torch.zeros(M, N, device=dev)
    lib = L.load()

    def call(**kw):
        base = dict(struct_bytes=C.sizeof(L.GemmFp8Args), M=M, N=N, K=K, A=aq.data_ptr(), a_scale=sa.data_ptr(), B=wq.data_ptr(),
                    b_scale=sw.data_ptr(), bias=None, out=out.data_ptr(), out_scale=None, gate=None, tok_idx=None, lda=K, lds=64,
                    ldb=K, ldo=N, ldos=0, gate_ld=0, epilogue=2, block_n=0)
        base.update(kw)
        return lib.yb_gemm_fp8(C.byref(L.GemmFp8Args(**base)), ops._stream())

    assert call() == 0
    assert call(struct_bytes=8) == -1
    assert call(K=200, lda=200, ldb=200) == -2          # K % 128
    assert call(N=96) == -2                             # N % 128
    assert call(epilogue=1) == -1                       # GELU_BF16 is not an fp8 epilogue
    assert call(epilogue=8) == -1                       # GELU_FP8 without out_scale
    assert call(lds=60) == -1                           # lds < M
    assert call(lda=K + 8) == -3                        # operand row pitch not 16-byte aligned
    assert call(block_n=256) == -1
    assert call(A=None) == -1
    torch.cuda.synchronize()


def _special_rows(M, K, dev, g):
    x = torch.randn(M, K, device=dev, generator=g) * torch.exp(2 * torch.randn(M, 1, device=dev, generator=g))
    x[0, :128] = 0.0                                   # zero group
    x[1, 128:256] = 1e-38                              # 448 / amax overflows: stored as zeros with scale 0
    x[2, 5] = float("nan")                             # NaN passes through, the group's other values are quantised
    x[3, :128] = 448.0 * 2.0 ** -7                     # exactly representable
    return x


@gpu
@pytest.mark.parametrize("rid", _ids("quant_rows_fp8") + ["odd_rows"])
def test_quant_rows_fp8_bit_identical_to_twin(rid):
    from yume_b200 import ops
    M, K = (37, 256) if rid == "odd_rows" else (_row(rid)["M"], _row(rid)["K"])
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(M)
    x = _special_rows(M, K, dev, g).to(torch.bfloat16)
    lds = (M + 3) // 4 * 4
    q = torch.empty(M, K, dtype=E4M3, device=dev)
    s = torch.full((K // 128, lds), float("nan"), device=dev)
    ops.quant_rows_fp8(x, q, s)
    torch.cuda.synchronize()
    tq, ts = quantize_act(x.float())
    _assert_twin(q, s[:, :M], tq, ts)


def _assert_twin(q, s, tq, ts):
    qb, tb = q.view(torch.uint8), tq.view(torch.uint8)
    nan = torch.isnan(tq.float())
    assert torch.equal(torch.isnan(q.float()), nan)
    assert torch.equal(qb[~nan], tb[~nan]), f"{int((qb != tb).sum())} bytes differ from the twin"
    assert torch.equal(s, ts)


@gpu
@pytest.mark.parametrize("rid", _ids("ln_modulate_fp8") + ["width1024.adaln", "width1024.affine"])
def test_ln_modulate_fp8_bit_identical_to_twin(rid):
    """The table's rows, plus the C = 1024 instance that only the 8-head test models run (the ragged rows cover C = 256)."""
    from yume_b200 import ops
    if rid.startswith("width"):
        C, form, L, use_tok = int(rid[5:].split(".")[0]), rid.split(".")[1], 300, True
    else:
        r = _row(rid)
        C, form, L, use_tok = r["C"], r["form"], r["L"], r["tok_idx"]
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(C + L)
    x = torch.randn(L, C, device=dev, generator=g) * 3 + 0.5
    tok = torch.randint(0, 2, (L,), device=dev, generator=g, dtype=torch.int32) if use_tok else None
    mod = torch.randn(2 if use_tok else 1, 6, C, device=dev, generator=g) * 0.3
    w, b = torch.randn(C, device=dev, generator=g), torch.randn(C, device=dev, generator=g)
    ref = torch.empty(L, C, device=dev)
    q = torch.empty(L, C, dtype=E4M3, device=dev)
    lds = (L + 3) // 4 * 4
    s = torch.full((C // 128, lds), float("nan"), device=dev)
    if form == "adaln":
        ops.ln_modulate(x, ref, mod[:, 1], mod[:, 0], tok)
        ops.ln_modulate_fp8(x, q, s, mod[:, 1], mod[:, 0], tok)
    else:
        ops.ln_modulate(x, ref, None, None, None, w, b)
        ops.ln_modulate_fp8(x, q, s, None, None, None, w, b)
    torch.cuda.synchronize()
    tq, ts = quantize_act(ref)
    _assert_twin(q, s[:, :L], tq, ts)


# ------------------------------------------------------------------------------------------------------------
# the table against the fp8 engine's launches
# ------------------------------------------------------------------------------------------------------------
def _record_fp8(monkeypatch):
    """Recording wrappers around every ops entry the fp8 engine's block can reach (they record, then call through)."""
    from yume_b200 import ops
    calls = []
    real = dict(gemm=ops.gemm, gemm_fp8=ops.gemm_fp8, ln_modulate=ops.ln_modulate, ln_modulate_fp8=ops.ln_modulate_fp8,
                quant_rows_fp8=ops.quant_rows_fp8)

    def gemm(a, w, bias, out, epilogue, **kw):
        calls.append(dict(entry="gemm", M=(kw.get("shape") or a.shape)[0], N=w.shape[0], K=w.shape[1], epi=epilogue))
        return real["gemm"](a, w, bias, out, epilogue, **kw)

    def gemm_fp8(a, a_scale, w, w_scale, bias, out, epilogue, gate=None, tok_idx=None, out_scale=None):
        flags = {n for n, t in (("gate", gate), ("tok_idx", tok_idx)) if t is not None}
        if out.stride(0) != w.shape[0]:
            flags.add("out_window")
        calls.append(dict(entry="gemm_fp8", M=a.shape[0], N=w.shape[0], K=w.shape[1], epi=epilogue, flags=frozenset(flags)))
        return real["gemm_fp8"](a, a_scale, w, w_scale, bias, out, epilogue, gate=gate, tok_idx=tok_idx, out_scale=out_scale)

    def ln_modulate(x, out, *args, **kw):
        calls.append(dict(entry="ln_modulate", L=x.shape[0], C=x.shape[1]))
        return real["ln_modulate"](x, out, *args, **kw)

    def ln_modulate_fp8(x, out, out_scale, scale, shift, tok_idx=None, weight=None, bias=None, eps=1e-6):
        calls.append(dict(entry="ln_modulate_fp8", L=x.shape[0], C=x.shape[1], form="affine" if weight is not None else "adaln",
                          tok_idx=tok_idx is not None))
        return real["ln_modulate_fp8"](x, out, out_scale, scale, shift, tok_idx, weight, bias, eps)

    def quant_rows_fp8(x, out, out_scale):
        calls.append(dict(entry="quant_rows_fp8", M=x.shape[0], K=x.shape[1]))
        return real["quant_rows_fp8"](x, out, out_scale)
    for name, fn in (("gemm", gemm), ("gemm_fp8", gemm_fp8), ("ln_modulate", ln_modulate), ("ln_modulate_fp8", ln_modulate_fp8),
                     ("quant_rows_fp8", quant_rows_fp8)):
        monkeypatch.setattr(ops, name, fn)
    return calls


def unmatched_fp8_launches(calls, cfg):
    """Recorded launches of configuration `cfg` without a row: fp8 launches against FP8_TABLE on every field; bf16 GEMMs (the
    all-layer cross K|V, recorded from a one-layer engine) against the production table of test_gpu_kernel_contract_prod;
    a bf16 LayerNorm inside an fp8 block has no row at all."""
    import test_gpu_kernel_contract_prod as P
    rows = [r for r in FP8_TABLE if r["cfg"] == cfg]
    bad = []
    for c in calls:
        if c["entry"] == "gemm":
            ok = any(r["entry"] == "gemm" and r["N"] // r["layers"] == c["N"] and r["K"] == c["K"] and r["epi"] == c["epi"]
                     and r["M"] == c["M"] for r in P.PROD_TABLE if r["cfg"] == cfg)
        else:
            keys = [k for k in c if k != "entry"]
            ok = any(r["entry"] == c["entry"] and all(r.get(k) == c[k] for k in keys) for r in rows)
        if not ok and c not in bad:
            bad.append(c)
    return bad


@gpu
@pytest.mark.parametrize("cfg_name", list(DIT_CFGS))
def test_fp8_table_covers_the_engines_launches(monkeypatch, cfg_name):
    """One real-width, one-layer WanDiT(precision="fp8") block (the engine's own _block, after its all-layer cross K|V GEMM) at
    the production L of the configuration, with recording wrappers around the ops entries: every launch must have a row."""
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
    eng = WanDiT(sd, variant, device="cuda", precision="fp8", **kw)
    del sd
    L, C = P.production_L(cfg_name), d["C"]                    # derived from the latent, not from the table
    g = torch.Generator(device="cuda").manual_seed(L)
    xs = torch.randn(L, C, generator=g, device="cuda")
    ctx = torch.randn((257 if d["img"] else 0) + 512, C, generator=g, device="cuda").to(torch.bfloat16)
    t_unique = torch.tensor([0.0, 900.0] if cfg_name == "5b" else [500.0], device="cuda")
    _, mod, _ = eng._time_tables(t_unique)
    tok_idx = (torch.arange(L, device="cuda") >= L // 3).to(torch.int32) if cfg_name == "5b" else None
    rope = eng._rope_table([(1, 1, L, 0)])
    calls = _record_fp8(monkeypatch)
    kv = eng._cross_kv(ctx)
    eng._block(0, xs, mod, tok_idx, rope, L, kv, L)
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert any(c["entry"] == "gemm_fp8" for c in calls), "the fp8 engine made no fp8 GEMM launch"
    bad = unmatched_fp8_launches(calls, cfg_name)
    assert not bad, f"{cfg_name}: {len(bad)} launch(es) without a table row: {bad}"
    assert torch.isfinite(xs).all()
