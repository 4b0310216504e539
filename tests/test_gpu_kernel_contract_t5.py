"""Per-element kernel contract of include/yume_b200_t5.h (`-m gpu`): yb_t5_attention, yb_t5_rmsnorm and yb_t5_geglu against
fp64 references computed on the device from the same bf16 / f32 inputs, with the bounds derived below, on NaN-poisoned outputs
inside guard-banded buffers; plus the encoder's production shapes (attention at L = 512 with 64 heads for B = 1 and 2, the
norms and the gated GELU at the real width, and the four GEMM launches at M = 512 and 1024 with the block_n the engine picks,
checked with the sampled machinery of tests/test_gpu_kernel_contract_prod.py), and a recording run of a one-layer real-width
engine that fails on any launch without a row of T5_TABLE.

Machinery (guarded / assert_within / _gen) is that of tests/test_gpu_kernel_contract.py. The reference and bound helpers above
the fixtures need no GPU; tests/test_t5_cpu.py runs them on the CPU, including the defects each bound must reject (the bias
with the sign of j - i flipped, a masked key included, a 1/8 score scale; the erf GELU, u and g swapped; the mean subtracted).
u16 = 2^-8, u32 = 2^-24.
"""
import pytest
import torch
import torch.nn.functional as F

import test_gpu_kernel_contract_prod as KP
from test_gpu_kernel_contract import U16, U32, _gen, assert_within, bf16_out_bound, guarded

pytestmark = pytest.mark.gpu

HD = 64
RMS_WIDTHS = (128, 256, 512, 768, 1024, 2048, 4096)        # the yb_t5_rmsnorm instances
EPI = KP.EPI
XXL = dict(dim=4096, dim_attn=4096, dim_ffn=10240, num_heads=64)


# ------------------------------------------------------------------------------------------------------------
# references and bounds (no GPU needed)
# ------------------------------------------------------------------------------------------------------------
def rel_index(L, device="cpu"):
    """[L, L] column of bias[h] for (query i, key j): j - i + L - 1."""
    ar = torch.arange(L, device=device)
    return ar[None, :] - ar[:, None] + L - 1


def t5_attention_ref(q, k, v, bias, keep, B, heads, flip=False, scale=1.0):
    """fp64 reference and bound of yb_t5_attention. q, k, v [B*L, heads*64] (any dtype); bias [heads, 2L-1]; keep bool
    [B, L] or None. flip / scale build defects (bias at i - j + L - 1; scores * scale).
    The kernel, per (b, h, query i), with e_i the largest logit error over the kept keys j:
      s_ij = q_i.k_j     fp32 sum of 64 exact bf16 products, in-core partial sums may truncate: 2*64*u32*(|q||k|^T)_ij
      + bias             one rounding: u32*|s_ij|
      exp(s - m)         the subtraction and the log2(e) multiply of __expf round once each (2*u32*(|s_ij| + |m_i|)), and
                         ex2.approx is within 2^-22 relative (4*u32 taken)
    so every p_ij moves by a relative e_i at most and the normalised weights by 2*e_i: 2*e_i * sum_j p_ij |v_j|.
      u16*|ref|          output rounding to bf16
      2*u16 * sum p|v|   P rounded to bf16 as the A operand of P.V while the normaliser sums the fp32 p_ij
      (28*nkv + 40)*u32 * sum p|v|   fp32 terms that grow with the nkv = ceil(L/64) K/V tiles: the normaliser (16 p per lane
                         and tile added in order, the rescale and the tile sum: 18*nkv, 2 shuffle levels), the rescales of l
                         and o (nkv each), o += P.V over 4 chained k16 mma steps per tile, in-core sums truncating
                         (2*(4*nkv + 16)), the final reciprocal and multiply (2)
    Masked keys have weight 0 exactly (the reference's finfo.min fill underflows to 0 in the softmax)."""
    BL = q.shape[0]
    L = BL // B
    nkv = -(-L // 64)
    dev = q.device
    idx = rel_index(L, dev)
    if flip:
        idx = 2 * (L - 1) - idx                                     # i - j + L - 1
    ref = torch.empty(BL, heads * HD, dtype=torch.float64, device=dev)
    bound = torch.empty_like(ref)
    for b in range(B):
        rows = slice(b * L, (b + 1) * L)
        kb = None if keep is None else keep[b].to(dev)
        for h in range(heads):
            cols = slice(h * HD, (h + 1) * HD)
            qh, kh, vh = q[rows, cols].double(), k[rows, cols].double(), v[rows, cols].double()
            s = (qh @ kh.t()) * scale + bias[h].double()[idx]
            if kb is not None:
                s = s.masked_fill(~kb[None, :], float("-inf"))
            p = torch.softmax(s, dim=-1)
            o = p @ vh
            pv = p @ vh.abs()
            sf = torch.where(torch.isinf(s), torch.zeros_like(s), s)
            m = sf.amax(dim=-1, keepdim=True).abs()
            e = 2 * HD * U32 * (qh.abs() @ kh.abs().t()) + U32 * sf.abs() + 2 * U32 * (sf.abs() + m) + 4 * U32
            if kb is not None:
                e = e.masked_fill(~kb[None, :], 0.0)
            e = e.amax(dim=-1, keepdim=True)
            ref[rows, cols] = o
            bound[rows, cols] = U16 * o.abs() + (2 * U16 + 2 * e + (28 * nkv + 40) * U32) * pv
    return ref, bound


def rmsnorm_ref(x, w, eps=1e-6, subtract_mean=False):
    """fp64 reference and fp32 error term of yb_t5_rmsnorm (x f32 [L, C], w f32 [C]); subtract_mean builds a defect.
    Kernel: sum of squares with per-lane runs of C/32 products and a 5-level shuffle, each product and addition rounded once:
    relative (C/32 + 8)*u32; / C and + eps: 2*u32; rsqrtf <= 2 ulp: the rstd is off by a relative (C/64 + 4)*u32 + 3*u32
    (half the mean-square error, through the square root); then x*rstd and *w round once each. So
      |y32 - ref| <= ((C/64 + 7) + 2) * u32 * |ref|,
    and the bf16 output adds bf16_out_bound on top. Returns (ref, f32_err)."""
    xd = x.double()
    if subtract_mean:
        xd = xd - xd.mean(dim=1, keepdim=True)
    C = x.shape[1]
    ref = xd * torch.rsqrt(xd.pow(2).mean(dim=1, keepdim=True) + eps) * w.double()
    return ref, (C / 64 + 9) * U32 * ref.abs()


def gelu_tanh64(g):
    return 0.5 * g * (1.0 + torch.tanh(0.7978845608028654 * (g + 0.044715 * g ** 3)))


def geglu_ref(ug, F_, erf=False, swap=False):
    """fp64 reference and bound of yb_t5_geglu (ug bf16 [L, 2F]); erf / swap build defects.
    Kernel in fp32: z = k0 * (g + k1 * g^3): g^3 (2 roundings), k1 * g^3, the sum, k0 * (...) and the fp32 constants k0, k1
    themselves (1 each): |dz| <= 7*u32 * k0 * (|g| + k1*|g|^3). tanhf is within 2 ulp, |tanh'| <= 1: |dt| <= |dz| + 2*u32.
    1 + t rounds once (<= 2*u32 absolute); 0.5*g*(1+t) once (u32 * |gelu|): |dgelu| <= 0.5*|g|*(|dz| + 4*u32) + u32*|gelu|.
    u * gelu rounds once: f32 error |u|*|dgelu| + u32*|ref|; then bf16_out_bound. Returns (ref, bound)."""
    u, g = ug[:, :F_].double(), ug[:, F_:2 * F_].double()
    if swap:
        u, g = g, u
    act = 0.5 * g * (1.0 + torch.erf(g / 2 ** 0.5)) if erf else gelu_tanh64(g)
    ref = u * act
    gg = ug[:, F_:2 * F_].double().abs() if not swap else ug[:, :F_].double().abs()
    dz = 7 * U32 * 0.7978845608028654 * (gg + 0.044715 * gg ** 3)
    dgelu = 0.5 * gg * (dz + 4 * U32) + U32 * act.abs()
    uu = (ug[:, :F_] if not swap else ug[:, F_:2 * F_]).double().abs()
    f32 = uu * dgelu + U32 * ref.abs()
    return ref, bf16_out_bound(ref, f32)


def attention_inputs(g, B, L, heads, mask_kind, device="cpu", q_scale=0.5):
    """q, k, v as column slices of one [B*L, 3*heads*64] bf16 buffer (the fused q|k|v GEMM output), a bias table with the
    magnitude of trained T5 biases (N(0, 2^2)), and the key mask: 'prefix' (B = 1: L//3 + 1 kept; B = 2: that and L),
    'holed' (seeded 60 % kept, key 0 kept) or 'none'."""
    W = heads * HD
    buf = torch.randn(B * L, 3 * W, generator=g)
    buf[:, :W] *= q_scale
    buf = buf.to(torch.bfloat16).to(device)
    bias = (2.0 * torch.randn(heads, 2 * L - 1, generator=g)).to(device)
    if mask_kind == "none":
        keep = None
    elif mask_kind == "prefix":
        keep = torch.zeros(B, L, dtype=torch.bool)
        for b, n in enumerate([L // 3 + 1, L][:B]):
            keep[b, :n] = True
    else:
        keep = torch.rand(B, L, generator=g) < 0.6
        keep[:, 0] = True
    return buf[:, :W], buf[:, W:2 * W], buf[:, 2 * W:], bias, None if keep is None else keep.to(device)


# ------------------------------------------------------------------------------------------------------------
# fixtures
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()
    return "cuda"


def _run_attention(q, k, v, bias, keep, B, heads, tag):
    from yume_b200 import ops
    out = guarded((q.shape[0], heads * HD), torch.bfloat16, pad=(64, 64))
    km = None if keep is None else keep.to(torch.uint8).contiguous()
    ops.t5_attention(q, k, v, out.view, B, heads, bias, km)
    torch.cuda.synchronize()
    out.check(tag)
    return out.view


# ------------------------------------------------------------------------------------------------------------
# yb_t5_attention
# ------------------------------------------------------------------------------------------------------------
ATT_CASES = [(1, 1, 1, "none"), (1, 3, 2, "prefix"), (7, 2, 1, "none"), (7, 5, 2, "holed"), (64, 4, 1, "holed"),
             (64, 64, 1, "prefix"), (77, 3, 2, "prefix"), (77, 16, 1, "holed"), (512, 8, 1, "prefix"), (512, 2, 2, "holed"),
             (600, 4, 2, "prefix"), (600, 1, 1, "none"), (600, 3, 1, "holed")]


@pytest.mark.parametrize("L,heads,B,mask", ATT_CASES)
def test_t5_attention_per_element(dev, L, heads, B, mask):
    """Lengths around the 64-row query and key tiles (1, 7, 64, 77, 512, 600), 1 to 64 heads, B = 1 and 2, prefix / holed /
    no masks. q, k, v are column slices of one fused buffer; the output a NaN-poisoned column window with guard rows and
    columns. Bound: t5_attention_ref (every row, including queries past a prefix mask, which the reference also returns)."""
    g = _gen("t5att", L, heads, B, mask)
    q, k, v, bias, keep = attention_inputs(g, B, L, heads, mask, dev)
    tag = f"t5_attention L{L} h{heads} B{B} {mask}"
    got = _run_attention(q, k, v, bias, keep, B, heads, tag)
    ref, bound = t5_attention_ref(q, k, v, bias, keep, B, heads)
    assert_within(got, ref, bound, tag, "t5_attention")


@pytest.mark.parametrize("B", [1, 2])
def test_t5_attention_production(dev, B):
    """The umT5-XXL launch: L = 512, 64 heads, q|k|v slices of the [B*512, 3*4096] buffer, the 120-token prompt mask (B = 2:
    a 120-token and a full 512-token prompt), bias magnitudes of trained T5 tables. Full fp64 reference, every row."""
    g = _gen("t5att_prod", B)
    q, k, v, bias, _ = attention_inputs(g, B, 512, 64, "none", dev)
    keep = torch.zeros(B, 512, dtype=torch.bool, device=dev)
    keep[0, :120] = True
    if B == 2:
        keep[1] = True
    tag = f"t5_attention production B{B} L512 h64"
    got = _run_attention(q, k, v, bias, keep, B, 64, tag)
    ref, bound = t5_attention_ref(q, k, v, bias, keep, B, 64)
    assert_within(got, ref, bound, tag, "t5_attention")


# ------------------------------------------------------------------------------------------------------------
# yb_t5_rmsnorm / yb_t5_geglu
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("L,C", [(77, c) for c in RMS_WIDTHS] + [(1, 4096), (512, 4096), (1024, 4096)])
def test_t5_rmsnorm_per_element(dev, L, C, out_dtype):
    """Every width instance and the production rows (L = 512 and 1024 at 4096). x is a column window of a wider fp32 stream
    with a nonzero row mean and rows of very different scale; the output a NaN-poisoned window. Bound: rmsnorm_ref."""
    from yume_b200 import ops
    g = _gen("t5rms", L, C, str(out_dtype))
    xs = (torch.randn(L, C + 16, generator=g) + 0.5) * torch.exp(2 * torch.randn(L, 1, generator=g))
    x = xs.to(dev)[:, 8:8 + C]
    w = (1.0 + 0.3 * torch.randn(C, generator=g)).to(dev)
    out = guarded((L, C), out_dtype, pad=(8, 8))
    ops.t5_rmsnorm(x, out.view, w, 1e-6)
    torch.cuda.synchronize()
    tag = f"t5_rmsnorm L{L} C{C} {out_dtype}"
    out.check(tag)
    ref, f32 = rmsnorm_ref(x, w)
    bound = bf16_out_bound(ref, f32) if out_dtype == torch.bfloat16 else f32 + U32 * ref.abs()
    assert_within(out.view, ref, bound, tag, "t5_rmsnorm")


@pytest.mark.parametrize("L,F_", [(1, 8), (77, 640), (3, 1000), (512, 10240), (1024, 10240)])
def test_t5_geglu_per_element(dev, L, F_):
    """The gated GELU on the [L, 2F] fc1|gate GEMM output (a row window of a wider buffer), production rows at F = 10240.
    Gate values span [-6, 6] so the tanh saturates on both sides. Bound: geglu_ref."""
    from yume_b200 import ops
    g = _gen("t5geglu", L, F_)
    ugf = torch.randn(L, 2 * F_ + 64, generator=g) * 2
    ug = ugf.to(torch.bfloat16).to(dev)[:, 32:32 + 2 * F_]
    out = guarded((L, F_), torch.bfloat16, pad=(8, 8))
    ops.t5_geglu(ug, out.view)
    torch.cuda.synchronize()
    tag = f"t5_geglu L{L} F{F_}"
    out.check(tag)
    ref, bound = geglu_ref(ug, F_)
    assert_within(out.view, ref, bound, tag, "t5_geglu")


def test_t5_entry_points_reject_bad_arguments(dev):
    """Return codes only, no launch: NULL pointers and non-positive sizes (YB_ERR_ARG), an rmsnorm width without an instance,
    F % 8 != 0 and a row stride below the row (YB_ERR_SHAPE), a misaligned pointer or stride (YB_ERR_ALIGNMENT)."""
    from yume_b200 import _lib
    lib = _lib.load()
    x = torch.zeros(64, 1024, device=dev)
    b = torch.zeros(64, 1024, device=dev, dtype=torch.bfloat16)
    p, pb = x.data_ptr(), b.data_ptr()
    assert lib.yb_t5_attention(None, 64, pb, 64, pb, 64, pb, 64, 1, 8, 1, p, None, None) == -1
    assert lib.yb_t5_attention(pb, 64, pb, 64, pb, 64, pb, 64, 1, 0, 1, p, None, None) == -1
    assert lib.yb_t5_attention(pb, 32, pb, 64, pb, 64, pb, 64, 1, 8, 1, p, None, None) == -2
    assert lib.yb_t5_attention(pb + 2, 64, pb, 64, pb, 64, pb, 64, 1, 8, 1, p, None, None) == -3
    assert lib.yb_t5_attention(pb, 68, pb, 68, pb, 68, pb, 68, 1, 8, 1, p, None, None) == -3
    assert lib.yb_t5_rmsnorm(None, 1024, p, 1024, 1, p, 8, 1024, 1e-6, None) == -1
    assert lib.yb_t5_rmsnorm(p, 1024, p, 1024, 1, p, 8, 1000, 1e-6, None) == -2
    assert lib.yb_t5_rmsnorm(p, 1024, p, 1024, 1, p, 8, 8192, 1e-6, None) == -2
    assert lib.yb_t5_rmsnorm(p + 4, 1024, p, 1024, 1, p, 8, 512, 1e-6, None) == -3
    assert lib.yb_t5_geglu(None, 1024, pb, 512, 8, 512, None) == -1
    assert lib.yb_t5_geglu(pb, 1024, pb, 512, 8, 500, None) == -2
    assert lib.yb_t5_geglu(pb, 512, pb, 512, 8, 512, None) == -2
    assert lib.yb_t5_geglu(pb + 2, 1024, pb, 512, 8, 512, None) == -3
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------
# production GEMM rows and the launch table
# ------------------------------------------------------------------------------------------------------------
def _t5_gemm_rows():
    from yume_b200.t5 import gemm_block_n
    C, A, Fd = XXL["dim"], XXL["dim_attn"], XXL["dim_ffn"]
    rows = []
    for M in (512, 1024):
        for name, N, K, epi in (("qkv", 3 * A, C, "BF16"), ("o", C, A, "GATE_RES"), ("fc1_gate", 2 * Fd, C, "BF16"),
                                ("fc2", C, Fd, "GATE_RES")):
            rows.append(dict(id=f"umt5_M{M}_{name}", entry="gemm", M=M, N=N, K=K, epi=EPI[epi],
                             block_n=gemm_block_n(M, N, KP.SMS)))
    return rows


T5_GEMM_ROWS = _t5_gemm_rows()
# every launch of the umT5-XXL encoder at B = 1 and 2 prompts of 512 tokens
T5_TABLE = T5_GEMM_ROWS + [dict(entry="t5_attention", B=B, L=512, heads=64) for B in (1, 2)] + \
    [dict(entry="t5_rmsnorm", L=M, C=4096, out=dt) for M in (512, 1024) for dt in (torch.bfloat16, torch.float32)] + \
    [dict(entry="t5_geglu", L=M, F=10240) for M in (512, 1024)]


@pytest.mark.parametrize("rid", [r["id"] for r in T5_GEMM_ROWS])
def test_t5_prod_gemm(dev, rid):
    """The four GEMM launches of an umT5-XXL layer at M = 512 (B = 1) and 1024 (B = 2) with the engine's block_n: NaN-poisoned
    (BF16) or seeded (GATE_RES, in place, then once more under F32 into a NaN buffer) outputs with guard rows, the fp64
    reference on the sampled rows and columns (test_gpu_kernel_contract_prod.gemm_sample: every tile of either block_n)."""
    from yume_b200 import ops
    row = next(r for r in T5_GEMM_ROWS if r["id"] == rid)
    M, N, K, epi, bn = row["M"], row["N"], row["K"], row["epi"], row["block_n"]
    g = KP._cuda_gen(rid)
    A = KP._rand(g, M, K)
    B = KP._rand(g, N, K, 1 / K ** 0.5)
    rows, cols = KP.gemm_sample(M, N, rid)
    tag = f"t5 prod gemm {rid} M{M} N{N} K{K} bn{bn}"
    if epi == EPI["GATE_RES"]:
        x0 = KP._rand(g, M, N, dtype=torch.float32)
        out = KP.Lean(M, N, torch.float32, fill=x0)
        ops.gemm(A, B, None, out.view, epi, block_n=bn)
        torch.cuda.synchronize()
        out.check(tag + " GATE_RES")
        KP._check_gemm_sampled(out.view, A, B, rows, cols, epi, tag + " GATE_RES", "t5_prod_gemm", x0=x0)
        o32 = KP.Lean(M, N, torch.float32)
        ops.gemm(A, B, None, o32.view, EPI["F32"], block_n=bn)
        torch.cuda.synchronize()
        o32.check(tag + " F32 coverage run")
        KP._check_gemm_sampled(o32.view, A, B, rows, cols, EPI["F32"], tag + " F32 coverage run", "t5_prod_gemm")
        return
    out = KP.Lean(M, N, torch.bfloat16)
    ops.gemm(A, B, None, out.view, epi, block_n=bn)
    torch.cuda.synchronize()
    out.check(tag)
    KP._check_gemm_sampled(out.view, A, B, rows, cols, epi, tag, "t5_prod_gemm")


def _record(monkeypatch):
    from yume_b200 import ops
    calls = []
    real = dict(gemm=ops.gemm, t5_attention=ops.t5_attention, t5_rmsnorm=ops.t5_rmsnorm, t5_geglu=ops.t5_geglu)

    def gemm(a, w, bias, out, epilogue, **kw):
        calls.append(dict(entry="gemm", M=a.shape[0], N=w.shape[0], K=w.shape[1], epi=epilogue, block_n=kw.get("block_n", 0)))
        return real["gemm"](a, w, bias, out, epilogue, **kw)

    def t5_attention(q, k, v, out, B, heads, bias, key_mask=None):
        calls.append(dict(entry="t5_attention", B=B, L=q.shape[0] // B, heads=heads))
        return real["t5_attention"](q, k, v, out, B, heads, bias, key_mask)

    def t5_rmsnorm(x, out, weight, eps=1e-6):
        calls.append(dict(entry="t5_rmsnorm", L=x.shape[0], C=x.shape[1], out=out.dtype))
        return real["t5_rmsnorm"](x, out, weight, eps)

    def t5_geglu(ug, out):
        calls.append(dict(entry="t5_geglu", L=ug.shape[0], F=out.shape[1]))
        return real["t5_geglu"](ug, out)
    for name, fn in (("gemm", gemm), ("t5_attention", t5_attention), ("t5_rmsnorm", t5_rmsnorm), ("t5_geglu", t5_geglu)):
        monkeypatch.setattr(ops, name, fn)
    return calls


def unmatched_t5_launches(calls):
    keys = {"gemm": ("M", "N", "K", "epi", "block_n"), "t5_attention": ("B", "L", "heads"), "t5_rmsnorm": ("L", "C", "out"),
            "t5_geglu": ("L", "F")}
    bad = []
    for c in calls:
        ok = any(r["entry"] == c["entry"] and all(r[k] == c[k] for k in keys[c["entry"]]) for r in T5_TABLE)
        if not ok and c not in bad:
            bad.append(c)
    return bad


@pytest.mark.parametrize("B", [1, 2])
def test_t5_table_covers_the_engines_launches(dev, monkeypatch, B):
    """A one-layer umT5-XXL-width engine (bf16 weights generated on the device, vocabulary cut to 4096 rows: only the gather
    depends on it) encodes B prompts of 512 tokens with recording wrappers around ops.gemm / t5_attention / t5_rmsnorm /
    t5_geglu: every launch must have a row in T5_TABLE (shape, epilogue and block_n)."""
    from oracle import t5 as ot5
    from yume_b200.t5 import T5TextEncoder
    assert KP.SMS == torch.cuda.get_device_properties(0).multi_processor_count, "the table's block_n assumes 132 SMs"
    cfg = dict(ot5.UMT5_XXL, vocab=4096, num_layers=1)
    sd = ot5.make_state_dict(77, **cfg, device=dev, dtype=torch.bfloat16)
    enc = T5TextEncoder(sd, **cfg, device=dev)
    del sd
    ids = torch.randint(0, 4096, (B, 512), generator=torch.Generator().manual_seed(3))
    mask = torch.zeros(B, 512, dtype=torch.long)
    mask[:, :120] = 1
    calls = _record(monkeypatch)
    enc(ids.to(dev), mask.to(dev))
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert len(calls) == 9, calls
    bad = unmatched_t5_launches(calls)
    assert not bad, f"{len(bad)} launch(es) without a T5_TABLE row: {bad}"


# entry point -> tests that exercise it (tests/test_t5_cpu.py applies the entry-point guard to include/yume_b200_t5.h)
COVERS = {
    "yb_t5_attention": ["test_t5_attention_per_element", "test_t5_attention_production",
                        "test_t5_entry_points_reject_bad_arguments", "test_t5_table_covers_the_engines_launches"],
    "yb_t5_rmsnorm": ["test_t5_rmsnorm_per_element", "test_t5_entry_points_reject_bad_arguments",
                      "test_t5_table_covers_the_engines_launches"],
    "yb_t5_geglu": ["test_t5_geglu_per_element", "test_t5_entry_points_reject_bad_arguments",
                    "test_t5_table_covers_the_engines_launches"],
}
