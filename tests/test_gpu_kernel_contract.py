"""Per-element kernel contract (`-m gpu`): every dispatch path of the CUDA kernels against a plain fp64 reference computed on the
device from the same bf16 / f32 inputs the kernel saw, with a per-element error bound derived from the arithmetic (never fitted to
the data), on outputs that are NaN-poisoned views inside larger guard-banded buffers.

Why not one relative-Frobenius number: a 64-wide K block dropped from one tail tile, eight columns never written in one row or a
wrong gate row for a few tokens move the global norm by less than bf16 rounding does. Here every element must satisfy
|got - ref| <= bound, every element of the output view must have been written (it starts as NaN, or as seeded finite data for
in-place and accumulating ops), and the guard band around the view (same allocation, so a stray store never reaches memory the
test does not own) must keep its bit pattern. Outputs are column windows / row offsets of larger buffers and operands are the
strided views production passes (qkv column slices, row / column offsets of B, ldb > K).

The worst |err| / bound of each case is printed and kept per kernel family; with YB_CONTRACT_REPORT=<path> the per-family worst
ratios are also written there as JSON at the end of the module.

Symbols: u16 = 2^-8 (unit roundoff of bf16), u32 = 2^-24 (of fp32). The helpers at the top need no GPU and are exercised on the
CPU by tests/test_kernel_contract_cpu.py, including one realistic defect per bound that the bound must reject.
"""
import json
import math
import os
import zlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U16 = 2.0 ** -8
U32 = 2.0 ** -24
YB_ERR_SHAPE = -2     # include/yume_b200.h

# dispatch width tables: tests/test_kernel_contract_cpu.py checks them against the template instances in the .cu sources
LN_WARP_WIDTHS = (256, 1024, 3072, 5120)              # YB_LN_WARP(2, 8, 24, 40): C = 128 * NV
LN_GENERAL_WIDTHS = (1280, 1536, 8192)                # ln_modulate_kernel (also every ada + affine call)
RR_WARP_WIDTHS = (256, 1024, 3072, 5120)              # YB_RR_FAST / YB_RR_WARP / YB_QK_WARP(1, 4, 12, 20): C = 256 * NCH
RR_GENERAL_WIDTHS = (384,)                            # rmsnorm_rope_kernel
SC_WIDTHS = (256, 1024, 3072, 5120)                   # YB_SC(1, 4, 12, 20); other widths are rejected (no general kernel)

# ------------------------------------------------------------------------------------------------------------
# shared machinery (no GPU needed)
# ------------------------------------------------------------------------------------------------------------
_GUARD_BITS = {torch.bfloat16: (torch.int16, 0x5A5B), torch.float32: (torch.int32, 0x5A5B5C5D),
               torch.float64: (torch.int64, 0x5A5B5C5D5E5F6061)}
_INT_VIEW = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}
WORST = {}           # kernel family -> worst |err| / bound over the passing cases of this module


class Guarded:
    """A view the kernel writes, inside a backing buffer whose other elements (the guard band) hold a fixed bit pattern."""

    def __init__(self, view, backing, mask):
        self.view, self.backing, self.mask = view, backing, mask
        self.bits = backing.view(_INT_VIEW[backing.dtype]).clone()

    def check(self, what, allow_nan=False):
        """The guard band is bit-identical to what it was before the call, and the view holds no NaN (every element written)."""
        now = self.backing.view(_INT_VIEW[self.backing.dtype])
        moved = (now != self.bits) & self.mask
        n = int(moved.sum())
        if n:
            idx = tuple(int(i) for i in moved.nonzero()[0])
            raise AssertionError(f"{what}: {n} guard-band element(s) changed, first at backing index {idx}")
        if not allow_nan:
            bad = torch.isnan(self.view)
            n = int(bad.sum())
            if n:
                idx = tuple(int(i) for i in bad.nonzero()[0])
                raise AssertionError(f"{what}: {n} output element(s) never written (still NaN), first at {idx}")


def guarded(shape, dtype, pad=(0, 0), fill=None, device="cuda"):
    """Backing buffer with `pad[0]` guard rows above and below the view and `pad[1]` guard columns left and right of it (the
    view's row stride is then shape[-1] + 2 * pad[1]; keep pad[1] % 8 == 0 for 16-byte alignment). The view is NaN, or a copy
    of `fill` (in-place / accumulating ops). Returns a Guarded with .view, .backing and .check()."""
    pr, pc = pad
    full = (shape[0] + 2 * pr,) + tuple(shape[1:-1]) + (shape[-1] + 2 * pc,)
    itype, pattern = _GUARD_BITS[dtype]
    backing = torch.full(full, pattern, dtype=itype, device=device).view(dtype)
    view = backing[pr:pr + shape[0], ..., pc:pc + shape[-1]]
    if fill is None:
        view.fill_(float("nan"))
    else:
        view.copy_(fill)
    mask = torch.ones(full, dtype=torch.bool, device=device)
    mask[pr:pr + shape[0], ..., pc:pc + shape[-1]] = False
    return Guarded(view, backing, mask)


def assert_within(got, ref, bound, what, family=None):
    """Per element |got - ref| <= bound (fp64). On failure: how many elements fail, the worst one in tensor coordinates and its
    |err| / bound. Returns (and records under `family`) the worst ratio of a passing case."""
    g = got.double()
    r = ref.double().to(g.device)
    b = bound.double().to(g.device)
    err = (g - r).abs()
    ratio = torch.where(b > 0, err / b, torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    ratio = torch.where(torch.isnan(err), torch.full_like(err, math.inf), ratio)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if not worst <= 1.0:
        fail = ratio > 1.0
        i = int(ratio.argmax())
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), ratio.shape))
        raise AssertionError(f"{what}: {int(fail.sum())} of {ratio.numel()} elements out of bound; worst at {idx}: "
                             f"got {float(g[idx]):.6g} ref {float(r[idx]):.6g} bound {float(b[idx]):.3g} "
                             f"(|err|/bound = {worst:.3g})")
    print(f"[contract] {what}: worst |err|/bound = {worst:.3f}")
    if family is not None:
        WORST[family] = max(WORST.get(family, 0.0), worst)
    return worst


def record_exact(family):
    """A bit-exact family passed a case (its |err| / bound is 0 by definition)."""
    WORST.setdefault(family, 0.0)


# ---- bounds ------------------------------------------------------------------------------------------------------------
def gemm_bounds(A, B, K):
    """fp32 accumulation of K bf16 products (exact in fp32) in any order, rounding or truncating each partial sum:
    |acc32 - acc| <= 2*K*u32 * (|A| |B|^T)_ij (the factor 2 covers truncation). Returns that term in fp64."""
    return 2.0 * K * U32 * (A.double().abs() @ B.double().abs().t())


def bf16_out_bound(ref, f32_err):
    """An fp32 value within f32_err of ref, rounded to bf16 (to nearest): |bf16(v) - ref| <= u16*(|ref| + f32_err) + f32_err."""
    return U16 * (ref.abs() + f32_err) + f32_err


def attention_bound(q, k, v, scale, ref):
    """Flash attention with fp32 logits / softmax, P rounded to bf16 as the A operand of P.V, bf16 output:
      u16*|ref|                      output rounding
      2*u16 * sum_j p_ij |v_j|       P rounded to bf16 (relative u16 per p_ij) while the normaliser sums the fp32 p_ij
      2*e_i * sum_j p_ij |v_j|       logit error e_i = max_j (2*128*u32*scale*(|q||k|^T)_ij + 4*u32*|s_ij|) moves each p_ij by a
                                     relative 2*e_i at most (fp32 Q.K^T accumulation, the scale / log2(e) multiply, exp2)
    p_ij from the fp64 softmax. q, k, v [L, 128] of one head (fp64)."""
    s = (q @ k.t()) * scale
    p = torch.softmax(s, dim=-1)
    pv = p @ v.abs()
    e = (2 * 128 * U32 * scale * (q.abs() @ k.abs().t()) + 4 * U32 * s.abs()).amax(dim=-1, keepdim=True)
    return U16 * ref.abs() + (2 * U16 + 2 * e) * pv


def _sum_err(C):
    """fp32 row sums in these kernels are per-thread runs of at most C/128 terms followed by a <= 8-level tree: the error of
    such a sum is <= (C/128 + 10) * u32 * sum |terms|."""
    return (C / 128 + 10) * U32


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


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("[contract] worst |err|/bound per family: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(WORST.items())))
        path = os.environ.get("YB_CONTRACT_REPORT")
        if path:
            info = {}
            if torch.cuda.is_available():
                info["device"] = torch.cuda.get_device_name(0)
            with open(path, "w") as f:
                json.dump({"worst_ratio": WORST, **info}, f, indent=1, sort_keys=True)


def _gen(*key):
    """CPU generator seeded from the case's parameters with a stable hash (str hashes are salted per process), so every case
    draws the same data in every run and a failure replays from its test id alone."""
    return torch.Generator(device="cpu").manual_seed(zlib.crc32(repr(key).encode()))


def _randn(g, *shape, scale=1.0, dev="cuda"):
    return (torch.randn(*shape, generator=g) * scale).to(dev)


# ------------------------------------------------------------------------------------------------------------
# GEMM yb_gemm_bf16
# ------------------------------------------------------------------------------------------------------------
GEMM_SHAPES = [(1, 32, 3072), (127, 96, 72), (129, 160, 144), (255, 3072, 120), (257, 96, 14336), (1000, 3072, 3072),
               (1000, 160, 1096)]                     # K % 64: 0, 8, 16, 56, 0, 0, 8
GEMM_LAYOUTS = ["dense", "production", "b_col_window"]


def _gemm_operands(g, M, N, K, layout, dev):
    """A, B as production lays them out. dense: contiguous A / B, out rows offset only (ldo = N). production: A a column slice
    (qkv[:, C:2C]-style, column offset 64, lda > K), B a row block of a larger weight (k[f*Lf:(f+1)*Lf]), out a column window
    (ldo > N) at a row offset. b_col_window: B a column window with ldb > K (vT[:, f*Lf:(f+1)*Lf]), A a column slice at offset 8."""
    a_full = _randn(g, M, K + 136, dev=dev).bfloat16()
    if layout == "dense":
        b_full = _randn(g, N, K, scale=1 / math.sqrt(K), dev=dev).bfloat16()
        A, B, pad = a_full[:, :K].contiguous(), b_full, (256, 0)
    elif layout == "production":
        b_full = _randn(g, N + 96, K, scale=1 / math.sqrt(K), dev=dev).bfloat16()      # rows 32 .. 32+N of a [N+96, K] weight
        A, B, pad = a_full[:, 64:64 + K], b_full[32:32 + N], (256, 256)
    else:
        b_full = _randn(g, N, K + 72, scale=1 / math.sqrt(K), dev=dev).bfloat16()
        A, B, pad = a_full[:, 8:8 + K], b_full[:, 64:64 + K], (256, 256)
    return A, B, pad


@pytest.mark.parametrize("layout", GEMM_LAYOUTS)
@pytest.mark.parametrize("kernel,block_n", [(1, 0), (1, 128), (1, 256), (2, 0), (2, 128), (2, 256)])
@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_every_epilogue_per_element(dev, M, N, K, kernel, block_n, layout):
    """Every epilogue on one operand set. acc = A.B^T + bias in fp64; F = 2*K*u32*(|A||B|^T) (gemm_bounds); every fp32 epilogue
    op adds at most u32 * |its operands|, covered by 4*u32*(sum of operand magnitudes). Bounds:
      BF16 / RES_BF16   bf16_out_bound(ref, F + 4*u32*(|acc| + |bias| + |res|))
      GELU tanh / erf   |gelu'| <= 1.13 carries the fp32 error of acc through; tanh.approx.f32 has relative error <= 2^-11, so
                        0.5*|x|*(1+tanh) is off by <= 2^-12*|x| (erff: a few ulp, 2^-20*|x| taken); then bf16 rounding
      F32               F + 4*u32*(|acc| + |bias|)
      GATE_RES          |gate| * (F + 4*u32*(|acc|+|bias|)) + 4*u32*(|x0| + |gate*acc|) (fp32 residual, no output rounding)"""
    from yume_b200 import ops
    g = _gen("gemm", M, N, K, kernel, block_n, layout)
    A, B, pad = _gemm_operands(g, M, N, K, layout, dev)
    bias = _randn(g, N, dev=dev)
    Ad, Bd = A.double(), B.double()
    acc = Ad @ Bd.t()
    Fb = gemm_bounds(A, B, K)
    accb = acc + bias.double()
    tag = f"gemm M{M} N{N} K{K} cta{kernel} bn{block_n} {layout}"
    kw = dict(cta_pair=kernel, block_n=block_n)

    def run(epi, dtype, fill=None, **extra):
        out = guarded((M, N), dtype, pad, fill=fill)
        ops.gemm(A, B, extra.pop("bias", bias), out.view, epi, **kw, **extra)
        torch.cuda.synchronize()
        return out

    o = run(ops.YB_EPI_BF16, torch.bfloat16)
    o.check(tag + " BF16")
    assert_within(o.view, accb, bf16_out_bound(accb, Fb + 4 * U32 * (acc.abs() + bias.double().abs())), tag + " BF16", "gemm")
    for epi, name in ((ops.YB_EPI_GELU_BF16, "GELU_TANH"), (ops.YB_EPI_GELU_ERF_BF16, "GELU_ERF")):
        o = run(epi, torch.bfloat16)
        o.check(tag + " " + name)
        ref = F.gelu(accb, approximate="tanh") if name == "GELU_TANH" else F.gelu(accb)
        ev = (2.0 ** -12 if name == "GELU_TANH" else 2.0 ** -20) * accb.abs()
        f32 = 1.13 * (Fb + 4 * U32 * (acc.abs() + bias.double().abs())) + ev + 4 * U32 * accb.abs()
        assert_within(o.view, ref, bf16_out_bound(ref, f32), tag + " " + name, "gemm")
    o = run(ops.YB_EPI_F32, torch.float32, bias=None)
    o.check(tag + " F32")
    assert_within(o.view, acc, Fb + 4 * U32 * acc.abs(), tag + " F32", "gemm")
    res = _randn(g, M, N + 16, dev=dev).bfloat16()[:, 8:8 + N]
    o = run(ops.YB_EPI_RES_BF16, torch.bfloat16, res=res)
    o.check(tag + " RES_BF16")
    ref = accb + res.double()
    assert_within(o.view, ref, bf16_out_bound(ref, Fb + 4 * U32 * (acc.abs() + bias.double().abs() + res.double().abs())),
                  tag + " RES_BF16", "gemm")
    U = 3
    gate6 = _randn(g, U, 6, N, dev=dev)
    tok = torch.randint(0, U, (M,), generator=g).to(dev, torch.int32)
    for gated in (True, False):
        x0 = _randn(g, M, N, dev=dev)
        extra = dict(gate=gate6[:, 2], tok_idx=tok) if gated else {}
        o = run(ops.YB_EPI_GATE_RES, torch.float32, fill=x0, **extra)
        o.check(tag + f" GATE_RES gate={gated}")
        gt = gate6[tok.long(), 2].double() if gated else torch.ones_like(acc)
        ref = x0.double() + accb * gt
        bound = gt.abs() * (Fb + 4 * U32 * (acc.abs() + bias.double().abs())) + 4 * U32 * (x0.double().abs() + (gt * accb).abs())
        assert_within(o.view, ref, bound, tag + f" GATE_RES gate={gated}", "gemm")


# ------------------------------------------------------------------------------------------------------------
# attention yb_attention_ex
# ------------------------------------------------------------------------------------------------------------
def _attention_ref(q, k, v, heads, scale):
    """fp64 reference and bound, per head; q [Lq, heads*128], k / v [Lk, heads*128] (any dtype)."""
    Lq = q.shape[0]
    ref = torch.empty(Lq, heads * 128, dtype=torch.float64, device=q.device)
    bound = torch.empty_like(ref)
    for h in range(heads):
        sl = slice(h * 128, (h + 1) * 128)
        qh, kh, vh = q[:, sl].double(), k[:, sl].double(), v[:, sl].double()
        o = torch.softmax((qh @ kh.t()) * scale, dim=-1) @ vh
        ref[:, sl] = o
        bound[:, sl] = attention_bound(qh, kh, vh, scale, o)
    return ref, bound


def _qkv_slices(g, Lq, Lk, heads, dev, q_scale=1.0):
    """q, k, v as column slices of one [L, 3*heads*128] buffer (the fused QKV GEMM output, dit.py)."""
    W = heads * 128
    buf = _randn(g, max(Lq, Lk), 3 * W, dev=dev).bfloat16()
    buf[:, :W] = (buf[:, :W].float() * q_scale).bfloat16()
    return buf[:Lq, :W], buf[:Lk, W:2 * W], buf[:Lk, 2 * W:]


def _run_attention(q, k, v, heads, scale, variant, split, accumulate, fill, tag):
    from yume_b200 import ops
    Lq = q.shape[0]
    out = guarded((Lq, heads * 128), torch.bfloat16, (128, 64), fill=fill)
    ops.attention(q, k, v, out.view, heads, scale=scale, variant=variant, accumulate=accumulate, split=split)
    torch.cuda.synchronize()
    out.check(tag)
    return out.view


@pytest.mark.parametrize("Lk", [1, 127, 128, 129, 383])
@pytest.mark.parametrize("Lq", [1, 255, 257])
@pytest.mark.parametrize("heads", [1, 5])
def test_attention_tails_scales_variants(dev, heads, Lq, Lk):
    """Query / key tails around the 128-row tiles, both kernel variants, three softmax scales (1/sqrt(128), and the
    `softmax_scale` the flash_attention seam passes through). Bound: attention_bound."""
    g = _gen("att", heads, Lq, Lk)
    q, k, v = _qkv_slices(g, Lq, Lk, heads, dev)
    for scale in (1 / math.sqrt(128.0), 0.05, 0.2):
        ref, bound = _attention_ref(q, k, v, heads, scale)
        for variant in (0, 1):
            tag = f"attention h{heads} Lq{Lq} Lk{Lk} scale{scale:.3g} variant{variant}"
            got = _run_attention(q, k, v, heads, scale, variant, 1, False, None, tag)
            assert_within(got, ref, bound, tag, "attention")


@pytest.mark.parametrize("Lq,Lk", [(257, 383), (1, 129), (255, 128)])
@pytest.mark.parametrize("heads", [24, 40])
def test_attention_production_heads(dev, heads, Lq, Lk):
    """The 5B (24 heads) and 14B (40 heads) head counts, short lengths, automatic split policy."""
    g = _gen("atth", heads, Lq, Lk)
    q, k, v = _qkv_slices(g, Lq, Lk, heads, dev)
    for scale in (1 / math.sqrt(128.0), 0.2):
        ref, bound = _attention_ref(q, k, v, heads, scale)
        tag = f"attention h{heads} Lq{Lq} Lk{Lk} scale{scale:.3g}"
        assert_within(_run_attention(q, k, v, heads, scale, 0, 0, False, None, tag), ref, bound, tag, "attention")


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("split", [1, 2, 4])
@pytest.mark.parametrize("Lq,Lk,heads", [(257, 383, 5), (255, 1000, 2)])
def test_attention_split_and_accumulate(dev, Lq, Lk, heads, split, accumulate):
    """Forced KV split (partials + combine kernel) and out += result on seeded finite data. Accumulating adds one more bf16
    rounding of the attention result before the add at most: + u16*|o|."""
    g = _gen("atts", Lq, Lk, heads, split, accumulate)
    q, k, v = _qkv_slices(g, Lq, Lk, heads, dev, q_scale=2.0)
    scale = 1 / math.sqrt(128.0)
    ref, bound = _attention_ref(q, k, v, heads, scale)
    fill = _randn(g, Lq, heads * 128, dev=dev).bfloat16() if accumulate else None
    if accumulate:
        bound = bound + U16 * ref.abs() + U16 * (ref + fill.double()).abs()
        ref = ref + fill.double()
    for variant in (0, 1):
        tag = f"attention Lq{Lq} Lk{Lk} h{heads} split{split} acc{int(accumulate)} variant{variant}"
        assert_within(_run_attention(q, k, v, heads, scale, variant, split, accumulate, fill, tag), ref, bound, tag, "attention")


# ------------------------------------------------------------------------------------------------------------
# norms
# ------------------------------------------------------------------------------------------------------------
def _ln_ref(x, C, eps, w, b, sc, sh):
    """fp64 LayerNorm (+ affine) (+ modulate) and its bound. The kernels compute mean and (two-pass) variance with fp32 sums
    (_sum_err), rsqrtf (<= 2 ulp), then per element (x - mean) * rstd [* w + b] [* (1 + sc) + sh] in fp32:
      d_mean = s*sum|x|/C + u32*|mean|                                  s = _sum_err(C)
      d_rstd/rstd = 0.5*((s + 3*u32) + (d_mean*rstd)^2) + 2^-22
      d_n  = rstd*d_mean + |n|*(d_rstd/rstd + 2*u32)                     n = (x - mean)*rstd
      f32  = |g|*d_n + 4*u32*(|n*w|*|1+sc| + |b|*|1+sc| + |y|)            g = w*(1+sc)
    then bf16 rounding (bf16_out_bound) or none (f32 out)."""
    xd = x.double()
    mean = xd.mean(dim=1, keepdim=True)
    var = (xd - mean).pow(2).mean(dim=1, keepdim=True)
    rstd = torch.rsqrt(var + eps)
    n = (xd - mean) * rstd
    one = torch.ones_like(n)
    wd = w.double() if w is not None else one
    bd = b.double() if b is not None else 0 * one
    scd = sc.double() if sc is not None else 0 * one
    shd = sh.double() if sh is not None else 0 * one
    y = (n * wd + bd) * (1 + scd) + shd
    s = _sum_err(C)
    dmean = s * xd.abs().sum(dim=1, keepdim=True) / C + U32 * mean.abs()
    drel = 0.5 * ((s + 3 * U32) + (dmean * rstd) ** 2) + 2.0 ** -22
    dn = rstd * dmean + n.abs() * (drel + 2 * U32)
    g = (wd * (1 + scd)).abs()
    f32 = g * dn + 4 * U32 * ((n * wd).abs() * (1 + scd).abs() + bd.abs() * (1 + scd).abs() + y.abs())
    return y, f32


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("mode", ["ada_table", "ada_1d", "affine", "ada_affine"])
@pytest.mark.parametrize("C", LN_WARP_WIDTHS + LN_GENERAL_WIDTHS)
def test_ln_modulate_every_instance(dev, C, mode, out_dtype):
    """yb_ln_modulate at every warp instance and the general kernel; ada with a [U, 6, C] table row per token (tok_idx), ada with
    1-D scale / shift, affine, and ada + affine (always the general kernel). x is a column window (ldx > C), out a guarded
    window (ldo > C), L % 8 != 0, and half the rows have mean ~1e3 with unit spread (variance cancellation)."""
    from yume_b200 import ops
    g = _gen("ln", C, mode, str(out_dtype))
    L, U = 203, 3
    xs = torch.randn(L, C + 16, generator=g)
    xs[::2] += 1000.0 + 10 * torch.rand(L // 2 + 1, 1, generator=g)
    x = xs.to(dev)[:, 8:8 + C]
    table = _randn(g, U, 6, C, scale=0.5, dev=dev)
    tok = torch.randint(0, U, (L,), generator=g).to(dev, torch.int32)
    w, b = _randn(g, C, dev=dev), _randn(g, C, dev=dev)
    sc = sh = tk = wt = bt = None
    if mode == "ada_table":
        sc, sh, tk = table[:, 1], table[:, 0], tok
        rsc, rsh = table[tok.long(), 1], table[tok.long(), 0]
    elif mode in ("ada_1d", "ada_affine"):
        sc, sh = table[0, 1], table[0, 0]
        rsc, rsh = sc.expand(L, C), sh.expand(L, C)
    else:
        rsc = rsh = None
    if mode in ("affine", "ada_affine"):
        wt, bt = w, b
    out = guarded((L, C), out_dtype, (8, 8))
    ops.ln_modulate(x, out.view, sc, sh, tk, wt, bt)
    torch.cuda.synchronize()
    tag = f"ln_modulate C{C} {mode} {'f32' if out_dtype == torch.float32 else 'bf16'}"
    out.check(tag)
    y, f32 = _ln_ref(x, C, 1e-6, wt, bt, rsc, rsh)
    bound = bf16_out_bound(y, f32) if out_dtype == torch.bfloat16 else f32
    assert_within(out.view, y, bound, tag, "ln_modulate")


def _rr_ref(x, weight, rope, rope_len, D, eps=1e-6):
    """fp64 RMSNorm * weight + RoPE (adjacent pairs of every head, rows < rope_len) and its bound: sum of squares in fp32
    (_sum_err(C) + u32 relative per square), rsqrtf 2 ulp, then per pair a = x*rstd*w, b likewise (2 roundings each) and the
    rotation a*c - b*s (3 roundings): f32 = (0.5*(s + 2*u32) + 2^-22 + 4*u32) * (|a*c| + |b*s|), m = |a| when not rotated."""
    L, C = x.shape
    xd = x.double()
    rstd = torch.rsqrt(xd.pow(2).mean(dim=1, keepdim=True) + eps)
    n = xd * rstd * weight.double()
    y, mag = n.clone(), n.abs()
    if rope is not None and rope_len > 0:
        r = min(rope_len, L)
        v = n[:r].view(r, C // D, D // 2, 2)
        cs = rope[:r].double()[:, None]
        c, s = cs[..., 0], cs[..., 1]
        rot = torch.stack([v[..., 0] * c - v[..., 1] * s, v[..., 0] * s + v[..., 1] * c], -1)
        m = torch.stack([(v[..., 0] * c).abs() + (v[..., 1] * s).abs(), (v[..., 0] * s).abs() + (v[..., 1] * c).abs()], -1)
        y[:r], mag[:r] = rot.reshape(r, C), m.reshape(r, C)
    f32 = (0.5 * (_sum_err(C) + 2 * U32) + 2.0 ** -22 + 4 * U32) * mag
    return y, bf16_out_bound(y, f32)


def _pieces(t, L, C, pc, ld):
    """Logical [L, C] rows of a peer-major buffer: column c is element c % pc of piece c // pc; pieces L*ld apart."""
    return torch.as_strided(t, (C // pc, L, pc), (L * ld, ld, 1), t.storage_offset()).permute(1, 0, 2).reshape(L, C)


@pytest.mark.parametrize("entry", ["rmsnorm_rope", "qk_norm_rope"])
@pytest.mark.parametrize("split", [1, 2, 4, 8])
@pytest.mark.parametrize("rope_mode", ["none", "0", "L-37", "L"])
@pytest.mark.parametrize("C", RR_WARP_WIDTHS + RR_GENERAL_WIDTHS)
def test_rmsnorm_rope_every_instance(dev, C, rope_mode, split, entry):
    """yb_rmsnorm_rope_pieces / yb_qk_norm_rope against the fp64 formula (not against each other): every YB_RR_FAST / YB_RR_WARP /
    YB_QK_WARP width plus the general kernel (384), rope NULL (the cross-attention q / k) and rope_len 0, L - 37, L; plain rows
    (split 1: q | k | v of the fused [L, 3C] buffer) and pieces of C / split columns laid out as the Ulysses send buffer
    [split, L, q|k|v of C/split]. The untouched v columns and the guard band must keep their bits. Bound: _rr_ref."""
    from yume_b200 import ops
    D, L = 128, 333
    g = _gen("rr", C, rope_mode, split, entry)
    pc = C // split
    data = _randn(g, split * L, 3 * pc, dev=dev).bfloat16()
    buf = guarded((split * L, 3 * pc), torch.bfloat16, (8, 8), fill=data)
    ld = buf.view.stride(0)                                             # 3 * pc + 16: rows of the send buffer inside the backing
    wq, wk = (torch.rand(C, generator=g) + 0.5).to(dev), (torch.rand(C, generator=g) + 0.5).to(dev)
    rope = None
    rope_len = 0
    if rope_mode != "none":
        ang = torch.rand(L, D // 2, generator=g, dtype=torch.float64) * 6.28
        rope = torch.stack([ang.cos(), ang.sin()], -1).float().contiguous().to(dev)
        rope_len = {"0": 0, "L-37": L - 37, "L": L}[rope_mode]
    q0, k0 = _pieces(buf.view, L, C, pc, ld).clone(), _pieces(buf.view[:, pc:], L, C, pc, ld).clone()
    v0 = buf.view[:, 2 * pc:].clone()
    pieces = (L, C, pc, L * ld)
    qv, kv = buf.view[:L, :pc], buf.view[:L, pc:2 * pc]
    if entry == "rmsnorm_rope":
        ops.rmsnorm_rope(qv, wq, rope, D, rope_len=rope_len, pieces=pieces)
        ops.rmsnorm_rope(kv, wk, rope, D, rope_len=rope_len, pieces=pieces)
    else:
        ops.qk_norm_rope(qv, kv, wq, wk, rope, D, rope_len=rope_len, pieces=pieces)
    torch.cuda.synchronize()
    tag = f"{entry} C{C} rope={rope_mode} pieces={split}"
    buf.check(tag)
    assert torch.equal(buf.view[:, 2 * pc:], v0), tag + ": v columns changed"
    for name, x0, w, off in (("q", q0, wq, 0), ("k", k0, wk, pc)):
        y, bound = _rr_ref(x0, w, rope, rope_len, D)
        assert_within(_pieces(buf.view[:, off:], L, C, pc, ld), y, bound, f"{tag} {name}", "rmsnorm_rope")


# ------------------------------------------------------------------------------------------------------------
# Ulysses kernels with P ranks emulated on one GPU
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,C", [(2, 256), (2, 1024), (4, 3072), (8, 1024), (8, 5120), (4, 5120)])
def test_sp_scatter_qkv_on_one_gpu(dev, P, C):
    """yb_sp_scatter_qkv: rank r normalises + rotates q, k of its Lp local tokens and stores q|k|v of head block p into
    peers[p][r]. Receive buffers [P(src), Lp, 3*Wh] are guarded; v must be bit-exact, q / k within _rr_ref of the fp64 formula
    on the GLOBAL token rows (rope rows and rope_len of the global sequence, cut per rank)."""
    from yume_b200 import _lib, ops
    D, Lp = 128, 67
    L = P * Lp
    Wh = C // P
    g = _gen("sc", P, C)
    qkv = _randn(g, L, 3 * C + 64, dev=dev).bfloat16()[:, 32:32 + 3 * C]
    wq, wk = (torch.rand(C, generator=g) + 0.5).to(dev), (torch.rand(C, generator=g) + 0.5).to(dev)
    ang = torch.rand(L, D // 2, generator=g, dtype=torch.float64) * 6.28
    rope = torch.stack([ang.cos(), ang.sin()], -1).float().contiguous().to(dev)
    rope_len = L - 37
    bufs = [guarded((P * Lp, 3 * Wh), torch.bfloat16, (8, 0)) for _ in range(P)]     # dense [P, Lp, 3*Wh] rows
    ptrs = [b.view.data_ptr() for b in bufs]
    for r in range(P):
        rl = max(0, min(Lp, rope_len - r * Lp))
        ops.sp_scatter_qkv(qkv[r * Lp:(r + 1) * Lp], wq, wk, rope[r * Lp:(r + 1) * Lp].contiguous(), rl, D, 1e-6, ptrs, r, Lp)
    torch.cuda.synchronize()
    yq, bq = _rr_ref(qkv[:, :C], wq, rope, rope_len, D)
    yk, bk = _rr_ref(qkv[:, C:2 * C], wk, rope, rope_len, D)
    for p in range(P):
        tag = f"sp_scatter_qkv P{P} C{C} receiver{p}"
        bufs[p].check(tag)
        rb = bufs[p].view
        cols = slice(p * Wh, (p + 1) * Wh)
        assert torch.equal(rb[:, 2 * Wh:], qkv[:, 2 * C:][:, cols]), tag + ": v not bit-exact"
        assert_within(rb[:, :Wh], yq[:, cols], bq[:, cols], tag + " q", "sp_scatter_qkv")
        assert_within(rb[:, Wh:2 * Wh], yk[:, cols], bk[:, cols], tag + " k", "sp_scatter_qkv")
    # widths without a template instance are rejected before any launch
    lib = _lib.load()
    arr = ops._ptr_array(ptrs)
    other = next(c for c in (3 * 128 * P, 2 * 128 * P) if c not in SC_WIDTHS)
    assert lib.yb_sp_scatter_qkv(qkv.data_ptr(), qkv.stride(0), wq.data_ptr(), wk.data_ptr(), None, 0, Lp, other, D,
                                 1e-6, arr, P, 0, Lp, None) == YB_ERR_SHAPE


@pytest.mark.parametrize("split", [1, 3])
@pytest.mark.parametrize("P,heads,Lp,pad", [(2, 2, 129, 0), (4, 8, 100, 7), (8, 8, 64, 37), (4, 24, 70, 5)])
def test_attention_sp_on_one_gpu(dev, P, heads, Lp, pad, split):
    """yb_attention_sp: rank r attends over all P*Lp gathered query rows for its heads/P heads and stores output row g into
    out_peers[g // Lp][r][g % Lp]. Keys past L_true = P*Lp - pad are absent (the padded sequence: Lk < Lq). split 3 forces the
    KV split (partials + peer-scatter combine). As in dit.py, q, k, v are column slices of each rank's gathered [P*Lp, 3*Wh]
    q|k|v buffer (row stride 3*Wh), k and v cut to L_true rows. Compared per element with the fp64 reference
    (attention_bound); the output receive buffers [P(src), Lp, heads/P*128] are guarded."""
    from yume_b200 import _lib, ops
    Hl = heads // P
    Lq, Lk = P * Lp, P * Lp - pad
    g = _gen("asp", P, heads, Lp, pad, split)
    scale = 1 / math.sqrt(128.0)
    q_all, k_all, v_all = (_randn(g, Lq, heads * 128, dev=dev).bfloat16() for _ in range(3))
    ref, bound = _attention_ref(q_all, k_all[:Lk], v_all[:Lk], heads, scale)
    Wh = Hl * 128
    bufs = [guarded((P * Lp, Hl * 128), torch.bfloat16, (128, 0)) for _ in range(P)]
    arr = ops._ptr_array([b.view.data_ptr() for b in bufs])
    lib = _lib.load()
    flags = (split & 7) << 4
    for r in range(P):
        cols = slice(r * Wh, (r + 1) * Wh)
        full = torch.cat([q_all[:, cols], k_all[:, cols], v_all[:, cols]], dim=1)          # rank r's gathered [P*Lp, 3*Wh]
        q, k, v = full[:, :Wh], full[:Lk, Wh:2 * Wh], full[:Lk, 2 * Wh:]
        ws, ws_bytes = ops._attention_ws(Lq, Lk, Hl, flags, q.device)
        rc = lib.yb_attention_sp(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), arr,
                                 Hl * 128, Lq, Lk, Hl, scale, P, r, Lp, flags, ops._ptr(ws), ws_bytes,
                                 ops._stream())
        assert rc == 0, rc
        torch.cuda.synchronize()
    for p in range(P):
        tag = f"attention_sp P{P} heads{heads} Lp{Lp} Lk{Lk} split{split} receiver{p}"
        bufs[p].check(tag)
        got = bufs[p].view.view(P, Lp, Hl * 128)
        for src in range(P):
            cols = slice(src * Hl * 128, (src + 1) * Hl * 128)
            rows = slice(p * Lp, (p + 1) * Lp)
            assert_within(got[src], ref[rows, cols], bound[rows, cols], f"{tag} src{src}", "attention_sp")


# ------------------------------------------------------------------------------------------------------------
# VAE glue
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("up", [(1, 1, 1), (1, 2, 2), (2, 2, 2)])
@pytest.mark.parametrize("pad", [0, 1])
def test_vae_pad_act(dev, pad, up, norm, silu):
    """yb_vae_pad_act: [GroupNorm from the stats] [SiLU] nearest upsample (first frame spatial only) and replicate padding, from
    a column window x (ldx > C) into a guarded [T(+2), H(+2), W(+2), Cp] buffer with zero channel padding C < Cp. Without norm
    and SiLU the pass is a copy: bit-exact. Otherwise: GroupNorm as one fp32 fma per element with a, b from fp64 stats
    (|a*x| + |b| carries <= 4*u32 relative, rsqrtf 2^-22), SiLU x/(1+__expf(-x)) with __expf relative error
    <= 2^-21*(2 + 1.16*|x|) (|silu'| <= 1.1) and the fast division 2 ulp, then bf16 rounding. Reference and bound are fp64
    values placed by the CPU stand-in's index logic (it maps each output voxel to its source voxel)."""
    from yume_b200 import ops
    g = _gen("pad", pad, up, norm, silu)
    Ts, Hs, Ws, C, Cp, G = 3, 5, 7, 64, 128, 32
    xs = (torch.randn(Ts * Hs * Ws, C + 64, generator=g) * 2 + 0.5).to(dev).bfloat16()
    x = xs[:, 32:32 + C]
    gamma, beta = _randn(g, C, dev=dev), _randn(g, C, dev=dev)
    stats = ops.gn_stats(x, G) if norm else None
    ft, fh, fw = up
    T, H, W = (1 + 2 * (Ts - 1) if ft == 2 else Ts), Hs * fh, Ws * fw
    shape = (T + 2 * pad, H + 2 * pad, W + 2 * pad, Cp)
    out = guarded(shape, torch.bfloat16, (2, 0))
    ops.vae_pad_act(x, (Ts, Hs, Ws), out.view, bool(pad), up, stats, gamma if norm else None, beta if norm else None, G, 1e-6,
                    silu)
    torch.cuda.synchronize()
    tag = f"vae_pad_act pad{pad} up{up} norm{int(norm)} silu{int(silu)}"
    out.check(tag)
    from helpers import torch_ops as T_
    xd = x.double().view(Ts, Hs, Ws, C)
    if norm:
        cnt = Ts * Hs * Ws * (C // G)
        st = stats.double()
        mean = st[:, 0] / cnt
        var = st[:, 1] / cnt - mean * mean
        a = torch.rsqrt(var + 1e-6).repeat_interleave(C // G) * gamma.double()
        b = beta.double() - mean.repeat_interleave(C // G) * a
        y = xd * a + b
        f32 = 4 * U32 * ((xd * a).abs() + b.abs()) + 2.0 ** -22 * (xd * a).abs()
    else:
        y, f32 = xd, torch.zeros_like(xd)
    if silu:
        sig = torch.sigmoid(y)
        f32 = 1.1 * f32 + (2.0 ** -21 * (2 + 1.16 * y.abs()) + 4 * U32) * (y * sig).abs() + 2 * U32 * (y * sig).abs()
        y = y * sig
    # source voxel of every output voxel, from the stand-in run on voxel numbers (exact in fp32 below 2^24)
    src = torch.arange(Ts * Hs * Ws, dtype=torch.float64, device=dev)[:, None].expand(-1, 8)
    where = torch.zeros(shape[:-1] + (8,), dtype=torch.float64, device=dev)
    T_.vae_pad_act(src, (Ts, Hs, Ws), where, bool(pad), up)
    where = where[..., 0].long()
    ref = torch.zeros(shape, dtype=torch.float64, device=dev)
    bnd = torch.zeros(shape, dtype=torch.float64, device=dev)
    ref[..., :C] = y.reshape(-1, C)[where]
    bnd[..., :C] = f32.reshape(-1, C)[where]
    if not (norm or silu):
        assert torch.equal(out.view.double(), ref), tag + ": copy path not bit-exact"
        record_exact("vae_pad_act_copy")
        return
    assert torch.equal(out.view[..., C:], torch.zeros_like(out.view[..., C:])), tag + ": channel padding not zero"
    assert_within(out.view[..., :C], ref[..., :C], bf16_out_bound(ref[..., :C], bnd[..., :C]), tag, "vae_pad_act")


@pytest.mark.parametrize("clamp", [None, (-1.0, 1.0)])
@pytest.mark.parametrize("N,Cn,ldx", [(1000, 3, 32), (777, 12, 16), (4096, 16, 64)])
def test_nhwc_to_nchw_f32(dev, N, Cn, ldx, clamp):
    """yb_nhwc_to_nchw_f32 / _clamp: channels-last [N, ldx] (ldx > Cn, the head conv output) -> [Cn, N], bit-exact."""
    from yume_b200 import ops
    g = _gen("nhwc", N, Cn, ldx, clamp)
    x = _randn(g, N, ldx, scale=1.5, dev=dev)
    out = guarded((Cn, N), torch.float32, (1, 0))
    ops.nhwc_to_nchw_f32(x, out.view, clamp)
    torch.cuda.synchronize()
    tag = f"nhwc_to_nchw N{N} Cn{Cn} ldx{ldx} clamp{clamp}"
    out.check(tag)
    want = x[:, :Cn].t()
    if clamp is not None:
        want = want.clamp(*clamp)
    assert torch.equal(out.view, want), tag
    record_exact("nhwc_to_nchw")


def _tile_plan(sizes, limit):
    """Output covered by tiles of the given sizes: sum(min(limit, s))."""
    return sum(min(limit, s) for s in sizes)


@pytest.mark.parametrize("nt", [1, 3])
@pytest.mark.parametrize("grid,th,tw,limit,extent", [
    ((1, 1), (24,), (40,), 0, 0),
    ((2, 3), (24, 24), (24, 24, 8), 16, 8),
    ((3, 2), (24, 24, 10), (32, 16), 18, 6),
    ((2, 3), (20, 6), (24, 24, 8), 12, 12),          # blend extent larger than the last row / column of tiles
])
def test_vae_assemble_tiles_is_the_reference_blend_sequence(dev, nt, grid, th, tw, limit, extent):
    """yb_vae_assemble_tiles against the CPU stand-in's in-place blend_v / blend_h / crop / cat / blend_t sequence (the
    reference's own order) run on the same f32 tiles on the device: bit-exact. Spatial grids 1x1, 2x3, 3x2 and 1 or 3
    temporal windows, tiles of unequal size with extents clamped by narrow edge tiles."""
    from yume_b200 import ops
    from helpers import torch_ops as T_
    g = _gen("asm", nt, grid, th, tw, limit, extent)
    Cc = 3
    ni, nj = grid
    tlen = [9] + [8] * (nt - 1) if nt > 1 else [9]
    t_blend, t_limit = 3, 5
    keep = [min(n, t_limit + (1 if i == 0 else 0)) for i, n in enumerate(tlen)] if nt > 1 else [tlen[0]]
    tf0 = [sum(keep[:i]) for i in range(nt)]
    tiles = [[[_randn(g, Cc, tlen[a] + (1 if a > 0 else 0), th[i], tw[j], dev=dev) for j in range(nj)] for i in range(ni)]
             for a in range(nt)]
    spatial = ni > 1 or nj > 1
    Ho = _tile_plan(th, limit) if spatial else th[0]
    Wo = _tile_plan(tw, limit) if spatial else tw[0]
    out = guarded((Cc, sum(keep), Ho, Wo), torch.float32, (1, 0))
    ops.vae_assemble_tiles(tiles, th, tw, tlen, tf0, out.view, limit, extent, t_limit, t_blend)
    torch.cuda.synchronize()
    tag = f"assemble_tiles nt{nt} grid{grid} th{th} tw{tw} limit{limit} extent{extent}"
    out.check(tag)
    want = torch.empty_like(out.view)
    T_.vae_assemble_tiles(tiles, th, tw, tlen, tf0, want, limit, extent, t_limit, t_blend)
    diff = (out.view != want)
    assert not bool(diff.any()), f"{tag}: {int(diff.sum())} voxels differ, first at {tuple(int(i) for i in diff.nonzero()[0])}"
    record_exact("assemble_tiles")
    if ni * nj > 1:     # an extent that would read a tile back inside its own blended region is refused before any launch
        from yume_b200._lib import YumeB200Error
        with pytest.raises(YumeB200Error, match="overlaps itself"):
            ops.vae_assemble_tiles(tiles, th, tw, tlen, tf0, out.view, limit, max(max(th), max(tw)), t_limit, t_blend)


@pytest.mark.parametrize("N,C,dist,mean,spread", [(1 << 20, 128, "normal", 1000.0, 16.0), (1_200_000, 64, "normal", -300.0, 2.0),
                                                  (1 << 20, 128, "lognormal", 0.0, 2.0)])
def test_gn_stats_large_n_mean_much_larger_than_spread(dev, N, C, dist, mean, spread):
    """yb_gn_stats over >= 1e6 rows whose group mean is far larger than the spread (bf16 values then sit on the grid of
    ulp(mean), and per-thread fp32 partials of fewer than 2^10 of them are exact: the recorded ratio is 0), plus one case
    (lognormal: randn * exp(spread * randn), magnitudes over ~2^16, zero mean) where the partials do round. Sums: fp32 partials
    of at most n_t voxels per thread, then fp64: |d sum| <= n_t*u32*sum|x|, |d sumsq| <= (n_t + 1)*u32*sum x^2 per group.
    n_t follows yb_gn_stats' launch (256/(C/8) voxels per block, at most 8 blocks per SM, grid-stride over the rest): a change
    of that launch policy must update n_t here, or the bound is wrong. The GroupNorm variance
    sumsq/n - mean^2 derived from the kernel's stats must then be within (d sumsq + 2|mean| d sum)/n of the fp64 variance, and
    — what GroupNorm needs from it — within 2^-9 relative (half a bf16 rounding of the normalised output)."""
    from yume_b200 import ops
    G = 32
    g = _gen("gn", N, C, dist, mean, spread)
    if dist == "normal":
        x = (torch.randn(N, C + 8, generator=g) * spread + mean).to(dev).bfloat16()[:, :C]
    else:
        x = (torch.randn(N, C + 8, generator=g) * torch.exp(spread * torch.randn(N, C + 8, generator=g)) + mean)
        x = x.to(dev).bfloat16()[:, :C]
    st = ops.gn_stats(x, G)
    xd = x.double().view(N, G, C // G)
    s, q = xd.sum((0, 2)), (xd * xd).sum((0, 2))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    vpb = 256 // (C // 8)                                     # the launch of yb_gn_stats (vae_elementwise.cu)
    blocks = min((N + vpb - 1) // vpb, sms * 8)
    n_t = -(-N // (blocks * vpb))
    ds = n_t * U32 * xd.abs().sum((0, 2))
    dq = (n_t + 1) * U32 * q
    tag = f"gn_stats N{N} C{C} {dist} mean{mean} spread{spread}"
    assert_within(st[:, 0], s, ds, tag + " sum", "gn_stats")
    assert_within(st[:, 1], q, dq, tag + " sumsq", "gn_stats")
    n = N * (C // G)
    var_ref = q / n - (s / n) ** 2
    var = st[:, 1] / n - (st[:, 0] / n) ** 2
    assert_within(var, var_ref, (dq + 2 * (s / n).abs() * ds) / n, tag + " variance (derived)", "gn_stats")
    assert_within(var, var_ref, 2.0 ** -9 * var_ref, tag + " variance (GroupNorm need)", "gn_stats")


@pytest.mark.parametrize("T,H,W,ci,co", [(3, 8, 8, 64, 64), (2, 6, 10, 128, 128), (1, 18, 32, 128, 96), (9, 4, 4, 64, 32),
                                         (2, 3, 200, 64, 128), (3, 9, 17, 128, 384)])
@pytest.mark.parametrize("fuse_w,cta_pair", [(1, 0), (2, 0), (1, 1)])
def test_conv3d_causal_per_element(dev, T, H, W, ci, co, fuse_w, cta_pair):
    """The replicate-padded causal conv shapes of test_gpu_parity under the per-element bound of the GEMM (K = 27*ci, F from
    |x| * |w|), RES_BF16 into a guarded NaN-poisoned window with ldo > Cout, and F32 out."""
    from yume_b200 import ops
    g = _gen("conv", T, H, W, ci, co, fuse_w, cta_pair)
    x = _randn(g, T * H * W, ci, dev=dev).bfloat16()
    wt = _randn(g, co, ci, 3, 3, 3, scale=1 / math.sqrt(27 * ci), dev=dev).bfloat16()
    b = _randn(g, co, dev=dev)
    res = _randn(g, T * H * W, co, dev=dev).bfloat16()
    xpad = torch.empty(T + 2, H + 2, W + 2, ci, device=dev, dtype=torch.bfloat16)
    ops.vae_pad_act(x, (T, H, W), xpad, True)
    wk = wt.permute(0, 2, 3, 4, 1).reshape(co, 27 * ci).contiguous()
    xp = xpad.double().permute(3, 0, 1, 2)[None]
    acc = F.conv3d(xp, wt.double())[0].permute(1, 2, 3, 0).reshape(T * H * W, co)
    Fb = 2.0 * 27 * ci * U32 * F.conv3d(xp.abs(), wt.double().abs())[0].permute(1, 2, 3, 0).reshape(T * H * W, co)
    tag = f"conv3d T{T} H{H} W{W} ci{ci} co{co} fuse_w{fuse_w} cta_pair{cta_pair}"
    out = guarded((T * H * W, co), torch.bfloat16, (128, 64))
    ops.conv3d_causal(xpad, wk, b, out.view, T, H, W, ops.YB_EPI_RES_BF16, res, fuse_w=fuse_w, cta_pair=cta_pair)
    torch.cuda.synchronize()
    out.check(tag + " RES_BF16")
    ref = acc + b.double() + res.double()
    f32 = Fb + 4 * U32 * (acc.abs() + b.double().abs() + res.double().abs())
    assert_within(out.view, ref, bf16_out_bound(ref, f32), tag + " RES_BF16", "conv3d")
    o32 = guarded((T * H * W, co), torch.float32, (128, 32))
    ops.conv3d_causal(xpad, wk, None, o32.view, T, H, W, ops.YB_EPI_F32, fuse_w=fuse_w, cta_pair=cta_pair)
    torch.cuda.synchronize()
    o32.check(tag + " F32")
    assert_within(o32.view, acc, Fb + 4 * U32 * acc.abs(), tag + " F32", "conv3d")


# ------------------------------------------------------------------------------------------------------------
# entry point -> tests that exercise it (tests/test_kernel_contract_cpu.py: every C-ABI entry point is in a COVERS table)
# ------------------------------------------------------------------------------------------------------------
COVERS = {
    "yb_gemm_bf16": ["test_gemm_every_epilogue_per_element"],
    "yb_attention_ex": ["test_attention_tails_scales_variants", "test_attention_production_heads",
                        "test_attention_split_and_accumulate"],
    "yb_ln_modulate": ["test_ln_modulate_every_instance"],
    "yb_rmsnorm_rope_pieces": ["test_rmsnorm_rope_every_instance"],
    "yb_qk_norm_rope": ["test_rmsnorm_rope_every_instance"],
    "yb_sp_scatter_qkv": ["test_sp_scatter_qkv_on_one_gpu"],
    "yb_attention_sp": ["test_attention_sp_on_one_gpu"],
    "yb_vae_pad_act": ["test_vae_pad_act", "test_conv3d_causal_per_element"],
    "yb_nhwc_to_nchw_f32": ["test_nhwc_to_nchw_f32"],
    "yb_nhwc_to_nchw_f32_clamp": ["test_nhwc_to_nchw_f32"],
    "yb_vae_assemble_tiles": ["test_vae_assemble_tiles_is_the_reference_blend_sequence"],
    "yb_gn_stats": ["test_gn_stats_large_n_mean_much_larger_than_spread", "test_vae_pad_act"],
    "yb_conv3d_causal": ["test_conv3d_causal_per_element"],
}
