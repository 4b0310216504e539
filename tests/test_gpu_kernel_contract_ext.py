"""Per-element kernel contract, part two (`-m gpu`): the production paths tests/test_gpu_kernel_contract.py does not reach —
the Ulysses GEMM layouts on the kernel production runs (1-CTA) and the SM-pair tail split-K, the fused QKV GEMM + all-to-all
chain, the Wan VAE conv modes (zero padding by TMA out-of-bounds fill, time_conv's frame interleave, the strided Resample
convs), the Wan VAE glue kernels, the fp32 DiT ops, and the two entry points ops.py does not call (yb_rmsnorm_rope,
yb_attention).

Same rules as part one, whose machinery this file imports: the fp64 reference is computed on the device from the same bf16 / f32
inputs the kernel saw; each bound is derived in the test's docstring from the kernel's arithmetic; outputs are NaN-poisoned
views inside guard-banded buffers (in-place outputs are seeded with finite data); every case draws its data from _gen(<its
parameters>). Index-only kernels are compared bit for bit. The worst |err| / bound per family is merged into the
YB_CONTRACT_REPORT file (max per family) at the end of the module.

The build compiles without fast-math (yume_b200/build.py), so sqrtf, `/` and 1/x are IEEE-rounded; __expf is the only
approximate transcendental below and its error is bounded explicitly. u16 = 2^-8, u32 = 2^-24.
"""
import json
import math
import os

import pytest
import torch
import torch.nn.functional as F

import test_gpu_kernel_contract as KC
from test_gpu_kernel_contract import (U32, Guarded, _gen, _randn, _rr_ref, assert_within, bf16_out_bound, gemm_bounds, guarded,
                                      record_exact)

pytestmark = pytest.mark.gpu

YB_ERR_SHAPE, YB_ERR_ALIGNMENT = -2, -3     # include/yume_b200.h

# yb_vae_rms_act width -> the YB_RMS_LAUNCH(NCH, G) instance it reaches (tests/test_kernel_contract_cpu.py checks this
# table against the instances and the width rule in vae_elementwise.cu)
RMS_WIDTHS = ((48, 64), (96, 128), (256, 256), (384, 384), (1024, 1024))


def _exp_err(x):
    """Relative error of __expf(x) (ex2.approx of x*log2(e) with the product rounded): <= 2^-21 * (2 + 1.16*|x|)."""
    return 2.0 ** -21 * (2 + 1.16 * x.abs())


def _silu_bound(y, f32):
    """SiLU y / (1 + __expf(-y)) of an fp32 value within f32 of y: |silu'| <= 1.1 carries f32 through, __expf's error
    moves 1 + e by at most its own relative error, the add and the IEEE division round once each."""
    s = y * torch.sigmoid(y)
    return 1.1 * f32 + (_exp_err(y) + 4 * U32) * s.abs() + 2 * U32 * s.abs()


def _chunked(P, rows, cols, gap, dtype, fill=None, gap_value=None):
    """P chunks of [rows, cols] in one backing buffer, `gap` guard rows before, between and after the chunks (chunk stride
    (rows + gap) * cols elements). Returns a Guarded whose .view is the strided [P, rows, cols] chunk view. Chunks are NaN or
    `fill`; the gap rows hold the guard pattern, or `gap_value` (e.g. NaN: memory a wrong extent would read)."""
    itype, pattern = KC._GUARD_BITS[dtype]
    n = P * (rows + gap) + gap
    backing = torch.full((n, cols), pattern, dtype=itype, device="cuda").view(dtype)
    if gap_value is not None:
        backing.fill_(gap_value)
    view = backing[gap:gap + P * (rows + gap)].view(P, rows + gap, cols)[:, :rows]
    if fill is None:
        view.fill_(float("nan"))
    else:
        view.copy_(fill)
    mask = torch.ones(n, cols, dtype=torch.bool, device="cuda")
    mask[gap:gap + P * (rows + gap)].view(P, rows + gap, cols)[:, :rows] = False
    return Guarded(view, backing, mask)


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
    if KC.WORST:
        print("[contract] worst |err|/bound per family: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(KC.WORST.items())))
        path = os.environ.get("YB_CONTRACT_REPORT")
        if path:
            data = {"worst_ratio": {}}
            if os.path.exists(path):
                with open(path) as f:
                    data = json.load(f)
            worst = data.setdefault("worst_ratio", {})
            for k, v in KC.WORST.items():
                worst[k] = max(worst.get(k, 0.0), v)
            if torch.cuda.is_available():
                data["device"] = torch.cuda.get_device_name(0)
            with open(path, "w") as f:
                json.dump(data, f, indent=1, sort_keys=True)


# ------------------------------------------------------------------------------------------------------------
# GEMM: Ulysses layouts and tail split-K
# ------------------------------------------------------------------------------------------------------------
KERNELS = [(0, 0), (1, 128), (1, 256), (2, 0), (2, 128), (2, 256)]     # (cta_pair, block_n); 0 = automatic


@pytest.mark.parametrize("Lp", [67, 129, 300])
@pytest.mark.parametrize("W3,P", [(384, 4), (1152, 2), (1920, 2), (2304, 2)])
@pytest.mark.parametrize("cta_pair,block_n", KERNELS)
def test_gemm_n_split_layout(dev, cta_pair, block_n, W3, P, Lp):
    """n_split (the nccl transport's QKV GEMM, dit.py): output column block j of width W3 goes to chunk j of a [P, Lp, W3]
    buffer whose chunks are split_stride > Lp*W3 apart with guard rows between them. W3 = 1152 (5B, 8 ranks) and 1920 (14B)
    are not multiples of the 256-column tile, so some tiles straddle two chunks. Bound: bf16_out_bound of the fp64 GEMM + bias
    with F = gemm_bounds and one fp32 bias add (4*u32*(|acc| + |bias|)), mapped through the layout."""
    from yume_b200 import ops
    K = 264
    N = P * W3
    g = _gen("nsplit", cta_pair, block_n, W3, P, Lp)
    A = _randn(g, Lp, K, dev=dev).bfloat16()
    B = _randn(g, N, K, scale=1 / math.sqrt(K), dev=dev).bfloat16()
    bias = _randn(g, N, dev=dev)
    out = _chunked(P, Lp, W3, 8, torch.bfloat16)
    stride = (Lp + 8) * W3
    ops.gemm(A, B, bias, out.view[0], ops.YB_EPI_BF16, n_split=W3, split_stride=stride, shape=(Lp, K), cta_pair=cta_pair,
             block_n=block_n)
    torch.cuda.synchronize()
    tag = f"gemm n_split W3{W3} P{P} Lp{Lp} cta{cta_pair} bn{block_n}"
    out.check(tag)
    acc = A.double() @ B.double().t()
    ref = acc + bias.double()
    bound = bf16_out_bound(ref, gemm_bounds(A, B, K) + 4 * U32 * (acc.abs() + bias.double().abs()))
    got = out.view.permute(1, 0, 2).reshape(Lp, N)
    assert_within(got, ref, bound, tag, "gemm_split_layout")


def _epilogue_cases(g, A, B, M, N, K, tag, family, out_pad, **kw):
    """Every epilogue of yb_gemm_bf16 for logical operands A [M, K] (bf16, any layout the kwargs describe) and B [N, K],
    with the bounds of test_gpu_kernel_contract.test_gemm_every_epilogue_per_element; GATE_RES with a [U, 6, N] gate table
    row per token (tok_idx, the o-projection) and without gate."""
    from yume_b200 import ops
    Al = kw.pop("logical")
    bias = _randn(g, N, dev="cuda")
    acc = Al.double() @ B.double().t()
    Fb = gemm_bounds(Al, B, K)
    accb = acc + bias.double()
    f32 = Fb + 4 * U32 * (acc.abs() + bias.double().abs())

    def run(epi, dtype, fill=None, **extra):
        out = guarded((M, N), dtype, out_pad, fill=fill)
        ops.gemm(A, B, extra.pop("bias", bias), out.view, epi, **kw, **extra)
        torch.cuda.synchronize()
        return out

    o = run(ops.YB_EPI_BF16, torch.bfloat16)
    o.check(tag + " BF16")
    assert_within(o.view, accb, bf16_out_bound(accb, f32), tag + " BF16", family)
    for epi, name in ((ops.YB_EPI_GELU_BF16, "GELU_TANH"), (ops.YB_EPI_GELU_ERF_BF16, "GELU_ERF")):
        o = run(epi, torch.bfloat16)
        o.check(tag + " " + name)
        ref = F.gelu(accb, approximate="tanh") if name == "GELU_TANH" else F.gelu(accb)
        ev = (2.0 ** -12 if name == "GELU_TANH" else 2.0 ** -20) * accb.abs()
        assert_within(o.view, ref, bf16_out_bound(ref, 1.13 * f32 + ev + 4 * U32 * accb.abs()), tag + " " + name, family)
    o = run(ops.YB_EPI_F32, torch.float32, bias=None)
    o.check(tag + " F32")
    assert_within(o.view, acc, Fb + 4 * U32 * acc.abs(), tag + " F32", family)
    res = _randn(g, M, N + 16, dev="cuda").bfloat16()[:, 8:8 + N]
    o = run(ops.YB_EPI_RES_BF16, torch.bfloat16, res=res)
    o.check(tag + " RES_BF16")
    ref = accb + res.double()
    assert_within(o.view, ref, bf16_out_bound(ref, f32 + 4 * U32 * res.double().abs()), tag + " RES_BF16", family)
    gate6 = _randn(g, 3, 6, N, dev="cuda")
    tok = torch.randint(0, 3, (M,), generator=g).to("cuda", torch.int32)
    for gated in (True, False):
        x0 = _randn(g, M, N, dev="cuda")
        extra = dict(gate=gate6[:, 2], tok_idx=tok) if gated else {}
        o = run(ops.YB_EPI_GATE_RES, torch.float32, fill=x0, **extra)
        o.check(tag + f" GATE_RES gate={gated}")
        gt = gate6[tok.long(), 2].double() if gated else torch.ones_like(acc)
        ref = x0.double() + accb * gt
        bound = gt.abs() * f32 + 4 * U32 * (x0.double().abs() + (gt * accb).abs())
        assert_within(o.view, ref, bound, tag + f" GATE_RES gate={gated}", family)


@pytest.mark.parametrize("P", [2, 4, 8])
@pytest.mark.parametrize("a_split", [128, 384, 640])
@pytest.mark.parametrize("cta_pair", [0, 1, 2])
def test_gemm_a_split_layout_every_epilogue(dev, cta_pair, a_split, P):
    """a_split (every transport's o-projection, dit.py, and its GATE_RES + gate + tok_idx epilogue): A is the [P, Lp, a_split]
    buffer the all-to-all delivers, logical column k = element k % a_split of chunk k // a_split. The chunks are
    a_split_stride > Lp*a_split apart and the rows between and after them hold NaN: a tensor map with a wrong chunk stride or
    base reads NaN into the result instead of silently reading valid memory. (A wrong row extent would not show here: A rows
    past M only reach accumulator rows >= M, which are never stored, and no 64-wide K block crosses a chunk since
    a_split % 64 == 0.) Every epilogue, bounds as in part one."""
    Lp, N = 129, 256
    K = P * a_split
    g = _gen("asplit", cta_pair, a_split, P)
    chunks = _randn(g, P, Lp, a_split, dev=dev).bfloat16()
    a = _chunked(P, Lp, a_split, 8, torch.bfloat16, fill=chunks, gap_value=float("nan"))
    B = _randn(g, N, K, scale=1 / math.sqrt(K), dev=dev).bfloat16()
    logical = chunks.permute(1, 0, 2).reshape(Lp, K)
    tag = f"gemm a_split{a_split} P{P} cta{cta_pair}"
    _epilogue_cases(g, a.view[0], B, Lp, N, K, tag, "gemm_split_layout", (64, 32), logical=logical, a_split=a_split,
                    a_split_stride=(Lp + 8) * a_split, shape=(Lp, K), cta_pair=cta_pair)


@pytest.mark.parametrize("split_k", [0, 2, 3, 12])
@pytest.mark.parametrize("gated", [True, False])
def test_gemm_pair_tail_split_k(dev, gated, split_k):
    """SM-pair GATE_RES launch with the last wave's tiles cut into K segments (fp32 partials in the workspace, then
    gemm_splitk_combine_kernel adds them and applies the epilogue). The [M, N] shape leaves the last wave partly empty on an
    H100, so yb_gemm_workspace_bytes > 0 for the forced splits. Bound: the GATE_RES bound of part one with the K term widened
    by the segment count ns (the combine adds ns fp32 partials: ns more roundings of a partial sum, each <= u32*(|A||B|^T);
    split_k = 0 lets the planner choose, so ns is taken at its maximum, 12):
      |gate| * (F + (ns + 4)*u32*(|A||B|^T + |bias|)) + 4*u32*(|x0| + |gate*acc|)
    The residual stream is a guarded window: the rows and columns around it must keep their bits."""
    from yume_b200 import _lib, ops
    M, N, K = 300, 3072, 3072
    g = _gen("splitk", gated, split_k)
    A = _randn(g, M, K, dev=dev).bfloat16()
    B = _randn(g, N, K, scale=1 / math.sqrt(K), dev=dev).bfloat16()
    bias = _randn(g, N, dev=dev)
    ws = _lib.load().yb_gemm_workspace_bytes(M, N, K, ops.YB_EPI_GATE_RES, 2, split_k)
    if split_k > 1:
        assert ws > 0, f"split_k={split_k} does not split this launch"
    ns = split_k if split_k > 1 else 12
    gate6 = _randn(g, 3, 6, N, dev=dev)
    tok = torch.randint(0, 3, (M,), generator=g).to(dev, torch.int32)
    x0 = _randn(g, M, N, dev=dev)
    out = guarded((M, N), torch.float32, (64, 32), fill=x0)
    extra = dict(gate=gate6[:, 2], tok_idx=tok) if gated else {}
    ops.gemm(A, B, bias, out.view, ops.YB_EPI_GATE_RES, cta_pair=2, split_k=split_k, **extra)
    torch.cuda.synchronize()
    tag = f"gemm pair GATE_RES split_k{split_k} gate={gated} ws{ws}"
    out.check(tag)
    acc = A.double() @ B.double().t()
    accb = acc + bias.double()
    gt = gate6[tok.long(), 2].double() if gated else torch.ones_like(acc)
    ab = A.double().abs() @ B.double().abs().t()
    bound = gt.abs() * (gemm_bounds(A, B, K) + (ns + 4) * U32 * (ab + bias.double().abs())) + \
        4 * U32 * (x0.double().abs() + (gt * accb).abs())
    assert_within(out.view, x0.double() + accb * gt, bound, tag, "gemm_splitk")


# ------------------------------------------------------------------------------------------------------------
# fused QKV GEMM + all-to-all (the p2p_gemm transport), P ranks emulated on one GPU
# ------------------------------------------------------------------------------------------------------------
def _post_norm_ref(x, S, C, w, rope, rope_len, D, eps=1e-6):
    """fp64 x * rstd * w + RoPE with rstd = 1/sqrt(S/C + eps) from the GIVEN fp32 sums S (inputs here, so no sum term).
    The kernel: rsqrtf(S/C + eps) (division and add: 2 roundings, so rstd carries u32 relative; rsqrtf 2^-22), then _rr_ref's
    per-pair arithmetic (x*rstd*w: 2 roundings; rotation: 3): f32 = (u32 + 2^-22 + 4*u32) * (|a*c| + |b*s|)."""
    L, Wc = x.shape
    rstd = torch.rsqrt(S.double()[:, None] / C + eps)
    n = x.double() * rstd * w.double()
    y, mag = n.clone(), n.abs()
    r = min(rope_len, L)
    v = n[:r].view(r, Wc // D, D // 2, 2)
    cs = rope[:r].double()[:, None]
    c, s = cs[..., 0], cs[..., 1]
    y[:r] = torch.stack([v[..., 0] * c - v[..., 1] * s, v[..., 0] * s + v[..., 1] * c], -1).reshape(r, Wc)
    mag[:r] = torch.stack([(v[..., 0] * c).abs() + (v[..., 1] * s).abs(), (v[..., 0] * s).abs() + (v[..., 1] * c).abs()],
                          -1).reshape(r, Wc)
    return y, bf16_out_bound(y, (U32 + 2.0 ** -22 + 4 * U32) * mag)


def sumsq_bound(xsq, n):
    """fp32 sum of n non-negative terms in ANY order (per-lane runs, shuffles, atomics across tiles), each square rounded:
    |err| <= n * u32 * sum(x^2) (first order; (n - 1) for the sum plus 1 for the squares)."""
    return n * U32 * xsq


@pytest.mark.parametrize("P,C,Lp,Lp_rows", [(2, 1024, 129, 129), (4, 1024, 67, 67), (8, 1024, 67, 67), (2, 3072, 100, 100),
                                            (8, 3072, 67, 67), (4, 5120, 67, 67), (8, 5120, 40, 40), (4, 1024, 67, 50)])
def test_gemm_sp_qkv_chain_on_one_gpu(dev, P, C, Lp, Lp_rows):
    """yb_gemm_sp_qkv -> yb_sp_bcast_sums -> yb_sp_post_norm_rope, each stage against its own inputs. Rank r projects its
    Lp_rows local tokens (q|k|v of all heads) and stores head block p into receiver p's guarded [P(src), Lp, 3*Wh] buffer,
    accumulating each token's [sum q^2, sum k^2] of the bf16-rounded columns into `local`; yb_sp_bcast_sums copies those into
    slot r of every receiver's guarded [P*Lp, 2] table and zeroes `local`. Checked on a snapshot taken before the norm:
      q|k|v columns   bf16_out_bound of the fp64 GEMM (F = gemm_bounds + one bias add)
      table rows      the fp64 sum of squares of the RECEIVED bf16 row (all receivers' q / k columns), sumsq_bound(C);
                      every receiver's table identical; `local` zero again
    Then yb_sp_post_norm_rope on the snapshot against _post_norm_ref (rstd from the snapshot's f32 sums); v bit-exact.
    Lp_rows < Lp: the padding rows of every source block are never written (stay NaN)."""
    from yume_b200 import ops
    D, K = 128, 1024
    Wh, L = C // P, P * Lp
    g = _gen("spqkv", P, C, Lp, Lp_rows)
    h = _randn(g, L, K, dev=dev).bfloat16()
    w = _randn(g, 3 * C, K, scale=1 / math.sqrt(K), dev=dev).bfloat16()
    bias = _randn(g, 3 * C, dev=dev)
    nq, nk = (torch.rand(C, generator=g) + 0.5).to(dev), (torch.rand(C, generator=g) + 0.5).to(dev)
    ang = torch.rand(L, D // 2, generator=g, dtype=torch.float64) * 6.28
    rope = torch.stack([ang.cos(), ang.sin()], -1).float().contiguous().to(dev)
    rope_len = L - 37
    bufs = [guarded((P * Lp, 3 * Wh), torch.bfloat16, (8, 0)) for _ in range(P)]
    tables = [guarded((P * Lp, 2), torch.float32, (4, 0)) for _ in range(P)]
    local = guarded((Lp, 2), torch.float32, (4, 0), fill=torch.zeros(Lp, 2))
    for r in range(P):
        ops.gemm_sp_qkv(h[r * Lp:r * Lp + Lp_rows], w, bias, [b.view.data_ptr() for b in bufs], r, Lp, local.view)
        ops.sp_bcast_sums(local.view, [t.view.data_ptr() for t in tables], r, Lp)
    torch.cuda.synchronize()
    tag = f"gemm_sp_qkv P{P} C{C} Lp{Lp} rows{Lp_rows}"
    local.check(tag + " local")
    assert float(local.view.abs().max()) == 0.0, tag + ": local sums not cleared"
    valid = (torch.arange(L, device=dev) % Lp) < Lp_rows
    snap = [b.view.clone() for b in bufs]
    for p in range(P):
        bufs[p].check(tag + f" receiver{p}", allow_nan=Lp_rows < Lp)
        tables[p].check(tag + f" table{p}")
        assert bool(torch.isnan(snap[p][~valid]).all()), tag + ": a padding row was written"
        assert torch.equal(tables[p].view, tables[0].view), tag + f": table {p} differs from table 0"
    hv = h[valid]
    acc = hv.double() @ w.double().t()
    ref = acc + bias.double()
    bound = bf16_out_bound(ref, gemm_bounds(hv, w, K) + 4 * U32 * (acc.abs() + bias.double().abs()))
    for p in range(P):
        for part in range(3):
            cols = slice(part * C + p * Wh, part * C + (p + 1) * Wh)
            assert_within(snap[p][valid][:, part * Wh:(part + 1) * Wh], ref[:, cols], bound[:, cols],
                          f"{tag} receiver{p} part{part}", "gemm_sp_qkv")
    S = tables[0].view[valid].double()
    for part, name in ((0, "q"), (1, "k")):
        xsq = torch.cat([snap[p][valid][:, part * Wh:(part + 1) * Wh] for p in range(P)], 1).double().pow(2).sum(1)
        assert_within(S[:, part], xsq, sumsq_bound(xsq, C), f"{tag} sum {name}^2", "gemm_sp_qkv")
    for p in range(P):
        ops.sp_post_norm_rope(bufs[p].view, tables[p].view, nq[p * Wh:(p + 1) * Wh], nk[p * Wh:(p + 1) * Wh], rope, rope_len, L,
                              Wh, C, D, 1e-6)
    torch.cuda.synchronize()
    rot = (torch.nonzero(valid).flatten() < rope_len)[:, None]        # buffer row = global token row: rotated below rope_len
    for p in range(P):
        t2 = f"sp_post_norm_rope P{P} C{C} Lp{Lp} rows{Lp_rows} receiver{p}"
        bufs[p].check(t2, allow_nan=Lp_rows < Lp)
        got = bufs[p].view
        assert torch.equal(got[valid][:, 2 * Wh:], snap[p][valid][:, 2 * Wh:]), t2 + ": v not bit-exact"
        for part, wt in ((0, nq), (1, nk)):
            args = (snap[p][valid][:, part * Wh:(part + 1) * Wh], tables[p].view[valid][:, part].float(), C,
                    wt[p * Wh:(p + 1) * Wh], rope[valid])
            yr, br = _post_norm_ref(*args, int(valid.sum()), D)
            y0, b0 = _post_norm_ref(*args, 0, D)
            assert_within(got[valid][:, part * Wh:(part + 1) * Wh], torch.where(rot, yr, y0), torch.where(rot, br, b0),
                          f"{t2} part{part}", "sp_post_norm_rope")


# ------------------------------------------------------------------------------------------------------------
# Wan VAE conv modes (yb_conv3d_causal with oob_zero_pad)
# ------------------------------------------------------------------------------------------------------------
def _conv_ref(x, wt, taps, stride_t=1, stride_hw=1):
    """fp64 conv of x bf16 [T, H, W, Cp] with wt [co, Cp, kt, kh, kw] on the EXPLICITLY zero-padded input (unit stride: kt-1
    frames in front, kh//2 / kw//2 around; stride_hw 2: one zero row / column behind, vae2_2.py's ZeroPad2d((0,1,0,1));
    stride_t 2: no padding). Returns (acc [To*Ho*Wo, co], F = 2*K*u32*conv(|x|, |w|) with K = kt*kh*kw*Cp, (To, Ho, Wo))."""
    kt, kh, kw = taps
    xd = x.double().permute(3, 0, 1, 2)[None]
    if stride_hw > 1:
        xd = F.pad(xd, (0, 1, 0, 1, 0, 0))
    elif stride_t == 1:
        xd = F.pad(xd, (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0))
    wd = wt.double()
    st = (stride_t, stride_hw, stride_hw)
    acc = F.conv3d(xd, wd, stride=st)[0]
    K = kt * kh * kw * x.shape[-1]
    Fb = 2.0 * K * U32 * F.conv3d(xd.abs(), wd.abs(), stride=st)[0]
    dims = tuple(acc.shape[1:])
    co = wt.shape[0]
    return acc.permute(1, 2, 3, 0).reshape(-1, co), Fb.permute(1, 2, 3, 0).reshape(-1, co), dims


def _conv_operands(g, T, H, W, Cp, co, taps, dev):
    kt, kh, kw = taps
    x = _randn(g, T, H, W, Cp, dev=dev).bfloat16()
    wt = _randn(g, co, Cp, kt, kh, kw, scale=1 / math.sqrt(kt * kh * kw * Cp), dev=dev).bfloat16()
    wk = wt.permute(0, 2, 3, 4, 1).reshape(co, kt * kh * kw * Cp).contiguous()
    return x, wt, wk


CONV_WAN_SHAPES = [(3, 9, 17, 64, 96), (1, 8, 40, 128, 128), (2, 5, 130, 64, 256), (4, 3, 7, 192, 64), (2, 4, 12, 1024, 128)]


@pytest.mark.parametrize("T,H,W,Cp,co", CONV_WAN_SHAPES)
@pytest.mark.parametrize("taps", [(3, 3, 3), (1, 3, 3), (3, 1, 1)])
@pytest.mark.parametrize("fuse_w,cta_pair", [(1, 0), (2, 0), (1, 1)])
def test_conv3d_wan_zero_pad_per_element(dev, taps, T, H, W, Cp, co, fuse_w, cta_pair):
    """The Wan VAE conv forms (3x3x3, Conv2d 3x3 = (1,3,3), time_conv = (3,1,1)) with the causal zero padding taken from
    TMA out-of-bounds fill on the unpadded activation, kw-fused and un-fused tiles and the SM-pair kernel, H / W not multiples
    of the tile, T = 1, and Cp up to 1024 (the Wan2.2 decoder width: K = 27 648). Epilogues BF16 and RES_BF16 into guarded
    windows with ldo > Cout, F32 likewise. Bound: the GEMM's, F = 2*K*u32*conv(|x|,|w|) (_conv_ref), plus one fp32 add per
    epilogue operand (4*u32*(|acc| + |bias| + |res|)), then bf16 rounding for the bf16 outputs."""
    from yume_b200 import ops
    g = _gen("convwan", taps, T, H, W, Cp, co, fuse_w, cta_pair)
    x, wt, wk = _conv_operands(g, T, H, W, Cp, co, taps, dev)
    b = _randn(g, co, dev=dev)
    acc, Fb, _ = _conv_ref(x, wt, taps)
    M = T * H * W
    res = _randn(g, M, co + 16, dev=dev).bfloat16()[:, 8:8 + co]
    bd, rd = b.double(), res.double()
    tag = f"conv3d_wan taps{taps} T{T} H{H} W{W} Cp{Cp} co{co} fuse_w{fuse_w} cta_pair{cta_pair}"
    kw = dict(taps=taps, oob_zero_pad=True, fuse_w=fuse_w, cta_pair=cta_pair)
    for epi, name in ((ops.YB_EPI_BF16, "BF16"), (ops.YB_EPI_RES_BF16, "RES_BF16")):
        out = guarded((M, co), torch.bfloat16, (128, 64))
        ops.conv3d_causal(x, wk, b, out.view, T, H, W, epi, res if name == "RES_BF16" else None, **kw)
        torch.cuda.synchronize()
        out.check(tag + " " + name)
        ref = acc + bd + (rd if name == "RES_BF16" else 0)
        f32 = Fb + 4 * U32 * (acc.abs() + bd.abs() + (rd.abs() if name == "RES_BF16" else 0))
        assert_within(out.view, ref, bf16_out_bound(ref, f32), tag + " " + name, "conv3d_wan")
    o32 = guarded((M, co), torch.float32, (128, 32))
    ops.conv3d_causal(x, wk, None, o32.view, T, H, W, ops.YB_EPI_F32, **kw)
    torch.cuda.synchronize()
    o32.check(tag + " F32")
    assert_within(o32.view, acc, Fb + 4 * U32 * acc.abs(), tag + " F32", "conv3d_wan")


@pytest.mark.parametrize("T,H,W,C", [(3, 6, 10, 128), (5, 4, 33, 64)])
def test_conv3d_wan_time_conv_interleave(dev, T, H, W, C):
    """time_conv as vae22.py runs it: frame 0 of x is copied to output frame 0, then the two channel groups of the (3,1,1)
    conv over frames 1.. write output frames 1 + 2(t-1) + g (out_t_mul = 2, out_t_add = 1 + g) of one NaN-poisoned
    [(2T-1)*H*W, C] buffer. After the first launch the second group's frames must still be NaN and the guard intact; after
    both every frame is within the conv bound of its group (BF16 epilogue)."""
    from yume_b200 import ops
    g = _gen("timeconv", T, H, W, C)
    HW = H * W
    x = _randn(g, T * HW, C, dev=dev).bfloat16()
    xin = x[HW:].view(T - 1, H, W, C)
    ws = [_conv_operands(g, 1, 1, 1, C, C, (3, 1, 1), dev)[1:] for _ in range(2)]
    bs = [_randn(g, C, dev=dev) for _ in range(2)]
    out = guarded(((2 * T - 1) * HW, C), torch.bfloat16, (64, 0))
    out.view[:HW].copy_(x[:HW])
    frames = out.view.view(2 * T - 1, HW, C)
    tag = f"time_conv T{T} H{H} W{W} C{C}"
    for grp in (0, 1):
        ops.conv3d_causal(xin, ws[grp][1], bs[grp], out.view, T - 1, H, W, ops.YB_EPI_BF16, taps=(3, 1, 1), oob_zero_pad=True,
                          out_t_mul=2, out_t_add=1 + grp)
        torch.cuda.synchronize()
        if grp == 0:
            out.check(tag + " after group 0", allow_nan=True)
            assert bool(torch.isnan(frames[2::2]).all()), tag + ": group 0 wrote into group 1's frames"
            assert not bool(torch.isnan(frames[1::2]).any()), tag + ": group 0 left frames unwritten"
    out.check(tag)
    assert torch.equal(frames[0], x[:HW]), tag + ": frame 0 changed"
    for grp in (0, 1):
        acc, Fb, _ = _conv_ref(xin, ws[grp][0], (3, 1, 1))
        ref = acc + bs[grp].double()
        bound = bf16_out_bound(ref, Fb + 4 * U32 * (acc.abs() + bs[grp].double().abs()))
        assert_within(frames[1 + grp::2].reshape(-1, C), ref, bound, f"{tag} group {grp}", "conv3d_wan")


@pytest.mark.parametrize("mode,T,H,W,C,co", [("hw", 2, 9, 13, 64, 128), ("hw", 1, 17, 31, 128, 96), ("hw", 3, 5, 130, 64, 64),
                                             ("t", 5, 4, 6, 128, 128), ("t", 8, 3, 40, 64, 96)])
def test_conv3d_wan_strided_resample(dev, mode, T, H, W, C, co):
    """The Encoder3d Resample convs. mode hw: Conv2d 3x3 stride 2 behind ZeroPad2d((0,1,0,1)) (stride_hw = 2, taps (1,3,3))
    with odd H / W, so the last output row / column reads the zero pad. mode t: time_conv (3,1,1) stride 2, no padding
    (stride_t = 2), written one frame behind (out_t_add = 1) into [1 + To, Ho*Wo, co] whose frame 0 holds seeded data that
    must keep its bits. Bound: the conv bound of _conv_ref, F32 accumulation then BF16 output."""
    from yume_b200 import ops
    g = _gen("strided", mode, T, H, W, C, co)
    taps = (1, 3, 3) if mode == "hw" else (3, 1, 1)
    x, wt, wk = _conv_operands(g, T, H, W, C, co, taps, dev)
    b = _randn(g, co, dev=dev)
    st = dict(stride_hw=2) if mode == "hw" else dict(stride_t=2)
    acc, Fb, (To, Ho, Wo) = _conv_ref(x, wt, taps, **st)
    assert (To, Ho, Wo) == ops.conv_out_dims(T, H, W, taps, **st)
    lead = 0 if mode == "hw" else 1
    rows = (lead + To) * Ho * Wo
    seed = _randn(g, rows, co, dev=dev).bfloat16()
    out = guarded((rows, co), torch.bfloat16, (64, 32))
    out.view[:lead * Ho * Wo].copy_(seed[:lead * Ho * Wo])
    ops.conv3d_causal(x, wk, b, out.view, T, H, W, ops.YB_EPI_BF16, taps=taps, oob_zero_pad=True, out_t_add=lead, **st)
    torch.cuda.synchronize()
    tag = f"conv3d_wan strided {mode} T{T} H{H} W{W} C{C} co{co}"
    out.check(tag)
    assert torch.equal(out.view[:lead * Ho * Wo], seed[:lead * Ho * Wo]), tag + ": the frame in front was overwritten"
    ref = acc + b.double()
    bound = bf16_out_bound(ref, Fb + 4 * U32 * (acc.abs() + b.double().abs()))
    assert_within(out.view[lead * Ho * Wo:], ref, bound, tag, "conv3d_wan")


# ------------------------------------------------------------------------------------------------------------
# Wan VAE glue
# ------------------------------------------------------------------------------------------------------------
def rms_act_bound(x, gamma, C, nch, G, silu):
    """yb_vae_rms_act in fp64 and its bound. Per voxel each of G lanes sums 8*NCH squares in fp32, then log2(G) shuffle
    levels: relative error of the sum of squares <= (8*NCH + log2 G + 1)*u32 (+1: the squares). sqrtf (IEEE, no fast-math)
    halves that and adds u32; sqrtf(C) and the division add u32 each, so the scale sqrt(C)/||x|| carries
    e = 0.5*(8*NCH + log2 G + 1)*u32 + 3*u32 relative; y = x*scale*gamma rounds twice more: f32 = (e + 2*u32)*|y|. SiLU:
    _silu_bound. The caller adds the bf16 rounding. x fp64 [N, C]."""
    y = x * math.sqrt(C) / x.pow(2).sum(1, keepdim=True).sqrt().clamp_min(1e-12) * gamma.double()
    e = 0.5 * (8 * nch + math.log2(G) + 1) * U32 + 3 * U32
    f32 = (e + 2 * U32) * y.abs()
    if silu:
        f32 = _silu_bound(y, f32)
        y = y * torch.sigmoid(y)
    return y, f32


def rms_instance(C, Cp):
    """The (NCH, G) template instance yb_vae_rms_act launches for C / Cp (its width rule, vae_elementwise.cu)."""
    nch = 1 if C <= 256 else (2 if C <= 512 else 4)
    return nch, (32 if nch > 1 else (8 if Cp <= 64 else (16 if Cp <= 128 else 32)))


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("up", [1, 2])
@pytest.mark.parametrize("C,Cp", RMS_WIDTHS)
def test_vae_rms_act_every_instance(dev, C, Cp, up, silu):
    """yb_vae_rms_act at one width per YB_RMS_LAUNCH instance, from a column window x (ldx > C) into a guarded
    [T, Hs*up, Ws*up, Cp] buffer; reference values placed by the CPU stand-in's index logic (it maps each output voxel to its
    source voxel). Bound: rms_act_bound + bf16 rounding. The pad columns [C, Cp) must be exactly 0; gamma = None with SiLU off
    is a copy and must be bit-exact."""
    from helpers import torch_ops as T_
    from yume_b200 import ops
    g = _gen("rms", C, Cp, up, silu)
    T, Hs, Ws = 2, 5, 7
    N = T * Hs * Ws
    x = (torch.randn(N, C + 16, generator=g) * 2 + 0.3).to(dev).bfloat16()[:, 8:8 + C]
    gamma = (torch.rand(C, generator=g) + 0.5).to(dev)
    shape = (T, Hs * up, Ws * up, Cp)
    src = torch.arange(N, dtype=torch.float64, device=dev)[:, None].expand(-1, 8)
    where = torch.zeros(shape[:-1] + (8,), dtype=torch.float64, device=dev)
    T_.vae_rms_act(src, (T, Hs, Ws), where, None, up=up, silu=False)
    where = where[..., 0].long()
    tag = f"vae_rms_act C{C} Cp{Cp} up{up} silu{int(silu)}"
    nch, G = rms_instance(C, Cp)
    out = guarded(shape, torch.bfloat16, (1, 0))
    ops.vae_rms_act(x, (T, Hs, Ws), out.view, gamma, up=up, silu=silu)
    torch.cuda.synchronize()
    out.check(tag)
    assert torch.equal(out.view[..., C:], torch.zeros_like(out.view[..., C:])), tag + ": channel padding not zero"
    y, f32 = rms_act_bound(x.double(), gamma, C, nch, G, silu)
    assert_within(out.view[..., :C], y[where], bf16_out_bound(y[where], f32[where]), tag, "vae_rms_act")
    if not silu:
        cp = guarded(shape, torch.bfloat16, (1, 0))
        ops.vae_rms_act(x, (T, Hs, Ws), cp.view, None, up=up, silu=False)
        torch.cuda.synchronize()
        cp.check(tag + " copy")
        want = torch.zeros(shape, dtype=torch.bfloat16, device=dev)
        want[..., :C] = x[where]
        assert torch.equal(cp.view, want), tag + ": copy path not bit-exact"
        record_exact("vae_rms_act_copy")


@pytest.mark.parametrize("ft,in_c,out_c", [(2, 1024, 1024), (1, 1024, 1024), (2, 1024, 512), (1, 1024, 512), (1, 512, 256)])
def test_vae_dupup_add_bit_exact(dev, ft, in_c, out_c):
    """yb_vae_dupup_add: main += DupUp3D(x) (fs = 2; rep = out_c*ft*4/in_c = 2, 4 and 8, ft 1 and 2). The kernel adds the two
    bf16 values in fp32 and rounds once, as torch does: bit-exact against (main.float() + src.float()).bfloat16(), with the
    source element of every (voxel, channel) taken from the CPU stand-in run on index numbers. main is seeded and guarded."""
    from helpers import torch_ops as T_
    from yume_b200 import ops
    g = _gen("dupup", ft, in_c, out_c)
    Ts, Hs, Ws, fs = 3, 3, 5, 2
    To = ft * Ts - (ft - 1)
    shape = (To, Hs * fs, Ws * fs, out_c)
    x = _randn(g, Ts * Hs * Ws, in_c, dev=dev).bfloat16()
    m0 = _randn(g, *shape, dev=dev).bfloat16()
    main = guarded(shape, torch.bfloat16, (1, 0), fill=m0)
    ops.vae_dupup_add(main.view, x, (Ts, Hs, Ws), in_c, out_c, ft, fs)
    torch.cuda.synchronize()
    tag = f"vae_dupup_add ft{ft} in_c{in_c} out_c{out_c}"
    main.check(tag)
    idx = torch.zeros(shape, dtype=torch.float64, device=dev)
    T_.vae_dupup_add(idx, torch.arange(x.numel(), dtype=torch.float64, device=dev).view(x.shape), (Ts, Hs, Ws), in_c, out_c,
                     ft, fs)
    want = (m0.float() + x.flatten()[idx.long()].float()).bfloat16()
    diff = main.view != want
    assert not bool(diff.any()), f"{tag}: {int(diff.sum())} elements differ, first at {tuple(diff.nonzero()[0].tolist())}"
    record_exact("vae_dupup_add")


def avgdown_ref(x, dims, in_c, out_c, ft, fs):
    """fp64 AvgDown3D (the stand-in's rearrangement in double): returns (mean, sum |x| / G) per output element, both
    [To, Ho, Wo, out_c]."""
    T, H, W = dims
    xn = x.double().view(T, H, W, in_c).permute(3, 0, 1, 2)[None]
    pad_t = (ft - T % ft) % ft
    xn = F.pad(xn, (0, 0, 0, 0, pad_t, 0))
    B, C, Tp, _, _ = xn.shape
    xn = xn.view(B, C, Tp // ft, ft, H // fs, fs, W // fs, fs).permute(0, 1, 3, 5, 7, 2, 4, 6).contiguous()
    xn = xn.view(out_c, C * ft * fs * fs // out_c, Tp // ft, H // fs, W // fs)
    return xn.mean(1).permute(1, 2, 3, 0), xn.abs().mean(1).permute(1, 2, 3, 0)


@pytest.mark.parametrize("T", [4, 5])
@pytest.mark.parametrize("ft,fs,in_c,out_c", [(1, 2, 160, 320), (2, 2, 320, 640), (2, 2, 640, 640), (1, 1, 640, 640),
                                              (2, 2, 64, 64)])
def test_vae_avgdown_add_per_element(dev, ft, fs, in_c, out_c, T):
    """yb_vae_avgdown_add: main += mean over G = in_c*ft*fs^2/out_c elements (odd T: (ft - T % ft) % ft zero frames in
    front). G is a power of two, so 1/G and acc/G are exact in fp32; the G-term sequential fp32 sum is off by at most
    (G-1)*u32*sum|x|; main + mean rounds once (u32), then bf16: bound = bf16_out_bound(ref, (G-1)*u32*sum|x|/G + u32*|ref|).
    G = 1 (no down-sampling) has no sum at all: its ratio is only the final roundings."""
    from yume_b200 import ops
    G = in_c * ft * fs * fs // out_c
    assert G & (G - 1) == 0, G
    g = _gen("avgdown", ft, fs, in_c, out_c, T)
    H, W = 4, 6
    x = _randn(g, T * H * W, in_c, dev=dev).bfloat16()
    To = (T + (ft - T % ft) % ft) // ft
    shape = (To, H // fs, W // fs, out_c)
    m0 = _randn(g, *shape, dev=dev).bfloat16()
    main = guarded(shape, torch.bfloat16, (1, 0), fill=m0)
    ops.vae_avgdown_add(main.view, x, (T, H, W), in_c, out_c, ft, fs)
    torch.cuda.synchronize()
    tag = f"vae_avgdown_add ft{ft} fs{fs} in_c{in_c} out_c{out_c} T{T}"
    main.check(tag)
    mean, absmean = avgdown_ref(x, (T, H, W), in_c, out_c, ft, fs)
    ref = m0.double() + mean
    assert_within(main.view, ref, bf16_out_bound(ref, (G - 1) * U32 * absmean + U32 * ref.abs()), tag, "vae_avgdown")


def _rup(v, m):
    return (v + m - 1) // m * m


def softmax_bound(s, L, hw):
    """Frame-causal softmax in fp64 and the f32 error of the kernel: arguments a_j = s_j - max (one rounding: u32*|a_j|
    absolute, so exp moves by that relative), __expf (_exp_err); the fp32 sum of at most L/256 per-thread terms, a 5-level
    shuffle and 8 partials (depth L/256 + 16, relative to the sum of positive terms); the IEEE 1/sum and the product: 2*u32.
    Per element p_i: f32 = (e_i + max_j e_j + (L/256 + 18)*u32) * p_i with e_j = _exp_err(a_j) + u32*|a_j|. Masked -> 0."""
    Lq = s.shape[0]
    rows = torch.arange(Lq, device=s.device)[:, None] // hw
    cols = torch.arange(s.shape[1], device=s.device)[None, :]
    keep = (cols // hw <= rows) & (cols < L)
    sm = s.double().masked_fill(~keep, -math.inf)
    p = torch.softmax(sm, dim=-1)
    a = (sm - sm.amax(1, keepdim=True)).masked_fill(~keep, 0.0)
    e = _exp_err(a) + U32 * a.abs()
    f32 = (e + e.masked_fill(~keep, 0).amax(1, keepdim=True) + (L / 256 + 18) * U32) * p
    return p, f32, keep


@pytest.mark.parametrize("ld_mode", ["L", "rup32"])
@pytest.mark.parametrize("hw,mult,short", [(40, 1, 0), (40, 3, 0), (40, 3, 5), (200, 3, 0), (200, 3, 5)])
def test_masked_softmax_per_element(dev, hw, mult, short, ld_mode):
    """yb_masked_softmax with L = hw, 3*hw and 3*hw - 5 (a short last frame) and ldP = L or rup(L, 32) (the Wan2.2
    mid-attention passes ldP = Lf > L and relies on columns >= L being exact zeros, vae22.py). Logits spread with sigma = 8,
    so __expf's argument-dependent error matters. Bound: softmax_bound + bf16 rounding; every masked entry and every column
    in [L, ldP) must be exactly 0; S is a window with ldS > ldP; P's guard rows must keep their bits."""
    from yume_b200 import ops
    L = hw * mult - short
    ldP = L if ld_mode == "L" else _rup(L, 32)
    g = _gen("msm", hw, mult, short, ld_mode)
    S = _randn(g, L, ldP + 24, scale=8.0, dev=dev)[:, :ldP]
    P = guarded((L, ldP), torch.bfloat16, (4, 0))
    ops.masked_softmax(S, P.view, L, hw)
    torch.cuda.synchronize()
    tag = f"masked_softmax hw{hw} L{L} ldP{ldP}"
    P.check(tag)
    p, f32, keep = softmax_bound(S, L, hw)
    assert bool((P.view[~keep] == 0).all()), tag + ": a masked entry (next frame / column >= L) is not exactly 0"
    assert_within(P.view, p, bf16_out_bound(p, f32), tag, "masked_softmax")


@pytest.mark.parametrize("T,H,W,ldo", [(1, 8, 12, 12), (3, 6, 10, 64), (2, 34, 18, 16)])
def test_vae_patchify2_bf16_bit_exact(dev, T, H, W, ldo):
    """yb_vae_patchify2_bf16: video f32 [3, T, H, W] -> bf16 [T*(H/2)*(W/2), ldo], channel (c r q), columns >= 12 zero.
    One bf16 rounding per element, as torch's .to(bfloat16): bit-exact against the CPU stand-in run on the device."""
    from helpers import torch_ops as T_
    from yume_b200 import ops
    g = _gen("pf2", T, H, W, ldo)
    video = _randn(g, 3, T, H, W, scale=1.5, dev=dev)
    N = T * (H // 2) * (W // 2)
    out = guarded((N, ldo), torch.bfloat16, (2, 0))
    ops.vae_patchify2_bf16(video, out.view)
    torch.cuda.synchronize()
    tag = f"vae_patchify2 T{T} H{H} W{W} ldo{ldo}"
    out.check(tag)
    want = T_.vae_patchify2_bf16(video, torch.empty(N, ldo, dtype=torch.bfloat16, device=dev))
    assert torch.equal(out.view, want), tag
    record_exact("vae_patchify2")


@pytest.mark.parametrize("T,H,W,ldy", [(1, 4, 6, 16), (3, 5, 7, 24), (2, 17, 9, 64)])
def test_vae_unpatchify2_clamp_bit_exact(dev, T, H, W, ldy):
    """yb_vae_unpatchify2_clamp: y f32 [T*H*W, ldy] (a 12-channel window, ldy > 12, values beyond +-1) -> guarded f32
    [3, T, 2H, 2W] clamped to [-1, 1]: bit-exact against the CPU stand-in run on the device."""
    from helpers import torch_ops as T_
    from yume_b200 import ops
    g = _gen("upf2", T, H, W, ldy)
    y = _randn(g, T * H * W, ldy, scale=1.5, dev=dev)[:, 4:16]
    out = guarded((3, T, 2 * H, 2 * W), torch.float32, (1, 0))
    ops.vae_unpatchify2_clamp(y, out.view, T, H, W)
    torch.cuda.synchronize()
    tag = f"vae_unpatchify2_clamp T{T} H{H} W{W} ldy{ldy}"
    out.check(tag)
    want = T_.vae_unpatchify2_clamp(y, torch.empty(3, T, 2 * H, 2 * W, device=dev), T, H, W)
    assert torch.equal(out.view, want), tag
    assert bool((want.abs() == 1).any()), tag + ": no value was clamped"
    record_exact("vae_unpatchify2_clamp")


@pytest.mark.parametrize("N,Cn,ldo", [(1000, 3, 64), (777, 16, 16), (4096, 12, 72)])
def test_nchw_to_nhwc_bf16_bit_exact(dev, N, Cn, ldo):
    """yb_nchw_to_nhwc_bf16: f32 [Cn, N] -> guarded bf16 [N, ldo], columns >= Cn zero: bit-exact."""
    from yume_b200 import ops
    g = _gen("nchw", N, Cn, ldo)
    x = _randn(g, Cn, N, scale=3.0, dev=dev)
    out = guarded((N, ldo), torch.bfloat16, (2, 0))
    ops.nchw_to_nhwc_bf16(x, out.view)
    torch.cuda.synchronize()
    tag = f"nchw_to_nhwc N{N} Cn{Cn} ldo{ldo}"
    out.check(tag)
    want = torch.zeros(N, ldo, dtype=torch.bfloat16, device=dev)
    want[:, :Cn] = x.t().bfloat16()
    assert torch.equal(out.view, want), tag
    record_exact("nchw_to_nhwc")


@pytest.mark.parametrize("dim,ext", [(1, 3), (2, 8), (3, 7), (3, 16)])
def test_blend_is_the_reference_expression(dev, dim, ext):
    """yb_blend in place on b: for y < ext, b[y] = a[ea - ext + y] * (1 - y/ext) + b[y] * (y/ext), evaluated as the reference
    evaluates it (f32 tensors times Python-float weights: the weights computed in double and rounded to f32, each product and
    the sum rounded separately). Bit-exact; b is seeded and guarded."""
    from yume_b200 import ops
    g = _gen("blend", dim, ext)
    shp_a, shp_b = [3, 9, 20, 24], [3, 9, 20, 24]
    shp_a[dim] += 5
    a = _randn(g, *shp_a, dev=dev)
    b0 = _randn(g, *shp_b, dev=dev)
    b = guarded(tuple(shp_b), torch.float32, (1, 0), fill=b0)
    ops.blend(a, b.view, dim, ext)
    torch.cuda.synchronize()
    tag = f"blend dim{dim} ext{ext}"
    b.check(tag)
    want = b0.clone()
    e = min(a.shape[dim], want.shape[dim], ext)
    for y in range(e):
        want.select(dim, y).copy_(a.select(dim, a.shape[dim] - e + y) * (1 - y / e) + want.select(dim, y) * (y / e))
    diff = b.view != want
    assert not bool(diff.any()), f"{tag}: {int(diff.sum())} elements differ, first at {tuple(diff.nonzero()[0].tolist())}"
    record_exact("blend")


# ------------------------------------------------------------------------------------------------------------
# fp32 DiT ops
# ------------------------------------------------------------------------------------------------------------
def sinusoidal_ref(t, dim):
    """(ref, bound) of yb_sinusoidal on f32 timesteps t [U] (test_sinusoidal_per_element derives the bound)."""
    half = dim // 2
    s = torch.outer(t.double(), torch.pow(10000.0, -torch.arange(half, device=t.device, dtype=torch.float64) / half))
    ref = torch.cat([s.cos(), s.sin()], 1)
    e = 2.0 ** -50 * (1 + t.double().abs())[:, None]
    return ref, U32 * (ref.abs() + e) + e


def linear_f32_small_ref(x, w, bias, silu):
    """(ref, bound) of yb_linear_f32_small on x [M, K], w [N, K] (test_linear_f32_small_per_element derives the bound)."""
    K, N = x.shape[1], w.shape[0]
    a = x.double()
    if silu:
        a = a * torch.sigmoid(a)
    ref = a @ w.double().t()
    bd = bias.double() if bias is not None else torch.zeros(N, dtype=torch.float64, device=x.device)
    aw = a.abs() @ w.double().abs().t()
    return ref + bd, (K / 32 + 6 + (6 if silu else 0)) * U32 * aw + U32 * (ref + bd).abs()


def linear_f32_ref(x, w, bias):
    """(ref, bound) of yb_linear_f32 on x [M, K], w [N, K] (test_linear_f32_per_element derives the bound)."""
    K = x.shape[1]
    ref = x.double() @ w.double().t()
    if bias is not None:
        ref = ref + bias.double()
    return ref, K * U32 * (x.double().abs() @ w.double().abs().t()) + U32 * ref.abs()


def test_sinusoidal_per_element(dev):
    """yb_sinusoidal: t = 0, integers up to 1000 and non-integer sampler timesteps; dim 256. The kernel evaluates
    pos * 10000^(-i/half), cos and sin in fp64 (each within a few fp64 ulps: the argument |a| <= |t| is off by <= 4*2^-53*|t|,
    and cos / sin add 2^-53) and rounds to f32: |out - ref| <= u32*(|ref| + e) + e with e = 2^-50*(1 + |t|)."""
    from yume_b200 import _lib, ops
    t = torch.tensor([0.0, 1.0, 2.0, 17.0, 250.0, 999.0, 1000.0, 0.5, 3.25, 937.8125, 12.3456, 999.999, 0.001],
                     device=dev, dtype=torch.float32)
    dim = 256
    out = guarded((t.numel(), dim), torch.float32, (2, 0))
    assert _lib.load().yb_sinusoidal(t.data_ptr(), out.view.data_ptr(), t.numel(), dim, ops._stream()) == 0
    torch.cuda.synchronize()
    out.check("sinusoidal")
    ref, bound = sinusoidal_ref(t, dim)
    assert_within(out.view, ref, bound, "sinusoidal dim256", "sinusoidal")


@pytest.mark.parametrize("silu,with_bias", [(False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M", [1, 2, 3, 16])
@pytest.mark.parametrize("K,N", [(256, 3072), (3072, 18432), (5120, 5120), (256, 1004)])
def test_linear_f32_small_per_element(dev, K, N, M, silu, with_bias):
    """yb_linear_f32_small (time MLP / projection, M <= 16, N = C or 6C; N = 1004 is not a multiple of the 8 columns a block
    owns, so the last block has idle warps). One warp per column: each lane runs K/32 fmaf terms, a 5-level shuffle, then
    + bias: |err| <= (K/32 + 6) * u32 * sum|a'*w| + u32*|bias|, a' = SiLU(a) when silu_in, computed with expf (<= 2 ulp), the add and the IEEE division: a' carries
    <= 6*u32 relative, adding 6*u32*sum|a'*w|. The wrapper allocates its output, so the C ABI is called with a guarded one."""
    from yume_b200 import _lib, ops
    g = _gen("lfs", K, N, M, silu, with_bias)
    x = _randn(g, M, K, dev=dev)
    w = _randn(g, N, K, scale=1 / math.sqrt(K), dev=dev)
    bias = _randn(g, N, dev=dev) if with_bias else None
    out = guarded((M, N), torch.float32, (2, 0))
    assert _lib.load().yb_linear_f32_small(x.data_ptr(), w.data_ptr(), ops._ptr(bias), out.view.data_ptr(), M, N, K,
                                           int(silu), ops._stream()) == 0
    torch.cuda.synchronize()
    tag = f"linear_f32_small M{M} N{N} K{K} silu{int(silu)} bias{int(with_bias)}"
    out.check(tag)
    ref, bound = linear_f32_small_ref(x, w, bias, silu)
    assert_within(out.view, ref, bound, tag, "linear_f32_small")


@pytest.mark.parametrize("N", [64, 100, 192])
@pytest.mark.parametrize("K", [3072, 5120])
@pytest.mark.parametrize("M", [1, 63, 130])
def test_linear_f32_per_element(dev, M, K, N):
    """yb_linear_f32 (the Head): x a column window (ldi = K + 16 > K), out a guarded window (ldo > N), M tails (1, 63, 130) and an
    N tail (100) of the 64x64 tile. Each output is one sequential fmaf chain over K then + bias:
    |err| <= K*u32*sum|a*w| + u32*|ref|."""
    from yume_b200 import ops
    g = _gen("lf", M, K, N)
    x = _randn(g, M, K + 16, dev=dev)[:, 8:8 + K]
    w = _randn(g, N, K, scale=1 / math.sqrt(K), dev=dev)
    bias = _randn(g, N, dev=dev)
    out = guarded((M, N), torch.float32, (8, 8))
    ops.linear_f32(x, w, bias, out.view)
    torch.cuda.synchronize()
    tag = f"linear_f32 M{M} K{K} N{N}"
    out.check(tag)
    ref, bound = linear_f32_ref(x, w, bias)
    assert_within(out.view, ref, bound, tag, "linear_f32")


def test_linear_f32_rejects_misaligned_and_bad_shapes(dev):
    """yb_linear_f32 reads in and W as float4: a pointer off 16 bytes, or N % 4 != 0, is refused before any launch (the
    return codes only; nothing misaligned is launched)."""
    from yume_b200 import _lib, ops
    lib = _lib.load()
    x = torch.zeros(4, 64, device=dev)
    w = torch.zeros(8, 64, device=dev)
    out = torch.zeros(4, 8, device=dev)
    s = ops._stream()
    assert lib.yb_linear_f32(x.data_ptr() + 4, 64, w.data_ptr(), None, out.data_ptr(), 8, 4, 8, 60, s) == YB_ERR_ALIGNMENT
    assert lib.yb_linear_f32(x.data_ptr(), 64, w.data_ptr() + 8, None, out.data_ptr(), 8, 4, 8, 60, s) == YB_ERR_ALIGNMENT
    assert lib.yb_linear_f32(x.data_ptr(), 64, w.data_ptr(), None, out.data_ptr(), 8, 4, 6, 64, s) == YB_ERR_SHAPE
    assert lib.yb_linear_f32(x.data_ptr(), 62, w.data_ptr(), None, out.data_ptr(), 8, 4, 8, 60, s) == YB_ERR_SHAPE


def test_bcast_add_bit_exact(dev):
    """yb_bcast_add: out[r1][r2][:] = a[r1] + b[r2] (one fp32 add, as torch's): bit-exact into a guarded output."""
    from yume_b200 import _lib, ops
    g = _gen("bcast")
    R1, R2, n = 30, 3, 6 * 1000
    a, b = _randn(g, R1, n, dev=dev), _randn(g, R2, n, dev=dev)
    out = guarded((R1, R2, n), torch.float32, (1, 0))
    assert _lib.load().yb_bcast_add(a.data_ptr(), b.data_ptr(), out.view.data_ptr(), R1, R2, n, ops._stream()) == 0
    torch.cuda.synchronize()
    out.check("bcast_add")
    assert torch.equal(out.view, a[:, None] + b[None]), "bcast_add"
    record_exact("bcast_add")


@pytest.mark.parametrize("Cin,F_,H,W,ph,pw", [(16, 3, 9, 13, 2, 2), (48, 2, 8, 8, 2, 2), (4, 1, 5, 7, 1, 2)])
def test_patchify_bit_exact(dev, Cin, F_, H, W, ph, pw):
    """yb_patchify from a strided input (a permuted, cropped view of a larger tensor) into a guarded [L, ldo] buffer with
    ldo > Cin*ph*pw: columns < Cin*ph*pw bit-exact against the CPU stand-in (H, W not multiples of the patch: zero fill);
    the kernel does not write the columns past Cin*ph*pw, which must keep their NaN."""
    from helpers import torch_ops as T_
    from yume_b200 import ops
    g = _gen("patchify", Cin, F_, H, W, ph, pw)
    big = _randn(g, F_, Cin + 2, H + 3, W + 5, dev=dev)
    x = big.permute(1, 0, 2, 3)[1:1 + Cin, :, 2:2 + H, 1:1 + W]
    Kc = Cin * ph * pw
    L = F_ * (-(-H // ph)) * (-(-W // pw))
    out = guarded((L, Kc + 8), torch.bfloat16, (2, 0))
    ops.patchify(x, out.view, ph, pw)
    torch.cuda.synchronize()
    tag = f"patchify Cin{Cin} F{F_} H{H} W{W} p{ph}x{pw}"
    out.check(tag, allow_nan=True)
    assert bool(torch.isnan(out.view[:, Kc:]).all()), tag + ": columns past Cin*ph*pw were written"
    want = T_.patchify(x, torch.empty(L, Kc, dtype=torch.bfloat16, device=dev), ph, pw)
    assert torch.equal(out.view[:, :Kc], want), tag
    record_exact("patchify")


@pytest.mark.parametrize("Cout,F_,Hp,Wp,ph,pw", [(48, 3, 5, 7, 2, 2), (16, 2, 4, 9, 2, 2), (3, 1, 6, 5, 1, 2)])
def test_unpatchify_bit_exact(dev, Cout, F_, Hp, Wp, ph, pw):
    """yb_unpatchify: y f32 [L, ldy] window (ldy > ph*pw*Cout) -> guarded [Cout, F, Hp*ph, Wp*pw]: bit-exact."""
    from helpers import torch_ops as T_
    from yume_b200 import ops
    g = _gen("unpatchify", Cout, F_, Hp, Wp, ph, pw)
    L, Kc = F_ * Hp * Wp, ph * pw * Cout
    y = _randn(g, L, Kc + 12, dev=dev)[:, 4:4 + Kc]
    shape = (Cout, F_, Hp * ph, Wp * pw)
    out = guarded(shape, torch.float32, (1, 0))
    ops.unpatchify(y, out.view, F_, Hp, Wp, ph, pw)
    torch.cuda.synchronize()
    tag = f"unpatchify Cout{Cout} F{F_} Hp{Hp} Wp{Wp} p{ph}x{pw}"
    out.check(tag)
    assert torch.equal(out.view, T_.unpatchify(y, torch.empty(shape, device=dev), F_, Hp, Wp, ph, pw)), tag
    record_exact("unpatchify")


# ------------------------------------------------------------------------------------------------------------
# direct entry points ops.py does not call
# ------------------------------------------------------------------------------------------------------------
def test_rmsnorm_rope_plain_entry(dev):
    """yb_rmsnorm_rope (the plain form) on the q columns of a guarded [L, 3C] buffer, C = 3072, rope_len = L - 37: q within
    _rr_ref, k and v columns and the guard band keep their bits."""
    from yume_b200 import _lib, ops
    D, L, C = 128, 333, 3072
    g = _gen("rr_plain")
    data = _randn(g, L, 3 * C, dev=dev).bfloat16()
    buf = guarded((L, 3 * C), torch.bfloat16, (8, 8), fill=data)
    w = (torch.rand(C, generator=g) + 0.5).to(dev)
    ang = torch.rand(L, D // 2, generator=g, dtype=torch.float64) * 6.28
    rope = torch.stack([ang.cos(), ang.sin()], -1).float().contiguous().to(dev)
    q = buf.view[:, :C]
    assert _lib.load().yb_rmsnorm_rope(q.data_ptr(), q.stride(0), w.data_ptr(), rope.data_ptr(), L - 37, L, C, D, 1e-6,
                                       ops._stream()) == 0
    torch.cuda.synchronize()
    buf.check("rmsnorm_rope plain")
    assert torch.equal(buf.view[:, C:], data[:, C:]), "rmsnorm_rope plain: k / v columns changed"
    y, bound = _rr_ref(data[:, :C], w, rope, L - 37, D)
    assert_within(buf.view[:, :C], y, bound, "rmsnorm_rope plain C3072", "rmsnorm_rope")


@pytest.mark.parametrize("flags", [0, 1])
def test_attention_plain_entry(dev, flags):
    """yb_attention (the form INTEGRATION.md documents; no workspace, so no automatic split) on qkv column slices, 5 heads,
    Lq 257, Lk 383, into a guarded window: attention_bound of part one."""
    from yume_b200 import _lib, ops
    g = _gen("att_plain", flags)
    heads, Lq, Lk = 5, 257, 383
    q, k, v = KC._qkv_slices(g, Lq, Lk, heads, dev)
    scale = 1 / math.sqrt(128.0)
    ref, bound = KC._attention_ref(q, k, v, heads, scale)
    out = guarded((Lq, heads * 128), torch.bfloat16, (128, 64))
    assert _lib.load().yb_attention(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                                    out.view.data_ptr(), out.view.stride(0), Lq, Lk, heads, scale, flags, ops._stream()) == 0
    torch.cuda.synchronize()
    tag = f"attention plain entry flags{flags}"
    out.check(tag)
    assert_within(out.view, ref, bound, tag, "attention")


# ------------------------------------------------------------------------------------------------------------
# entry point -> tests that exercise it (tests/test_kernel_contract_cpu.py: every C-ABI entry point is in a COVERS table)
# ------------------------------------------------------------------------------------------------------------
COVERS = {
    "yb_gemm_bf16": ["test_gemm_n_split_layout", "test_gemm_a_split_layout_every_epilogue", "test_gemm_pair_tail_split_k"],
    "yb_gemm_sp_qkv": ["test_gemm_sp_qkv_chain_on_one_gpu"],
    "yb_sp_bcast_sums": ["test_gemm_sp_qkv_chain_on_one_gpu"],
    "yb_sp_post_norm_rope": ["test_gemm_sp_qkv_chain_on_one_gpu"],
    "yb_conv3d_causal": ["test_conv3d_wan_zero_pad_per_element", "test_conv3d_wan_time_conv_interleave",
                         "test_conv3d_wan_strided_resample"],
    "yb_vae_rms_act": ["test_vae_rms_act_every_instance"],
    "yb_vae_dupup_add": ["test_vae_dupup_add_bit_exact"],
    "yb_vae_avgdown_add": ["test_vae_avgdown_add_per_element"],
    "yb_masked_softmax": ["test_masked_softmax_per_element"],
    "yb_vae_patchify2_bf16": ["test_vae_patchify2_bf16_bit_exact"],
    "yb_vae_unpatchify2_clamp": ["test_vae_unpatchify2_clamp_bit_exact"],
    "yb_nchw_to_nhwc_bf16": ["test_nchw_to_nhwc_bf16_bit_exact"],
    "yb_blend": ["test_blend_is_the_reference_expression"],
    "yb_sinusoidal": ["test_sinusoidal_per_element"],
    "yb_linear_f32_small": ["test_linear_f32_small_per_element"],
    "yb_linear_f32": ["test_linear_f32_per_element", "test_linear_f32_rejects_misaligned_and_bad_shapes"],
    "yb_bcast_add": ["test_bcast_add_bit_exact"],
    "yb_patchify": ["test_patchify_bit_exact"],
    "yb_unpatchify": ["test_unpatchify_bit_exact"],
    "yb_rmsnorm_rope": ["test_rmsnorm_rope_plain_entry"],
    "yb_attention": ["test_attention_plain_entry"],
}
