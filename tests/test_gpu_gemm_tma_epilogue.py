"""The 1-CTA GEMM's TMA epilogue (gemm.cu: staged 128-byte boxes leave through TMA stores, and GATE_RES through bulk reduce-adds
into the fp32 residual) against the SM-pair kernel, which keeps the register epilogue and accumulates in the same order along K.

- BF16, GELU tanh / erf, F32 and the ungated residual update are bit-identical between the two.
- The gated residual update rounds the product (acc + b) * g before the add in L2, where the register epilogue contracts the two
  into one FMA: the two differ by at most that rounding plus one ulp of the result, and both lie within the fp64 contract bound.
- The output may be a column window of a wider buffer: the guard columns and the rows past M keep their bits.
"""
from __future__ import annotations

import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
# the ragged M / N shapes of the pair-vs-1-CTA parity test; N = 96 and 704 run 128-wide tiles on the 1-CTA kernel, the rest 256
SHAPES = [(256, 256, 64), (300, 512, 192), (4097, 768, 256), (1000, 3072, 3072), (2310, 3072, 512), (1500, 704, 320),
          (513, 96, 128), (1029, 1184, 192)]
GUARD_L, GUARD_R, GUARD_ROWS = 8, 24, 3


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()
    return "cuda"


def _operands(dev, M, N, K, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = torch.randn(M, K, generator=g).to(dev).bfloat16()
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dev).bfloat16()
    b = torch.randn(N, generator=g).to(dev)
    return g, a, w, b


def _windowed(M, N, dtype, dev, fill):
    """[M, N] column window of a [M + GUARD_ROWS, GUARD_L + N + GUARD_R] buffer (row pitch > N), guards set to `fill`."""
    buf = torch.full((M + GUARD_ROWS, GUARD_L + N + GUARD_R), fill, dtype=dtype, device=dev)
    return buf, buf[:M, GUARD_L:GUARD_L + N]


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _guards_kept(buf, M, N, fill):
    ref = torch.full_like(buf, fill)
    keep = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    keep[:M, GUARD_L:GUARD_L + N] = False
    return torch.equal(_bits(buf)[keep], _bits(ref)[keep])


@pytest.mark.parametrize("epi", ["BF16", "GELU_BF16", "GELU_ERF_BF16", "F32", "GATE_RES"])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_tma_epilogue_matches_register_epilogue(dev, M, N, K, epi):
    """1-CTA kernel (TMA epilogue) == SM-pair kernel (register epilogue), bit for bit, into a windowed output whose guard columns
    and trailing rows keep their bits; GATE_RES here is the ungated update (cross-attention o): x + (acc + b) rounds once either way."""
    from yume_b200 import ops
    e = getattr(ops, "YB_EPI_" + epi)
    g, a, w, b = _operands(dev, M, N, K, M + N + K)
    f32 = epi in ("F32", "GATE_RES")
    dtype = torch.float32 if f32 else torch.bfloat16
    fill = 7.0
    buf1, one = _windowed(M, N, dtype, dev, fill)
    two = torch.full((M, N), -3.0, dtype=dtype, device=dev)
    if epi == "GATE_RES":
        x0 = torch.randn(M, N, generator=g).to(dev)
        one.copy_(x0)
        two.copy_(x0)
    ops.gemm(a, w, b, one, e, cta_pair=1)
    ops.gemm(a, w, b, two, e, cta_pair=2, split_k=1)   # unsplit: the same K order as the 1-CTA kernel
    torch.cuda.synchronize()
    assert torch.equal(_bits(one.contiguous()), _bits(two)), f"{epi}: TMA and register epilogues differ"
    assert _guards_kept(buf1, M, N, fill), f"{epi}: a store left the [M, N] window"


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_tma_gated_residual_within_bounds(dev, M, N, K):
    """Gated x += (acc + b) * gate[tok]: per element within u32*|(acc + b)*g| + ulp(result) of the register epilogue (the product's
    own rounding, then one ulp of the sum — a bound of one ulp alone fails where x and the update cancel), and within the fp64
    contract bound |g|*(F + 4u(|acc| + |b|)) + 4u(|x0| + |g*acc|) with F = 2*K*u*(|A||B|^T)."""
    from yume_b200 import ops
    g, a, w, b = _operands(dev, M, N, K, 7 * M + N + K)
    U = 5
    gate = torch.randn(U, N, generator=g).to(dev)
    tok = torch.randint(0, U, (M,), generator=g).to(dev, torch.int32)
    x0 = torch.randn(M, N, generator=g).to(dev)
    buf, one = _windowed(M, N, torch.float32, dev, 7.0)
    one.copy_(x0)
    two = x0.clone()
    ops.gemm(a, w, b, one, ops.YB_EPI_GATE_RES, gate=gate, tok_idx=tok, cta_pair=1)
    ops.gemm(a, w, b, two, ops.YB_EPI_GATE_RES, gate=gate, tok_idx=tok, cta_pair=2, split_k=1)
    torch.cuda.synchronize()
    assert _guards_kept(buf, M, N, 7.0)
    gt = gate.double()[tok.long()]
    acc = a.double() @ w.double().t()
    accb = acc + b.double()
    res = one.double()
    F = 2.0 * K * U32 * (a.double().abs() @ w.double().abs().t())
    e_accb = F + 4 * U32 * (acc.abs() + b.double().abs())   # |fp32 (acc + b) - accb|
    # both kernels form the same fp32 p = (acc + b) * g; this one rounds it (<= u32 * |p|) before the add, then each sum rounds
    _, ex = torch.frexp(torch.maximum(one.abs(), two.abs()))
    ulp = torch.ldexp(torch.ones_like(one), ex.to(torch.int32) - 24).double()
    d_pair = (res - two.double()).abs()
    bound_pair = U32 * gt.abs() * (accb.abs() + e_accb) + ulp
    assert bool((d_pair <= bound_pair).all()), f"max |diff|/bound against the register epilogue {float((d_pair / bound_pair).max()):.3f}"
    want = x0.double() + accb * gt
    bound = gt.abs() * e_accb + 4 * U32 * (x0.double().abs() + (gt * accb).abs())
    d = (res - want).abs()
    assert bool((d <= bound).all()), f"max |err|/bound {float((d / bound).max()):.3f}"


def test_misaligned_output_pitch_is_rejected(dev):
    """Every accepted launch has a 16-byte row pitch and base, so the TMA epilogue can always describe a plain output; a pitch
    that is not a multiple of 16 bytes is refused rather than written some other way."""
    from yume_b200 import ops
    from yume_b200._lib import YumeB200Error
    M, N, K = 130, 256, 64
    _, a, w, b = _operands(dev, M, N, K, 1)
    buf = torch.zeros(M, N + 4, dtype=torch.bfloat16, device=dev)   # pitch N + 4 bf16 = 520 B
    with pytest.raises(YumeB200Error):
        ops.gemm(a, w, b, buf[:, :N], ops.YB_EPI_BF16, cta_pair=1)
