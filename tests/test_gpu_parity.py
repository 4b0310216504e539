"""GPU parity tests (`-m gpu`): the CUDA path, called through the C ABI, against (a) the CPU oracle, (b) the
golden vectors generated from the reference's own code, (c) size-independent properties at full 5B size.

Tolerances (bf16 path vs fp32-weight oracle, SURVEY.md §8c / BASELINE.md §3):
  * index / gather ops (patchify, unpatchify): bit-exact
  * single kernels vs an fp32 torch reference: bf16 output rounding, rel-Frobenius <= 4e-3
  * one WanAttentionBlock (delta y - x): rel-Frobenius <= 1e-2, max-abs <= 3e-2 on unit-variance inputs
  * whole tiny model output: rel-Frobenius <= 5e-3 (measured ~2e-3)
"""
import math
import os

import pytest
import torch

from oracle import synth
from oracle.wan_dit import WanOracle, grid_freqs

pytestmark = pytest.mark.gpu

KERNEL_TOL = 4e-3
BLOCK_TOL_REL, BLOCK_TOL_ABS = 1e-2, 3e-2
MODEL_TOL = 5e-3     # measured ~2e-3 on every golden case (round 1); a 2.5x regression fails


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()  # fail loudly if the extension is missing
    return "cuda"


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ------------------------------------------------------------------------------------------------------------
# building blocks
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_umma_probe(dev, mode):
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(mode)
    a = torch.randn(128, 128, generator=g).to(dev).bfloat16()
    b = torch.randn(128, 128, generator=g).to(dev).bfloat16()
    d = ops.umma_probe(a, b, mode)
    ref = a.float() @ (b.float().t() if mode == 0 else b.float())
    assert rel(d, ref) < 1e-5


@pytest.mark.parametrize("M,N,K,bn", [(256, 256, 64, 0), (300, 512, 192, 0), (4097, 768, 256, 0), (1000, 3072, 3072, 0),
                                       (2310, 3072, 512, 0), (2310, 3072, 512, 224), (1500, 704, 320, 160), (513, 96, 128, 32),
                                       (1029, 1184, 192, 192)])
def test_gemm_pair_kernel_matches_1cta_kernel(dev, M, N, K, bn):
    """SM-pair (2-CTA cluster) kernel, forced, against the 1-CTA kernel (bit-identical: same products, same fp32 accumulation
    order along K) and fp32 — ragged M / N tails, runtime N tiles (auto and forced), every fused epilogue."""
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).to(dev).bfloat16()
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dev).bfloat16()
    b = torch.randn(N, generator=g).to(dev)
    one = ops.gemm(a, w, b, torch.empty(M, N, device=dev, dtype=torch.bfloat16), ops.YB_EPI_BF16, cta_pair=1)
    two = ops.gemm(a, w, b, torch.full((M, N), 7.0, device=dev, dtype=torch.bfloat16), ops.YB_EPI_BF16, cta_pair=2, block_n=bn)
    assert torch.equal(one, two)
    assert rel(two, a.float() @ w.float().t() + b) < KERNEL_TOL
    acc = a.float() @ w.float().t() + b
    o = ops.gemm(a, w, b, torch.empty(M, N, device=dev, dtype=torch.bfloat16), ops.YB_EPI_GELU_BF16, cta_pair=2, block_n=bn)
    assert rel(o, torch.nn.functional.gelu(acc, approximate="tanh")) < KERNEL_TOL
    U = 3
    gate = torch.randn(U, N, generator=g).to(dev)
    tok = torch.randint(0, U, (M,), generator=g).to(dev, torch.int32)
    x = torch.randn(M, N, generator=g).to(dev)
    want = x + acc * gate[tok.long()]
    ops.gemm(a, w, b, x, ops.YB_EPI_GATE_RES, gate=gate, tok_idx=tok, cta_pair=2, block_n=bn)
    assert rel(x, want) < 1e-5
    res = torch.randn(M, N, generator=g).to(dev).bfloat16()
    o = ops.gemm(a, w, b, torch.empty(M, N, device=dev, dtype=torch.bfloat16), ops.YB_EPI_RES_BF16, res=res, cta_pair=2, block_n=bn)
    assert rel(o, acc + res.float()) < KERNEL_TOL
    o32 = ops.gemm(a, w, None, torch.empty(M, N, device=dev), ops.YB_EPI_F32, cta_pair=2, block_n=bn)
    assert rel(o32, acc - b) < 1e-5


@pytest.mark.parametrize("M,N,K,split_k", [(1100, 256, 512, 2), (700, 288, 1024, 3), (4620, 3072, 14336, 0), (2310, 3072, 14336, 3),
                                           (4620, 3072, 3072, 0), (1280, 512, 640, 4)])
def test_gemm_tail_split_k(dev, M, N, K, split_k):
    """Tail split-K of the SM-pair gate+residual GEMM (the 4- / 8-GPU per-rank shapes leave a mostly idle last wave): K segments
    leave fp32 partials in a caller-owned workspace, a second kernel adds them in index order and applies the epilogue. Same
    result as the unsplit launch up to fp32 summation order; the residual rows outside the split tiles are untouched by it."""
    from yume_b200 import _lib, ops
    g = torch.Generator(device="cpu").manual_seed(M + N + K + split_k)
    a = torch.randn(M, K, generator=g).to(dev).bfloat16()
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dev).bfloat16()
    b = torch.randn(N, generator=g).to(dev)
    gate = torch.randn(2, N, generator=g).to(dev)
    tok = torch.randint(0, 2, (M,), generator=g).to(dev, torch.int32)
    x0 = torch.randn(M, N, generator=g).to(dev)
    if split_k == 0:   # the automatic plan must actually split these shapes (otherwise the test checks nothing)
        assert _lib.load().yb_gemm_workspace_bytes(M, N, K, ops.YB_EPI_GATE_RES, 2, 0) > 0
    plain = ops.gemm(a, w, b, x0.clone(), ops.YB_EPI_GATE_RES, gate=gate, tok_idx=tok, cta_pair=2, split_k=1)
    split = ops.gemm(a, w, b, x0.clone(), ops.YB_EPI_GATE_RES, gate=gate, tok_idx=tok, cta_pair=2, split_k=split_k)
    assert rel(split, plain) < 1e-5            # fp32 summation order along K (4e-6 measured at K = 14336)
    assert float((split - plain).abs().max()) < 1e-3 * float(plain.abs().max())
    assert not torch.equal(split, x0)
    if M * N * K < 2e10:
        want = x0 + (a.float() @ w.float().t() + b) * gate[tok.long()]
        assert rel(split, want) < 1e-5
    # gate-less form (cross-attention o-projection): x += acc + bias
    plain = ops.gemm(a, w, b, x0.clone(), ops.YB_EPI_GATE_RES, cta_pair=2, split_k=1)
    split = ops.gemm(a, w, b, x0.clone(), ops.YB_EPI_GATE_RES, cta_pair=2, split_k=split_k)
    assert rel(split, plain) < 1e-5


def test_gemm_pair_kernel_split_layouts(dev):
    """The Ulysses layouts through the SM-pair kernel: K-split A operand (a_split) and N-split output (n_split)."""
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(41)
    P, Lp, Wh, N = 4, 300, 128, 512
    a3 = torch.randn(P, Lp, Wh, generator=g).to(dev).bfloat16()                 # [P, Lp, Wh]: column k of row t = a3[k // Wh, t, k % Wh]
    w = (torch.randn(N, P * Wh, generator=g) / math.sqrt(P * Wh)).to(dev).bfloat16()
    a2 = a3.permute(1, 0, 2).reshape(Lp, P * Wh).contiguous()
    want = ops.gemm(a2, w, None, torch.empty(Lp, N, device=dev, dtype=torch.bfloat16), ops.YB_EPI_BF16, cta_pair=1)
    got = ops.gemm(a3, w, None, torch.empty(Lp, N, device=dev, dtype=torch.bfloat16), ops.YB_EPI_BF16, a_split=Wh,
                   a_split_stride=Lp * Wh, shape=(Lp, P * Wh), cta_pair=2)
    assert torch.equal(got, want)
    send = torch.zeros(P, Lp, N // P, device=dev, dtype=torch.bfloat16)         # n_split: column block j -> send[j]
    ops.gemm(a2, w, None, send, ops.YB_EPI_BF16, n_split=N // P, split_stride=Lp * (N // P), shape=(Lp, P * Wh), cta_pair=2)
    assert torch.equal(send.permute(1, 0, 2).reshape(Lp, N), want)


@pytest.mark.parametrize("P,Lp,C", [(2, 300, 1024), (4, 257, 1024), (8, 129, 3072)])
def test_fused_qkv_gemm_all_to_all_on_one_gpu(dev, P, Lp, C):
    """yb_gemm_sp_qkv / yb_sp_bcast_sums / yb_sp_post_norm_rope (the "p2p_gemm" Ulysses transport) with the P ranks emulated
    on ONE device: every "rank" runs the fused projection on its token shard with peer pointers to P receive buffers; after
    the sums exchange each receiver normalises + rotates in place. Must equal the plain path (one QKV GEMM over all tokens,
    yb_qk_norm_rope) column block by column block; v bit-exact, q/k up to the fp32 summation order of the row statistics."""
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(P * 1000 + Lp)
    D, K, Wh, L = 128, 256, C // P, P * Lp
    h = torch.randn(L, K, generator=g).to(dev).bfloat16()
    w = (torch.randn(3 * C, K, generator=g) / math.sqrt(K)).to(dev).bfloat16()
    bias = torch.randn(3 * C, generator=g).to(dev)
    nq, nk = (torch.rand(C, generator=g) + 0.5).to(dev), (torch.rand(C, generator=g) + 0.5).to(dev)
    rope = torch.randn(L, D // 2, 2, generator=g).to(dev)
    rope_len = L - 37
    ref = ops.gemm(h, w, bias, torch.empty(L, 3 * C, device=dev, dtype=torch.bfloat16), ops.YB_EPI_BF16)
    v_ref = ref[:, 2 * C:].clone()
    ops.qk_norm_rope(ref[:, :C], ref[:, C:2 * C], nq, nk, rope, D, rope_len=rope_len)
    bufs = [torch.zeros(P * Lp, 3 * Wh, device=dev, dtype=torch.bfloat16) for _ in range(P)]
    tables = [torch.zeros(P * Lp, 2, device=dev) for _ in range(P)]
    local = torch.zeros(Lp, 2, device=dev)
    for r in range(P):
        ops.gemm_sp_qkv(h[r * Lp:(r + 1) * Lp], w, bias, [b.data_ptr() for b in bufs], r, Lp, local)
        ops.sp_bcast_sums(local, [t.data_ptr() for t in tables], r, Lp)
        assert float(local.abs().max()) == 0.0                 # accumulator cleared for the next layer
    for p in range(P):
        ops.sp_post_norm_rope(bufs[p], tables[p], nq[p * Wh:(p + 1) * Wh], nk[p * Wh:(p + 1) * Wh], rope, rope_len, L, Wh, C, D, 1e-6)
        assert torch.equal(bufs[p][:, 2 * Wh:], v_ref[:, p * Wh:(p + 1) * Wh])
        assert rel(bufs[p][:, :Wh], ref[:, p * Wh:(p + 1) * Wh]) < 2e-3
        assert rel(bufs[p][:, Wh:2 * Wh], ref[:, C + p * Wh:C + (p + 1) * Wh]) < 2e-3


@pytest.mark.parametrize("shift", [1, 2, 3, 7, 8])
def test_umma_probe_row_shifted_a(dev, shift):
    """The conv kernel reuses one TMA halo box for the three kw taps by moving the A descriptor's start address by whole
    128-byte rows inside the 128B-swizzled tile; D[m] must equal A[m + shift] . B^T (rows past the end are TMA zeros)."""
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(30 + shift)
    a = torch.randn(128, 128, generator=g).to(dev).bfloat16()
    b = torch.randn(128, 128, generator=g).to(dev).bfloat16()
    d = ops.umma_probe(a, b, 2 + shift)
    ash = torch.zeros_like(a)
    ash[:128 - shift] = a[shift:]
    assert rel(d, ash.float() @ b.float().t()) < 1e-5


@pytest.mark.parametrize("M,N,K,bn", [(128, 256, 64, 0), (300, 384, 192, 0), (1000, 3072, 3072, 0), (512, 128, 4096, 128),
                                       (77, 96, 144, 0), (4097, 768, 256, 256)])
def test_gemm_bf16_matches_fp32_reference(dev, M, N, K, bn):
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M + N)
    a = (torch.randn(M, K, generator=g) * 0.5).to(dev).bfloat16()
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dev).bfloat16()
    bias = torch.randn(N, generator=g).to(dev)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    ops.gemm(a, w, bias, out, ops.YB_EPI_BF16, block_n=bn)
    assert rel(out, a.float() @ w.float().t() + bias) < KERNEL_TOL


def test_gemm_epilogues(dev):
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(5)
    M, N, K, U = 1000, 512, 320, 3
    a = (torch.randn(M, K, generator=g) * 0.5).to(dev).bfloat16()
    w = (torch.randn(N, K, generator=g) * 0.1).to(dev).bfloat16()
    bias = torch.randn(N, generator=g).to(dev)
    acc = a.float() @ w.float().t() + bias
    o = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    ops.gemm(a, w, bias, o, ops.YB_EPI_GELU_BF16)
    assert rel(o, torch.nn.functional.gelu(acc, approximate="tanh")) < KERNEL_TOL
    ops.gemm(a, w, bias, o, ops.YB_EPI_GELU_ERF_BF16)
    assert rel(o, torch.nn.functional.gelu(acc)) < KERNEL_TOL
    o32 = torch.empty(M, N, device=dev)
    ops.gemm(a, w, None, o32, ops.YB_EPI_F32)
    assert rel(o32, acc - bias) < 1e-5
    gate = torch.randn(U, 6, N, generator=g).to(dev)
    tok = torch.randint(0, U, (M,), generator=g).to(dev, torch.int32)
    x = torch.randn(M, N, generator=g).to(dev)
    want = x + acc * gate[tok.long(), 2]
    ops.gemm(a, w, bias, x, ops.YB_EPI_GATE_RES, gate=gate[:, 2], tok_idx=tok)
    assert rel(x, want) < 1e-5
    x2 = torch.randn(M, N, generator=g).to(dev)
    want2 = x2 + acc
    ops.gemm(a, w, bias, x2, ops.YB_EPI_GATE_RES)
    assert rel(x2, want2) < 1e-5


def _sdpa(q, k, v, heads):
    Lq, Lk = q.shape[0], k.shape[0]
    f = lambda t, L: t.reshape(L, heads, 128).transpose(0, 1).float()[None]  # noqa: E731
    o = torch.nn.functional.scaled_dot_product_attention(f(q, Lq), f(k, Lk), f(v, Lk))[0]
    return o.transpose(0, 1).reshape(Lq, heads * 128)


@pytest.mark.parametrize("split", [2, 3, 4])
@pytest.mark.parametrize("Lq,Lk,heads", [(300, 1000, 2), (1000, 777, 3), (257, 2049, 1), (512, 512, 2)])
def test_attention_kv_split_matches_unsplit(dev, Lq, Lk, heads, split):
    """KV-split path (partial O / max / sum per segment + combine kernel) against the single-pass kernel and fp32."""
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(Lq + Lk + split)
    q = torch.randn(Lq, heads * 128, generator=g).to(dev).bfloat16()
    k = torch.randn(Lk, heads * 128, generator=g).to(dev).bfloat16()
    v = torch.randn(Lk, heads * 128, generator=g).to(dev).bfloat16()
    one = ops.attention(q, k, v, torch.empty_like(q), heads, split=1)
    two = ops.attention(q, k, v, torch.full_like(q, 9.0), heads, split=split)
    assert rel(two, one) < 3e-3                      # both bf16-rounded; segments change the fp32 summation order only
    qh, kh, vh = (x.float().view(-1, heads, 128).transpose(0, 1) for x in (q, k, v))
    ref = torch.softmax(qh @ kh.transpose(1, 2) / math.sqrt(128.0), dim=-1) @ vh
    assert rel(two, ref.transpose(0, 1).reshape(Lq, heads * 128)) < KERNEL_TOL


def test_attention_auto_tail_split_full_size_properties(dev):
    """A full-length shape whose last wave is mostly idle (2 heads, L = 18 480: 146 units on the 132 SMs of an H100) takes the
    automatic tail split; compare the whole output with the never-split launch."""
    from yume_b200 import _lib, ops
    g = torch.Generator(device=dev).manual_seed(5)
    L, heads = 18480, 2
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    assert _lib.load().yb_attention_workspace_bytes(L, L, heads, sms, 0) > 0   # the automatic plan splits this launch
    q, k, v = (torch.randn(L, heads * 128, generator=g, device=dev).bfloat16() for _ in range(3))
    a = ops.attention(q, k, v, torch.empty_like(q), heads, split=1)
    b = ops.attention(q, k, v, torch.full_like(q, 7.0), heads, split=0)
    assert bool(torch.isfinite(b.float()).all()) and rel(b, a) < 3e-3


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("Lq,Lk,heads", [(128, 128, 1), (300, 200, 2), (1000, 512, 3), (777, 1500, 2), (257, 257, 2),
                                         (1, 1, 1), (130, 769, 2)])
def test_attention_matches_sdpa(dev, variant, Lq, Lk, heads):
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(Lq * 7 + Lk)
    qkv = torch.randn(max(Lq, Lk), 3 * heads * 128, generator=g).to(dev).bfloat16()
    q, k, v = qkv[:Lq, :heads * 128], qkv[:Lk, heads * 128:2 * heads * 128], qkv[:Lk, 2 * heads * 128:]
    out = torch.zeros(Lq, heads * 128, device=dev, dtype=torch.bfloat16)
    ops.attention(q, k, v, out, heads, variant=variant)
    assert torch.isfinite(out.float()).all()
    assert rel(out, _sdpa(q, k, v, heads)) < KERNEL_TOL


def test_attention_large_logits_and_accumulate(dev):
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(11)
    Lq, Lk, heads = 512, 1024, 2
    q = (torch.randn(Lq, heads * 128, generator=g) * 4).to(dev).bfloat16()
    k = (torch.randn(Lk, heads * 128, generator=g) * 4).to(dev).bfloat16()
    v = torch.randn(Lk, heads * 128, generator=g).to(dev).bfloat16()
    out = torch.zeros(Lq, heads * 128, device=dev, dtype=torch.bfloat16)
    ops.attention(q, k, v, out, heads)            # row maxima jump by >> 2^8: exercises the lazy O rescale
    ref = _sdpa(q, k, v, heads)
    assert rel(out, ref) < KERNEL_TOL
    k2 = torch.randn(257, heads * 128, generator=g).to(dev).bfloat16()
    v2 = torch.randn(257, heads * 128, generator=g).to(dev).bfloat16()
    ops.attention(q, k2, v2, out, heads, accumulate=True)
    assert rel(out, ref + _sdpa(q, k2, v2, heads)) < 2 * KERNEL_TOL


def test_elementwise_kernels(dev):
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(3)
    L, C, D, U = 1000, 3072, 128, 2
    x = (torch.randn(L, C, generator=g) * 2 + 0.3).to(dev)
    mod = (torch.randn(U, 6, C, generator=g) * 0.5).to(dev)
    tok = torch.randint(0, U, (L,), generator=g).to(dev, torch.int32)
    out = torch.empty(L, C, device=dev, dtype=torch.bfloat16)
    ops.ln_modulate(x, out, mod[:, 1], mod[:, 0], tok)
    ln = torch.nn.functional.layer_norm(x, (C,), eps=1e-6)
    assert rel(out, ln * (1 + mod[tok.long(), 1]) + mod[tok.long(), 0]) < KERNEL_TOL
    w, b = torch.randn(C, generator=g).to(dev), torch.randn(C, generator=g).to(dev)
    ops.ln_modulate(x, out, None, None, None, w, b)
    assert rel(out, ln * w + b) < KERNEL_TOL
    o32 = torch.empty(L, C, device=dev)
    ops.ln_modulate(x, o32, mod[0, 1], mod[0, 0])
    assert rel(o32, ln * (1 + mod[0, 1]) + mod[0, 0]) < 1e-5
    # RMSNorm + RoPE against the reference formula (fp64 complex multiply, wan23/modules/model.py:62-72)
    qkv = torch.randn(L, 3 * C, generator=g).to(dev).bfloat16()
    q0, v0 = qkv[:, :C].clone(), qkv[:, 2 * C:].clone()
    wq = (torch.rand(C, generator=g) + 0.5).to(dev)
    ang = (torch.rand(L, D // 2, generator=g, dtype=torch.float64) * 6.28).to(dev)
    rope = torch.stack([ang.cos(), ang.sin()], -1).float().contiguous()
    ops.rmsnorm_rope(qkv[:, :C], wq, rope, D, rope_len=L - 100)
    xf = q0.float()
    n = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6) * wq
    c = torch.view_as_complex(n.double().view(L, C // D, D // 2, 2)) * torch.polar(torch.ones_like(ang), ang)[:, None]
    want = torch.view_as_real(c).flatten(1).float()
    want[L - 100:] = n[L - 100:]                      # tokens past the grid are not rotated (model.py:73)
    assert rel(qkv[:, :C], want) < KERNEL_TOL
    assert torch.equal(qkv[:, 2 * C:], v0)            # neighbours untouched
    # q and k in ONE launch (yb_qk_norm_rope) == the two single launches, bit for bit (same arithmetic, same order)
    for Cw in (3072, 5120, 1024, 256, 384):             # warp-per-row instances and the general fallback (384)
        qkv2 = torch.randn(333, 3 * Cw, generator=g).to(dev).bfloat16()
        ref2 = qkv2.clone()
        w_q, w_k = (torch.rand(Cw, generator=g) + 0.5).to(dev), (torch.rand(Cw, generator=g) + 0.5).to(dev)
        rope2 = torch.randn(333, D // 2, 2, generator=g).to(dev)
        ops.rmsnorm_rope(ref2[:, :Cw], w_q, rope2, D, rope_len=300)
        ops.rmsnorm_rope(ref2[:, Cw:2 * Cw], w_k, rope2, D, rope_len=300)
        ops.qk_norm_rope(qkv2[:, :Cw], qkv2[:, Cw:2 * Cw], w_q, w_k, rope2, D, rope_len=300)
        assert torch.equal(qkv2, ref2), Cw
    # small fp32 pieces
    t = torch.tensor([0.0, 999.0, 500.5], device=dev)
    half = 128
    s = torch.outer(t.double(), torch.pow(10000, -torch.arange(half, device=dev).double().div(half)))
    assert (ops.sinusoidal(t, 256) - torch.cat([s.cos(), s.sin()], 1).float()).abs().max() < 1e-6
    xi, w1, b1 = torch.randn(3, 256, generator=g).to(dev), (torch.randn(512, 256, generator=g) * 0.05).to(dev), torch.randn(512, generator=g).to(dev)
    assert rel(ops.linear_f32_small(xi, w1, b1), xi @ w1.t() + b1) < 1e-5
    assert rel(ops.linear_f32_small(xi, w1, None, True), torch.nn.functional.silu(xi) @ w1.t()) < 1e-5
    xa, wh = torch.randn(1000, 3072, generator=g).to(dev), (torch.randn(192, 3072, generator=g) * 0.02).to(dev)
    oh = torch.empty(1000, 192, device=dev)
    ops.linear_f32(xa, wh, None, oh)
    assert rel(oh, xa.double() @ wh.double().t()) < 1e-5
    a2, b2 = torch.randn(5, 64, generator=g).to(dev), torch.randn(3, 64, generator=g).to(dev)
    assert torch.equal(ops.bcast_add(a2, b2), a2[:, None] + b2[None])


def test_patchify_unpatchify_are_bit_exact(dev):
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(4)
    for (cin, F, H, W, p) in [(48, 3, 10, 12, 2), (48, 2, 9, 11, 4), (36, 2, 7, 33, 32), (48, 21, 44, 80, 2)]:
        x = torch.randn(cin, F, H, W, generator=g).to(dev)
        hp, wp = -(-H // p), -(-W // p)
        out = torch.empty(F * hp * wp, cin * p * p, device=dev, dtype=torch.bfloat16)
        ops.patchify(x, out, p, p)
        xp = torch.nn.functional.pad(x, (0, wp * p - W, 0, hp * p - H)).bfloat16().float()
        want = torch.nn.functional.unfold(xp.permute(1, 0, 2, 3), p, stride=p).permute(0, 2, 1).reshape(F * hp * wp, cin * p * p)
        assert torch.equal(out.float(), want)
        xs = x[:, 1:]                                  # frame slice = non-contiguous channel stride
        out2 = torch.empty((F - 1) * hp * wp, cin * p * p, device=dev, dtype=torch.bfloat16)
        ops.patchify(xs, out2, p, p)
        assert torch.equal(out2, out[hp * wp:])
    F, hp, wp, co = 3, 5, 6, 48
    y = torch.randn(F * hp * wp, 4 * co, generator=g).to(dev)
    uo = torch.empty(co, F, hp * 2, wp * 2, device=dev)
    ops.unpatchify(y, uo, F, hp, wp, 2, 2)
    want = torch.einsum("fhwpqrc->cfphqwr", y.view(F, hp, wp, 1, 2, 2, co)).reshape(co, F, hp * 2, wp * 2)
    assert torch.equal(uo, want)


# ------------------------------------------------------------------------------------------------------------
# block and model parity vs the oracle and the reference-generated golden vectors
# ------------------------------------------------------------------------------------------------------------
def _engine(cfg, sd, dev):
    from yume_b200.dit import WanDiT
    kw = synth.oracle_kwargs(cfg)
    variant = kw.pop("variant")
    return WanDiT(sd, variant, device=dev, **kw)


@pytest.fixture(scope="module")
def tiny5(dev, golden_dir):
    g = torch.load(golden_dir / "wan23_tiny.pt", weights_only=False)
    sd = synth.make_state_dict(g["cfg"], g["seed_w"])
    return g, sd, _engine(g["cfg"], sd, dev)


@pytest.fixture(scope="module")
def tiny14(dev, golden_dir):
    g = torch.load(golden_dir / "wan21_tiny.pt", weights_only=False)
    sd = synth.make_state_dict(g["cfg"], g["seed_w"])
    return g, sd, _engine(g["cfg"], sd, dev)


def test_single_block_config0(tiny5):
    """BASELINE.json configs[0]: one WanAttentionBlock, 128 tokens (grid 2x8x8), vs the reference output."""
    g, sd, eng = tiny5
    cfg, b = g["cfg"], g["block"]
    gen = torch.Generator().manual_seed(b["seed"])
    L, C = b["L"], cfg["dim"]
    x = torch.randn(1, L, C, generator=gen)
    e = 0.5 * torch.randn(1, L, 6, C, generator=gen)
    ctx = torch.randn(1, cfg["text_len"], C, generator=gen)
    y = eng.block_forward(0, x[0], e[0], b["grid"], ctx[0]).cpu()
    delta_ref = b["out"][0] - x[0]
    delta = y - x[0]
    assert float((delta - delta_ref).norm() / delta_ref.norm()) < BLOCK_TOL_REL
    # bf16-rounded context differs from the fp32 one the reference saw; abs tolerance covers it
    assert float((y - b["out"][0]).abs().max()) < BLOCK_TOL_ABS * max(1.0, float(b["out"].abs().mean()))


@pytest.mark.parametrize("case", ["5b_grid", "5b_grid_padded", "5b_pack_h3", "5b_pack_h1", "5b_pack_h10",
                                  "5b_pack_h30", "5b_pack_h100", "5b_pack_h400"])
def test_5b_forward_vs_reference_golden(tiny5, case):
    g, sd, eng = tiny5
    c, cfg = g["cases"][case], g["cfg"]
    inp = synth.make_inputs(cfg, c["seed"], c["frames"], c["H"], c["W"], c["ctx_len"])
    out = eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], latent_frame_zero=c["lfz"],
                      packed=c["flag"])
    assert out.shape == c["out"].shape
    assert rel(out, c["out"]) < MODEL_TOL


@pytest.mark.parametrize("case", ["14b_grid", "14b_pack_h4", "14b_pack_lfz8", "14b_pack_h12"])
def test_14b_forward_vs_reference_golden(tiny14, case):
    g, sd, eng = tiny14
    c, cfg = g["cases"][case], g["cfg"]
    inp = synth.make_inputs(cfg, c["seed"], c["frames"], c["H"], c["W"], c["ctx_len"])
    out = eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], y=inp["y"], clip_fea=inp["clip_fea"],
                      latent_frame_zero=c["lfz"], packed=c["rand_num_img"] >= 0.4)
    assert out.shape == c["out"].shape
    assert rel(out, c["out"]) < MODEL_TOL


@pytest.mark.parametrize("fname,case", [("wan23_h8.pt", "5b_grid"), ("wan23_h8.pt", "5b_grid_padded"), ("wan23_h8.pt", "5b_pack_h10"),
                                        ("wan23_h8.pt", "5b_pack_h30"), ("wan21_h8.pt", "14b_grid"),
                                        ("wan21_h8.pt", "14b_grid_padded"), ("wan21_h8.pt", "14b_pack_lfz8")])
def test_h8_forward_vs_reference_golden(dev, golden_dir, fname, case):
    """8-head (dim 1024) models: the goldens the Ulysses parity at world 2/4/8 uses, on one GPU. 14b_grid_padded has
    seq_len > F*H*W: the 14B tree masks the padded rows as keys (wan/modules/model.py:311-314), the 5B tree does not."""
    g = torch.load(golden_dir / fname, weights_only=False)
    cfg, c = g["cfg"], g["cases"][case]
    eng = _engine(cfg, synth.make_state_dict(cfg, g["seed_w"]), dev)
    inp = synth.make_inputs(cfg, c["seed"], c["frames"], c["H"], c["W"], c["ctx_len"])
    if cfg["variant"] == "5b":
        out = eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], latent_frame_zero=c["lfz"],
                          packed=c["flag"])
    else:
        out = eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], y=inp["y"], clip_fea=inp["clip_fea"],
                          latent_frame_zero=c["lfz"], packed=c["rand_num_img"] >= 0.4)
    assert out.shape == c["out"].shape
    assert rel(out, c["out"]) < MODEL_TOL


def test_mirror_module_keeps_reference_signature(tiny5, dev):
    """WanModel5B built on the meta device + install(state_dict): forward(x list, t, context list, seq_len, ...)."""
    from yume_b200.model import WanModel5B
    g, sd, _ = tiny5
    cfg, c = g["cfg"], g["cases"]["5b_pack_h10"]
    with torch.device("meta"):
        m = WanModel5B(model_type="ti2v", text_len=cfg["text_len"], in_dim=cfg["in_dim"], dim=cfg["dim"],
                       ffn_dim=cfg["ffn_dim"], freq_dim=cfg["freq_dim"], text_dim=cfg["text_dim"], out_dim=cfg["out_dim"],
                       num_heads=cfg["num_heads"], num_layers=cfg["num_layers"])
    m.install(dev, state_dict=sd)
    inp = synth.make_inputs(cfg, c["seed"], c["frames"], c["H"], c["W"], c["ctx_len"])
    outs = m([inp["x"]], torch.tensor(c["t"]), [inp["context"]], seq_len=c["seq_len"], latent_frame_zero=c["lfz"], flag=True)
    assert isinstance(outs, list) and outs[0].dtype == torch.float32
    assert rel(outs[0], c["out"]) < MODEL_TOL
    with pytest.raises(NotImplementedError):
        m([inp["x"]], torch.tensor(c["t"]), [inp["context"]], seq_len=c["seq_len"], enable_mask=True)


def _mirror5(cfg, sd, dev):
    from yume_b200.model import WanModel5B
    with torch.device("meta"):
        m = WanModel5B(model_type="ti2v", text_len=cfg["text_len"], in_dim=cfg["in_dim"], dim=cfg["dim"],
                       ffn_dim=cfg["ffn_dim"], freq_dim=cfg["freq_dim"], text_dim=cfg["text_dim"], out_dim=cfg["out_dim"],
                       num_heads=cfg["num_heads"], num_layers=cfg["num_layers"])
    return m.install(dev, state_dict=sd)


def test_block_and_self_attention_seams_keep_reference_signatures(tiny5, dev):
    """SURVEY.md §8(b): `WanAttentionBlock.forward` / `WanSelfAttention.forward` with the reference's argument lists,
    bound by install_seams. Block seam vs the reference block output (configs[0] fixture, grid path) and vs the oracle on
    the FramePack path (per-token complex freqs); self-attention seam vs the oracle's self_attn."""
    import yume_b200
    from oracle.wan_dit import grid_freqs
    g, sd, _ = tiny5
    cfg, b = g["cfg"], g["block"]
    m = yume_b200.install_seams(_mirror5(cfg, sd, dev))
    gen = torch.Generator().manual_seed(b["seed"])
    L, C = b["L"], cfg["dim"]
    x = torch.randn(1, L, C, generator=gen)
    e = 0.5 * torch.randn(1, L, 6, C, generator=gen)
    ctx = torch.randn(1, cfg["text_len"], C, generator=gen)
    orc = WanOracle(sd, **synth.oracle_kwargs(cfg))
    tables = torch.cat(orc.tables, dim=1)                                  # the [1024, 64] table the reference passes on the grid path
    y = m.blocks[0](x.to(dev), e.to(dev), torch.tensor([L]), torch.tensor([[2, 8, 8]]), tables, ctx.to(dev), None, flag=False)
    assert y.shape == (1, L, C) and y.dtype == torch.float32
    d_ref, d = b["out"][0] - x[0], y[0].cpu() - x[0]
    assert float((d - d_ref).norm() / d_ref.norm()) < BLOCK_TOL_REL
    # FramePack path: per-token complex table (model.py:101-105), a temporal offset so it differs from the plain grid
    fr = grid_freqs(orc.tables, 2, 8, 8, f0=3)
    want = orc.block(1, x, e, fr, ctx)[0]
    got = m.blocks[1](x.to(dev), e.to(dev), torch.tensor([L]), None, fr.to(dev), ctx.to(dev), None, flag=True)[0].cpu()
    assert float(((got - x[0]) - (want - x[0])).norm() / (want - x[0]).norm()) < BLOCK_TOL_REL
    # self-attention seam: o(attention(rope(norm(q)), rope(norm(k)), v))
    h = torch.randn(1, L, C, generator=gen)
    want_sa = orc.self_attn("blocks.0.self_attn", h, fr)[0]
    got_sa = m.blocks[0].self_attn(h.to(dev), torch.tensor([L]), None, fr.to(dev), None, None, None, True)[0]
    assert got_sa.dtype == torch.bfloat16 and rel(got_sa, want_sa) < 1e-2
    with pytest.raises(NotImplementedError):
        m.blocks[0](x.to(dev), e.to(dev), torch.tensor([L]), None, fr.to(dev), ctx.to(dev), None, ids_keep=torch.zeros(1, 4))


def test_flash_attention_shim_keeps_reference_contract(dev):
    """`flash_attention(q, k, v, k_lens=...)` with the reference's layout [B, L, N, D], dtype behaviour (fp32 in -> fp32
    out, computed in bf16) and k_lens masking (wan23/modules/attention.py:24-130), B = 2."""
    import yume_b200
    g = torch.Generator(device="cpu").manual_seed(17)
    B, Lq, Lk, N = 2, 200, 333, 2
    q, k, v = (torch.randn(B, L_, N, 128, generator=g).to(dev) for L_ in (Lq, Lk, Lk))
    k_lens = torch.tensor([333, 150])
    out = yume_b200.flash_attention(q, k, v, k_lens=k_lens)
    assert out.shape == (B, Lq, N, 128) and out.dtype == torch.float32
    for i in range(B):
        kl = int(k_lens[i])
        ref = _sdpa(q[i].bfloat16().reshape(Lq, N * 128), k[i, :kl].bfloat16().reshape(kl, N * 128),
                    v[i, :kl].bfloat16().reshape(kl, N * 128), N)
        assert rel(out[i].reshape(Lq, N * 128), ref) < KERNEL_TOL
    half = yume_b200.flash_attention(q.bfloat16(), k.bfloat16(), v.bfloat16(), softmax_scale=0.05)
    assert half.dtype == torch.bfloat16 and bool(torch.isfinite(half.float()).all())
    with pytest.raises(NotImplementedError):
        yume_b200.flash_attention(q, k, v, causal=True)
    with pytest.raises(AssertionError):
        yume_b200.flash_attention(q.cpu(), k.cpu(), v.cpu())               # the reference asserts CUDA too (attention.py:54)


def test_sampler_loop_cache_and_cuda_graph_match_plain_forwards(tiny5, dev):
    """Sampler-loop fusion (SURVEY.md §8(f) rank 2): the 4-step 5B loop with the context cache on, and again replayed from a
    CUDA graph, gives the result of the same loop with every forward computed from scratch."""
    from yume_b200 import sampler
    g, sd, _ = tiny5
    cfg = g["cfg"]
    m = _mirror5(cfg, sd, dev)
    eng = m._yb_engine
    gen = torch.Generator().manual_seed(23)
    hist = torch.randn(48, 5, 6, 10, generator=gen).to(dev)
    noise = torch.randn(48, 2, 6, 10, generator=gen).to(dev)
    ctx = torch.randn(20, cfg["text_dim"], generator=gen).to(dev).bfloat16()
    arg_c = dict(context=[ctx], seq_len=0)

    def loop():
        return sampler.denoise_chunk_5b(m, torch.cat([hist, noise], 1), hist, 2, 4, arg_c, shift=7.0)
    eng.context_cache, eng.use_cuda_graph = False, False
    plain = loop()
    eng.context_cache = True
    cached = loop()
    assert torch.equal(cached, plain)
    eng.use_cuda_graph = True
    graphed = loop()
    graphed2 = loop()                                                      # second pass replays the captured graphs
    assert torch.equal(graphed, plain) and torch.equal(graphed2, plain)
    assert len(eng._graphs) >= 1
    ctx2 = (ctx.float() * 0.5).bfloat16()                                  # a NEW context tensor must not hit the old entry
    other = sampler.denoise_chunk_5b(m, torch.cat([hist, noise], 1), hist, 2, 4, dict(context=[ctx2], seq_len=0), shift=7.0)
    assert not torch.equal(other, plain)
    ctx.mul_(0.5)                                                          # in-place edit bumps _version: recomputed, same as ctx2
    assert torch.equal(loop(), other)


def test_oracle_block_at_real_width(dev):
    """One block at the real 5B width (C=3072, 24 heads, F=14336), L=256: CUDA vs oracle (seconds on CPU)."""
    cfg = dict(synth.CFG_5B, num_layers=1, text_len=64)
    sd = synth.make_state_dict(cfg, 77, num_layers=1)
    eng = _engine(cfg, sd, dev)
    gen = torch.Generator().manual_seed(9)
    L, C = 256, cfg["dim"]
    x = torch.randn(1, L, C, generator=gen)
    e = 0.5 * torch.randn(1, L, 6, C, generator=gen)
    ctx = torch.randn(1, 64, C, generator=gen).bfloat16().float()
    m = WanOracle(sd, **synth.oracle_kwargs(cfg))
    want = m.block(0, x, e, grid_freqs(m.tables, 4, 8, 8), ctx)[0]
    got = eng.block_forward(0, x[0], e[0], (4, 8, 8), ctx[0]).cpu()
    d_ref, d = want - x[0], got - x[0]
    assert float((d - d_ref).norm() / d_ref.norm()) < BLOCK_TOL_REL
    assert float((got - want).abs().max()) < BLOCK_TOL_ABS * max(1.0, float(want.abs().mean()))


def test_oracle_block_at_real_width_14b(dev):
    """One block at the real 14B width (C=5120, 40 heads, F=13824, 257 CLIP + 64 text context rows -> the k_img/v_img
    branch and the C=5120 template instances of the glue kernels), L=256: CUDA vs oracle. Same bar as configs[0]."""
    cfg = dict(synth.CFG_14B, num_layers=1, text_len=64)
    sd = synth.make_state_dict(cfg, 78, num_layers=1)
    eng = _engine(cfg, sd, dev)
    gen = torch.Generator().manual_seed(10)
    L, C = 256, cfg["dim"]
    x = torch.randn(1, L, C, generator=gen)
    e = 0.5 * torch.randn(1, 6, C, generator=gen)                      # 14B: per-sample modulation [B, 6, C]
    ctx = torch.randn(1, 257 + 64, C, generator=gen).bfloat16().float()
    m = WanOracle(sd, **synth.oracle_kwargs(cfg))
    want = m.block(0, x, e, grid_freqs(m.tables, 4, 8, 8), ctx)[0]
    got = eng.block_forward(0, x[0], e[0], (4, 8, 8), ctx[0]).cpu()
    d_ref, d = want - x[0], got - x[0]
    assert float((d - d_ref).norm() / d_ref.norm()) < BLOCK_TOL_REL
    assert float((got - want).abs().max()) < BLOCK_TOL_ABS * max(1.0, float(want.abs().mean()))


# ------------------------------------------------------------------------------------------------------------
# full-size properties (BASELINE.json configs[1] geometry: L = 18480, 24 heads) — no oracle needed
# ------------------------------------------------------------------------------------------------------------
def test_fullsize_attention_is_key_permutation_invariant(dev):
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(21)
    L, heads = 18480, 2
    q = torch.randn(L, heads * 128, generator=g).to(dev).bfloat16()
    k = torch.randn(L, heads * 128, generator=g).to(dev).bfloat16()
    v = torch.randn(L, heads * 128, generator=g).to(dev).bfloat16()
    o1 = torch.empty_like(q)
    o2 = torch.empty_like(q)
    ops.attention(q, k, v, o1, heads)
    perm = torch.randperm(L, generator=g).to(dev)
    ops.attention(q, k[perm].contiguous(), v[perm].contiguous(), o2, heads)
    assert rel(o1, o2) < 5e-3                          # two independently bf16-rounded outputs: sqrt(2) x rounding noise
    idx = torch.randint(0, L, (256,), generator=g).to(dev)
    assert rel(o1[idx], _sdpa(q[idx].contiguous(), k, v, heads)) < KERNEL_TOL


def test_fullsize_gemm_linearity_and_row_independence(dev):
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(22)
    M, N, K = 18480, 3072, 3072
    a1 = (torch.randn(M, K, generator=g) * 0.5).to(dev).bfloat16()
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dev).bfloat16()
    o1 = torch.empty(M, N, device=dev)
    ops.gemm(a1, w, None, o1, ops.YB_EPI_F32)
    o2 = torch.empty(M, N, device=dev)
    ops.gemm((a1.float() * 2).bfloat16(), w, None, o2, ops.YB_EPI_F32)     # exact scaling by 2 in bf16
    assert torch.equal(o2, o1 * 2)
    rows = torch.randint(0, M, (300,), generator=g).to(dev)
    sub = torch.empty(300, N, device=dev)
    ops.gemm(a1[rows].contiguous(), w, None, sub, ops.YB_EPI_F32)
    assert torch.equal(sub, o1[rows])                                      # a row's result does not depend on its tile
    assert rel(o1[rows], a1[rows].float() @ w.float().t()) < 1e-4


@pytest.mark.parametrize("world,transport,split", [(2, "p2p", "0"), (2, "p2p_gemm", "0"), (2, "nccl", "0"), (4, "p2p", "0"),
                                                   (4, "p2p_gemm", "0"), (4, "nccl", "0"), (8, "p2p", "0"), (8, "p2p_gemm", "0"),
                                                   (8, "nccl", "0"), (2, "p2p", "2"), (8, "p2p_gemm", "2")])
def test_ulysses_matches_golden(dev, world, transport, split):
    """Sequence-parallel forward on `world` GPUs (torchrun) vs the reference-generated golden outputs: the 2-head tiny
    models at world 2, the 8-head (dim 1024) models at world 2 / 4 / 8; every transport (NVLink peer-memory kernels with the
    q|k|v exchange in the norm/RoPE pass or in the QKV GEMM's epilogue, NCCL all-to-all); split = forced KV tail split of the attention launch through the peer-scatter combine kernel.
    Skipped on boxes with fewer GPUs — bench.py's `parity_vs_n1` carries the same check on every multi-GPU bench line."""
    import subprocess
    import sys
    from pathlib import Path
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    root = Path(__file__).resolve().parents[1]
    env = dict(os.environ, YB_SP_TRANSPORT=transport)
    if split != "0":
        env["YB_ATT_FORCE_SPLIT"] = split
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29533 + world), str(root / "tools" / "sp_parity.py")],
                       capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


# ------------------------------------------------------------------------------------------------------------
# hyvideo causal 3D VAE decode (SURVEY.md §8 a17-a19)
# ------------------------------------------------------------------------------------------------------------
VAE_TOL = 3e-2   # ~35 bf16 conv/norm layers deep; fp32 oracle / reference fixtures
VAE_PSNR_DB = 40.0   # the same bar as an image metric: decoded video lives in [-1, 1] (peak-to-peak 2); rel-Fro 3e-2 on an output
                     # of RMS ~0.5 is ~42 dB. The Wan VAEs run in fp32 in the reference (vae2_2.py:918): this is the error budget
                     # of multiplying in bf16 (fp32 accumulation, fp32 norms / softmax) instead.


def psnr(got, want):
    """PSNR in dB against the reference's own dynamic range (2 for a clamped [-1, 1] video; random-init fixtures can be wider)."""
    want = want.float().cpu()
    mse = float((got.float().cpu() - want).pow(2).mean())
    peak = max(2.0, float(want.max() - want.min()))
    return 10.0 * math.log10(peak * peak / max(mse, 1e-20))


@pytest.mark.parametrize("T,H,W,ci,co", [(3, 8, 8, 64, 64), (2, 6, 10, 128, 128), (5, 32, 32, 64, 256), (1, 18, 32, 128, 96),
                                         (9, 4, 4, 64, 32), (2, 3, 200, 64, 128), (3, 2, 256, 128, 256), (2, 10, 24, 64, 192),
                                         (3, 9, 17, 128, 384)])
@pytest.mark.parametrize("fuse_w", [1, 2])
def test_conv3d_causal_matches_torch(dev, T, H, W, ci, co, fuse_w):
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(T * 100 + H)
    x = torch.randn(T * H * W, ci, generator=g).to(dev).bfloat16()
    wt = (torch.randn(co, ci, 3, 3, 3, generator=g) / math.sqrt(27 * ci)).to(dev).bfloat16()
    b = torch.randn(co, generator=g).to(dev)
    res = torch.randn(T * H * W, co, generator=g).to(dev).bfloat16()
    xpad = torch.empty(T + 2, H + 2, W + 2, ci, device=dev, dtype=torch.bfloat16)
    ops.vae_pad_act(x, (T, H, W), xpad, True)
    xn = x.float().view(T, H, W, ci).permute(3, 0, 1, 2)[None]
    want_pad = torch.nn.functional.pad(xn, (1, 1, 1, 1, 2, 0), mode="replicate")
    assert torch.equal(xpad.float().permute(3, 0, 1, 2)[None], want_pad)            # replicate padding is bit-exact
    wk = wt.permute(0, 2, 3, 4, 1).reshape(co, 27 * ci).contiguous()
    out = torch.empty(T * H * W, co, device=dev, dtype=torch.bfloat16)
    ops.conv3d_causal(xpad, wk, b, out, T, H, W, ops.YB_EPI_RES_BF16, res, fuse_w=fuse_w, cta_pair=2)   # 1-CTA kernel
    ref = torch.nn.functional.conv3d(want_pad, wt.float(), b)[0].permute(1, 2, 3, 0).reshape(T * H * W, co) + res.float()
    assert rel(out, ref) < KERNEL_TOL
    o32 = torch.empty(T * H * W, co, device=dev)
    ops.conv3d_causal(xpad, wk, None, o32, T, H, W, ops.YB_EPI_F32, fuse_w=fuse_w, cta_pair=2)
    assert rel(o32, ref - res.float() - b) < 1e-4
    if fuse_w == 1:   # SM-pair conv kernel (forced; automatic for 192 / 384 outputs): the 1-CTA un-fused result bit for bit
        pair = torch.full_like(out, 3.0)
        ops.conv3d_causal(xpad, wk, b, pair, T, H, W, ops.YB_EPI_RES_BF16, res, cta_pair=1)
        assert torch.equal(pair, out)
        p32 = torch.empty_like(o32)
        ops.conv3d_causal(xpad, wk, None, p32, T, H, W, ops.YB_EPI_F32, cta_pair=1)
        assert torch.equal(p32, o32)


def test_vae_glue_kernels(dev):
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(8)
    Ts, Hs, Ws, C, G = 3, 5, 6, 64, 32
    x = (torch.randn(Ts * Hs * Ws, C, generator=g) * 2 + 0.5).to(dev).bfloat16()
    gamma, beta = torch.randn(C, generator=g).to(dev), torch.randn(C, generator=g).to(dev)
    st = ops.gn_stats(x, G)
    xg = x.float().view(-1, G, C // G)
    assert torch.allclose(st[:, 0], xg.sum((0, 2)).double(), rtol=1e-4, atol=1e-2)
    assert torch.allclose(st[:, 1], (xg * xg).sum((0, 2)).double(), rtol=1e-4)
    # GroupNorm + SiLU + (2,2,2) upsample + replicate pad in one pass vs the four torch ops
    T, H, W = 1 + 2 * (Ts - 1), 2 * Hs, 2 * Ws
    out = torch.empty(T + 2, H + 2, W + 2, C, device=dev, dtype=torch.bfloat16)
    ops.vae_pad_act(x, (Ts, Hs, Ws), out, True, (2, 2, 2), st, gamma, beta, G, 1e-6, True)
    xn = x.float().view(Ts, Hs, Ws, C).permute(3, 0, 1, 2)[None]
    y = torch.nn.functional.silu(torch.nn.functional.group_norm(xn, G, gamma, beta, eps=1e-6))
    first = torch.nn.functional.interpolate(y[:, :, 0], scale_factor=(2, 2), mode="nearest")[:, :, None]
    other = torch.nn.functional.interpolate(y[:, :, 1:], scale_factor=(2, 2, 2), mode="nearest")
    want = torch.nn.functional.pad(torch.cat([first, other], 2), (1, 1, 1, 1, 2, 0), mode="replicate")
    assert rel(out.float().permute(3, 0, 1, 2)[None], want) < KERNEL_TOL
    # frame-causal softmax
    L, hw = 96, 32
    S = torch.randn(L, L, generator=g).to(dev)
    P = torch.empty(L, L, device=dev, dtype=torch.bfloat16)
    ops.masked_softmax(S, P, L, hw)
    fr = torch.arange(L, device=dev) // hw
    wantP = torch.where(fr[:, None] >= fr[None, :], S, torch.full_like(S, float("-inf"))).softmax(-1)
    assert rel(P, wantP) < KERNEL_TOL
    # cross-fade and layout converters
    a, b = torch.randn(1, 3, 4, 10, 7, generator=g).to(dev), torch.randn(1, 3, 4, 6, 7, generator=g).to(dev)
    want = b.clone()
    for yy in range(4):
        want[:, :, :, yy] = a[:, :, :, -4 + yy] * (1 - yy / 4) + want[:, :, :, yy] * (yy / 4)
    assert torch.allclose(ops.blend(a, b, 3, 4), want, atol=1e-6)
    z = torch.randn(16, 40, generator=g).to(dev)
    zl = torch.empty(40, 64, device=dev, dtype=torch.bfloat16)
    ops.nchw_to_nhwc_bf16(z, zl)
    assert torch.equal(zl[:, :16].float(), z.t().bfloat16().float()) and not zl[:, 16:].any()


@pytest.fixture(scope="module")
def vae_gold(dev, golden_dir):
    from oracle import hyvae
    g = torch.load(golden_dir / "hyvae_tiny.pt", weights_only=False)
    return g, hyvae.make_state_dict(g["seed_w"], **g["cfg"])


@pytest.mark.parametrize("case", ["untiled", "untiled_t1", "spatial_tiled", "temporal_spatial_tiled"])
def test_vae_decode_vs_reference_golden(dev, vae_gold, case):
    from yume_b200.vae import HyVaeDecoder
    g, sd = vae_gold
    c = g["cases"][case]
    eng = HyVaeDecoder(sd, sample_size=c["sample_size"], sample_tsize=c["sample_tsize"], device=dev, **g["cfg"])
    eng.enable_tiling(c["tiling"])
    z = torch.randn(1, 16, c["T"], c["H"], c["W"], generator=torch.Generator().manual_seed(c["seed"]))
    out = eng.decode(z).cpu()
    assert tuple(out.shape) == c["shape"]
    for name, got in (("sample", out[..., ::3, ::3]), ("rowsum", out.sum(-1)), ("colsum", out.sum(-2))):
        assert float((got - c[name]).norm() / c[name].norm()) < VAE_TOL, name
        assert psnr(got, c[name]) > VAE_PSNR_DB, name


def test_vae_decode_real_width_tile_vs_oracle(dev):
    """One small tile at the REAL channel widths (128/256/512/512) against the fp32 oracle."""
    from oracle import hyvae
    from yume_b200.vae import HyVaeDecoder
    cfg = dict(block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=16, out_channels=3)
    sd = hyvae.make_state_dict(99, **cfg)
    z = torch.randn(1, 16, 2, 4, 4, generator=torch.Generator().manual_seed(5))
    want = hyvae.HyVaeOracle(sd, **cfg).decode(z)
    got = HyVaeDecoder(sd, device=dev, **cfg).decode(z).cpu()
    assert got.shape == want.shape and rel(got, want) < VAE_TOL and psnr(got, want) > VAE_PSNR_DB


# ---- Wan2.2 VAE (wan23/modules/vae2_2.py) -------------------------------------------------------------------------
@pytest.mark.parametrize("taps,T,H,W,ci,co,tm,ta", [((3, 3, 3), 3, 8, 8, 64, 64, 1, 0), ((1, 3, 3), 4, 6, 10, 128, 96, 1, 0),
                                                     ((3, 1, 1), 3, 5, 8, 64, 128, 2, 1), ((3, 1, 1), 3, 5, 8, 64, 128, 2, 2),
                                                     ((3, 3, 3), 1, 18, 32, 128, 32, 1, 0), ((3, 3, 3), 5, 40, 24, 64, 64, 1, 0),
                                                     ((1, 3, 3), 2, 130, 9, 64, 64, 1, 0), ((3, 3, 3), 2, 5, 300, 128, 256, 1, 0),
                                                     ((1, 3, 3), 3, 4, 129, 64, 96, 1, 0)])
@pytest.mark.parametrize("fuse_w", [1, 2])
def test_conv3d_zero_pad_tap_modes(dev, taps, T, H, W, ci, co, tm, ta, fuse_w):
    """CausalConv3d with ZERO padding taken from TMA out-of-bounds fill, (kt,kh,kw) taps and interleaved output frames."""
    from yume_b200 import ops
    kt, kh, kw = taps
    g = torch.Generator(device="cpu").manual_seed(T * 100 + H + kt)
    x = torch.randn(T, H, W, ci, generator=g).to(dev).bfloat16()
    wt = (torch.randn(co, ci, kt, kh, kw, generator=g) / math.sqrt(kt * kh * kw * ci)).to(dev).bfloat16()
    b = torch.randn(co, generator=g).to(dev)
    wk = wt.permute(0, 2, 3, 4, 1).reshape(co, kt * kh * kw * ci).contiguous()
    To = (T - 1) * tm + ta + 1
    out = torch.full((To * H * W, co), 7.0, device=dev, dtype=torch.bfloat16)
    ops.conv3d_causal(x, wk, b, out, T, H, W, ops.YB_EPI_BF16, taps=taps, oob_zero_pad=True, out_t_mul=tm, out_t_add=ta,
                      fuse_w=fuse_w)
    xn = torch.nn.functional.pad(x.float().permute(3, 0, 1, 2)[None], (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0))
    ref = torch.nn.functional.conv3d(xn, wt.float(), b)[0].permute(1, 2, 3, 0)             # [T, H, W, co]
    got = out.view(To, H, W, co).float()
    written = torch.zeros(To, dtype=torch.bool)
    written[ta::tm][:T] = True
    assert rel(got[written.to(dev)], ref) < KERNEL_TOL
    assert bool((got[(~written).to(dev)] == 7.0).all())                                     # other frames untouched


def test_wan22_vae_glue_kernels(dev):
    from oracle import wan22vae
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(21)
    T, H, W, C = 3, 4, 6, 96
    x = (torch.randn(T * H * W, C, generator=g) * 1.5).to(dev).bfloat16()
    gamma = (1 + 0.1 * torch.randn(C, generator=g)).to(dev)
    xn = x.float().view(T, H, W, C).permute(3, 0, 1, 2)[None]                              # [1, C, T, H, W]
    # RMS_norm * gamma, SiLU, nearest-exact 2x, channel pad to 128
    out = torch.empty(T, 2 * H, 2 * W, 128, device=dev, dtype=torch.bfloat16)
    ops.vae_rms_act(x, (T, H, W), out, gamma, 2, True)
    y = torch.nn.functional.silu(wan22vae.rms_norm(xn, gamma))[0].permute(1, 0, 2, 3)       # [T, C, H, W]
    y = torch.nn.functional.interpolate(y, scale_factor=(2.0, 2.0), mode="nearest-exact").permute(0, 2, 3, 1)
    assert rel(out[..., :C], y) < 6e-3 and bool((out[..., C:] == 0).all())
    out1 = torch.empty(T, H, W, 128, device=dev, dtype=torch.bfloat16)
    ops.vae_rms_act(x, (T, H, W), out1, None, 1, False)                                     # plain channel-pad copy
    assert torch.equal(out1[..., :C].reshape(-1, C), x)
    # DupUp3D shortcut add, both factor_t, against the oracle's whole-sequence form
    for ft, co in ((2, 48), (1, 96), (2, 96)):
        To = ft * T - (ft - 1)
        main = torch.randn(To * 2 * H * 2 * W, co, generator=g).to(dev).bfloat16()
        want = main.float().view(To, 2 * H, 2 * W, co) + wan22vae.Wan22VaeOracle.dup_up(xn, co, ft, 2)[0].permute(1, 2, 3, 0)
        ops.vae_dupup_add(main, x, (T, H, W), C, co, ft, 2)
        assert rel(main.view(To, 2 * H, 2 * W, co), want) < 6e-3
    # head: [N, 32] f32 (12 used) -> unpatchify(2) + clamp
    yh = (torch.randn(T * H * W, 32, generator=g) * 0.8).to(dev)
    o = torch.empty(3, T, 2 * H, 2 * W, device=dev)
    ops.vae_unpatchify2_clamp(yh, o, T, H, W)
    v = yh[:, :12].view(T, H, W, 12).permute(3, 0, 1, 2)[None]
    want = v.view(1, 3, 2, 2, T, H, W).permute(0, 1, 4, 5, 3, 6, 2).reshape(3, T, 2 * H, 2 * W).clamp(-1, 1)
    assert torch.equal(o, want)


@pytest.fixture(scope="module")
def vae22_gold(dev, golden_dir):
    from oracle import wan22vae
    g = torch.load(golden_dir / "wan22vae_tiny.pt", weights_only=False)
    return g, wan22vae.make_state_dict(g["seed_w"], **g["cfg"])


@pytest.mark.parametrize("case", ["t1", "t2", "t5", "t3_wide"])
def test_wan22_vae_decode_vs_reference_golden(dev, vae22_gold, case):
    """One-pass whole-sequence decode on the GPU against the reference's own chunked / feature-cached decode."""
    from yume_b200.vae22 import Wan22VaeDecoder
    g, sd = vae22_gold
    c = g["cases"][case]
    eng = Wan22VaeDecoder(sd, mean=g["mean"], std=g["std"], device=dev, **g["cfg"])
    z = torch.randn(g["cfg"]["z_dim"], c["T"], c["H"], c["W"], generator=torch.Generator().manual_seed(c["seed"]))
    out = eng.decode(z).cpu()
    assert tuple(out.shape) == c["shape"]
    for name, got in (("sample", out[..., ::3, ::3]), ("rowsum", out.sum(-1)), ("colsum", out.sum(-2))):
        assert float((got - c[name]).norm() / c[name].norm()) < VAE_TOL, name
        assert psnr(got, c[name]) > VAE_PSNR_DB, name


def test_wan22_vae_decode_real_width_vs_oracle(dev):
    """Real channel widths (dec_dim 256, z_dim 48 -> 1024/1024/1024/512/256) on a small latent against the fp32 oracle."""
    from oracle import wan22vae
    from yume_b200.vae22 import Wan22VaeDecoder
    cfg = dict(dec_dim=256, z_dim=48, dim_mult=(1, 2, 4, 4), num_res_blocks=2, temperal_upsample=(True, True, False))
    sd = wan22vae.make_state_dict(31, **cfg)
    gen = torch.Generator().manual_seed(6)
    mean, std = 0.2 * torch.randn(48, generator=gen), 0.5 + torch.rand(48, generator=gen)
    z = torch.randn(48, 2, 2, 4, generator=gen)
    want = wan22vae.Wan22VaeOracle(sd, mean=mean, std=std, **cfg).decode(z)
    got = Wan22VaeDecoder(sd, mean=mean, std=std, device=dev, **cfg).decode(z).cpu()
    assert got.shape == want.shape and rel(got, want) < VAE_TOL and psnr(got, want) > VAE_PSNR_DB


# ---- Wan2.1 VAE (wan/modules/vae.py) ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def vae21_gold(dev, golden_dir):
    from oracle import wan21vae
    g = torch.load(golden_dir / "wan21vae_tiny.pt", weights_only=False)
    return g, wan21vae.make_state_dict(g["seed_w"], **g["cfg"])


@pytest.mark.parametrize("case", ["t1", "t2", "t5", "t3_wide"])
def test_wan21_vae_decode_vs_reference_golden(dev, vae21_gold, case):
    from yume_b200.vae21 import Wan21VaeDecoder
    g, sd = vae21_gold
    c = g["cases"][case]
    eng = Wan21VaeDecoder(sd, mean=g["mean"], std=g["std"], device=dev, **g["cfg"])
    z = torch.randn(g["cfg"]["z_dim"], c["T"], c["H"], c["W"], generator=torch.Generator().manual_seed(c["seed"]))
    out = eng.decode(z).cpu()
    assert tuple(out.shape) == c["shape"]
    for name, got in (("sample", out[..., ::3, ::3]), ("rowsum", out.sum(-1)), ("colsum", out.sum(-2))):
        assert float((got - c[name]).norm() / c[name].norm()) < VAE_TOL, name
        assert psnr(got, c[name]) > VAE_PSNR_DB, name


def test_wan21_vae_decode_real_width_vs_oracle(dev):
    """Real channel widths (dim 96 -> 384/192/96, z16) on a small latent against the fp32 oracle."""
    from oracle import wan21vae
    from yume_b200.vae21 import Wan21VaeDecoder
    cfg = dict(dim=96, z_dim=16, dim_mult=(1, 2, 4, 4), num_res_blocks=2, temperal_upsample=(True, True, False))
    sd = wan21vae.make_state_dict(41, **cfg)
    gen = torch.Generator().manual_seed(7)
    mean, std = 0.2 * torch.randn(16, generator=gen), 0.5 + torch.rand(16, generator=gen)
    z = torch.randn(16, 3, 4, 6, generator=gen)
    want = wan21vae.Wan21VaeOracle(sd, mean=mean, std=std, **cfg).decode(z)
    got = Wan21VaeDecoder(sd, mean=mean, std=std, device=dev, **cfg).decode(z).cpu()
    assert got.shape == want.shape and rel(got, want) < VAE_TOL and psnr(got, want) > VAE_PSNR_DB
    assert float(got.min()) >= -1.0 and float(got.max()) <= 1.0


# ---- Wan VAE ENCODE (SURVEY.md §8(f) rank 3): strided Resample convs, AvgDown3D shortcut, whole-sequence encoders ------------
@pytest.mark.parametrize("T,H,W,ci,co", [(1, 16, 32, 64, 32), (3, 9, 14, 64, 64), (2, 44, 80, 128, 96), (5, 8, 258, 192, 160),
                                         (1, 130, 6, 64, 320)])
def test_conv3d_stride2_spatial_matches_torch(dev, T, H, W, ci, co):
    """`Resample(downsample2d)`: ZeroPad2d((0,1,0,1)) + Conv2d(3x3, stride 2) per frame (vae2_2.py:101-104), the stride taken by
    the tensor map (TMA elementStrides), the pad row / column behind the data by out-of-bounds fill; odd H / W included."""
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(T * 1000 + H * 10 + W)
    x = torch.randn(T, H, W, ci, generator=g).to(dev).bfloat16()
    wt = (torch.randn(co, ci, 3, 3, generator=g) / math.sqrt(9 * ci)).to(dev).bfloat16()
    b = torch.randn(co, generator=g).to(dev)
    wk = wt.permute(0, 2, 3, 1).reshape(co, 9 * ci).contiguous()
    To, Ho, Wo = ops.conv_out_dims(T, H, W, (1, 3, 3), 1, 2)
    ref = torch.nn.functional.conv2d(torch.nn.functional.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1)), wt.float(), b, stride=2)
    assert (To, Ho, Wo) == (T, ref.shape[-2], ref.shape[-1])
    out = torch.empty(To * Ho * Wo, co, device=dev, dtype=torch.bfloat16)
    ops.conv3d_causal(x, wk, b, out, T, H, W, ops.YB_EPI_BF16, taps=(1, 3, 3), oob_zero_pad=True, stride_hw=2)
    assert rel(out.view(T, Ho, Wo, co), ref.permute(0, 2, 3, 1)) < KERNEL_TOL


@pytest.mark.parametrize("T,H,W,ci,co", [(3, 4, 8, 64, 64), (5, 6, 10, 128, 96), (9, 3, 40, 192, 160), (17, 2, 6, 64, 320)])
def test_conv3d_stride2_temporal_matches_torch(dev, T, H, W, ci, co):
    """`Resample(downsample3d).time_conv`: CausalConv3d((3,1,1), stride (2,1,1), padding 0) over the frames it is given
    (vae2_2.py:105-110, 158-170), output written one frame behind a frame 0 the caller copied."""
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(T * 100 + W)
    x = torch.randn(T, H, W, ci, generator=g).to(dev).bfloat16()
    wt = (torch.randn(co, ci, 3, 1, 1, generator=g) / math.sqrt(3 * ci)).to(dev).bfloat16()
    b = torch.randn(co, generator=g).to(dev)
    wk = wt.permute(0, 2, 3, 4, 1).reshape(co, 3 * ci).contiguous()
    ref = torch.nn.functional.conv3d(x.float().permute(3, 0, 1, 2)[None], wt.float(), b, stride=(2, 1, 1))[0].permute(1, 2, 3, 0)
    To = (T - 3) // 2 + 1
    assert ops.conv_out_dims(T, H, W, (3, 1, 1), 2, 1) == (To, H, W) and ref.shape[0] == To
    out = torch.full(((1 + To) * H * W, co), 7.0, device=dev, dtype=torch.bfloat16)
    ops.conv3d_causal(x, wk, b, out, T, H, W, ops.YB_EPI_BF16, taps=(3, 1, 1), oob_zero_pad=True, stride_t=2, out_t_add=1)
    got = out.view(1 + To, H, W, co)
    assert rel(got[1:], ref) < KERNEL_TOL and bool((got[0] == 7.0).all())


def test_wan22_vae_encode_glue_kernels(dev):
    from oracle import wan22vae_enc
    from yume_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(33)
    # patchify(2): f32 [3, T, H, W] -> bf16 [T*H/2*W/2, 64], 12 channels (c r q), the rest zero — bit-exact after the bf16 rounding
    T, H, W = 3, 8, 12
    video = torch.randn(3, T, H, W, generator=g).to(dev)
    out = torch.full((T * (H // 2) * (W // 2), 64), 7.0, device=dev, dtype=torch.bfloat16)
    ops.vae_patchify2_bf16(video, out)
    want = wan22vae_enc.patchify2(video[None].cpu())[0].permute(1, 2, 3, 0).reshape(-1, 12).to(dev).bfloat16()
    assert torch.equal(out[:, :12], want) and bool((out[:, 12:] == 0).all())
    # AvgDown3D shortcut add against the oracle's whole-sequence form: every (ft, fs) / width ratio the encoder uses, odd T
    for Tn, Hn, Wn, ci, co, ft, fs in ((5, 4, 6, 32, 32, 1, 2), (5, 4, 6, 32, 64, 2, 2), (1, 4, 6, 32, 64, 2, 2), (9, 2, 4, 64, 128, 2, 2),
                                       (3, 4, 6, 128, 128, 1, 1), (5, 2, 2, 160, 320, 2, 2)):
        x = torch.randn(Tn * Hn * Wn, ci, generator=g).to(dev).bfloat16()
        short = wan22vae_enc.avg_down(x.float().cpu().view(Tn, Hn, Wn, ci).permute(3, 0, 1, 2)[None], co, ft, fs)[0]   # [co, To, Ho, Wo]
        To, Ho, Wo = short.shape[1:]
        main = torch.randn(To * Ho * Wo, co, generator=g).to(dev).bfloat16()
        want = main.float().view(To, Ho, Wo, co) + short.permute(1, 2, 3, 0).to(dev)
        ops.vae_avgdown_add(main, x, (Tn, Hn, Wn), ci, co, ft, fs)
        assert rel(main.view(To, Ho, Wo, co), want) < 6e-3, (Tn, ci, co, ft, fs)


def _enc_gold(golden_dir, name, mod):
    g = torch.load(golden_dir / name, weights_only=False)
    sd = mod.make_state_dict(g["seed_w"], **g["cfg"])
    got = float(sum(v.abs().sum() for v in sd.values()))
    if abs(got - g["weight_abs_sum"]) > 1e-3 * g["weight_abs_sum"]:
        pytest.skip("torch CPU RNG stream differs from the one that generated the golden weights")
    return g, sd


ENC_PSNR_DB = 35.0   # latents are unbounded: PSNR against the fixture's own range


@pytest.mark.parametrize("case", ["t1", "t5", "t9", "t17_wide"])
def test_wan21_vae_encode_vs_reference_golden(dev, golden_dir, case):
    """One-pass whole-sequence ENCODE on the GPU against the reference's own chunked / feature-cached `WanVAE_.encode`."""
    from oracle import wan21vae_enc
    from yume_b200.vae_enc import Wan21VaeEncoder
    g, sd = _enc_gold(golden_dir, "wan21vae_enc_tiny.pt", wan21vae_enc)
    c = g["cases"][case]
    eng = Wan21VaeEncoder(sd, mean=g["mean"], std=g["std"], device=dev, **g["cfg"])
    x = torch.randn(3, c["T"], c["H"], c["W"], generator=torch.Generator().manual_seed(c["seed"])).clamp_(-1, 1)
    mu = eng.encode(x).cpu()
    assert tuple(mu.shape) == c["shape"]
    assert rel(mu, c["mu"]) < VAE_TOL and psnr(mu, c["mu"]) > ENC_PSNR_DB


@pytest.mark.parametrize("case", ["t1", "t5", "t9", "t17_wide"])
def test_wan22_vae_encode_vs_reference_golden(dev, golden_dir, case):
    from oracle import wan22vae_enc
    from yume_b200.vae_enc import Wan22VaeEncoder
    g, sd = _enc_gold(golden_dir, "wan22vae_enc_tiny.pt", wan22vae_enc)
    c = g["cases"][case]
    eng = Wan22VaeEncoder(sd, mean=g["mean"], std=g["std"], device=dev, **g["cfg"])
    x = torch.randn(3, c["T"], c["H"], c["W"], generator=torch.Generator().manual_seed(c["seed"])).clamp_(-1, 1)
    mu = eng.encode(x).cpu()
    assert tuple(mu.shape) == c["shape"]
    assert rel(mu, c["mu"]) < VAE_TOL and psnr(mu, c["mu"]) > ENC_PSNR_DB


@pytest.mark.parametrize("which", ["wan21", "wan22"])
def test_wan_vae_encode_real_width_vs_oracle(dev, which):
    """Real channel widths (2.1: 96/192/384/384, z16; 2.2: 160/320/640/640, z48) on a small clip against the fp32 oracle; a
    frame count that is not 1 + 4k is truncated like the reference's chunk loop (vae2_2.py:802-803)."""
    from oracle import wan21vae_enc, wan22vae_enc
    from yume_b200.vae_enc import Wan21VaeEncoder, Wan22VaeEncoder
    gen = torch.Generator().manual_seed(9)
    if which == "wan21":
        cfg = dict(dim=96, z_dim=16, dim_mult=(1, 2, 4, 4), num_res_blocks=2, temperal_downsample=(False, True, True))
        mod, Oracle, Engine, hw = wan21vae_enc, wan21vae_enc.Wan21VaeEncodeOracle, Wan21VaeEncoder, (32, 48)
    else:
        cfg = dict(dim=160, z_dim=48, dim_mult=(1, 2, 4, 4), num_res_blocks=2, temperal_downsample=(False, True, True))
        mod, Oracle, Engine, hw = wan22vae_enc, wan22vae_enc.Wan22VaeEncodeOracle, Wan22VaeEncoder, (64, 96)
    sd = mod.make_state_dict(51, **cfg)
    z = cfg["z_dim"]
    mean, std = 0.2 * torch.randn(z, generator=gen), 0.5 + torch.rand(z, generator=gen)
    video = torch.randn(3, 7, *hw, generator=gen).clamp_(-1, 1)            # 7 frames -> the first 5 are encoded
    want = Oracle(sd, mean=mean, std=std, **cfg).encode(video[:, :5])
    got = Engine(sd, mean=mean, std=std, device=dev, **cfg).encode(video).cpu()
    assert got.shape == want.shape == (z, 2, hw[0] // (8 if which == "wan21" else 16), hw[1] // (8 if which == "wan21" else 16))
    assert rel(got, want) < VAE_TOL and psnr(got, want) > ENC_PSNR_DB
