"""Diagnostic run of every kernel against torch references on the GPU box (prints, never asserts).
Usage: python tools/gpu_check_kernels.py [section ...]"""
import math
import sys
import time
import traceback

import torch

sys.path.insert(0, ".")
from yume_b200 import ops  # noqa: E402

dev = "cuda"
torch.manual_seed(0)


def rel(a, b):
    a = a.float(); b = b.float()
    return ((a - b).norm() / (b.norm() + 1e-30)).item(), (a - b).abs().max().item()


def timeit(fn, n=5):
    fn(); torch.cuda.synchronize()
    t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(n):
        fn()
    t1.record(); torch.cuda.synchronize()
    return t0.elapsed_time(t1) / n


def sec_probe():
    a = torch.randn(128, 128, device=dev).bfloat16()
    b = torch.randn(128, 128, device=dev).bfloat16()
    for mode in (0, 1, 2):
        d = ops.umma_probe(a, b, mode)
        torch.cuda.synchronize()
        ref = a.float() @ (b.float().t() if mode == 0 else b.float())
        alt = a.float() @ (b.float() if mode == 0 else b.float().t())
        print(f"probe mode {mode}: rel/max vs expected {rel(d, ref)}  vs transposed-B {rel(d, alt)}  finite={torch.isfinite(d).all().item()}")
        if mode == 2:
            # hypothesis check: swapped bf16 halves in the register A operand
            a_sw = a.view(128, 64, 2).flip(-1).reshape(128, 128)
            print("   vs half-swapped A:", rel(d, a_sw.float() @ b.float()))


def sec_gemm():
    for (M, N, K, bn) in [(128, 256, 64, 0), (256, 256, 256, 0), (300, 384, 192, 0), (1000, 3072, 3072, 0),
                          (512, 128, 4096, 128), (18480, 3072, 3072, 0), (18480, 9216, 3072, 0), (18480, 14336, 3072, 0),
                          (18480, 3072, 14336, 0)]:
        a = (torch.randn(M, K, device=dev) * 0.5).bfloat16()
        w = (torch.randn(N, K, device=dev) * 0.05).bfloat16()
        bias = torch.randn(N, device=dev)
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        try:
            ops.gemm(a, w, bias, out, ops.YB_EPI_BF16, block_n=bn)
            torch.cuda.synchronize()
            ref = (a @ w.t()).float() + bias
            r = rel(out, ref)
            ms = timeit(lambda: ops.gemm(a, w, bias, out, ops.YB_EPI_BF16, block_n=bn))
            ms_t = timeit(lambda: torch.matmul(a, w.t()))
            print(f"gemm bf16 M={M} N={N} K={K} bn={bn}: rel={r[0]:.3e} max={r[1]:.3e}  {ms:.3f} ms = {2*M*N*K/ms/1e9:.0f} TF/s  (torch {ms_t:.3f} ms = {2*M*N*K/ms_t/1e9:.0f} TF/s)")
        except Exception as e:
            print(f"gemm M={M} N={N} K={K} FAILED: {e}")
            raise
    # epilogues
    M, N, K = 1000, 512, 320
    a = (torch.randn(M, K, device=dev) * 0.5).bfloat16(); w = (torch.randn(N, K, device=dev) * 0.1).bfloat16()
    bias = torch.randn(N, device=dev)
    accref = a.float() @ w.float().t() + bias
    o = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    ops.gemm(a, w, bias, o, ops.YB_EPI_GELU_BF16)
    print("gemm gelu:", rel(o, torch.nn.functional.gelu(accref, approximate="tanh")))
    o32 = torch.empty(M, N, device=dev)
    ops.gemm(a, w, None, o32, ops.YB_EPI_F32)
    print("gemm f32 nobias:", rel(o32, accref - bias))
    U = 3
    gate = torch.randn(U, 6, N, device=dev)
    tok = torch.randint(0, U, (M,), device=dev, dtype=torch.int32)
    x = torch.randn(M, N, device=dev)
    xr = x + accref * gate[tok.long(), 2]
    ops.gemm(a, w, bias, x, ops.YB_EPI_GATE_RES, gate=gate[:, 2], tok_idx=tok)
    print("gemm gate_res:", rel(x, xr))
    x2 = torch.randn(M, N, device=dev); x2r = x2 + accref
    ops.gemm(a, w, bias, x2, ops.YB_EPI_GATE_RES)
    print("gemm res nogate:", rel(x2, x2r))
    # strided A (column slice of a wider buffer)
    big = (torch.randn(M, 3 * K, device=dev) * 0.5).bfloat16()
    av = big[:, K:2 * K]
    ops.gemm(av, w, bias, o, ops.YB_EPI_BF16)
    print("gemm strided A:", rel(o, av.float() @ w.float().t() + bias))


def sdpa_ref(q, k, v, heads):
    Lq, Lk = q.shape[0], k.shape[0]
    qh = q.view(Lq, heads, 128).transpose(0, 1).float()
    kh = k.view(Lk, heads, 128).transpose(0, 1).float()
    vh = v.view(Lk, heads, 128).transpose(0, 1).float()
    o = torch.nn.functional.scaled_dot_product_attention(qh[None], kh[None], vh[None])[0]
    return o.transpose(0, 1).reshape(Lq, heads * 128)


def sec_attention():
    for variant in (0, 1):
        for (Lq, Lk, heads) in [(128, 128, 1), (256, 256, 2), (300, 200, 2), (1000, 512, 3), (2048, 2048, 4), (777, 1500, 2)]:
            qkv = (torch.randn(max(Lq, Lk), 3 * heads * 128, device=dev)).bfloat16()
            q = qkv[:Lq, : heads * 128]; k = qkv[:Lk, heads * 128: 2 * heads * 128]; v = qkv[:Lk, 2 * heads * 128:]
            out = torch.zeros(Lq, heads * 128, device=dev, dtype=torch.bfloat16)
            try:
                ops.attention(q, k, v, out, heads, variant=variant)
                torch.cuda.synchronize()
                ref = sdpa_ref(q, k, v, heads)
                print(f"attention v{variant} Lq={Lq} Lk={Lk} H={heads}: rel/max {rel(out, ref)} finite={torch.isfinite(out.float()).all().item()}")
            except Exception as e:
                print(f"attention v{variant} Lq={Lq} Lk={Lk} FAILED: {e}")
                raise
        # large-magnitude logits exercise the lazy rescale path
        Lq, Lk, heads = 512, 1024, 2
        q = (torch.randn(Lq, heads * 128, device=dev) * 4).bfloat16(); k = (torch.randn(Lk, heads * 128, device=dev) * 4).bfloat16()
        v = torch.randn(Lk, heads * 128, device=dev).bfloat16(); out = torch.zeros(Lq, heads * 128, device=dev, dtype=torch.bfloat16)
        ops.attention(q, k, v, out, heads, variant=variant); torch.cuda.synchronize()
        print(f"attention v{variant} peaky: rel/max {rel(out, sdpa_ref(q, k, v, heads))}")
    for variant in (0, 1):
        heads, L = 24, 18480
        qkv = torch.randn(L, 3 * heads * 128, device=dev).bfloat16()
        q = qkv[:, : heads * 128]; k = qkv[:, heads * 128: 2 * heads * 128]; v = qkv[:, 2 * heads * 128:]
        out = torch.empty(L, heads * 128, device=dev, dtype=torch.bfloat16)
        ms = timeit(lambda: ops.attention(q, k, v, out, heads, variant=variant), n=3)
        fl = 4.0 * L * L * heads * 128
        print(f"attention v{variant} self 5B L={L}: {ms:.2f} ms = {fl/ms/1e9:.0f} TF/s")
        idx = torch.randint(0, L, (512,), device=dev)
        ref = sdpa_ref(q[idx].contiguous(), k, v, heads)
        print("   sample rows rel/max:", rel(out[idx], ref))
        kc = torch.randn(512, 2 * heads * 128, device=dev).bfloat16()
        ms = timeit(lambda: ops.attention(q, kc[:, : heads * 128], kc[:, heads * 128:], out, heads, variant=variant), n=3)
        print(f"attention v{variant} cross 5B Lk=512: {ms:.3f} ms = {4.0*L*512*heads*128/ms/1e9:.0f} TF/s")
    try:
        qh = q.view(L, heads, 128).transpose(0, 1)[None].contiguous(); kh = k.view(L, heads, 128).transpose(0, 1)[None].contiguous(); vh = v.view(L, heads, 128).transpose(0, 1)[None].contiguous()
        ms = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(qh, kh, vh), n=3)
        print(f"torch SDPA self 5B: {ms:.2f} ms = {fl/ms/1e9:.0f} TF/s")
        from flash_attn import flash_attn_func
        q4 = q.reshape(1, L, heads, 128).contiguous(); k4 = k.reshape(1, L, heads, 128).contiguous(); v4 = v.reshape(1, L, heads, 128).contiguous()
        ms = timeit(lambda: flash_attn_func(q4, k4, v4), n=3)
        print(f"flash_attn FA2 self 5B: {ms:.2f} ms = {fl/ms/1e9:.0f} TF/s")
    except Exception as e:
        print("baseline attention timing failed:", e)


def sec_elementwise():
    L, Cdim, D = 1000, 3072, 128
    x = torch.randn(L, Cdim, device=dev) * 2 + 0.3
    U = 2
    mod = torch.randn(U, 6, Cdim, device=dev) * 0.5
    tok = torch.randint(0, U, (L,), device=dev, dtype=torch.int32)
    out = torch.empty(L, Cdim, device=dev, dtype=torch.bfloat16)
    ops.ln_modulate(x, out, mod[:, 1], mod[:, 0], tok)
    ln = torch.nn.functional.layer_norm(x, (Cdim,), eps=1e-6)
    ref = ln * (1 + mod[tok.long(), 1]) + mod[tok.long(), 0]
    print("ln_modulate:", rel(out, ref))
    w = torch.randn(Cdim, device=dev); b = torch.randn(Cdim, device=dev)
    ops.ln_modulate(x, out, None, None, None, w, b)
    print("ln affine:", rel(out, ln * w + b))
    o32 = torch.empty(L, Cdim, device=dev)
    ops.ln_modulate(x, o32, mod[0, 1], mod[0, 0])
    print("ln_modulate f32 U=1:", rel(o32, ln * (1 + mod[0, 1]) + mod[0, 0]))
    # rmsnorm + rope
    qkv = torch.randn(L, 3 * Cdim, device=dev).bfloat16()
    q0 = qkv[:, :Cdim].clone()
    wq = torch.rand(Cdim, device=dev) + 0.5
    ang = torch.rand(L, D // 2, device=dev, dtype=torch.float64) * 6.28
    rope = torch.stack([ang.cos(), ang.sin()], -1).float().contiguous()
    ops.rmsnorm_rope(qkv[:, :Cdim], wq, rope, D)
    xf = q0.float(); n = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6) * wq
    c = torch.view_as_complex(n.double().view(L, Cdim // D, D // 2, 2)) * torch.polar(torch.ones_like(ang), ang)[:, None]
    refq = torch.view_as_real(c).flatten(1).float()
    print("rmsnorm_rope:", rel(qkv[:, :Cdim], refq), " untouched k:", (qkv[:, Cdim:] != qkv[:, Cdim:]).any().item())
    k0 = qkv[:, Cdim:2 * Cdim].clone()
    ops.rmsnorm_rope(qkv[:, Cdim:2 * Cdim], wq, None, D)
    kf = k0.float(); print("rmsnorm only:", rel(qkv[:, Cdim:2 * Cdim], kf * torch.rsqrt(kf.pow(2).mean(-1, keepdim=True) + 1e-6) * wq))
    # patchify / unpatchify
    Cin, F, H, W = 48, 3, 10, 12
    xin = torch.randn(Cin, F, H, W, device=dev)
    conv = torch.nn.Conv3d(Cin, 64, (1, 2, 2), (1, 2, 2)).to(dev)
    pa = torch.empty(F * 5 * 6, Cin * 4, device=dev, dtype=torch.bfloat16)
    ops.patchify(xin, pa, 2, 2)
    refp = torch.nn.functional.unfold(xin.bfloat16().float().permute(1, 0, 2, 3), 2, stride=2)  # [F, Cin*4, 30]
    refp = refp.permute(0, 2, 1).reshape(F * 30, Cin * 4)
    print("patchify exact:", torch.equal(pa.float(), refp))
    xin2 = torch.randn(Cin, 2, 9, 11, device=dev)
    pa2 = torch.empty(2 * 3 * 3, Cin * 16, device=dev, dtype=torch.bfloat16)
    ops.patchify(xin2, pa2, 4, 4)
    xp = torch.nn.functional.pad(xin2, (0, 1, 0, 3))
    refp2 = torch.nn.functional.unfold(xp.bfloat16().float().permute(1, 0, 2, 3), 4, stride=4).permute(0, 2, 1).reshape(18, Cin * 16)
    print("patchify padded exact:", torch.equal(pa2.float(), refp2))
    y = torch.randn(F * 5 * 6, 4 * 48, device=dev)
    uo = torch.empty(48, F, 10, 12, device=dev)
    ops.unpatchify(y, uo, F, 5, 6, 2, 2)
    refu = torch.einsum("fhwpqrc->cfphqwr", y.view(F, 5, 6, 1, 2, 2, 48)).reshape(48, F, 10, 12)
    print("unpatchify exact:", torch.equal(uo, refu))
    t = torch.tensor([0.0, 999.0, 500.5], device=dev)
    se = ops.sinusoidal(t, 256)
    half = 128
    sin = torch.outer(t.double(), torch.pow(10000, -torch.arange(half, device=dev).double().div(half)))
    print("sinusoidal max err:", (se - torch.cat([sin.cos(), sin.sin()], 1).float()).abs().max().item())
    xi = torch.randn(3, 256, device=dev); w1 = torch.randn(3072, 256, device=dev) * 0.05; b1 = torch.randn(3072, device=dev)
    print("linear_f32_small:", rel(ops.linear_f32_small(xi, w1, b1), xi @ w1.t() + b1))
    xs = torch.randn(3, 3072, device=dev); w2 = torch.randn(1024, 3072, device=dev) * 0.02
    print("linear_f32_small silu:", rel(ops.linear_f32_small(xs, w2, None, True), torch.nn.functional.silu(xs) @ w2.t()))
    xa = torch.randn(1000, 3072, device=dev); wh = torch.randn(192, 3072, device=dev) * 0.02; bh = torch.randn(192, device=dev)
    oh = torch.empty(1000, 192, device=dev)
    ops.linear_f32(xa, wh, bh, oh)
    print("linear_f32:", rel(oh, xa.double() @ wh.double().t() + bh.double()))
    L2 = 18480
    xb = torch.randn(L2, Cdim, device=dev); ob = torch.empty(L2, Cdim, device=dev, dtype=torch.bfloat16); tk = torch.zeros(L2, device=dev, dtype=torch.int32)
    ms = timeit(lambda: ops.ln_modulate(xb, ob, mod[:, 1], mod[:, 0], tk))
    print(f"ln_modulate L={L2}: {ms*1e3:.1f} us = {L2*Cdim*6/ms/1e6:.0f} GB/s")
    qb = torch.randn(L2, 3 * Cdim, device=dev).bfloat16(); rp = torch.randn(L2, 64, 2, device=dev)
    ms = timeit(lambda: ops.rmsnorm_rope(qb[:, :Cdim], wq, rp, D))
    print(f"rmsnorm_rope L={L2}: {ms*1e3:.1f} us = {L2*Cdim*4/ms/1e6:.0f} GB/s")
    ms = timeit(lambda: ops.qk_norm_rope(qb[:, :Cdim], qb[:, Cdim:2 * Cdim], wq, wq, rp, D))
    print(f"qk_norm_rope (q+k, one launch) L={L2}: {ms*1e3:.1f} us = {L2*Cdim*8/ms/1e6:.0f} GB/s")
    wln = torch.randn(Cdim, device=dev); bln = torch.randn(Cdim, device=dev)
    ms = timeit(lambda: ops.ln_modulate(xb, ob, None, None, None, wln, bln))
    print(f"ln affine L={L2}: {ms*1e3:.1f} us = {L2*Cdim*6/ms/1e6:.0f} GB/s")


def sec_atttune():
    heads, L = 24, 18480
    qkv = torch.randn(L, 3 * heads * 128, device=dev).bfloat16()
    q = qkv[:, : heads * 128]; k = qkv[:, heads * 128: 2 * heads * 128]; v = qkv[:, 2 * heads * 128:]
    out = torch.empty(L, heads * 128, device=dev, dtype=torch.bfloat16)
    idx = torch.randint(0, L, (256,), device=dev)
    ref = sdpa_ref(q[idx].contiguous(), k, v, heads)
    fl = 4.0 * L * L * heads * 128
    ms = min(timeit(lambda: ops.attention(q, k, v, out, heads), n=5) for _ in range(3))
    print(f"attention: {ms:.3f} ms = {fl/ms/1e9:.0f} TF/s   rel/max {rel(out[idx], ref)}")


def sec_attsplit():
    """Tail split of the attention launch: the per-rank shape of 8-GPU Ulysses (3 of 24 heads) and neighbours."""
    from yume_b200 import ops
    L = 18480
    for heads in (3, 6, 24):
        g = torch.Generator(device=dev).manual_seed(heads)
        q, k, v = (torch.randn(L, heads * 128, generator=g, device=dev).bfloat16() for _ in range(3))
        o = torch.empty_like(q)
        fl = 4.0 * L * L * heads * 128
        line = f"attsplit heads={heads} units={heads * ((L + 255) // 256)}:"
        for name, split in (("never", 1), ("auto", 0), ("force2", 2)):
            ms = timeit(lambda: ops.attention(q, k, v, o, heads, split=split), 10)
            line += f"  {name} {ms:.3f} ms ({fl / ms / 1e9:.0f} TF/s)"
        print(line, flush=True)


def sec_attmodes():
    """Softmax schedules of the attention kernel at the 5B self-attention shape, the 8-GPU per-rank shape and 14B."""
    for heads, L in ((24, 18480), (3, 18480), (40, 21930)):
        qkv = torch.randn(L, 3 * heads * 128, device=dev).bfloat16()
        q = qkv[:, : heads * 128]; k = qkv[:, heads * 128: 2 * heads * 128]; v = qkv[:, 2 * heads * 128:]
        out = torch.empty(L, heads * 128, device=dev, dtype=torch.bfloat16)
        idx = torch.randint(0, L, (256,), device=dev)
        ref = sdpa_ref(q[idx].contiguous(), k, v, heads)
        fl = 4.0 * L * L * heads * 128
        ms = min(timeit(lambda: ops.attention(q, k, v, out, heads), n=5) for _ in range(3))
        print(f"attmodes heads={heads} L={L}: {ms:.3f} ms = {fl/ms/1e9:.0f} TF/s   rel/max {rel(out[idx], ref)}", flush=True)
    try:
        heads, L = 24, 18480
        qkv = torch.randn(L, 3 * heads * 128, device=dev).bfloat16()
        q = qkv[:, : heads * 128]; k = qkv[:, heads * 128: 2 * heads * 128]; v = qkv[:, 2 * heads * 128:]
        fl = 4.0 * L * L * heads * 128
        qh = q.view(L, heads, 128).transpose(0, 1)[None].contiguous(); kh = k.view(L, heads, 128).transpose(0, 1)[None].contiguous(); vh = v.view(L, heads, 128).transpose(0, 1)[None].contiguous()
        ms = min(timeit(lambda: torch.nn.functional.scaled_dot_product_attention(qh, kh, vh), n=5) for _ in range(3))
        print(f"attmodes comparator torch SDPA (cuDNN/flash backend) self 5B: {ms:.3f} ms = {fl/ms/1e9:.0f} TF/s", flush=True)
    except Exception as e:
        print("SDPA comparator failed:", e)


def sec_gemmpair():
    """SM-pair (cta_group::2) GEMM against the 1-CTA kernel and cuBLAS: the DiT shapes at N = 1 and the per-rank shapes of 8-GPU
    Ulysses (M = 2310), plain and GATE_RES epilogues, automatic and forced N tiles."""
    C, F = 3072, 14336
    for L in (18480, 2310):
        for name, (M, N, K) in (("qkv", (L, 3 * C, C)), ("o", (L, C, C)), ("ffn1", (L, F, C)), ("ffn2", (L, C, F))):
            a = torch.randn(M, K, device=dev).bfloat16()
            w = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
            o1, o2 = torch.empty(M, N, device=dev, dtype=torch.bfloat16), torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            fl = 2.0 * M * N * K
            t1 = timeit(lambda: ops.gemm(a, w, None, o1, ops.YB_EPI_BF16, cta_pair=1), 5)
            t2 = timeit(lambda: ops.gemm(a, w, None, o2, ops.YB_EPI_BF16, cta_pair=2), 5)
            t256 = timeit(lambda: ops.gemm(a, w, None, o2, ops.YB_EPI_BF16, cta_pair=2, block_n=256), 5)
            t3 = timeit(lambda: torch.matmul(a, w.t()), 5)
            line = (f"gemmpair L={L} {name}: 1-CTA {t1:.3f} ms ({fl/t1/1e9:.0f} TF/s)  pair(auto bn) {t2:.3f} ms ({fl/t2/1e9:.0f} TF/s)  "
                    f"pair(bn=256) {t256:.3f} ms ({fl/t256/1e9:.0f})  cuBLAS {t3:.3f} ms ({fl/t3/1e9:.0f} TF/s)  equal={torch.equal(o1, o2)}")
            if name in ("o", "ffn2"):
                x = torch.randn(M, N, device=dev); gate = torch.randn(1, N, device=dev)
                g1 = timeit(lambda: ops.gemm(a, w, None, x, ops.YB_EPI_GATE_RES, gate=gate, cta_pair=1), 5)
                g2 = timeit(lambda: ops.gemm(a, w, None, x, ops.YB_EPI_GATE_RES, gate=gate, cta_pair=2), 5)
                line += f"  GATE_RES: 1-CTA {g1:.3f} ms ({fl/g1/1e9:.0f})  pair {g2:.3f} ms ({fl/g2/1e9:.0f})"
            print(line, flush=True)


def sec_gemmsplit():
    """Tail split-K of the SM-pair gate+residual GEMM at the per-rank shapes of 8-, 4- and 2-GPU Ulysses (and the full shape)."""
    C, F = 3072, 14336
    for L in (2310, 4620, 9240, 18480):
        for name, (M, N, K) in (("o", (L, C, C)), ("ffn2", (L, C, F))):
            a = torch.randn(M, K, device=dev).bfloat16()
            w = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
            x = torch.randn(M, N, device=dev); gate = torch.randn(1, N, device=dev)
            fl = 2.0 * M * N * K
            ws = _lib_ws(M, N, K)
            t0 = min(timeit(lambda: ops.gemm(a, w, None, x, ops.YB_EPI_GATE_RES, gate=gate, cta_pair=2, split_k=1), 10) for _ in range(3))
            t1 = min(timeit(lambda: ops.gemm(a, w, None, x, ops.YB_EPI_GATE_RES, gate=gate, cta_pair=2, split_k=0), 10) for _ in range(3))
            t3 = timeit(lambda: torch.matmul(a, w.t()), 10)
            print(f"gemmsplit L={L} {name}: unsplit {t0*1e3:.1f} us ({fl/t0/1e9:.0f} TF/s)  auto {t1*1e3:.1f} us ({fl/t1/1e9:.0f} TF/s, workspace {ws/1e6:.1f} MB)  "
                  f"cuBLAS plain {t3*1e3:.1f} us ({fl/t3/1e9:.0f})", flush=True)


def _lib_ws(M, N, K):
    from yume_b200 import _lib
    return _lib.load().yb_gemm_workspace_bytes(M, N, K, ops.YB_EPI_GATE_RES, 2, 0)


def sec_convpair():
    """Causal conv as implicit GEMM: 1-CTA un-fused / 1-CTA kw-fused / SM-pair kernel on the widths of the three VAE decoders."""
    shapes = [("hy 128->128 @17x256x256", 17, 256, 256, 128, 128), ("hy 256->256 @17x128x128", 17, 128, 128, 256, 256),
              ("hy 512->512 @9x64x64", 9, 64, 64, 512, 512), ("w21 96->96 @21x272x480", 21, 272, 480, 128, 96),
              ("w21 192->192 @21x136x240", 21, 136, 240, 192, 192), ("w22 256->256 @21x176x320", 21, 176, 320, 256, 256),
              ("w21 384->384 @11x68x120", 11, 68, 120, 384, 384)]
    for name, T, H, W, ci, co in shapes:
        x = torch.randn(T + 2, H + 2, W + 2, ci, device=dev).bfloat16()
        wk = (torch.randn(co, 27 * ci, device=dev) / math.sqrt(27 * ci)).bfloat16()
        outs, line = [], f"convpair {name}:"
        fl = 2.0 * T * H * W * 27 * ci * co
        for label, kw in (("1cta", dict(fuse_w=1, cta_pair=2)), ("1cta-kwfused", dict(fuse_w=2, cta_pair=2)), ("pair", dict(cta_pair=1))):
            o = torch.empty(T * H * W, co, device=dev, dtype=torch.bfloat16)
            ms = timeit(lambda: ops.conv3d_causal(x, wk, None, o, T, H, W, ops.YB_EPI_BF16, **kw), 3)
            outs.append(o)
            line += f"  {label} {ms:.3f} ms ({fl/ms/1e9:.0f} TF/s)"
        print(line + f"  equal={torch.equal(outs[0], outs[2])} fused_rel={rel(outs[1], outs[0])[0]:.1e}", flush=True)


SECTIONS = {"attmodes": sec_attmodes, "gemmpair": sec_gemmpair, "gemmsplit": sec_gemmsplit, "convpair": sec_convpair, "attsplit": sec_attsplit, "atttune": sec_atttune, "probe": sec_probe, "gemm": sec_gemm, "attention": sec_attention, "elementwise": sec_elementwise}
if __name__ == "__main__":
    names = sys.argv[1:] or [n for n in SECTIONS if n not in ("gemmpair", "attmodes", "convpair", "gemmsplit")]   # experimental sections only on request
    print(torch.cuda.get_device_name(0))
    for n in names:
        print(f"===== {n} =====", flush=True)
        t0 = time.time()
        try:
            SECTIONS[n]()
            torch.cuda.synchronize()
        except Exception:
            traceback.print_exc()
            print(f"section {n} aborted", flush=True)
            break  # a CUDA fault poisons the context
        print(f"----- {n} done in {time.time()-t0:.1f}s", flush=True)
