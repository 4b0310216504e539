"""CPU half of the per-element kernel contract (tests/test_gpu_kernel_contract.py):
  * its checker and bounds reject the defects they exist for (one element 4 bf16 ulp off, a row never written, a guard cell
    overwritten, a 64-wide K block dropped from a GEMM tile, a 128-key tile dropped from an attention row), and accept the same
    results without the defect — computed here the way the kernels compute them (fp32 accumulation, bf16 P, bf16 output);
  * every template instance the .cu sources dispatch to (YB_LN_WARP, YB_RR_FAST, YB_RR_WARP, YB_QK_WARP, YB_SC) is in the GPU
    file's width tables, with at least one width that reaches each general kernel — a new instance without a test fails here.
"""
import math
import re
from pathlib import Path

import pytest
import torch

import test_gpu_kernel_contract as K

CSRC = Path(__file__).resolve().parents[1] / "yume_b200" / "csrc"


def _bf16_step(x, steps):
    """x (bf16) moved by `steps` units in the last place."""
    bits = x.view(torch.int16).clone()
    bits += steps if float(x) >= 0 else -steps
    return bits.view(torch.bfloat16)


def _gemm_case(M=128, N=128, Kd=512, drop_block=None):
    g = torch.Generator().manual_seed(7)
    A = torch.randn(M, Kd, generator=g).bfloat16()
    B = (torch.randn(N, Kd, generator=g) / math.sqrt(Kd)).bfloat16()
    keep = torch.ones(Kd, dtype=torch.bool)
    if drop_block is not None:
        keep[drop_block * 64:(drop_block + 1) * 64] = False
    got = (A.float()[:, keep] @ B.float()[:, keep].t()).bfloat16()          # fp32 accumulation, bf16 output
    ref = A.double() @ B.double().t()
    return got, ref, K.bf16_out_bound(ref, K.gemm_bounds(A, B, Kd))


def test_gemm_bound_accepts_the_kernel_arithmetic():
    got, ref, bound = _gemm_case()
    assert K.assert_within(got, ref, bound, "gemm 128x128x512") <= 1.0


def test_gemm_bound_rejects_one_element_moved_by_4_ulp():
    got, ref, bound = _gemm_case()
    got[37, 101] = _bf16_step(got[37, 101], 4)
    with pytest.raises(AssertionError, match=r"1 of 16384 elements out of bound; worst at \(37, 101\)"):
        K.assert_within(got, ref, bound, "gemm one element +4 ulp")


def test_gemm_bound_rejects_a_dropped_k_block():
    got, ref, bound = _gemm_case(drop_block=5)
    with pytest.raises(AssertionError, match="out of bound"):
        K.assert_within(got, ref, bound, "gemm K block 5 dropped")


def _attention_case(Lk=512, drop_tile=None, scale=1 / math.sqrt(128.0)):
    """One head, computed as the kernel does: fp32 logits and softmax, P rounded to bf16 for P.V, fp32 normaliser, bf16 out."""
    g = torch.Generator().manual_seed(3)
    q, k, v = (torch.randn(L, 128, generator=g).bfloat16() for L in (4, Lk, Lk))
    keep = torch.ones(Lk, dtype=torch.bool)
    if drop_tile is not None:
        keep[drop_tile * 128:(drop_tile + 1) * 128] = False
    s = (q.float() @ k.float()[keep].t()) * scale
    p = torch.exp(s - s.amax(-1, keepdim=True))
    got = ((p.bfloat16().float() @ v.float()[keep]) / p.sum(-1, keepdim=True)).bfloat16()
    qd, kd, vd = q.double(), k.double(), v.double()
    ref = torch.softmax((qd @ kd.t()) * scale, -1) @ vd
    return got, ref, K.attention_bound(qd, kd, vd, scale, ref)


@pytest.mark.parametrize("scale", [1 / math.sqrt(128.0), 0.05, 0.2])
def test_attention_bound_accepts_the_kernel_arithmetic(scale):
    got, ref, bound = _attention_case(scale=scale)
    assert K.assert_within(got, ref, bound, f"attention scale {scale:.3g}") <= 1.0


def test_attention_bound_rejects_a_dropped_key_tile():
    got, ref, bound = _attention_case(drop_tile=2)
    with pytest.raises(AssertionError, match="out of bound"):
        K.assert_within(got, ref, bound, "attention key tile 2 dropped")


def test_norm_bounds_accept_fp32_arithmetic_and_reject_a_shifted_element():
    g = torch.Generator().manual_seed(5)
    L, C = 16, 1024
    x = torch.randn(L, C, generator=g) + 1000.0 * (torch.arange(L) % 2)[:, None]
    sc = torch.randn(L, C, generator=g) * 0.5
    mean = x.mean(1, keepdim=True)
    y32 = ((x - mean) * torch.rsqrt((x - mean).pow(2).mean(1, keepdim=True) + 1e-6)) * (1 + sc)
    ref, f32 = K._ln_ref(x, C, 1e-6, None, None, sc, None)
    bound = K.bf16_out_bound(ref, f32)
    got = y32.bfloat16()
    assert K.assert_within(got, ref, bound, "ln_modulate fp32 arithmetic") <= 1.0
    got[3, 200] = _bf16_step(got[3, 200], 4)
    with pytest.raises(AssertionError, match=r"worst at \(3, 200\)"):
        K.assert_within(got, ref, bound, "ln_modulate +4 ulp")
    q = torch.randn(L, C, generator=g).bfloat16()
    w = torch.rand(C, generator=g) + 0.5
    ang = torch.rand(L, 64, generator=g, dtype=torch.float64) * 6.28
    rope = torch.stack([ang.cos(), ang.sin()], -1).float()
    ref, bound = K._rr_ref(q, w, rope, L - 3, 128)
    qf = q.float()
    n = qf * torch.rsqrt(qf.pow(2).mean(1, keepdim=True) + 1e-6) * w
    v = n[:L - 3].view(L - 3, C // 128, 64, 2)
    c, s = rope[:L - 3, None, :, 0], rope[:L - 3, None, :, 1]
    n[:L - 3] = torch.stack([v[..., 0] * c - v[..., 1] * s, v[..., 0] * s + v[..., 1] * c], -1).reshape(L - 3, C)
    got = n.bfloat16()
    assert K.assert_within(got, ref, bound, "rmsnorm_rope fp32 arithmetic") <= 1.0
    got[L - 2, 5] = _bf16_step(got[L - 2, 5], 4)                            # an un-rotated row past rope_len
    with pytest.raises(AssertionError, match="out of bound"):
        K.assert_within(got, ref, bound, "rmsnorm_rope +4 ulp")


def test_guard_band_rejects_a_nan_row_and_a_changed_guard_cell():
    out = K.guarded((5, 16), torch.bfloat16, (2, 8), device="cpu")
    assert out.view.stride(0) == 32 and out.view.data_ptr() - out.backing.data_ptr() == (2 * 32 + 8) * 2
    out.view[:4] = 1.0                                                      # row 4 never written
    with pytest.raises(AssertionError, match=r"never written \(still NaN\), first at \(4, 0\)"):
        out.check("one NaN row")
    out.view[4] = 2.0
    out.check("all rows written")
    out.backing[2 + 4, 8 + 16] = 3.0                                        # one column past N: a guard cell
    with pytest.raises(AssertionError, match=r"1 guard-band element\(s\) changed, first at backing index \(6, 24\)"):
        out.check("one stray store")
    acc = K.guarded((3, 4, 8), torch.float32, (1, 0), fill=torch.ones(3, 4, 8), device="cpu")
    acc.view += 1.0
    acc.check("in-place update of seeded data")
    acc.backing[-1, 0, 0] = 0.0
    with pytest.raises(AssertionError, match="guard-band"):
        acc.check("store past the last row")


def test_assert_within_reports_count_index_and_ratio():
    ref = torch.zeros(3, 4, dtype=torch.float64)
    got = ref.clone()
    got[1, 2], got[2, 3] = 0.5, 3.0
    with pytest.raises(AssertionError, match=r"2 of 12 elements out of bound; worst at \(2, 3\).*\|err\|/bound = 12\)"):
        K.assert_within(got, ref, torch.full_like(ref, 0.25), "report")
    assert K.assert_within(got, ref, torch.full_like(ref, 6.0), "margin") == 0.5


def test_case_data_is_the_same_in_every_process():
    """Case data are drawn from a seed derived from the case's parameters; it must not depend on the per-process str hash salt,
    or a failing case could not be replayed from its test id."""
    import os
    import subprocess
    import sys
    code = ("import sys, torch; sys.path.insert(0, sys.argv[1]); import test_gpu_kernel_contract as K; "
            "print(torch.randn(4, generator=K._gen('gemm', 1, 32, 3072, 1, 0, 'dense')).tolist())")
    outs = {subprocess.run([sys.executable, "-c", code, str(Path(__file__).parent)], capture_output=True, text=True, check=True,
                           env=dict(os.environ, PYTHONHASHSEED=seed)).stdout for seed in ("1", "2")}
    assert len(outs) == 1, outs


# ------------------------------------------------------------------------------------------------------------
# dispatch coverage guard
# ------------------------------------------------------------------------------------------------------------
def _instances(macro, path):
    """Arguments of the instance lines `  MACRO(n)` (the #define line has a parameter name, not a number)."""
    return {int(n) for n in re.findall(rf"^\s*{macro}\((\d+)\)\s*$", path.read_text(), flags=re.M)}


def _coverage_problems(src):
    problems = []
    ln = {128 * n for n in _instances("YB_LN_WARP", src)}
    if not ln:
        problems.append("no YB_LN_WARP instances found")
    missing = ln - set(K.LN_WARP_WIDTHS)
    if missing:
        problems.append(f"YB_LN_WARP widths without a test: {sorted(missing)}")
    if not [c for c in K.LN_GENERAL_WIDTHS if c not in ln]:
        problems.append("no tested width reaches the general ln_modulate kernel")
    rr_all = set()
    for macro in ("YB_RR_FAST", "YB_RR_WARP", "YB_QK_WARP"):
        widths = {256 * n for n in _instances(macro, src)}
        if not widths:
            problems.append(f"no {macro} instances found")
        missing = widths - set(K.RR_WARP_WIDTHS)
        if missing:
            problems.append(f"{macro} widths without a test: {sorted(missing)}")
        rr_all |= widths
    if not [c for c in K.RR_GENERAL_WIDTHS if c not in rr_all]:
        problems.append("no tested width reaches the general rmsnorm_rope kernel")
    sc = {256 * n for n in _instances("YB_SC", src)}
    if not sc:
        problems.append("no YB_SC instances found")
    missing = sc - set(K.SC_WIDTHS)
    if missing:
        problems.append(f"YB_SC widths without a test: {sorted(missing)}")
    return problems


def test_every_dispatch_instance_has_a_width_in_the_gpu_tables():
    assert _coverage_problems(CSRC / "elementwise.cu") == []


def test_coverage_guard_notices_a_new_instance(tmp_path):
    text = (CSRC / "elementwise.cu").read_text()
    fake = tmp_path / "elementwise.cu"
    fake.write_text(text.replace("  YB_LN_WARP(2)\n", "  YB_LN_WARP(2)\n  YB_LN_WARP(16)\n", 1))
    assert _coverage_problems(fake) == ["YB_LN_WARP widths without a test: [2048]"]
    fake.write_text(text.replace("  YB_QK_WARP(1)\n", "  YB_QK_WARP(1)\n  YB_QK_WARP(6)\n", 1))
    assert _coverage_problems(fake) == ["YB_QK_WARP widths without a test: [1536]"]


def test_coverage_guard_notices_a_width_removed_from_a_table(monkeypatch):
    monkeypatch.setattr(K, "LN_WARP_WIDTHS", (256, 1024, 3072))
    monkeypatch.setattr(K, "RR_GENERAL_WIDTHS", (1024,))
    assert _coverage_problems(CSRC / "elementwise.cu") == ["YB_LN_WARP widths without a test: [5120]",
                                                          "no tested width reaches the general rmsnorm_rope kernel"]
