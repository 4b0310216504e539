"""CPU half of the per-element kernel contract (tests/test_gpu_kernel_contract.py):
  * its checker and bounds reject the defects they exist for (one element 4 bf16 ulp off, a row never written, a guard cell
    overwritten, a 64-wide K block dropped from a GEMM tile, a 128-key tile dropped from an attention row), and accept the same
    results without the defect — computed here the way the kernels compute them (fp32 accumulation, bf16 P, bf16 output);
  * every template instance the .cu sources dispatch to (YB_LN_WARP, YB_RR_FAST, YB_RR_WARP, YB_QK_WARP, YB_SC) is in the GPU
    file's width tables, with at least one width that reaches each general kernel — a new instance without a test fails here;
  * every C-ABI entry point of include/yume_b200.h is named in the COVERS table of one of the two GPU contract files (or is
    exempt, with its reason), every test a table names exists, and a tested width reaches each YB_RMS_LAUNCH instance;
  * the bounds of tests/test_gpu_kernel_contract_ext.py reject their defects (a next-frame key leaking into a masked softmax
    row, an AvgDown group element dropped, replicate instead of zero padding on one conv face, a straddling n_split tile
    sent to the wrong chunk, a token's sum of squares missing a head block) and accept the kernels' arithmetic;
  * the production-shape table of tests/test_gpu_kernel_contract_prod.py stays multi-wave (planned at 132 SMs), with 5B and 14B
    self-attention rows on the tail split; its sample sets hit every tile, conv box and (head, unit, query tile); and its sampled
    checker rejects, at production M x N with a tiny K, a tile written with its neighbour's coordinates, a GATE_RES tile with the
    wrong tok_idx row, KV tile 100 of 145 dropped in one unit the sampler covers by its per-tile rows only, and a unit whose second
    query tile was never written.
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


# ------------------------------------------------------------------------------------------------------------
# C-ABI entry-point coverage guard
# ------------------------------------------------------------------------------------------------------------
import test_gpu_kernel_contract_ext as KX  # noqa: E402

HEADER = Path(__file__).resolve().parents[1] / "include" / "yume_b200.h"
EXEMPT = {
    "yb_abi_version": "returns a constant; build() compares it with the Python side",
    "yb_debug_force_split": "process-global test hook of the multi-GPU parity tool; sets a flag, launches nothing",
    "yb_umma_probe": "self-test of the wgmma / TMA building blocks, not a product path (tests/test_gpu_parity.py)",
}
EXEMPT_SUFFIXES = {
    "_plan": "host-only planner: no device code (pinned by the host-logic tests)",
    "_workspace_bytes": "host-only workspace sizing: no device code",
}


def _entry_points(header):
    return re.findall(r"^(?:int|long long)\s+(yb_\w+)\(", header.read_text(), flags=re.M)


def _entry_problems(header, modules=(K, KX)):
    problems, covered = [], set()
    for mod in modules:
        for entry, tests in mod.COVERS.items():
            covered.add(entry)
            for name in tests:
                if not callable(getattr(mod, name, None)):
                    problems.append(f"{mod.__name__}.COVERS[{entry!r}] names a test that does not exist: {name}")
    entries = _entry_points(header)
    if not entries:
        problems.append("no entry points found in the header")
    for entry in entries:
        if entry in EXEMPT or any(entry.endswith(s) for s in EXEMPT_SUFFIXES):
            continue
        if entry not in covered:
            problems.append(f"entry point without a contract test: {entry}")
    return problems


def test_every_entry_point_has_a_contract_test():
    assert _entry_problems(HEADER) == []


def test_entry_point_guard_notices_a_new_entry_point_and_a_missing_test(tmp_path, monkeypatch):
    fake = tmp_path / "yume_b200.h"
    fake.write_text(HEADER.read_text().replace("int yb_bcast_add(", "int yb_new_kernel(const void* x, void* stream);\n"
                                               "int yb_bcast_add(", 1))
    assert _entry_problems(fake) == ["entry point without a contract test: yb_new_kernel"]
    covers = dict(KX.COVERS)
    covers["yb_blend"] = ["test_blend_renamed"]
    monkeypatch.setattr(KX, "COVERS", covers)
    assert _entry_problems(HEADER) == [
        "test_gpu_kernel_contract_ext.COVERS['yb_blend'] names a test that does not exist: test_blend_renamed"]
    del covers["yb_blend"]
    assert _entry_problems(HEADER) == ["entry point without a contract test: yb_blend"]


# ------------------------------------------------------------------------------------------------------------
# yb_vae_rms_act instance guard
# ------------------------------------------------------------------------------------------------------------
def _rms_problems(src, widths):
    text = src.read_text()
    problems = []
    inst = {(int(n), int(g)) for n, g in re.findall(r"YB_RMS_LAUNCH\((\d+),\s*(\d+)\);", text)}
    if not inst:
        problems.append("no YB_RMS_LAUNCH instances found")
    m1 = re.search(r"nch = C <= (\d+) \? 1 : \(C <= (\d+) \? 2 : 4\);", text)
    m2 = re.search(r"g = nch > 1 \? 32 : \(Cp <= (\d+) \? 8 : \(Cp <= (\d+) \? 16 : 32\)\);", text)
    if not (m1 and m2):
        return problems + ["the width rule of yb_vae_rms_act was not found (update this guard with it)"]
    c1, c2, p1, p2 = int(m1[1]), int(m1[2]), int(m2[1]), int(m2[2])
    reached = set()
    for C, Cp in widths:
        nch = 1 if C <= c1 else (2 if C <= c2 else 4)
        g = 32 if nch > 1 else (8 if Cp <= p1 else (16 if Cp <= p2 else 32))
        if KX.rms_instance(C, Cp) != (nch, g):
            problems.append(f"rms_instance({C}, {Cp}) = {KX.rms_instance(C, Cp)}, the kernel picks {(nch, g)}")
        reached.add((nch, g))
    for n, g in sorted(inst - reached):
        problems.append(f"YB_RMS_LAUNCH({n}, {g}) is reached by no tested width")
    return problems


def test_every_rms_act_instance_has_a_tested_width():
    assert _rms_problems(CSRC / "vae_elementwise.cu", KX.RMS_WIDTHS) == []


def test_rms_act_guard_notices_a_dropped_width():
    widths = tuple(w for w in KX.RMS_WIDTHS if w != (48, 64))
    assert _rms_problems(CSRC / "vae_elementwise.cu", widths) == ["YB_RMS_LAUNCH(1, 8) is reached by no tested width"]


# ------------------------------------------------------------------------------------------------------------
# the new bounds reject their defects and accept the kernels' arithmetic
# ------------------------------------------------------------------------------------------------------------
def _masked_softmax_f32(S, L, hw, leak=0):
    """fp32 frame-causal softmax as the kernel computes it (max, exp of the shifted logits, fp32 sum, 1/sum, bf16 out);
    leak = 1 moves every frame boundary one key late (one next-frame key enters the row)."""
    rows = torch.arange(S.shape[0])[:, None] // hw
    cols = torch.arange(S.shape[1])[None, :]
    keep = (cols < (torch.clamp((rows + 1) * hw + leak, max=L))) & (cols < L)
    s = S.masked_fill(~keep, -math.inf)
    e = torch.exp(s - s.amax(1, keepdim=True))
    return (e * (1.0 / e.sum(1, keepdim=True))).bfloat16()


def test_masked_softmax_bound_rejects_a_leaked_next_frame_key():
    g = torch.Generator().manual_seed(11)
    hw, L = 40, 115
    S = torch.randn(L, 128, generator=g) * 8
    p, f32, keep = KX.softmax_bound(S, L, hw)
    bound = K.bf16_out_bound(p, f32)
    assert K.assert_within(_masked_softmax_f32(S, L, hw), p, bound, "masked_softmax fp32") <= 1.0
    with pytest.raises(AssertionError, match="out of bound"):
        K.assert_within(_masked_softmax_f32(S, L, hw, leak=1), p, bound, "masked_softmax boundary one key late")


def test_avgdown_bound_rejects_a_dropped_group_element():
    g = torch.Generator().manual_seed(12)
    T, H, W, in_c, out_c, ft, fs = 5, 4, 4, 64, 64, 2, 2
    G = in_c * ft * fs * fs // out_c
    x = torch.randn(T * H * W, in_c, generator=g).bfloat16()
    m0 = torch.randn(3, 2, 2, out_c, generator=g).bfloat16()
    mean, absmean = KX.avgdown_ref(x, (T, H, W), in_c, out_c, ft, fs)
    ref = m0.double() + mean
    bound = K.bf16_out_bound(ref, (G - 1) * K.U32 * absmean + K.U32 * ref.abs())
    # the same grouping in fp32, as the kernel sums it: sequential over the G members, times the exact 1/G
    xn = torch.nn.functional.pad(x.float().view(T, H, W, in_c).permute(3, 0, 1, 2)[None], (0, 0, 0, 0, 1, 0))
    xn = xn.view(1, in_c, 3, ft, 2, fs, 2, fs).permute(0, 1, 3, 5, 7, 2, 4, 6).reshape(out_c, G, 3, 2, 2)
    acc = torch.zeros(out_c, 3, 2, 2)
    for j in range(G):
        acc = acc + xn[:, j]
    good = (m0.float() + (acc * (1.0 / G)).permute(1, 2, 3, 0)).bfloat16()
    assert K.assert_within(good, ref, bound, "avgdown fp32") <= 1.0
    bad = (m0.float() + ((acc - xn[:, G - 1]) * (1.0 / G)).permute(1, 2, 3, 0)).bfloat16()
    with pytest.raises(AssertionError, match="out of bound"):
        K.assert_within(bad, ref, bound, "avgdown one group element dropped")


def test_zero_pad_conv_bound_rejects_replicate_padding_on_one_face():
    g = torch.Generator().manual_seed(13)
    T, H, W, Cp, co, taps = 2, 5, 6, 64, 32, (3, 3, 3)
    x = (torch.randn(T, H, W, Cp, generator=g) + 1.0).bfloat16()
    wt = (torch.randn(co, Cp, 3, 3, 3, generator=g) / math.sqrt(27 * Cp)).bfloat16()
    acc, Fb, _ = KX._conv_ref(x, wt, taps)
    bound = K.bf16_out_bound(acc, Fb + 4 * K.U32 * acc.abs())
    xf = x.float().permute(3, 0, 1, 2)[None]
    zero = torch.nn.functional.pad(xf, (1, 1, 1, 1, 2, 0))
    good = torch.nn.functional.conv3d(zero, wt.float())[0].permute(1, 2, 3, 0).reshape(-1, co).bfloat16()
    assert K.assert_within(good, acc, bound, "conv zero pad fp32") <= 1.0
    rep = zero.clone()
    rep[..., 0] = rep[..., 1]                                     # the left W face replicated instead of zero
    bad = torch.nn.functional.conv3d(rep, wt.float())[0].permute(1, 2, 3, 0).reshape(-1, co).bfloat16()
    with pytest.raises(AssertionError, match="out of bound"):
        K.assert_within(bad, acc, bound, "conv replicate-padded left face")


def test_n_split_check_rejects_a_straddling_tile_sent_to_the_wrong_chunk():
    """W3 = 384, 256-column tiles: tile 1 covers columns 256..511, i.e. chunk 0 columns 256..383 and chunk 1 columns 0..127.
    The defect stores that second half into chunk 2 instead (chunk 1 keeps its NaN poison there)."""
    got, ref, bound = _gemm_case(M=64, N=4 * 384, Kd=128)
    P, W3 = 4, 384
    chunks = got.view(64, P, W3).permute(1, 0, 2).clone()              # [P, Lp, W3] as the kernel lays it out
    assert K.assert_within(chunks.permute(1, 0, 2).reshape(64, P * W3), ref, bound, "n_split layout") <= 1.0
    chunks[2, :, :128] = chunks[1, :, :128]
    chunks[1, :, :128] = float("nan")
    with pytest.raises(AssertionError, match="out of bound"):
        K.assert_within(chunks.permute(1, 0, 2).reshape(64, P * W3), ref, bound, "n_split straddling tile misplaced")


def test_sp_sums_bound_rejects_a_missing_head_block():
    g = torch.Generator().manual_seed(14)
    L, C = 16, 3072
    q = torch.randn(L, C, generator=g).bfloat16()
    xsq = q.double().pow(2).sum(1)
    bound = KX.sumsq_bound(xsq, C)
    sq = q.float().pow(2)
    good = sq.view(L, C // 256, 256).sum(2).sum(1)                    # per-tile partials, then across tiles (fp32)
    assert K.assert_within(good, xsq, bound, "sum q^2 fp32") <= 1.0
    bad = good.clone()
    bad[5] = sq[5, :C - 128].sum()
    with pytest.raises(AssertionError, match=r"1 of 16 elements out of bound; worst at \(5,\)"):
        K.assert_within(bad, xsq, bound, "sum q^2 without the last head block")


# ------------------------------------------------------------------------------------------------------------
# production-shape contract (tests/test_gpu_kernel_contract_prod.py): the table stays multi-wave, the sampler hits every
# tile, and the sampled checker rejects cross-tile defects at production M x N
# ------------------------------------------------------------------------------------------------------------
import test_gpu_kernel_contract_prod as KP  # noqa: E402


def _wave_problems(table):
    problems = []
    vae_cfgs = {r["cfg"] for r in table if r["entry"] == "conv"}
    multi = set()
    for r in table:
        p = KP.row_plan(r)
        if r["entry"] in ("attention", "attention_sp"):
            if r.get("self_attn") and p["nkv"] < 100:
                problems.append(f"{r['id']}: {p['nkv']} KV tiles < 100")
            if not r.get("self_attn") and p["per_cta"] < 3:
                problems.append(f"{r['id']}: {p['per_cta']:.2f} units per SM < 3")
        elif p["per_cta"] >= 3:
            multi.add(r["cfg"])
            if r["id"] in KP.WAVE_EXEMPT:
                problems.append(f"{r['id']}: exempt, but plans {p['per_cta']:.2f} tiles per CTA")
        elif r["id"] not in KP.WAVE_EXEMPT:
            problems.append(f"{r['id']}: {p['per_cta']:.2f} tiles per CTA < 3")
    for cfg in sorted(vae_cfgs - multi):
        problems.append(f"{cfg}: no conv / GEMM row with >= 3 tiles per CTA")
    for tree in ("5b", "14b"):
        if not any(r["entry"] == "attention" and r.get("self_attn") and r["cfg"].startswith(tree) and KP.row_plan(r)["tail"] > 0
                   for r in table):
            problems.append(f"no {tree} self-attention row takes the tail split")
    if not any(r["entry"] == "gemm" and r.get("raster") and KP.row_plan(r)["n_tiles"] >= 100 * KP.row_plan(r)["m_tiles"]
               for r in table):
        problems.append("no raster row with >= 100 N tiles per M tile")
    return problems


def test_production_table_is_multi_wave():
    assert _wave_problems(KP.PROD_TABLE) == []


def test_multi_wave_guard_notices_a_shrunk_table():
    t = KP.PROD_TABLE
    no_split = [r for r in t if not (r["entry"] == "attention" and r["id"] == "5b.self_attention")]
    assert _wave_problems(no_split) == ["no 5b self-attention row takes the tail split"]
    short = [dict(r, L=2310, M=2310) if r["id"] == "5b.o" else r for r in t]
    assert _wave_problems(short) == ["5b.o: 1.73 tiles per CTA < 3"]
    short_kv = [dict(r, Lk=8000) if r["id"] == "14b_grid.self_attention" else r for r in t]
    assert _wave_problems(short_kv) == ["14b_grid.self_attention: 63 KV tiles < 100"]
    no_raster = [r for r in t if not r.get("raster")]
    assert _wave_problems(no_raster) == ["no raster row with >= 100 N tiles per M tile"]
    grown = [dict(r, T=9) if r["id"] == "hy_tile.conv9_2x64x64_512to512_k333" else r for r in t]
    assert _wave_problems(grown) == ["hy_tile.conv9_2x64x64_512to512_k333: exempt, but plans 4.36 tiles per CTA"]


def _sample_problems(table, gemm_sample=None):
    gemm_sample = gemm_sample or KP.gemm_sample
    problems = []
    for r in table:
        p = KP.row_plan(r)
        if r["entry"] == "gemm":
            rows, cols = gemm_sample(r["M"], r["N"], r["id"])
            for bm in (128, 256):
                miss = KP.gemm_tiles_missed(rows, cols, r["M"], r["N"], bm, p["block_n"])
                if miss:
                    problems.append(f"{r['id']}: {len(miss)} {bm}-row tiles without samples, first {miss[0]}")
        elif r["entry"] == "gemm_sp_qkv":          # every rank's own 256-row SM-pair tiles and 256-wide N tiles
            rows, cols = KP.gemm_sp_qkv_sample(r)
            for rank in range(r["P"]):
                mine = rows[(rows // r["Lp"]) == rank] - rank * r["Lp"]
                miss = KP.gemm_tiles_missed(mine, cols, r["Lp"], 3 * r["C"], p["block_m"], p["block_n"])
                if miss:
                    problems.append(f"{r['id']}: rank {rank}: {len(miss)} tiles without samples, first {miss[0]}")
        elif r["entry"] == "conv":
            miss = KP.conv_boxes_missed(KP.conv_sample(p["dims"], p["box"], r["id"]), p["dims"], p["box"])
            if miss:
                problems.append(f"{r['id']}: {len(miss)} boxes without samples")
        elif r["entry"] in ("attention", "attention_sp"):
            miss = KP.attention_units_missed(KP.attention_sample(p["Lq"], p["heads"], r["id"]), p["Lq"], p["heads"])
            if miss:
                problems.append(f"{r['id']}: {len(miss)} (head, unit, query tile) without samples, first {miss[0]}")
    return problems


def test_sampler_hits_every_tile_box_and_unit():
    assert _sample_problems(KP.PROD_TABLE) == []


def test_sampler_guard_notices_a_band_without_samples():
    def broken(M, N, key):                                   # the rows of band 5 never sampled
        rows, cols = KP.gemm_sample(M, N, key)
        return rows[(rows // 128) != 5], cols[(cols // 256) != 3]
    rows = [r for r in KP.PROD_TABLE if r["id"] == "5b.qkv"]
    probs = _sample_problems(rows, broken)
    assert probs and "5b.qkv: 1 128-row tiles without samples, first (5, 3)" in probs[0]


def _prod_gemm_case(gated=False):
    """Production M x N (the 5B o-projection) with K = 16, computed the way the kernel does (fp32 accumulation)."""
    g = torch.Generator().manual_seed(21)
    M, N, Kd = 18480, 3072, 16
    A = torch.randn(M, Kd, generator=g).bfloat16()
    B = (torch.randn(N, Kd, generator=g) / 4).bfloat16()
    bias = torch.randn(N, generator=g)
    acc = A.float() @ B.float().t() + bias
    if not gated:
        return A, B, bias, acc, None
    gate6 = torch.randn(2, 6, N, generator=g)
    tok = (torch.arange(M) >= M // 3).long()
    return A, B, bias, acc, (gate6, tok)


@pytest.mark.parametrize("tile", [(0, 4), (77, 5), (144, 11)])     # first band, interior, last (partial: 48 rows) band
def test_prod_gemm_check_rejects_a_tile_written_with_its_neighbours_coordinates(tile):
    A, B, bias, acc, _ = _prod_gemm_case()
    got = acc.bfloat16()
    rows, cols = KP.gemm_sample(A.shape[0], B.shape[0], "defect")
    KP._check_gemm_sampled(got, A, B, rows, cols, KP.EPI["BF16"], "kernel arithmetic", None, bias=bias)
    i, j = tile
    jn = j + 1 if j + 1 < 12 else j - 1
    rs = slice(i * 128, min((i + 1) * 128, A.shape[0]))
    got[rs, j * 256:(j + 1) * 256] = got[rs, jn * 256:(jn + 1) * 256]
    with pytest.raises(AssertionError, match="out of bound"):
        KP._check_gemm_sampled(got, A, B, rows, cols, KP.EPI["BF16"], f"tile {tile} from its neighbour", None, bias=bias)


def test_prod_gemm_check_rejects_a_gate_res_tile_with_the_wrong_tok_idx_row():
    A, B, bias, acc, (gate6, tok) = _prod_gemm_case(gated=True)
    x0 = torch.randn(acc.shape, generator=torch.Generator().manual_seed(3))
    gate_rows = lambda ri: gate6[tok[ri if ri is not None else slice(None)], 2].double()      # noqa: E731
    good = x0 + acc * gate6[tok, 2]
    rows, cols = KP.gemm_sample(A.shape[0], B.shape[0], "defect")
    KP._check_gemm_sampled(good, A, B, rows, cols, KP.EPI["GATE_RES"], "GATE_RES kernel arithmetic", None, bias=bias, x0=x0,
                           gate_rows=gate_rows)
    bad = good.clone()
    rs, cs = slice(10 * 128, 11 * 128), slice(3 * 256, 4 * 256)          # a tile of history tokens used the new-token gate
    bad[rs, cs] = x0[rs, cs] + acc[rs, cs] * gate6[1, 2, cs]
    with pytest.raises(AssertionError, match="out of bound"):
        KP._check_gemm_sampled(bad, A, B, rows, cols, KP.EPI["GATE_RES"], "GATE_RES wrong tok_idx row", None, bias=bias, x0=x0,
                               gate_rows=gate_rows)


def _prod_attention_case(seed, drop_unit=None, Lq=1024, Lk=18480):
    """One head, Lq = 1024 (4 units), Lk = 18480 (145 KV tiles), data drawn like the GPU test's (q * 2, unit-variance k and v)
    and computed as the kernel does (fp32 logits and softmax, P in bf16, fp32 normaliser, bf16 out). drop_unit: KV tile 100
    is missing from every row of that unit."""
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(Lq, 128, generator=g) * 2).bfloat16()
    k, v = torch.randn(Lk, 128, generator=g).bfloat16(), torch.randn(Lk, 128, generator=g).bfloat16()
    scale = 1 / math.sqrt(128.0)
    s = (q.float() @ k.float().t()) * scale
    if drop_unit is not None:
        s[drop_unit * 256:(drop_unit + 1) * 256, 100 * 128:101 * 128] = -math.inf
    p = torch.exp(s - s.amax(-1, keepdim=True))
    got = ((p.bfloat16().float() @ v.float()) / p.sum(-1, keepdim=True)).bfloat16()
    return got, q, k, v, scale, dict(nkv=-(-Lk // 128), ns=1)


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_prod_attention_check_rejects_kv_tile_100_dropped_in_one_unit(seed):
    """The dropped tile is in a unit the sampler covers with its per-tile rows only (not the one whole unit per head)."""
    key = ("defect", seed)
    whole = int(torch.bincount(KP.attention_sample(1024, 1, key)[0] // 256).argmax())
    got, q, k, v, scale, plan = _prod_attention_case(seed)
    KP._check_attention_sampled(got, q, k, v, 1, scale, plan, key, "kernel arithmetic", None)
    got, q, k, v, scale, plan = _prod_attention_case(seed, drop_unit=(whole + 1) % 4)
    with pytest.raises(AssertionError, match=r"head0: \d+ of \d+ elements out of bound"):
        KP._check_attention_sampled(got, q, k, v, 1, scale, plan, key, "KV tile 100 dropped in one unit", None)


def test_prod_attention_check_rejects_a_tail_unit_with_an_unwritten_second_query_tile():
    got, q, k, v, scale, plan = _prod_attention_case(0)
    got[768 + 128:1024] = float("nan")                         # the last unit's second 128-row query tile
    with pytest.raises(AssertionError, match=r"\|err\|/bound = inf"):
        KP._check_attention_sampled(got, q, k, v, 1, scale, plan, "defect", "second query tile never written", None)
