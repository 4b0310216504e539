"""precision="fp8" without a GPU: the weight and activation quantisers against the numerics contract (include/yume_b200_fp8.h),
the engine's fp8 host logic over the torch stand-ins (tests/helpers/torch_ops_fp8.py) against the fp8-qdq oracle, the rejections,
the entry-point guard of the new header, and the GEMM bound of the GPU contract against realistic kernel defects."""
import contextlib
from pathlib import Path

import pytest
import torch

import test_gpu_kernel_contract_fp8 as KF
from helpers import torch_ops_fp8
from oracle import synth
from oracle.fp8 import WanOracleFp8, dequantize_act, quantize_act, quantize_weight
from test_kernel_contract_cpu import _entry_problems
from yume_b200 import dit
from yume_b200._lib import YumeB200Error

FP8_HEADER = Path(__file__).resolve().parents[1] / "include" / "yume_b200_fp8.h"
E4M3 = torch.float8_e4m3fn


# ------------------------------------------------------------------------------------------------------------
# quantisers
# ------------------------------------------------------------------------------------------------------------
def test_weight_quantisation_per_channel():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(64, 384, generator=g) * torch.exp(torch.randn(64, 1, generator=g))
    w[5] = 0.0
    wq, sw = dit.quantize_weight_fp8(w)
    assert wq.dtype == E4M3 and sw.dtype == torch.float32 and sw.shape == (64,)
    amax = w.abs().amax(dim=1)
    assert torch.equal(sw, amax / torch.full_like(amax, 448.0))
    assert sw[5] == 0 and (wq[5].float() == 0).all()
    rows = torch.arange(64) != 5
    assert (wq.float().abs().amax(dim=1)[rows] == 448).all(), "the row maximum lands exactly on 448"
    deq = wq.float() * sw[:, None]
    # e4m3 keeps 3 mantissa bits: half an ulp is 2^-4 of the value; below 2^-6 (subnormals) the step is 2^-9 of the scale
    tol = torch.maximum(w.abs() * 2.0 ** -4, sw[:, None] * 2.0 ** -10) * (1 + 1e-6)
    assert ((deq - w).abs() <= tol).all()
    oq, osw = quantize_weight(w)                     # the oracle's twin, written from the same contract
    assert torch.equal(oq.view(torch.uint8), wq.view(torch.uint8)) and torch.equal(osw, sw)


def test_activation_twin_group_edges():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 384, generator=g)
    x[0, 127], x[0, 128] = 1000.0, -30.0             # column 127 is the last of group 0, column 128 the first of group 1
    q, s = quantize_act(x)
    assert q.shape == (2, 384) and s.shape == (3, 2)
    assert s[0, 0] == torch.tensor(1000.0) / 448 and q[0, 127].float() == 448
    assert s[1, 0] == torch.tensor(30.0) / 448 and q[0, 128].float() == -448
    assert (q.float().abs().view(2, 3, 128).amax(dim=-1) == 448).all()


def test_activation_twin_zero_tiny_and_nan_groups():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(4, 384, generator=g)
    x[1, :128] = 0.0
    x[2, 128:256] = 1e-38                            # 448 / amax overflows: stored as zeros with scale 0
    x[3, 7] = float("nan")
    q, s = quantize_act(x)
    assert s[0, 1] == 0 and (q[1, :128].float() == 0).all()
    assert s[1, 2] == 0 and (q[2, 128:256].float() == 0).all()
    assert torch.isnan(q[3, 7].float()) and torch.isfinite(q[3, :7].float()).all()
    assert s[0, 3] == torch.cat([x[3, :7], x[3, 8:128]]).abs().max() / 448     # NaN takes no part in the group maximum
    deq = dequantize_act(q, s)
    ok = torch.isfinite(deq)
    ok[2, 128:256] = False                           # flushed to zero on purpose
    sc = s.t().repeat_interleave(128, dim=1)
    assert ((deq - x).abs()[ok] <= torch.maximum(x.abs() * 2.0 ** -4, sc * 2.0 ** -10)[ok] * (1 + 1e-6)).all()


# ------------------------------------------------------------------------------------------------------------
# the engine's fp8 host logic
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def cpu_fp8_engine(monkeypatch):
    monkeypatch.setattr(dit, "ops", torch_ops_fp8)
    monkeypatch.setattr(torch.cuda, "device", lambda *_a, **_k: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)

    def make(cfg, sd, precision="fp8"):
        kw = synth.oracle_kwargs(cfg)
        variant = kw.pop("variant")
        return dit.WanDiT(sd, variant, device="cpu", precision=precision, **kw)
    return make


def _forward(eng, cfg, c, inp):
    if cfg["variant"] == "5b":
        return eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], latent_frame_zero=c["lfz"], packed=c["flag"])
    return eng.forward(inp["x"], torch.tensor(c["t"]), inp["context"], c["seq_len"], y=inp["y"], clip_fea=inp["clip_fea"],
                       latent_frame_zero=c["lfz"], packed=c["rand_num_img"] >= 0.4)


def _oracle(orc, cfg, c, inp):
    if cfg["variant"] == "5b":
        return orc.forward([inp["x"]], torch.tensor(c["t"]), [inp["context"]], seq_len=c["seq_len"], latent_frame_zero=c["lfz"],
                           flag=c["flag"])
    return orc.forward([inp["x"]], torch.tensor(c["t"]), [inp["context"]], seq_len=c["seq_len"], y=[inp["y"]],
                       clip_fea=inp["clip_fea"], latent_frame_zero=c["lfz"], rand_num_img=c["rand_num_img"])


# measured worst over CASES: fp8 engine over the stand-ins vs the fp8-qdq oracle 1.54e-2, vs the reference's own bf16 forward
# 2.63e-2 (the cost of fp8: the bf16 engine is within 5e-3 of it). The qdq oracle cannot be much closer than that at the whole
# forward: the fp8 model is that sensitive to its input. The oracle against itself moves by 7.9e-3 when the latent is perturbed by
# 1e-7 (relative), 1.1e-2 at 2^-9: every perturbation moves some e4m3 roundings by a whole 2^-3 step, and two layers propagate
# them. Kernel defects are caught per GEMM by the per-element bound of tests/test_gpu_kernel_contract_fp8.py, not here.
QDQ_BAR = 3e-2
REF_BAR = 5e-2
CASES = [("wan23_tiny.pt", "5b_pack_h10"), ("wan23_tiny.pt", "5b_grid_padded"), ("wan21_tiny.pt", "14b_grid"),
         ("wan21_tiny.pt", "14b_pack_h4"), ("wan23_h8.pt", "5b_pack_h10"), ("wan21_h8.pt", "14b_pack_lfz8")]


@pytest.mark.parametrize("fname,case", CASES)
def test_fp8_engine_host_logic_matches_the_fp8_qdq_oracle(cpu_fp8_engine, golden_dir, fname, case):
    g = torch.load(golden_dir / fname, weights_only=False)
    cfg, c = g["cfg"], g["cases"][case]
    sd = synth.make_state_dict(cfg, g["seed_w"])
    inp = synth.make_inputs(cfg, c["seed"], c["frames"], c["H"], c["W"], c["ctx_len"])
    eng = cpu_fp8_engine(cfg, sd)
    assert all(eng.blocks[0][k][0].dtype == E4M3 for k in dit.FP8_WEIGHTS)
    got = _forward(eng, cfg, c, inp)
    want = _oracle(WanOracleFp8(sd, **synth.oracle_kwargs(cfg)), cfg, c, inp)
    rel = float((got - want).norm() / want.norm())
    ref = float((got - c["out"]).norm() / c["out"].norm())
    print(f"{fname}:{case}: vs fp8-qdq oracle {rel:.2e}, vs reference bf16 forward {ref:.2e}")
    assert rel < QDQ_BAR
    assert ref < REF_BAR


def test_fp8_rejections(cpu_fp8_engine):
    cfg = dict(synth.CFG_5B_TINY, ffn_dim=500)
    sd = synth.make_state_dict(synth.CFG_5B_TINY, 0)
    with pytest.raises(YumeB200Error, match="divisible by 128"):
        cpu_fp8_engine(cfg, sd)
    with pytest.raises(YumeB200Error, match="divisible by 128"):
        cpu_fp8_engine(dict(synth.CFG_5B_TINY, dim=200), sd)
    with pytest.raises(YumeB200Error, match="precision"):
        cpu_fp8_engine(synth.CFG_5B_TINY, sd, precision="fp16")
    eng = cpu_fp8_engine(synth.CFG_5B_TINY, sd)
    with pytest.raises(YumeB200Error, match="sequence parallel"):
        eng.enable_sequence_parallel(None)


def test_fp8_rejects_a_width_without_an_fp8_layernorm(cpu_fp8_engine):
    """dim 1536 is a multiple of 128 but has no yb_ln_modulate_fp8 instance: rejected when the engine is built, not at the first
    forward. The widths listed in the engine are exactly the kernel's instances."""
    import re
    cfg = dict(synth.CFG_5B_TINY, dim=1536, num_heads=12)
    with pytest.raises(YumeB200Error, match="fp8 LayerNorm"):
        cpu_fp8_engine(cfg, synth.make_state_dict(cfg, 0))
    src = (Path(__file__).resolve().parents[1] / "yume_b200" / "csrc" / "gemm_fp8.cu").read_text()
    assert sorted(128 * int(n) for n in re.findall(r"^\s*YB_LN8\((\d+)\)", src, flags=re.M)) == sorted(dit.FP8_LN_WIDTHS)


def _mirror_kwargs(cfg):
    return dict(text_len=cfg["text_len"], in_dim=cfg["in_dim"], dim=cfg["dim"], ffn_dim=cfg["ffn_dim"], freq_dim=cfg["freq_dim"],
                text_dim=cfg["text_dim"], out_dim=cfg["out_dim"], num_heads=cfg["num_heads"], num_layers=cfg["num_layers"])


def test_public_switches_and_the_self_attention_seam_in_fp8(cpu_fp8_engine, golden_dir):
    """install(model, precision="fp8") through both of its paths (state_dict, and WanDiT.from_module on a loaded module), the
    mirrors' .install(precision=), and the fp8 WanSelfAttention seam against the fp8-qdq oracle's self-attention."""
    import yume_b200
    from oracle.wan_dit import grid_freqs
    from yume_b200.model import WanModel5B, install
    g = torch.load(golden_dir / "wan23_tiny.pt", weights_only=False)
    cfg = g["cfg"]
    sd = synth.make_state_dict(cfg, g["seed_w"])

    def fp8_weights(m):
        eng = m._yb_engine
        return eng.precision == "fp8" and all(b[k][0].dtype == E4M3 and b[k][1].dtype == torch.float32
                                              for b in eng.blocks for k in dit.FP8_WEIGHTS)
    with torch.device("meta"):
        mirror = WanModel5B(model_type="ti2v", **_mirror_kwargs(cfg))
    m = mirror.install("cpu", state_dict=sd, precision="fp8")
    assert fp8_weights(m)
    loaded = WanModel5B(model_type="ti2v", **_mirror_kwargs(cfg))
    loaded.load_state_dict({k: v for k, v in sd.items() if k in loaded.state_dict()})
    assert fp8_weights(install(loaded, device="cpu", precision="fp8"))
    assert install(WanModel5B(model_type="ti2v", **_mirror_kwargs(cfg)), device="cpu")._yb_engine.precision == "bf16"

    m = yume_b200.install_seams(m)
    orc = WanOracleFp8(sd, **synth.oracle_kwargs(cfg))
    gen = torch.Generator().manual_seed(5)
    L, C = 2 * 8 * 8, cfg["dim"]
    h = torch.randn(1, L, C, generator=gen).to(torch.bfloat16).float()      # the seam's input is bf16
    fr = grid_freqs(orc.tables, 2, 8, 8, f0=3)
    want = orc.self_attn("blocks.0.self_attn", h, fr)[0]
    got = m.blocks[0].self_attn(h, torch.tensor([L]), None, fr, None, None, None, True)[0]
    rel = float((got.float() - want).norm() / want.norm())
    print(f"fp8 self-attention seam vs fp8-qdq oracle {rel:.2e}")
    assert got.dtype == torch.bfloat16 and rel < QDQ_BAR


# ------------------------------------------------------------------------------------------------------------
# C-ABI guards over include/yume_b200_fp8.h
# ------------------------------------------------------------------------------------------------------------
def test_fp8_header_symbols_are_bound():
    import re
    from yume_b200 import _lib
    declared = set(re.findall(r"^\s*(?:int|long long)\s+(yb_\w+)\s*\(", FP8_HEADER.read_text(), flags=re.M))
    assert declared == {"yb_gemm_fp8", "yb_ln_modulate_fp8", "yb_quant_rows_fp8"} == set(_lib.FP8_SIGNATURES)
    assert not declared & (set(_lib.SIGNATURES) | set(_lib.CLIP_SIGNATURES) | set(_lib.T5_SIGNATURES) | set(_lib.STREAM_SIGNATURES))


def test_every_fp8_entry_point_has_a_contract_test():
    assert _entry_problems(FP8_HEADER, modules=(KF,)) == []


def test_fp8_entry_point_guard_notices_a_missing_test(monkeypatch):
    covers = dict(KF.COVERS)
    del covers["yb_quant_rows_fp8"]
    monkeypatch.setattr(KF, "COVERS", covers)
    assert _entry_problems(FP8_HEADER, modules=(KF,)) == ["entry point without a contract test: yb_quant_rows_fp8"]


# ------------------------------------------------------------------------------------------------------------
# the GPU contract's GEMM bound rejects realistic defects
# ------------------------------------------------------------------------------------------------------------
def _truncate(x, bits):
    """x rounded toward zero to `bits` mantissa bits (a model of the fp8 tensor-core accumulator)."""
    m, e = torch.frexp(x)
    step = torch.ldexp(torch.ones_like(x), e - bits)
    return torch.trunc(x / step) * step


def _operands(M=128, N=128, K=2048, positive=False, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g, dtype=torch.float64) * (1 + 3 * torch.rand(M, 1, generator=g, dtype=torch.float64))
    w = torch.randn(N, K, generator=g, dtype=torch.float64) * 0.02
    if positive:
        x, w = x.abs(), w.abs()
    x = x * torch.exp(torch.randn(1, K // 128, generator=g, dtype=torch.float64)).repeat_interleave(128, dim=1)
    aq, sa = quantize_act(x.float())
    wq, sw = quantize_weight(w.float())
    return aq.double(), sa.double(), wq.double(), sw.double()


def _kernel_model(aq, sa, wq, sw, defect=None):
    """Per-group wgmma (ACC_BITS truncation after each k32 step) and fp32-exact promotion, with an optional defect."""
    M, K = aq.shape
    G = K // 128
    acc = torch.zeros(M, wq.shape[0], dtype=torch.float64)
    if defect == "no_promotion":              # the whole K in the fp8 accumulator, one scale (valid: the test uses equal scales)
        run = torch.zeros_like(acc)
        for k in range(0, K, 32):
            run = _truncate(run + aq[:, k:k + 32] @ wq[:, k:k + 32].t(), KF.ACC_BITS)
        return run * sa[0][:, None] * sw[None, :]
    for gi in range(G):
        if defect == "drop_group" and gi == G // 2:
            continue
        part = torch.zeros_like(acc)
        for k in range(gi * 128, gi * 128 + 128, 32):
            part = _truncate(part + aq[:, k:k + 32] @ wq[:, k:k + 32].t(), KF.ACC_BITS)
        s = sa[gi]
        if defect == "neighbour_row":
            s = torch.roll(s, 1)
        if defect == "neighbour_group":
            s = sa[(gi + 1) % G]
        acc = acc + s[:, None] * part
    return acc * (1.0 if defect == "no_weight_scale" else sw[None, :])


@pytest.mark.parametrize("defect", [None, "drop_group", "neighbour_row", "neighbour_group", "no_weight_scale", "no_promotion"])
def test_gemm_bound_accepts_the_kernel_model_and_rejects_defects(defect):
    positive = defect == "no_promotion"                        # ffn.2 reads GELU outputs: mostly positive
    aq, sa, wq, sw = _operands(K=14336 if positive else 2048, positive=positive)
    if positive:
        sa = sa[:1].expand_as(sa).clone()                      # one scale for every group, so that a single accumulator is valid
    ad = aq * sa.t().repeat_interleave(128, dim=1)
    wd = wq * sw[:, None]
    ref = ad @ wd.t()
    bound = KF.gemm_bound(ad.abs(), wd.abs(), aq.shape[1], 2.0 ** -24, ref)
    ratio = float(((_kernel_model(aq, sa, wq, sw, defect) - ref).abs() / bound).max())
    if defect is None:
        assert ratio <= 1.0
    else:
        assert ratio > 1.0, f"{defect} passes the bound (worst ratio {ratio:.3f})"
