"""CLIP image encoder (yume_b200/clip.py, oracle/clip.py, include/yume_b200_clip.h) without a GPU:
  * oracle/clip.py reproduces tests/golden/clip_tiny.pt, which tools/make_golden_clip.py wrote by running the reference's own
    CLIPModel.visual (fp32 on CPU), and its preprocessed-image sample;
  * the engine's host logic (weight re-packing with heads padded 80 -> 128, the embedding table, the patch K padding, the
    block sequence) reproduces the same fixtures over the torch stand-in of its ops (tests/helpers/torch_ops_clip.py);
  * the ViT-H/14 state-dict layout the engine reads is the reference's, and install_clip reads every key it needs;
  * configurations the engine does not implement raise, and non-list inputs behave as the reference's;
  * the C-ABI guards of include/yume_b200.h applied to include/yume_b200_clip.h, and the resample bound of
    tests/test_gpu_kernel_contract_clip.py rejects an unclamped tap, align_corners=True and an antialiased resample while
    accepting the kernel's arithmetic emulated in fp32.
"""
import re
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

import test_gpu_kernel_contract_clip as KC
from helpers import clip_standin, torch_ops_clip
from oracle import clip as oclip
from test_kernel_contract_cpu import _entry_problems

ROOT = Path(__file__).resolve().parents[1]
CLIP_HEADER = ROOT / "include" / "yume_b200_clip.h"


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(golden_dir / "clip_tiny.pt", weights_only=False)


def _images(gold, case):
    """The fixture's input images, regenerated from their seeds (tools/make_golden_clip.py:images)."""
    c = gold["cases"][case]
    out = []
    for (H, W), seed in zip(c["sizes"], c["seeds"]):
        g = torch.Generator().manual_seed(seed)
        out.append(torch.rand(3, 1, H, W, generator=g) * 2 - 1)
    assert abs(float(sum(u.abs().sum() for u in out)) - c["input_abs_sum"]) <= 1e-6 * c["input_abs_sum"], "input RNG drifted"
    return out


def _check_rows(out, c):
    """out [N, tokens, dim] against the fixture's stored rows: full shape, then rel-Frobenius over the stored token rows."""
    assert tuple(out.shape) == tuple(c["out_shape"]) and out.dtype == torch.float32
    return _rel(out[:, c["out_rows"].long()], c["out"])


def _sd(gold):
    sd = oclip.make_state_dict(gold["seed_w"], **gold["cfg"], out_dim=gold["out_dim"])
    got = float(sum(v.abs().sum() for v in sd.values()))
    assert abs(got - gold["weight_abs_sum"]) <= 1e-5 * gold["weight_abs_sum"], "weight RNG drifted"
    return sd


CASES = ["down_544x960", "identity_224", "up_150x200", "odd_33x47", "list_2"]


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference_fixture(gold, case):
    sd, cfg = _sd(gold), gold["cfg"]
    imgs = _images(gold, case)
    out = oclip.visual(sd, [u.clone() for u in imgs], **cfg)
    c = gold["cases"][case]
    err = _check_rows(out, c)
    assert err <= 2e-5, err
    pre = oclip.preprocess([u.clone() for u in imgs], cfg["image_size"])
    assert _rel(pre.reshape(-1)[c["pre_idx"].long()], c["pre_sample"]) <= 2e-5


def _engine(gold, monkeypatch, sd=None):
    from yume_b200 import clip as eng
    monkeypatch.setattr(eng, "ops", torch_ops_clip)
    cfg = gold["cfg"]
    return eng.ClipVisionEncoder(sd if sd is not None else _sd(gold), mean=gold["mean"], std=gold["std"], device="cpu", **cfg)


# The engine over the stand-in differs from the fixture by its bf16 GEMM / attention operands and bf16 LayerNorm outputs (the
# reference's fp32 path rounds only q, k, v to bf16). Measured worst rel-Frobenius over the cases: 3.7e-3; bar 7.5e-3 (2x margin).
ENGINE_BAR = 7.5e-3


@pytest.mark.parametrize("case", CASES)
def test_engine_host_logic_matches_reference_fixture(gold, monkeypatch, case):
    enc = _engine(gold, monkeypatch)
    imgs = _images(gold, case)
    err = _check_rows(enc.encode(imgs), gold["cases"][case])
    print(f"[clip] engine (stand-in ops) vs reference fixture {case}: rel-Frobenius {err:.3g}")
    assert err <= ENGINE_BAR


def test_engine_head_padding_is_exact(gold, monkeypatch):
    """The packed q|k|v weight holds each head's 80 rows then 48 zero rows (zero bias); the o-projection has zero columns at
    the padded positions; the patch weight's K padding (588 -> 592) is zero."""
    sd = _sd(gold)
    enc = _engine(gold, monkeypatch, sd)
    cfg = gold["cfg"]
    H, d, dim = cfg["heads"], cfg["dim"] // cfg["heads"], cfg["dim"]
    b = enc.blocks[1]
    w = b.w_qkv.float().view(3, H, 128, dim)
    assert torch.equal(w[:, :, :d], sd["transformer.1.attn.to_qkv.weight"].bfloat16().float().view(3, H, d, dim))
    assert not w[:, :, d:].any() and not b.b_qkv.view(3, H, 128)[:, :, d:].any()
    wo = b.w_o.float().view(dim, H, 128)
    assert torch.equal(wo[:, :, :d], sd["transformer.1.attn.proj.weight"].bfloat16().float().view(dim, H, d))
    assert not wo[:, :, d:].any()
    assert enc.w_patch.shape == (dim, 592) and not enc.w_patch[:, 588:].any()
    assert torch.equal(enc.table[1:], sd["pos_embedding"][0, 1:])
    assert torch.equal(enc.table[0], sd["cls_embedding"][0, 0] + sd["pos_embedding"][0, 0])
    assert len(enc.blocks) == cfg["layers"] - 1


def test_vit_h_14_layout_is_the_reference_layout(gold):
    cfg = gold["vit_h_14_cfg"]
    assert {k: cfg[k] for k in oclip.VIT_H_14} == oclip.VIT_H_14
    shapes = oclip.param_shapes(**oclip.VIT_H_14, out_dim=cfg["out_dim"])
    assert shapes == {k: tuple(v) for k, v in gold["vit_h_14_shapes"].items()}


class _Recording(dict):
    def __init__(self, *a):
        super().__init__(*a)
        self.read = set()

    def __getitem__(self, k):
        self.read.add(k)
        return super().__getitem__(k)


def test_engine_reads_every_key_it_needs(gold, monkeypatch):
    """Every weight of the embeddings, pre_norm and blocks 0 .. layers-2 is read; the last block, post_norm and head are not."""
    sd = _Recording(_sd(gold))
    _engine(gold, monkeypatch, sd)
    L = gold["cfg"]["layers"]
    unused = {k for k in sd if k.startswith(f"transformer.{L - 1}.") or k.startswith("post_norm") or k == "head"}
    assert sd.read == set(sd) - unused


def test_install_clip_rebinds_visual(gold, monkeypatch):
    from yume_b200 import clip as eng
    monkeypatch.setattr(eng, "ops", torch_ops_clip)
    sd = _sd(gold)
    clip = clip_standin.make_clip(sd, gold["cfg"], gold["out_dim"])
    enc = eng.install_clip(clip, device="cpu")
    assert enc.blocks_run == gold["cfg"]["layers"] - 1
    imgs = _images(gold, "list_2")
    assert _check_rows(clip.visual(imgs), gold["cases"]["list_2"]) <= ENGINE_BAR
    # shipped regime: fp16 autocast dtype over bf16 weights -> fp32 result (torch.promote_types)
    clip16 = clip_standin.make_clip(sd, gold["cfg"], gold["out_dim"], dtype=torch.float16, param_dtype=torch.bfloat16)
    eng.install_clip(clip16, device="cpu")
    assert clip16.visual(imgs[:1]).dtype == torch.float32


@pytest.mark.parametrize("variant,match", [(dict(activation="quick_gelu"), "QuickGELU"), (dict(activation="swi_glu"), "swi_glu"),
                                           (dict(post_norm=True), "post_norm"), (dict(pool_type="attn_pool"), "attn_pool")])
def test_install_clip_rejects_unimplemented_configs(gold, variant, match):
    from yume_b200 import clip as eng
    clip = clip_standin.make_clip(_sd(gold), gold["cfg"], gold["out_dim"], **variant)
    with pytest.raises(NotImplementedError, match=match):
        eng.install_clip(clip, device="cpu")


def test_interpolation_is_rejected(gold, monkeypatch):
    enc = _engine(gold, monkeypatch)
    with pytest.raises(NotImplementedError, match="interpolation"):
        enc.encode(_images(gold, "identity_224"), interpolation=True)


def test_non_list_inputs_behave_as_the_reference(gold, monkeypatch):
    """The reference iterates `videos`: a [N, 3, 1, H, W] tensor is N images, a single [3, 1, H, W] tensor yields [1, H, W]
    entries that F.interpolate rejects with ValueError; a tuple is a list."""
    enc = _engine(gold, monkeypatch)
    imgs = _images(gold, "odd_33x47")
    want = enc.encode(imgs)
    assert torch.equal(enc.encode(torch.stack(imgs)), want)
    assert torch.equal(enc.encode(tuple(imgs)), want)
    with pytest.raises(ValueError):
        oclip.preprocess(imgs[0], 224)
    with pytest.raises(ValueError):
        enc.encode(imgs[0])


# ------------------------------------------------------------------------------------------------------------
# C-ABI guards over include/yume_b200_clip.h
# ------------------------------------------------------------------------------------------------------------
def test_library_exports_every_clip_header_symbol():
    import yume_b200
    from yume_b200 import _lib
    declared = set(re.findall(r"^\s*(?:int|long long)\s+(yb_\w+)\s*\(", CLIP_HEADER.read_text(), flags=re.M))
    assert declared, "no declarations parsed"
    lib = yume_b200.load()
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/yume_b200_clip.h but not exported"
    assert declared == set(_lib.CLIP_SIGNATURES)
    assert not declared & set(_lib.SIGNATURES)


def test_every_clip_entry_point_has_a_contract_test():
    assert _entry_problems(CLIP_HEADER, modules=(KC,)) == []


def test_clip_entry_point_guard_notices_a_missing_test(monkeypatch):
    monkeypatch.setattr(KC, "COVERS", {})
    assert _entry_problems(CLIP_HEADER, modules=(KC,)) == ["entry point without a contract test: yb_resize_bicubic_normalize"]


# ------------------------------------------------------------------------------------------------------------
# the resample bound: accepts the kernel's fp32 arithmetic, rejects the defects
# ------------------------------------------------------------------------------------------------------------
def _emulate_kernel(x, S):
    """yb_resize_bicubic_normalize's arithmetic in fp32 torch ops: fmaf source coordinates (source_coords), fp32 Keys
    coefficients, the x pass then the y pass with separately rounded products and sums, then the fp32 normalize."""
    C, H, W = x.shape
    A = -0.75

    def coeffs(t):
        t = t.float()
        w1 = lambda v: ((A + 2) * v - (A + 3)) * v * v + 1            # noqa: E731
        w2 = lambda v: ((A * v - 5 * A) * v + 8 * A) * v - 4 * A      # noqa: E731
        return torch.stack([w2(t + 1), w1(t), w1(1 - t), w2((1 - t) + 1)], dim=-1)

    fy, ty = KC.source_coords(H, S)
    fx, tx = KC.source_coords(W, S)
    iy, _ = KC._taps(fy, H)
    ix, _ = KC._taps(fx, W)
    cy, cx = coeffs(ty), coeffs(tx)
    g = x[:, iy[:, :, None, None], ix[None, None, :, :]]            # [C, S, 4, S, 4]
    r = g[..., 0] * cx[None, None, None, :, 0]
    for j in range(1, 4):
        r = r + g[..., j] * cx[None, None, None, :, j]                 # [C, S, 4, S]
    v = r[:, :, 0] * cy[None, :, 0, None]
    for k in range(1, 4):
        v = v + r[:, :, k] * cy[None, :, k, None]
    m = torch.tensor(KC.MEAN, dtype=torch.float32).view(-1, 1, 1)
    s = torch.tensor(KC.STD, dtype=torch.float32).view(-1, 1, 1)
    return (v * 0.5 + 0.5 - m) / s


def _normalize(v):
    m = torch.tensor(KC.MEAN, dtype=torch.float32).view(-1, 1, 1)
    s = torch.tensor(KC.STD, dtype=torch.float32).view(-1, 1, 1)
    return (v.float() * 0.5 + 0.5 - m) / s


@pytest.fixture(scope="module")
def resize_case():
    g = torch.Generator().manual_seed(11)
    x = KC.strided_image(g, 150, 260, "cpu")[:, 0]
    ref, v, M = KC.resize_ref(x, 224)
    return x, ref, KC.resize_bound(x, 224, ref, v, M)


def test_keys_weights_sum_bound():
    t = torch.linspace(0, 1, 10001, dtype=torch.float64)
    w = KC.keys_weights(t)
    assert torch.allclose(w.sum(dim=-1), torch.ones_like(t))
    assert float(w.abs().sum(dim=-1).max()) <= KC.COEF_ABS_SUM


def test_resize_bound_accepts_the_kernel_arithmetic(resize_case):
    x, ref, bound = resize_case
    assert KC.assert_within(_emulate_kernel(x, 224), ref, bound, "resize emulated") <= 1.0
    xi = KC.strided_image(torch.Generator().manual_seed(3), 224, 224, "cpu")[:, 0]
    r, v, M = KC.resize_ref(xi, 224)
    assert KC.assert_within(_normalize(xi), r, KC.resize_bound(xi, 224, r, v, M), "resize identity") <= 1.0


def test_resize_bound_rejects_an_unclamped_tap(resize_case):
    x, ref, bound = resize_case
    bad, _, _ = KC.resize_ref(x, 224, clamp=False)                   # out-of-range taps read 0 instead of the border
    with pytest.raises(AssertionError, match="out of bound"):
        KC.assert_within(bad.float(), ref, bound, "resize unclamped")


def test_resize_bound_rejects_align_corners(resize_case):
    x, ref, bound = resize_case
    bad = _normalize(F.interpolate(x[None], size=(224, 224), mode="bicubic", align_corners=True)[0])
    with pytest.raises(AssertionError, match="out of bound"):
        KC.assert_within(bad, ref, bound, "resize align_corners")


def test_resize_bound_rejects_antialias(resize_case):
    x, ref, bound = resize_case
    bad = _normalize(F.interpolate(x[None], size=(224, 224), mode="bicubic", align_corners=False, antialias=True)[0])
    with pytest.raises(AssertionError, match="out of bound"):
        KC.assert_within(bad, ref, bound, "resize antialias")
