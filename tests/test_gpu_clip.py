"""CLIP image encoder on the GPU (`-m gpu`): yume_b200/clip.py on the sm_90a kernels against
  * the reference fixtures (tests/golden/clip_tiny.pt, the reference's own CLIPModel.visual in fp32, 2 heads of 80);
  * oracle/clip.py in fp32 on the device at the real ViT-H/14 width (1280, 16 heads of 80, 31 blocks run, seeded weights,
    a 544x960 image);
and checks that the padded attention columns are exactly zero, that CUDA-graph replay equals eager, and that install_clip on a
stand-in CLIPModel in the shipped regime (bf16 weights, fp16 autocast dtype) returns fp32 [1, 257, 1280].
Bars are set from the measured error with a stated margin; the engine's GEMM and attention operands are bf16 where the fp32
reference keeps fp32 (bar reasoning in each test)."""
import pytest
import torch

from helpers import clip_standin
from oracle import clip as oclip

pytestmark = pytest.mark.gpu

CASES = ["down_544x960", "identity_224", "up_150x200", "odd_33x47", "list_2"]


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()
    return "cuda"


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(golden_dir / "clip_tiny.pt", weights_only=False)


def _images(gold, case, device="cpu"):
    c = gold["cases"][case]
    out = []
    for (H, W), seed in zip(c["sizes"], c["seeds"]):
        g = torch.Generator().manual_seed(seed)
        out.append((torch.rand(3, 1, H, W, generator=g) * 2 - 1).to(device))
    return out


@pytest.fixture(scope="module")
def tiny(gold, dev):
    from yume_b200.clip import ClipVisionEncoder
    sd = oclip.make_state_dict(gold["seed_w"], **gold["cfg"], out_dim=gold["out_dim"])
    return ClipVisionEncoder(sd, mean=gold["mean"], std=gold["std"], device=dev, **gold["cfg"])


# Measured on the stand-in ops (same bf16 roundings, tests/test_clip_cpu.py): 3.7e-3; bar 7.5e-3 as there.
FIXTURE_BAR = 7.5e-3


@pytest.mark.parametrize("case", CASES)
def test_engine_matches_reference_fixture(tiny, gold, case):
    out = tiny.encode(_images(gold, case, "cuda")).cpu()
    c = gold["cases"][case]                      # the fixture stores a seeded subset of the token rows
    assert out.dtype == torch.float32 and tuple(out.shape) == tuple(c["out_shape"])
    err = _rel(out[:, c["out_rows"].long()], c["out"])
    print(f"[clip] engine vs reference fixture {case}: rel-Frobenius {err:.3g}")
    assert err <= FIXTURE_BAR


def test_padded_attention_columns_are_zero(tiny, gold):
    """q|k|v columns 80..127 of every head come from zero weight rows and zero bias; the attention output there is P.0."""
    tiny.encode(_images(gold, "identity_224", "cuda"))
    st = tiny._state[(3, 224, 224)]
    T, H = tiny.tokens, tiny.heads
    assert not st["qkv"].view(T, 3, H, 128)[..., tiny.head_dim:].any()
    assert not st["att"].view(T, H, 128)[..., tiny.head_dim:].any()


def test_graph_replay_equals_eager(tiny, gold):
    imgs = _images(gold, "list_2", "cuda")
    tiny.use_cuda_graph = False
    eager = tiny.encode(imgs)
    tiny.use_cuda_graph = True
    try:
        first = tiny.encode(imgs)                       # captures one graph per input shape
        again = tiny.encode([u.clone() for u in imgs])  # replays them
    finally:
        tiny.use_cuda_graph = False
    assert torch.equal(first, eager) and torch.equal(again, eager)


@pytest.fixture(scope="module")
def vit_h(dev):
    sd = oclip.make_state_dict(1234, **oclip.VIT_H_14)
    g = torch.Generator().manual_seed(99)
    img = torch.rand(3, 1, 544, 960, generator=g) * 2 - 1
    return sd, img


# The 31-block fp32 oracle against the bf16-operand engine at the real width. Measured on an H100: 6.0e-3 (the reference's own
# fp16-autocast regime measures 6.5e-3 against the same oracle, tools/bench_clip.py); bar 1.2e-2 (2x margin).
VIT_H_BAR = 1.2e-2


def test_engine_at_vit_h_14_width_matches_fp32_oracle(dev, vit_h):
    """Engine vs oracle/clip.py (fp32 weights and stream on the device; q, k, v bf16 as the reference's flash_attention rounds
    them) for one 544x960 image. The bar is twice the measured rel-Frobenius error (VIT_H_BAR)."""
    from yume_b200.clip import ClipVisionEncoder
    sd, img = vit_h
    enc = ClipVisionEncoder(sd, mean=oclip.MEAN, std=oclip.STD, device=dev, **oclip.VIT_H_14)
    out = enc.encode([img.to(dev)])
    del enc
    sdd = {k: v.to(dev) for k, v in sd.items()}
    with torch.no_grad():
        ref = oclip.visual(sdd, [img.to(dev)], **oclip.VIT_H_14)
    del sdd
    assert out.shape == ref.shape == (1, 257, 1280) and out.dtype == torch.float32
    err = _rel(out, ref)
    print(f"[clip] engine vs fp32 oracle at ViT-H/14 width (544x960): rel-Frobenius {err:.3g}")
    assert err <= VIT_H_BAR


def test_install_clip_on_standin_clip_model(dev, vit_h):
    from yume_b200.clip import install_clip
    sd, img = vit_h
    clip = clip_standin.make_clip(sd, oclip.VIT_H_14, out_dim=1024, dtype=torch.float16, param_dtype=torch.bfloat16)
    install_clip(clip, device=dev)
    out = clip.visual([img.to(dev)])
    assert out.dtype == torch.float32 and tuple(out.shape) == (1, 257, 1280) and torch.isfinite(out).all()
