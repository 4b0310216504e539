"""Generate tests/golden/clip_tiny.pt by running the REFERENCE's own `CLIPModel.visual` (wan/modules/clip.py:527-542) on CPU.

    python tools/make_golden_clip.py <reference root>

Recipe: register bare `wan` / `wan.modules` packages so their __init__ files never run; stub `.tokenizers` (it needs ftfy,
which the image path never uses) and `.attention` (its `flash_attention` asserts CUDA and calls flash_attn) with the SDPA
restatement of tools/make_golden.py; load xlm_roberta.py and clip.py by path. `CLIPModel.visual` is then called unbound on
a stand-in carrying a tiny `VisionTransformer` (image 224, patch 14, dim 160, 2 heads of 80 so the engine's head padding
is exercised, 3 layers) and the reference's own transforms from `_clip(return_transforms=True)`. On CPU the CUDA autocast
it enters is a no-op, so the fixture is the fp32 arithmetic. Weights come from oracle/clip.py (seeded); input images are
regenerated from their seeds by the tests (`images(case)` below). To keep the file small, each case stores a seeded sample of
the preprocessed images and of the output token rows (the cls row and 31 patch rows of every image, with their indices)
rather than the whole tensors.
"""
from __future__ import annotations

import importlib.util
import sys
import types
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from oracle import clip as oclip  # noqa: E402

TINY = dict(image_size=224, patch_size=14, dim=160, heads=2, layers=3, mlp_ratio=4, eps=1e-5)
TINY_OUT_DIM = 64
SEED_W = 4242
# name -> list of (H, W) images of one visual() call
CASES = {"down_544x960": [(544, 960)], "identity_224": [(224, 224)], "up_150x200": [(150, 200)], "odd_33x47": [(33, 47)],
         "list_2": [(480, 832), (33, 47)]}
SAMPLE = 1024          # preprocessed values stored per case
ROWS = 32              # output token rows stored per case: the cls row and 31 seeded patch rows


def image_seed(case, i):
    return 1000 + 17 * sorted(CASES).index(case) + i


def images(case):
    """The fp32 [3, 1, H, W] images in [-1, 1] of a case (uniform noise, seeded per image)."""
    out = []
    for i, (H, W) in enumerate(CASES[case]):
        g = torch.Generator().manual_seed(image_seed(case, i))
        out.append(torch.rand(3, 1, H, W, generator=g) * 2 - 1)
    return out


def load_reference_clip(ref_root: Path):
    from make_golden import _sdpa_flash_attention
    for pk in ("wan", "wan.modules"):
        if pk not in sys.modules:
            m = types.ModuleType(pk)
            m.__path__ = [str(ref_root / pk.replace(".", "/"))]
            sys.modules[pk] = m
    tok = types.ModuleType("wan.modules.tokenizers")
    tok.HuggingfaceTokenizer = object
    sys.modules["wan.modules.tokenizers"] = tok
    att = types.ModuleType("wan.modules.attention")
    att.flash_attention = _sdpa_flash_attention
    sys.modules["wan.modules.attention"] = att

    def load(modname, path):
        spec = importlib.util.spec_from_file_location(modname, path)
        mod = importlib.util.module_from_spec(spec)
        sys.modules[modname] = mod
        spec.loader.exec_module(mod)
        return mod

    load("wan.modules.xlm_roberta", ref_root / "wan" / "modules" / "xlm_roberta.py")
    return load("wan.modules.clip", ref_root / "wan" / "modules" / "clip.py")


def main(ref_root: Path):
    ref = load_reference_clip(ref_root)
    sd = oclip.make_state_dict(SEED_W, **TINY, out_dim=TINY_OUT_DIM)

    class Tiny(torch.nn.Module):           # what _clip builds, cut to the vision tower (clip.py:377-392)
        def __init__(self, **kw):
            super().__init__()
            self.image_size = TINY["image_size"]
            self.visual = ref.VisionTransformer(
                image_size=TINY["image_size"], patch_size=TINY["patch_size"], dim=TINY["dim"], mlp_ratio=TINY["mlp_ratio"],
                out_dim=TINY_OUT_DIM, num_heads=TINY["heads"], num_layers=TINY["layers"], pool_type="token", pre_norm=True,
                post_norm=False, activation="gelu", norm_eps=TINY["eps"])

    model, transforms = ref._clip(pretrained=False, pretrained_name="open-clip-xlm-roberta-large-vit-huge-14", model_cls=Tiny,
                                  return_transforms=True, dtype=torch.float32, device="cpu")
    missing, unexpected = model.visual.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    model.eval().requires_grad_(False)
    standin = types.SimpleNamespace(model=model, transforms=transforms, dtype=torch.float16)

    gold = {"cfg": TINY, "out_dim": TINY_OUT_DIM, "seed_w": SEED_W,
            "weight_abs_sum": float(sum(v.abs().sum() for v in sd.values())),
            "mean": list(transforms.transforms[-1].mean), "std": list(transforms.transforms[-1].std), "cases": {}}
    for case in CASES:
        imgs = images(case)
        with torch.no_grad():
            out = ref.CLIPModel.visual(standin, [u.clone() for u in imgs])      # visual() preprocesses in place
            pre = oclip.preprocess([u.clone() for u in imgs], TINY["image_size"])
        g = torch.Generator().manual_seed(image_seed(case, 99))
        idx = torch.randint(0, pre.numel(), (SAMPLE,), generator=g, dtype=torch.int32)
        rows = torch.cat([torch.zeros(1, dtype=torch.int64), torch.randperm(out.shape[1] - 1, generator=g)[:ROWS - 1].sort()[0] + 1])
        gold["cases"][case] = {"sizes": CASES[case], "seeds": [image_seed(case, i) for i in range(len(imgs))],
                               "input_abs_sum": float(sum(u.abs().sum() for u in imgs)),
                               "pre_idx": idx, "pre_sample": pre.reshape(-1)[idx.long()].clone(),
                               "out_shape": tuple(out.shape), "out_rows": rows.to(torch.int32),
                               "out": out.float()[:, rows].clone()}
        print(f"{case}: out {tuple(out.shape)} {out.dtype}")

    # keys and shapes of the real ViT-H/14 vision tower, built on the meta device (no memory, no weights)
    big = ref.clip_xlm_roberta_vit_h_14(pretrained=False, return_transforms=False, dtype=torch.float32, device="meta")
    gold["vit_h_14_shapes"] = {k: tuple(v.shape) for k, v in big.visual.state_dict().items()}
    gold["vit_h_14_cfg"] = dict(image_size=big.visual.image_size, patch_size=big.visual.patch_size, dim=big.visual.dim,
                                heads=big.visual.num_heads, layers=big.visual.num_layers, mlp_ratio=big.visual.mlp_ratio,
                                eps=big.visual.norm_eps, out_dim=big.visual.out_dim)
    dst = ROOT / "tests" / "golden" / "clip_tiny.pt"
    torch.save(gold, dst)
    print(f"wrote {dst} ({dst.stat().st_size / 1e6:.2f} MB)")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: python tools/make_golden_clip.py <reference root>")
    main(Path(sys.argv[1]))
