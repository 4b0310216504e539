"""Generate tests/golden/t5_tiny.pt by running the REFERENCE's own `T5Encoder.forward` (wan23/modules/t5.py:267-312) on CPU.

    python tools/make_golden_t5.py <reference root>

Recipe: register bare `wan23` / `wan23.modules` packages so their __init__ files never run, stub `.tokenizers` (it needs
ftfy, which the encoder never uses) and load wan23/modules/t5.py by path. (wan/modules/t5.py is the same code except that it
evaluates `torch.cuda.current_device()` as a default argument at import, which raises without a GPU.) Two tiny encoders are
built with the reference's class — vocab 1000, dim 256, 4 heads of 64, ffn 640, 32 buckets: 3 layers with per-layer position
embeddings (shared_pos=False, as umt5_xxl), and 2 layers with one shared embedding — loaded with the seeded weights of
oracle/t5.py and run in fp32, eval mode. To keep the file small, each case stores its ids and mask, the output's shape and a
seeded subset of its rows (ROWS per sample, with their indices). Also stored: the reference's [600, 600] bucket table
(int8) and the umt5_xxl encoder's state-dict keys and shapes, built on the meta device.
"""
from __future__ import annotations

import importlib.util
import sys
import types
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import t5 as ot5  # noqa: E402

TINY = dict(vocab=1000, dim=256, dim_attn=256, dim_ffn=640, num_heads=4, num_layers=3, num_buckets=32, shared_pos=False)
TINY_SHARED = dict(TINY, num_layers=2, shared_pos=True)
SEED_W = {"tiny": 5151, "tiny_shared": 5152}
ROWS = 24
# name -> (model, L, mask per sample: an int n = prefix of n ones, "holed" = a seeded non-prefix mask, None = mask=None)
CASES = {
    "L512_m1": ("tiny", 512, [1]),
    "L512_m37": ("tiny", 512, [37]),
    "L512_m512": ("tiny", 512, [512]),
    "B2_L77": ("tiny", 77, [17, 77]),
    "L64_none": ("tiny", 64, None),
    "L96_holed": ("tiny", 96, ["holed"]),
    "L600": ("tiny", 600, [451]),
    "shared_B2_L77": ("tiny_shared", 77, [30, 77]),
    "shared_L600_holed": ("tiny_shared", 600, ["holed"]),
}
BUCKET_L = 600


def case_seed(case):
    return 2000 + 31 * sorted(CASES).index(case)


def inputs(case):
    """ids int64 [B, L] (seeded, in [0, vocab)) and the mask (int64 [B, L] or None) of a case."""
    model, L, masks = CASES[case]
    g = torch.Generator().manual_seed(case_seed(case))
    B = 1 if masks is None else len(masks)
    ids = torch.randint(0, TINY["vocab"], (B, L), generator=g)
    if masks is None:
        return ids, None
    mask = torch.zeros(B, L, dtype=torch.long)
    for b, m in enumerate(masks):
        if m == "holed":
            mask[b] = (torch.rand(L, generator=g) < 0.6).long()
            mask[b, 0] = 1
        else:
            mask[b, :m] = 1
    return ids, mask


def load_reference_t5(ref_root: Path):
    for pk in ("wan23", "wan23.modules"):
        if pk not in sys.modules:
            m = types.ModuleType(pk)
            m.__path__ = [str(ref_root / pk.replace(".", "/"))]
            sys.modules[pk] = m
    tok = types.ModuleType("wan23.modules.tokenizers")
    tok.HuggingfaceTokenizer = object
    sys.modules["wan23.modules.tokenizers"] = tok
    spec = importlib.util.spec_from_file_location("wan23.modules.t5", ref_root / "wan23" / "modules" / "t5.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules["wan23.modules.t5"] = mod
    spec.loader.exec_module(mod)
    return mod


def main(ref_root: Path):
    ref = load_reference_t5(ref_root)
    cfgs = {"tiny": TINY, "tiny_shared": TINY_SHARED}
    models, sds = {}, {}
    for name, cfg in cfgs.items():
        sd = ot5.make_state_dict(SEED_W[name], **cfg)
        m = ref.T5Encoder(**cfg, dropout=0.1)
        missing, unexpected = m.load_state_dict(sd, strict=True)
        assert not missing and not unexpected
        models[name] = m.eval().requires_grad_(False)
        sds[name] = sd
    gold = {"cfg": cfgs, "seed_w": SEED_W, "eps": 1e-6, "max_dist": 128,
            "weight_abs_sum": {n: float(sum(v.abs().sum() for v in sd.values())) for n, sd in sds.items()}, "cases": {}}
    for case, (name, L, _) in CASES.items():
        ids, mask = inputs(case)
        with torch.no_grad():
            out = models[name](ids, mask)
        g = torch.Generator().manual_seed(case_seed(case) + 1)
        rows = torch.stack([torch.randperm(L, generator=g)[:min(ROWS, L)].sort()[0] for _ in range(ids.shape[0])])
        gold["cases"][case] = {"model": name, "ids": ids.to(torch.int16), "mask": None if mask is None else mask.to(torch.int8),
                               "out_shape": tuple(out.shape), "out_dtype": str(out.dtype), "out_rows": rows.to(torch.int16),
                               "out": torch.stack([out[b, rows[b]] for b in range(ids.shape[0])]).float().clone()}
        print(f"{case}: out {tuple(out.shape)} {out.dtype}")

    # the reference's bucket table, from its own method on the CPU
    rel_emb = models["tiny"].blocks[0].pos_embedding
    rel = torch.arange(BUCKET_L).unsqueeze(0) - torch.arange(BUCKET_L).unsqueeze(1)
    gold["buckets_L600"] = rel_emb._relative_position_bucket(rel).to(torch.int8)

    # keys and shapes of the real umt5_xxl encoder, built on the meta device (no memory, no weights)
    big = ref.umt5_xxl(encoder_only=True, return_tokenizer=False, dtype=torch.bfloat16, device="meta")
    gold["umt5_xxl_shapes"] = {k: tuple(v.shape) for k, v in big.state_dict().items()}
    gold["umt5_xxl_cfg"] = dict(vocab=big.token_embedding.num_embeddings, dim=big.dim, dim_attn=big.dim_attn,
                                dim_ffn=big.dim_ffn, num_heads=big.num_heads, num_layers=big.num_layers,
                                num_buckets=big.num_buckets, shared_pos=big.shared_pos)
    dst = ROOT / "tests" / "golden" / "t5_tiny.pt"
    torch.save(gold, dst)
    print(f"wrote {dst} ({dst.stat().st_size / 1e6:.2f} MB)")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: python tools/make_golden_t5.py <reference root>")
    main(Path(sys.argv[1]))
