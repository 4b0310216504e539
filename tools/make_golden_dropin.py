"""Writes tests/golden/dropin_forward.pt: the output of the REFERENCE's own WanModel.forward (both trees, tools/make_golden.py
recipe) called the way the samplers call it, on the seeded tiny configs and inputs of tests/test_host_logic_dit.py
(test_install_on_the_reference_wanmodel_is_a_drop_in). Usage: python tools/make_golden_dropin.py"""
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

import make_golden  # noqa: E402
from oracle import synth  # noqa: E402

FRAMES, H, W, LFZ, SEED_W, SEED_X = 12, 6, 10, 2, 2468, 77


def dropin_call(cfg):
    """(args, kwargs) of the sampler-style call on the seeded inputs"""
    inp = synth.make_inputs(cfg, SEED_X, FRAMES, H, W, ctx_len=20)
    if cfg["variant"] == "5b":   # packed path: seq_len is recomputed by the model
        return ([inp["x"]], torch.tensor([[0.0, 400.0]]), [inp["context"]]), dict(seq_len=10 ** 6, latent_frame_zero=LFZ, flag=True)
    L = FRAMES * (H // 2) * (W // 2)
    return ([inp["x"]], torch.tensor([300.0]), [inp["context"]]), dict(seq_len=L, clip_fea=inp["clip_fea"], y=[inp["y"]],
                                                                      rand_num_img=0.2, latent_frame_zero=LFZ)


def main():
    out = {}
    for tree, cfg_name in (("wan23", "CFG_5B_TINY"), ("wan", "CFG_14B_TINY")):
        cfg = getattr(synth, cfg_name)
        model = make_golden.build_reference_model(make_golden.load_reference(tree), cfg, synth.make_state_dict(cfg, SEED_W))
        args, kwargs = dropin_call(cfg)
        with torch.no_grad():
            r = model(*args, **kwargs)
        out[tree] = r[0].float().contiguous()   # 5B returns [tensor], 14B (tensor, cache)
    dst = ROOT / "tests" / "golden" / "dropin_forward.pt"
    torch.save(out, dst)
    print(f"wrote {dst}: " + ", ".join(f"{k} {tuple(v.shape)}" for k, v in out.items()))


if __name__ == "__main__":
    main()
