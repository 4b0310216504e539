"""Writes tests/golden/install_hooks.pt: what the install hooks of yume_b200 read from the REFERENCE's own objects, and what those
objects return, on the seeded tiny configs of tests/test_host_logic_vae_install.py and tests/test_host_logic.py:
  * wan22 / wan21: the `WanVAE_` attributes the hooks read, the state-dict keys and shapes, and the reference's own chunked
    encode / decode of the seeded video / latent;
  * hyvae: the `AutoencoderKLCausal3D` config fields, the tiling switches after enable_tiling() / disable_tiling(), the decoder
    state-dict keys and shapes, a fixed seeded sample of the tiled decode and the whole untiled decode of a small latent;
  * wanmodel: the state-dict keys and shapes of the reference's `WanModel` (both trees) on the tiny configs.
Usage: python tools/make_golden_install.py <reference root>"""
import importlib.util
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from oracle import hyvae, synth, wan21vae, wan21vae_enc, wan22vae, wan22vae_enc  # noqa: E402

HY_SAMPLE = 65536   # tiled hyvae decode: elements stored (the whole output is 0.5 M floats)


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, str(path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def wan_vae_inputs(tree):
    """seeded (mean, std, video, z) of the wan22 / wan21 cases"""
    g = torch.Generator().manual_seed(3 if tree == "wan22" else 4)
    mean, std = 0.3 * torch.randn(16, generator=g), 0.5 + torch.rand(16, generator=g)
    video = torch.randn(3, 5, 32, 64, generator=g).clamp_(-1, 1) if tree == "wan22" else torch.randn(3, 5, 16, 32, generator=g).clamp_(-1, 1)
    z = torch.randn(16, 2, 2, 4, generator=g)
    return mean, std, video, z


def wan22_state_dict():
    sd = dict(wan22vae_enc.make_state_dict(11, dim=32, z_dim=16, dim_mult=(1, 2, 4, 4), num_res_blocks=2,
                                           temperal_downsample=(False, True, True)))
    sd.update(wan22vae.make_state_dict(12, dec_dim=32, z_dim=16, dim_mult=(1, 2, 4, 4), num_res_blocks=2, temperal_upsample=(True, True, False)))
    return sd


def wan21_state_dict():
    cfg = dict(dim=32, z_dim=16, dim_mult=(1, 2, 4, 4), num_res_blocks=2)
    sd = dict(wan21vae_enc.make_state_dict(21, temperal_downsample=(False, True, True), **cfg))
    sd.update(wan21vae.make_state_dict(22, temperal_upsample=(True, True, False), **cfg))
    return sd


def hy_latents():
    return (torch.randn(1, 16, 6, 10, 12, generator=torch.Generator().manual_seed(5)),
            torch.randn(1, 16, 2, 4, 6, generator=torch.Generator().manual_seed(6)))


def hy_sample_index(numel):
    return torch.randint(0, numel, (HY_SAMPLE,), generator=torch.Generator().manual_seed(7)).sort().values


def _attrs(m, names):
    return {n: (list(getattr(m, n)) if isinstance(getattr(m, n), (list, tuple)) else getattr(m, n)) for n in names}


def _shapes(sd, keep=lambda k: True):
    return {k: tuple(v.shape) for k, v in sd.items() if keep(k)}


@torch.no_grad()
def main(ref_root: Path):
    out = {}
    for tree, path, make_sd in (("wan22", ref_root / "wan23" / "modules" / "vae2_2.py", wan22_state_dict),
                                ("wan21", ref_root / "wan" / "modules" / "vae.py", wan21_state_dict)):
        ref = _load(path, f"ref_{tree}_install")
        kw = dict(dim=32, z_dim=16, dim_mult=[1, 2, 4, 4], num_res_blocks=2, attn_scales=[], temperal_downsample=[False, True, True])
        if tree == "wan22":
            kw["dec_dim"] = 32
        model = ref.WanVAE_(**kw).eval()
        model.load_state_dict(make_sd(), strict=True)
        mean, std, video, z = wan_vae_inputs(tree)
        scale = [mean, 1.0 / std]
        out[tree] = {"attrs": _attrs(model, ("dim", "z_dim", "dim_mult", "num_res_blocks", "temperal_downsample", "temperal_upsample")),
                     "keys": _shapes(model.state_dict()),
                     "mu": model.encode(video.unsqueeze(0), scale).float().squeeze(0).clone(),
                     "x": model.decode(z.unsqueeze(0), scale).float().clamp_(-1, 1).squeeze(0).clone()}
    import make_golden_vae
    ak = make_golden_vae.load_reference_vae()
    cfg = make_golden_vae.TINY
    sd = hyvae.make_state_dict(99, **cfg)
    ref = ak.AutoencoderKLCausal3D(in_channels=3, out_channels=3, down_block_types=("DownEncoderBlockCausal3D",) * 4,
                                   up_block_types=("UpDecoderBlockCausal3D",) * 4, block_out_channels=cfg["block_out_channels"],
                                   layers_per_block=2, act_fn="silu", latent_channels=16, norm_num_groups=32, sample_size=64,
                                   sample_tsize=16, time_compression_ratio=4, spatial_compression_ratio=8, mid_block_add_attention=True)
    ref.load_state_dict(sd, strict=False)
    ref.eval()
    z, small = hy_latents()
    conf = ref.config
    get = (lambda k: conf.get(k)) if isinstance(conf, dict) else (lambda k: getattr(conf, k))
    ref.enable_tiling()
    on = (ref.use_spatial_tiling, ref.use_temporal_tiling)
    tiled = ref.decode(z, return_dict=False)[0]
    ref.disable_tiling()
    off = (ref.use_spatial_tiling, ref.use_temporal_tiling)
    untiled = ref.decode(small, return_dict=False)[0]
    idx = hy_sample_index(tiled.numel())
    out["hyvae"] = {"config": {k: (list(get(k)) if isinstance(get(k), (list, tuple)) else get(k)) for k in
                               ("block_out_channels", "layers_per_block", "norm_num_groups", "sample_size", "sample_tsize",
                                "latent_channels", "out_channels")},
                    "tiling_on": on, "tiling_off": off,
                    "keys": _shapes(ref.state_dict(), lambda k: k in sd),
                    "tiled_shape": tuple(tiled.shape), "tiled_sample": tiled.float().reshape(-1)[idx].clone(),
                    "untiled_small": untiled.float().clone()}
    import make_golden
    out["wanmodel"] = {}
    for tree, cfg_name in (("wan23", "CFG_5B_TINY"), ("wan", "CFG_14B_TINY")):
        cfg = getattr(synth, cfg_name)
        m = make_golden.build_reference_model(make_golden.load_reference(tree), cfg, synth.make_state_dict(cfg, 4321))
        out["wanmodel"][tree] = _shapes(m.state_dict())
    dst = ROOT / "tests" / "golden" / "install_hooks.pt"
    torch.save(out, dst)
    print(f"wrote {dst}")


if __name__ == "__main__":
    main(Path(sys.argv[1]))
