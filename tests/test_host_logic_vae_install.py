"""Drop-in hooks of the VAEs against the REFERENCE's own objects, on CPU. tools/make_golden_install.py built the reference's `WanVAE_`
(2.2 and 2.1 trees) and `AutoencoderKLCausal3D` with seeded weights and stored, in tests/golden/install_hooks.pt, what the hooks read
from them (the attributes, the state-dict keys and shapes, `config` and the tiling switches) and what their own encode / decode
returned. Here the hooks are installed on stand-ins that expose exactly that recorded interface, and `encode(list)` / `decode(list)`
/ `decode(z, return_dict=...)` must keep the reference's calling convention and land within the bf16 budget of its fp32 result. The
engines run over the torch stand-in for the C ABI (tests/helpers/torch_ops.py)."""
import sys
import types
from pathlib import Path

import pytest
import torch

from helpers import torch_ops
from yume_b200 import vae21, vae22, vae_enc

sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tools"))
import make_golden_install as recipe  # noqa: E402


@pytest.fixture()
def cpu_ops(monkeypatch):
    for mod in (vae22, vae21, vae_enc):
        monkeypatch.setattr(mod, "ops", torch_ops)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(golden_dir / "install_hooks.pt")


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def _wan_model(g, sd):
    """stand-in for the reference `WanVAE_`: its recorded attributes and a state dict with the recorded keys and shapes"""
    assert {k: tuple(v.shape) for k, v in sd.items()} == g["keys"]
    return types.SimpleNamespace(state_dict=lambda: dict(sd), **g["attrs"])


@torch.no_grad()
def test_wan22_wrapper_hooks_are_drop_ins(cpu_ops, golden):
    g = golden["wan22"]
    mean, std, video, z = recipe.wan_vae_inputs("wan22")
    wrapper = types.SimpleNamespace(model=_wan_model(g, recipe.wan22_state_dict()), scale=[mean, 1.0 / std], dtype=torch.float)
    vae_enc.install_wan22_vae_encoder(wrapper, device="cpu")
    vae22.install_wan22_vae(wrapper, device="cpu")
    got_mu, got_x = wrapper.encode([video]), wrapper.decode([z])
    assert isinstance(got_mu, list) and isinstance(got_x, list) and len(got_mu) == len(got_x) == 1
    assert got_mu[0].shape == g["mu"].shape and _rel(got_mu[0], g["mu"]) < 3e-2
    assert got_x[0].shape == g["x"].shape and _rel(got_x[0], g["x"]) < 3e-2
    assert wrapper.encode(video) is None and wrapper.decode(z) is None          # the reference logs a TypeError and returns None


@torch.no_grad()
def test_wan21_wrapper_hooks_are_drop_ins(cpu_ops, golden):
    g = golden["wan21"]
    mean, std, video, z = recipe.wan_vae_inputs("wan21")
    wrapper = types.SimpleNamespace(model=_wan_model(g, recipe.wan21_state_dict()), mean=mean, std=std, scale=[mean, 1.0 / std],
                                    dtype=torch.float)
    vae_enc.install_wan21_vae_encoder(wrapper, device="cpu")
    vae21.install_wan21_vae(wrapper, device="cpu")
    got_mu, got_x = wrapper.encode([video]), wrapper.decode([z])
    assert got_mu[0].shape == g["mu"].shape and _rel(got_mu[0], g["mu"]) < 3e-2
    assert got_x[0].shape == g["x"].shape and _rel(got_x[0], g["x"]) < 3e-2


@torch.no_grad()
def test_hyvideo_install_vae_is_a_drop_in(monkeypatch, golden):
    """`install_vae` on a stand-in with the reference `AutoencoderKLCausal3D`'s config, tiling switches and decoder state dict: the
    re-bound `decode(z, return_dict=...)` keeps the return convention, follows the module's tiling switches, and matches the reference's
    tiled decode (a fixed seeded sample of it) and its untiled decode of a small latent."""
    from oracle import hyvae
    from yume_b200 import vae as ybvae
    monkeypatch.setattr(ybvae, "ops", torch_ops)
    g = golden["hyvae"]
    import make_golden_vae
    sd = hyvae.make_state_dict(99, **make_golden_vae.TINY)
    sd = {k: v for k, v in sd.items() if k in g["keys"]}
    assert {k: tuple(v.shape) for k, v in sd.items()} == g["keys"]
    ref = types.SimpleNamespace(config=dict(g["config"]), state_dict=lambda: dict(sd))
    ref.use_spatial_tiling, ref.use_temporal_tiling = g["tiling_on"]                # what enable_tiling() leaves
    z, small = recipe.hy_latents()
    ybvae.install_vae(ref, device="cpu")
    got = ref.decode(z, return_dict=False)
    assert isinstance(got, tuple) and tuple(got[0].shape) == g["tiled_shape"]
    idx = recipe.hy_sample_index(got[0].numel())
    assert _rel(got[0].reshape(-1)[idx], g["tiled_sample"]) < 3e-2
    out = ref.decode(z)
    assert _rel(out.sample.reshape(-1)[idx], g["tiled_sample"]) < 3e-2
    ref.use_spatial_tiling, ref.use_temporal_tiling = g["tiling_off"]               # what disable_tiling() leaves
    small_out = ref.decode(small, return_dict=False)[0]
    assert small_out.shape == g["untiled_small"].shape == (1, 3, 5, 32, 48) and _rel(small_out, g["untiled_small"]) < 3e-2
