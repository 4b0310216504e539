"""yume_b200 — H100-native (sm_90a) implementation of YUME's denoise hot path behind the reference's own seams.

Public surface:
  yume_b200.install(model)          re-bind `WanModel.forward` of a live reference model (yume_b200.model)
  yume_b200.install_seams(model)    also bind `WanAttentionBlock.forward` / `WanSelfAttention.forward` (yume_b200.seams)
  yume_b200.flash_attention         drop-in for the reference's module-level `flash_attention`
  yume_b200.sampler                 the Euler / CFG / SDE denoising loops of the samplers over any such model
  yume_b200.install_vae / install_wan22_vae / install_wan21_vae              re-bind `decode` of the three VAE wrappers
  yume_b200.install_wan22_vae_encoder / install_wan21_vae_encoder            re-bind `encode` of the two Wan VAE wrappers
  yume_b200.install_clip            re-bind `visual` of the reference's CLIPModel (the 14B I2V image encoder, yume_b200.clip)
  yume_b200.install_t5              re-bind `model.forward` of the reference's T5EncoderModel (the umT5 text encoder, yume_b200.t5)
  yume_b200.ops                     tensor-level wrappers over the C ABI (include/yume_b200.h)
  yume_b200.build                   in-tree nvcc build of csrc/libyume_b200.so
The torch-dependent modules are imported lazily so that `import yume_b200; yume_b200.load()` stays a pure ctypes check.
"""
from ._lib import YumeB200Error, lib_path, load  # noqa: F401

__version__ = "0.2.0"

_LAZY = {"install": "model", "WanModel5B": "model", "WanModel14B": "model", "install_seams": "seams",
         "flash_attention": "seams", "patch_flash_attention": "seams", "install_vae": "vae", "install_wan22_vae": "vae22",
         "install_wan21_vae": "vae21", "install_wan22_vae_encoder": "vae_enc", "install_wan21_vae_encoder": "vae_enc",
         "install_clip": "clip", "install_t5": "t5"}


def __getattr__(name):
    mod = _LAZY.get(name)
    if mod is None:
        raise AttributeError(f"module 'yume_b200' has no attribute {name!r}")
    import importlib
    return getattr(importlib.import_module(f"{__name__}.{mod}"), name)
