"""Host-side mirror of the reference's WanModel interface, and `install()` — the drop-in seam.

Two ways in, both ending in the same WanDiT engine (yume_b200/dit.py):

1. `install(model)` — given a live *reference* `WanModel` instance (what `wan23.Yume(...).model` /
   `wan.Yume(...).model` own, sample_5b.py:1154 / sample.py:943), re-bind its `forward` with
   `types.MethodType`, exactly the mechanism the reference uses for its own sequence-parallel patch
   (wan23/textimage2video.py:190-194). Samplers, pipelines and checkpoints stay untouched.

2. `WanModel5B` / `WanModel14B` — parameter containers with the reference's constructor arguments, attribute
   names and state-dict keys (SURVEY.md §8b), for use where the reference package is not importable (tests,
   bench, the GPU box). Their `forward` keeps the reference signature, argument meaning and error behaviour:
     5B : wan23/modules/model.py:547-558  -> List[Tensor fp32]
     14B: wan/modules/model.py:723-738    -> (Tensor fp32, None)
"""
from __future__ import annotations

import types
from typing import List, Optional

import torch
import torch.nn as nn

from ._lib import YumeB200Error
from .dit import WanDiT

__all__ = ["WanModel5B", "WanModel14B", "install", "forward_5b", "forward_14b"]


# ------------------------------------------------------------------------------------------------------------
# forwards with the reference signatures (bound onto a module by install())
# ------------------------------------------------------------------------------------------------------------
def _engine(self) -> WanDiT:
    eng = getattr(self, "_yb_engine", None)
    if eng is None:
        raise YumeB200Error("yume_b200.install(model) has not been called on this WanModel")
    return eng


def forward_5b(self, x, t, context, seq_len, enable_mask=False, y=None, latent_frame_zero=8, input_ids=None,
               flag=True):
    """Drop-in for wan23 WanModel.forward (wan23/modules/model.py:547-865)."""
    if self.model_type == "i2v":
        assert y is not None                                            # model.py:578-579
    if enable_mask:
        raise NotImplementedError("enable_mask=True is the MVDT training path (model.py:764-800); inference only")
    eng = _engine(self)
    outs = []
    for i, u in enumerate(x):
        yi = y[i] if y is not None else None
        ti = t if t.dim() == 1 and t.numel() == 1 else (t[i] if t.dim() == 2 and t.size(0) == len(x) else t)
        outs.append(eng.forward(u, ti, context[i], seq_len, y=yi, latent_frame_zero=latent_frame_zero,
                                packed=bool(flag)))
    return [u.float() for u in outs]


def forward_14b(self, x, t, context, seq_len, clip_fea=None, y=None, rand_num_img=None, enable_mask=False,
                latent_frame_zero=9, cache_sample=False, cache=None, return_cache=False, cache_list=None):
    """Drop-in for wan WanModel.forward (wan/modules/model.py:723-1013). Returns (tensor, None) like the
    reference with caching off (:1010-1013)."""
    if self.model_type == "i2v":
        assert clip_fea is not None and y is not None                   # wan/modules/model.py:760-761
    if enable_mask:
        raise NotImplementedError("enable_mask=True is the MVDT training path; inference only")
    if cache_sample:
        raise NotImplementedError("the block-residual cache (cache_sample) is unused by the shipped samplers")
    if rand_num_img is None:
        # the reference then multiplies q/k by the [1024, 64] grid table on the packed path and fails with a shape
        # error unless L == 1024 (SURVEY.md Appendix A); keep that an error rather than guessing
        raise RuntimeError("rand_num_img must be set: < 0.4 regular grid, >= 0.4 FramePack (wan/modules/model.py:40-41)")
    if len(x) != 1:
        raise YumeB200Error("the 14B tree only handles batch 1 on the packed RoPE path (wan/modules/model.py:108)")
    eng = _engine(self)
    out = eng.forward(x[0], t, context[0], seq_len, y=y[0] if y is not None else None,
                      clip_fea=clip_fea, latent_frame_zero=latent_frame_zero, packed=rand_num_img >= 0.4)
    return out.float(), None


def install(model: nn.Module, variant: Optional[str] = None, device="cuda", state_dict=None, precision: str = "bf16") -> nn.Module:
    """Attach a WanDiT engine to `model` (reference WanModel or the mirrors below) and re-bind its forward.
    Weights are read from the live module at call time (or from `state_dict`, e.g. when the module was built on
    the meta device); call again after loading a new checkpoint. precision="fp8" runs the six block linears as e4m3 GEMMs,
    precision="fp8_attn" also the self-attention (WanDiT, DESIGN.md §3)."""
    if variant is None:
        variant = "14b" if hasattr(model, "img_emb") else "5b"
    if state_dict is not None:
        model._yb_engine = WanDiT(state_dict, variant, dim=model.dim, ffn_dim=model.ffn_dim, num_heads=model.num_heads,
                                  num_layers=model.num_layers, in_dim=model.in_dim, out_dim=model.out_dim,
                                  text_len=model.text_len, freq_dim=model.freq_dim, patch_size=model.patch_size,
                                  eps=model.eps, device=device, precision=precision)
    else:
        model._yb_engine = WanDiT.from_module(model, variant, device=device, precision=precision)
    model.forward = types.MethodType(forward_5b if variant == "5b" else forward_14b, model)
    return model


# ------------------------------------------------------------------------------------------------------------
# parameter containers with the reference's names
# ------------------------------------------------------------------------------------------------------------
class _RMS(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim))


class _Attn(nn.Module):
    def __init__(self, dim, img: bool):
        super().__init__()
        self.q, self.k, self.v, self.o = (nn.Linear(dim, dim) for _ in range(4))
        self.norm_q, self.norm_k = _RMS(dim), _RMS(dim)
        if img:
            self.k_img, self.v_img, self.norm_k_img = nn.Linear(dim, dim), nn.Linear(dim, dim), _RMS(dim)


class _Block(nn.Module):
    def __init__(self, dim, ffn_dim, img: bool):
        super().__init__()
        self.self_attn = _Attn(dim, False)
        self.norm3 = nn.LayerNorm(dim, eps=1e-6, elementwise_affine=True)
        self.cross_attn = _Attn(dim, img)
        self.ffn = nn.Sequential(nn.Linear(dim, ffn_dim), nn.GELU(approximate="tanh"), nn.Linear(ffn_dim, dim))
        self.modulation = nn.Parameter(torch.randn(1, 6, dim) / dim ** 0.5)


class _Head(nn.Module):
    def __init__(self, dim, out_dim, patch_size):
        super().__init__()
        self.head = nn.Linear(dim, out_dim * patch_size[0] * patch_size[1] * patch_size[2])
        self.modulation = nn.Parameter(torch.randn(1, 2, dim) / dim ** 0.5)


class _MLPProj(nn.Module):
    def __init__(self, in_dim, out_dim):
        super().__init__()
        self.proj = nn.Sequential(nn.LayerNorm(in_dim), nn.Linear(in_dim, in_dim), nn.GELU(), nn.Linear(in_dim, out_dim),
                                  nn.LayerNorm(out_dim))


class _WanBase(nn.Module):
    def __init__(self, variant, model_type, patch_size, text_len, in_dim, dim, ffn_dim, freq_dim, text_dim, out_dim,
                 num_heads, num_layers, window_size, qk_norm, cross_attn_norm, eps, clip_dim=1280):
        super().__init__()
        assert (dim % num_heads) == 0 and (dim // num_heads) % 2 == 0
        self.variant, self.model_type = variant, model_type
        self.patch_size, self.text_len, self.in_dim, self.dim, self.ffn_dim = tuple(patch_size), text_len, in_dim, dim, ffn_dim
        self.freq_dim, self.text_dim, self.out_dim, self.num_heads, self.num_layers = freq_dim, text_dim, out_dim, num_heads, num_layers
        self.window_size, self.qk_norm, self.cross_attn_norm, self.eps = window_size, qk_norm, cross_attn_norm, eps
        img = variant == "14b"
        self.patch_embedding = nn.Conv3d(in_dim, dim, kernel_size=patch_size, stride=patch_size)
        for name, k in (("patch_embedding_2x", 4), ("patch_embedding_4x", 8), ("patch_embedding_8x", 16),
                        ("patch_embedding_16x", 32)):
            setattr(self, name, nn.Conv3d(in_dim, dim, (1, k, k), (1, k, k)))
        self.patch_embedding_2x_f = nn.Conv3d(in_dim, in_dim, (1, 4, 4), (1, 4, 4))
        self.text_embedding = nn.Sequential(nn.Linear(text_dim, dim), nn.GELU(approximate="tanh"), nn.Linear(dim, dim))
        self.time_embedding = nn.Sequential(nn.Linear(freq_dim, dim), nn.SiLU(), nn.Linear(dim, dim))
        self.time_projection = nn.Sequential(nn.SiLU(), nn.Linear(dim, dim * 6))
        self.blocks = nn.ModuleList([_Block(dim, ffn_dim, img) for _ in range(num_layers)])
        self.head = _Head(dim, out_dim, self.patch_size)
        if img:
            self.img_emb = _MLPProj(clip_dim, dim)

    def install(self, device="cuda", state_dict=None, precision: str = "bf16"):
        return install(self, self.variant, device, state_dict, precision=precision)


class WanModel5B(_WanBase):
    """Mirror of wan23 `WanModel` (wan23/modules/model.py:369-498): same constructor arguments and state-dict keys."""

    def __init__(self, model_type="t2v", patch_size=(1, 2, 2), text_len=512, in_dim=16, dim=2048, ffn_dim=8192,
                 freq_dim=256, text_dim=4096, out_dim=16, num_heads=16, num_layers=32, window_size=(-1, -1),
                 qk_norm=True, cross_attn_norm=True, eps=1e-6):
        assert model_type in ["t2v", "i2v", "ti2v"]
        super().__init__("5b", model_type, patch_size, text_len, in_dim, dim, ffn_dim, freq_dim, text_dim, out_dim,
                         num_heads, num_layers, window_size, qk_norm, cross_attn_norm, eps)

    forward = forward_5b


class WanModel14B(_WanBase):
    """Mirror of wan `WanModel` (wan/modules/model.py:548-675; always the i2v cross-attention, :610,642)."""

    def __init__(self, model_type="i2v", patch_size=(1, 2, 2), text_len=512, in_dim=16, dim=2048, ffn_dim=8192,
                 freq_dim=256, text_dim=4096, out_dim=16, num_heads=16, num_layers=32, window_size=(-1, -1),
                 qk_norm=True, cross_attn_norm=True, eps=1e-6, clip_dim=1280):
        assert model_type in ["t2v", "i2v"]
        super().__init__("14b", "i2v", patch_size, text_len, in_dim, dim, ffn_dim, freq_dim, text_dim, out_dim,
                         num_heads, num_layers, window_size, qk_norm, cross_attn_norm, eps, clip_dim)

    forward = forward_14b
