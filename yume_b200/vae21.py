"""H100 decode path of the Wan2.1 VAE (`WanVAE.decode`) — the VAE the 14B sampler calls (wan/image2video.py:197,
fastvideo/sample/sample.py). SURVEY.md §8(f) "next" row, rank 1 (second half).

Reference: /root/reference/wan/modules/vae.py (≡ wan23/modules/vae2_1.py) — `WanVAE_.decode` (:544-568) decodes one
latent frame per `Decoder3d.forward` call through a per-conv feature cache. As for the 2.2 VAE (yume_b200/vae22.py, whose
decode side this engine shares) the cache logic unrolls to causal convs over the whole sequence, so the H100 path is a
single pass of wgmma implicit-GEMM convs with TMA zero fill as the padding. What differs from 2.2: the flat
`decoder.upsamples` Sequential (:395-414), `Resample`'s Conv2d halves the channels (:76-83) so blocks 1..3 start at
dims[i] // 2 (:398-399), there is no DupUp3D shortcut, and the head conv emits RGB directly (no unpatchify).
"""
from __future__ import annotations

import types
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import ops
from .vae22 import WanVaeDecoder, decoder_front
from .wan_vae import Layer, _rup

Tensor = torch.Tensor


def upsample_plan(dim: int = 96, dim_mult: Sequence[int] = (1, 2, 4, 4), num_res_blocks: int = 2,
                  temperal_upsample: Sequence[bool] = (True, True, False)) -> List[Tuple[int, str, int, int]]:
    """(sequential index, kind, in_dim, out_dim) for every module of `Decoder3d.upsamples` (vae.py:395-414)."""
    dims = [dim * u for u in [dim_mult[-1]] + list(dim_mult[::-1])]
    plan, n = [], 0
    for i in range(len(dim_mult)):
        ci, co = (dims[i] // 2 if i in (1, 2, 3) else dims[i]), dims[i + 1]
        for _ in range(num_res_blocks + 1):
            plan.append((n, "res", ci, co))
            n, ci = n + 1, co
        if i != len(dim_mult) - 1:
            plan.append((n, "upsample3d" if temperal_upsample[i] else "upsample2d", co, co // 2))
            n += 1
    return plan


def decoder_param_shapes(dim: int = 96, z_dim: int = 16, dim_mult: Sequence[int] = (1, 2, 4, 4), num_res_blocks: int = 2,
                         temperal_upsample: Sequence[bool] = (True, True, False)) -> Dict[str, tuple]:
    """State-dict keys / shapes of the decode-side modules of `WanVAE_` (conv2 + Decoder3d, vae.py:369-419, 503-506)."""
    d0 = dim * dim_mult[-1]
    s: Dict[str, tuple] = {}

    def conv(p, co, ci, *k):
        s[p + ".weight"], s[p + ".bias"] = (co, ci, *k), (co,)

    def res(p, ci, co):
        s[p + ".residual.0.gamma"] = (ci, 1, 1, 1)
        conv(p + ".residual.2", co, ci, 3, 3, 3)
        s[p + ".residual.3.gamma"] = (co, 1, 1, 1)
        conv(p + ".residual.6", co, co, 3, 3, 3)
        if ci != co:
            conv(p + ".shortcut", co, ci, 1, 1, 1)

    conv("conv2", z_dim, z_dim, 1, 1, 1)
    conv("decoder.conv1", d0, z_dim, 3, 3, 3)
    res("decoder.middle.0", d0, d0)
    s["decoder.middle.1.norm.gamma"] = (d0, 1, 1)
    conv("decoder.middle.1.to_qkv", 3 * d0, d0, 1, 1)
    conv("decoder.middle.1.proj", d0, d0, 1, 1)
    res("decoder.middle.2", d0, d0)
    last = d0
    for n, kind, ci, co in upsample_plan(dim, dim_mult, num_res_blocks, temperal_upsample):
        p = f"decoder.upsamples.{n}"
        if kind == "res":
            res(p, ci, co)
            last = co
        else:
            conv(p + ".resample.1", co, ci, 3, 3)
            if kind == "upsample3d":
                conv(p + ".time_conv", 2 * ci, ci, 3, 1, 1)
    s["decoder.head.0.gamma"] = (last, 1, 1, 1)
    conv("decoder.head.2", 3, last, 3, 3, 3)
    return s


class Wan21VaeDecoder(WanVaeDecoder):
    """`WanVAE.decode` (vae.py:655-663): z [z_dim, T, H, W] -> f32 [3, 4(T-1)+1, 8H, 8W]."""
    SCALE = 8

    def __init__(self, sd: Dict[str, Tensor], dim: int = 96, z_dim: int = 16, dim_mult: Sequence[int] = (1, 2, 4, 4),
                 num_res_blocks: int = 2, temperal_upsample: Sequence[bool] = (True, True, False),
                 mean: Optional[Tensor] = None, std: Optional[Tensor] = None, device="cuda", precision: str = "bf16",
                 resume: bool = False, **_):
        self.plan = upsample_plan(dim, dim_mult, num_res_blocks, temperal_upsample)
        layers = decoder_front(dim * dim_mult[-1])
        for n, kind, ci, co in self.plan:                        # Resample's Conv2d halves the channels (:76-83)
            p = f"decoder.upsamples.{n}"
            ft = 2 if kind == "upsample3d" else 1
            layers.append(Layer("res", p, ci, co) if kind == "res" else Layer("up", p, ci, co, ft, 2))
        layers.append(Layer("head", "decoder.head.2", self.plan[-1][3], _rup(3, 32)))
        super().__init__(sd, z_dim, layers, mean, std, device, precision, resume)

    def _write(self, y: Tensor, out: Tensor, dims) -> None:
        if self._rows is not None:
            _, hs, _ = dims
            r = self._row0(hs)
            ops.nhwc_to_nchw_f32_rows(y, out[:, :, r:r + hs], (-1.0, 1.0))
        elif self._one_pass:
            ops.nhwc_to_nchw_f32(y, out.view(3, -1), clamp=(-1.0, 1.0))
        else:
            ops.nhwc_to_nchw_f32_win(y, out, (-1.0, 1.0))


def install_wan21_vae(vae, device="cuda", precision: str = "bf16", resume: bool = False):
    """Attach a Wan21VaeDecoder to a live reference `WanVAE` wrapper and re-bind its `decode(zs)` (list in / list out,
    vae.py:655-663). precision: "bf16" only (Wan21VaeDecoder rejects "fp8"). resume: keep the last decode's state so that a
    latent extending it decodes only its new frames (WanVaeEngine._resumed)."""
    m = vae.model
    eng = Wan21VaeDecoder(dict(m.state_dict()), dim=m.dim, z_dim=m.z_dim, dim_mult=list(m.dim_mult),
                          num_res_blocks=m.num_res_blocks, temperal_upsample=list(m.temperal_upsample),
                          mean=vae.mean.detach().float(), std=vae.std.detach().float(), device=device, precision=precision,
                          resume=resume)
    vae._yb_decoder = eng

    def decode(self, zs):
        return [eng.decode(u) for u in zs]

    vae.decode = types.MethodType(decode, vae)
    return vae
