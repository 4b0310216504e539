"""H100 decode path of the Wan2.1 VAE (`WanVAE.decode`) — the VAE the 14B sampler calls (wan/image2video.py:197,
fastvideo/sample/sample.py). SURVEY.md §8(f) "next" row, rank 1 (second half).

Reference: /root/reference/wan/modules/vae.py (≡ wan23/modules/vae2_1.py) — `WanVAE_.decode` (:544-568) decodes one
latent frame per `Decoder3d.forward` call through a per-conv feature cache. As for the 2.2 VAE (yume_b200/vae22.py, whose
building blocks this engine reuses) the cache logic unrolls to causal convs over the whole sequence, so the H100 path is a
single pass of wgmma implicit-GEMM convs with TMA zero fill as the padding. What differs from 2.2: the flat
`decoder.upsamples` Sequential (:395-414), `Resample`'s Conv2d halves the channels (:76-83) so blocks 1..3 start at
dims[i] // 2 (:398-399), there is no DupUp3D shortcut, and the head conv emits RGB directly (no unpatchify).
"""
from __future__ import annotations

import types
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import ops
from .vae22 import _F32, Wan22VaeDecoder

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


class Wan21VaeDecoder(Wan22VaeDecoder):
    def __init__(self, sd: Dict[str, Tensor], dim: int = 96, z_dim: int = 16, dim_mult: Sequence[int] = (1, 2, 4, 4),
                 num_res_blocks: int = 2, temperal_upsample: Sequence[bool] = (True, True, False),
                 mean: Optional[Tensor] = None, std: Optional[Tensor] = None, device="cuda", **_):
        self.device = torch.device(device)
        self.z_dim = z_dim
        self.dims = [dim * dim_mult[-1]]                         # attention width (decoder.middle.1)
        self.plan = upsample_plan(dim, dim_mult, num_res_blocks, temperal_upsample)
        mean = torch.zeros(z_dim) if mean is None else mean
        std = torch.ones(z_dim) if std is None else std
        self._repack(sd, mean.detach().to(self.device, _F32), std.detach().to(self.device, _F32))

    def _t_ups(self) -> int:
        return sum(1 for _, kind, _, _ in self.plan if kind == "upsample3d")

    def _out_shape(self, T: int, H: int, W: int):
        return 3, 1 + (T - 1) * (1 << self._t_ups()), 8 * H, 8 * W

    def _decode_chunk(self, z: Tensor, out: Tensor) -> None:
        """One chunk of `decode` (WanVAE.decode :655-663) into `out`, its frame window of the video."""
        x, dims = self._front(z)
        x = self._res_block("decoder.middle.0", x, dims)
        x = self._attention("decoder.middle.1", x, dims)
        x = self._res_block("decoder.middle.2", x, dims)
        for n, kind, _, _ in self.plan:
            p = f"decoder.upsamples.{n}"
            if kind == "res":
                x = self._res_block(p, x, dims)
            else:
                x, dims = self._resample(p, x, dims, kind == "upsample3d")
        y = self._head(x, dims)
        if self._chunk == 0 and not self._more:
            ops.nhwc_to_nchw_f32(y, out.view(3, -1), clamp=(-1.0, 1.0))
        else:
            ops.nhwc_to_nchw_f32_win(y, out, (-1.0, 1.0))

    def _level_plan(self, H: int, W: int) -> List[tuple]:
        d0 = self.dims[0]
        plan: List[tuple] = [("in", 1, H, W, 64, d0), ("res", 1, H, W, d0, d0), ("attn", 1, H, W, d0, 0), ("res", 1, H, W, d0, d0)]
        s, h, w, last = 1, H, W, d0
        for _, kind, ci, co in self.plan:
            if kind == "res":
                plan.append(("res", s, h, w, ci, co))
            else:                                                # Resample's Conv2d halves the channels (:76-83)
                plan.append(("up", s, h, w, ci, co, kind == "upsample3d", 0))
                s, h, w = (2 * s if kind == "upsample3d" else s), 2 * h, 2 * w
            last = co
        plan.append(("head", s, h, w, last, self.conv["decoder.head.2"][0].shape[0]))
        return plan


def install_wan21_vae(vae, device="cuda"):
    """Attach a Wan21VaeDecoder to a live reference `WanVAE` wrapper and re-bind its `decode(zs)` (list in / list out,
    vae.py:655-663)."""
    m = vae.model
    eng = Wan21VaeDecoder(dict(m.state_dict()), dim=m.dim, z_dim=m.z_dim, dim_mult=list(m.dim_mult),
                          num_res_blocks=m.num_res_blocks, temperal_upsample=list(m.temperal_upsample),
                          mean=vae.mean.detach().float(), std=vae.std.detach().float(), device=device)
    vae._yb_decoder = eng

    def decode(self, zs):
        return [eng.decode(u) for u in zs]

    vae.decode = types.MethodType(decode, vae)
    return vae
