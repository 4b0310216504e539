"""H100 ENCODE paths of the two Wan VAEs — SURVEY.md §8(f) "next" row, rank 3: the conditioning / history encodes the samplers
run before the denoise loop (`Wan2_2_VAE.encode`, fastvideo/sample/sample_5b.py:892-893; `WanVAE.encode`,
wan/image2video.py:348-367).

Reference: /root/reference/wan23/modules/vae2_2.py `WanVAE_.encode` (:796-829) and /root/reference/wan/modules/vae.py (:515-542)
encode frame 0 alone and then 4 frames per `Encoder3d.forward` call, threading a feature cache through every `CausalConv3d`.
Unrolled (oracle/wan22vae_enc.py, oracle/wan21vae_enc.py, both pinned to the reference's chunked output) every conv is a causal
conv over the whole frame sequence, so the H100 path is the decoder's design run backwards: ONE pass over channels-last bf16
[T, H, W, C] tensors on the wgmma implicit-GEMM conv, with the two strided `Resample` convs done by the tensor map itself —
  * `Resample(downsample2d)`: ZeroPad2d((0,1,0,1)) + Conv2d(3x3, stride 2) (vae2_2.py:101-104) = `yb_conv3d_causal` with
    `stride_hw = 2`: TMA `elementStrides` sample every second voxel, the pad row/column behind the data is out-of-bounds fill;
  * `Resample(downsample3d)` (:105-110, :158-170): frame 0 bypasses `time_conv`, the rest is CausalConv3d((3,1,1),
    stride (2,1,1), padding 0) over [f0, f1, f2, ...] = `stride_t = 2`, written one output frame behind the copied frame 0;
  * Wan2.2 only: the `AvgDown3D` shortcut of `Down_ResidualBlock` (:320-373, :449-459) is one gather-add, the input `patchify`
    (:284-300) one gather;
  * `conv1` (1x1x1) with the latent normalisation (mu - mean) / std folded into its weights; only the mu half is computed.
No feature cache, no per-chunk launches, no padded or strided copy of any activation.
"""
from __future__ import annotations

import types
from typing import Dict, Optional, Sequence

import torch

from . import ops
from ._lib import YumeB200Error
from .vae22 import _BF16, _F32, Wan22VaeDecoder, _rup

Tensor = torch.Tensor

__all__ = ["Wan22VaeEncoder", "Wan21VaeEncoder", "install_wan22_vae_encoder", "install_wan21_vae_encoder",
           "encoder_param_shapes_22", "encoder_param_shapes_21"]


def _res_shapes(s: Dict[str, tuple], p: str, ci: int, co: int) -> None:
    s[p + ".residual.0.gamma"] = (ci, 1, 1, 1)
    s[p + ".residual.2.weight"], s[p + ".residual.2.bias"] = (co, ci, 3, 3, 3), (co,)
    s[p + ".residual.3.gamma"] = (co, 1, 1, 1)
    s[p + ".residual.6.weight"], s[p + ".residual.6.bias"] = (co, co, 3, 3, 3), (co,)
    if ci != co:
        s[p + ".shortcut.weight"], s[p + ".shortcut.bias"] = (co, ci, 1, 1, 1), (co,)


def _tail_shapes(s: Dict[str, tuple], d: int, z_dim: int) -> None:
    _res_shapes(s, "encoder.middle.0", d, d)
    s["encoder.middle.1.norm.gamma"] = (d, 1, 1)
    s["encoder.middle.1.to_qkv.weight"], s["encoder.middle.1.to_qkv.bias"] = (3 * d, d, 1, 1), (3 * d,)
    s["encoder.middle.1.proj.weight"], s["encoder.middle.1.proj.bias"] = (d, d, 1, 1), (d,)
    _res_shapes(s, "encoder.middle.2", d, d)
    s["encoder.head.0.gamma"] = (d, 1, 1, 1)
    s["encoder.head.2.weight"], s["encoder.head.2.bias"] = (2 * z_dim, d, 3, 3, 3), (2 * z_dim,)


def encoder_param_shapes_22(dim: int = 160, z_dim: int = 48, dim_mult: Sequence[int] = (1, 2, 4, 4), num_res_blocks: int = 2,
                            temperal_downsample: Sequence[bool] = (False, True, True)) -> Dict[str, tuple]:
    """State-dict keys / shapes of the encode-side modules of the 2.2 `WanVAE_` (conv1 + Encoder3d, vae2_2.py:506-620)."""
    dims = [dim * u for u in [1] + list(dim_mult)]
    s: Dict[str, tuple] = {"conv1.weight": (2 * z_dim, 2 * z_dim, 1, 1, 1), "conv1.bias": (2 * z_dim,),
                           "encoder.conv1.weight": (dims[0], 12, 3, 3, 3), "encoder.conv1.bias": (dims[0],)}
    for i, (ci, co) in enumerate(zip(dims[:-1], dims[1:])):
        p, c = f"encoder.downsamples.{i}.downsamples", ci
        for j in range(num_res_blocks):
            _res_shapes(s, f"{p}.{j}", c, co)
            c = co
        if i != len(dim_mult) - 1:
            q = f"{p}.{num_res_blocks}"
            s[q + ".resample.1.weight"], s[q + ".resample.1.bias"] = (co, co, 3, 3), (co,)
            if i < len(temperal_downsample) and temperal_downsample[i]:
                s[q + ".time_conv.weight"], s[q + ".time_conv.bias"] = (co, co, 3, 1, 1), (co,)
    _tail_shapes(s, dims[-1], z_dim)
    return s


def encoder_param_shapes_21(dim: int = 96, z_dim: int = 16, dim_mult: Sequence[int] = (1, 2, 4, 4), num_res_blocks: int = 2,
                            temperal_downsample: Sequence[bool] = (False, True, True)) -> Dict[str, tuple]:
    """State-dict keys / shapes of the encode-side modules of the 2.1 `WanVAE_` (conv1 + Encoder3d, vae.py:265-366, 500-502)."""
    dims = [dim * u for u in [1] + list(dim_mult)]
    s: Dict[str, tuple] = {"conv1.weight": (2 * z_dim, 2 * z_dim, 1, 1, 1), "conv1.bias": (2 * z_dim,),
                           "encoder.conv1.weight": (dims[0], 3, 3, 3, 3), "encoder.conv1.bias": (dims[0],)}
    n = 0
    for i, (ci, co) in enumerate(zip(dims[:-1], dims[1:])):
        for _ in range(num_res_blocks):
            _res_shapes(s, f"encoder.downsamples.{n}", ci, co)
            n, ci = n + 1, co
        if i != len(dim_mult) - 1:
            q = f"encoder.downsamples.{n}"
            s[q + ".resample.1.weight"], s[q + ".resample.1.bias"] = (co, co, 3, 3), (co,)
            if temperal_downsample[i]:
                s[q + ".time_conv.weight"], s[q + ".time_conv.bias"] = (co, co, 3, 1, 1), (co,)
            n += 1
    _tail_shapes(s, dims[-1], z_dim)
    return s


class Wan22VaeEncoder(Wan22VaeDecoder):
    """`Wan2_2_VAE.encode` for one video: f32 [3, T, H, W] -> mu f32 [z_dim, 1 + (T-1)//4, H/16, W/16]. The building blocks
    (`_conv`, `_act`, `_res_block`, `_attention`) are the decoder's."""

    def __init__(self, sd: Dict[str, Tensor], dim: int = 160, z_dim: int = 48, dim_mult: Sequence[int] = (1, 2, 4, 4),
                 num_res_blocks: int = 2, temperal_downsample: Sequence[bool] = (False, True, True),
                 mean: Optional[Tensor] = None, std: Optional[Tensor] = None, device="cuda", **_):
        self.device = torch.device(device)
        self.z_dim, self.nrb = z_dim, num_res_blocks
        self.dims = [dim * u for u in [1] + list(dim_mult)]                         # vae2_2.py:527
        self.t_down, self.n_down = list(temperal_downsample), len(dim_mult)
        mean = torch.zeros(z_dim) if mean is None else mean
        std = torch.ones(z_dim) if std is None else std
        self._repack_encoder(sd, mean.detach().to(self.device, _F32), std.detach().to(self.device, _F32), self.dims[-1])

    def _repack_encoder(self, sd: Dict[str, Tensor], mean: Tensor, std: Tensor, width: int) -> None:
        dev = self.device
        sd = self._pack_side(sd, ("encoder.", "conv1."), "conv1", "encoder.middle.1", width, False)
        # conv1 (1x1x1, 2z -> 2z), mu half only (`.chunk(2, dim=1)[0]`, :822), normalisation folded in:
        # (W x + b - mean) / std = (diag(1/std) W) x + (b - mean) / std
        zd = self.z_dim
        W1 = sd["conv1.weight"].detach().float().reshape(2 * zd, 2 * zd)[:zd]
        w = torch.zeros(_rup(zd, 32), _rup(2 * zd, 32), dtype=_F32, device=dev)
        w[:zd, :2 * zd] = W1 / std[:, None]
        b = torch.zeros(_rup(zd, 32), dtype=_F32, device=dev)
        b[:zd] = (sd["conv1.bias"].detach().float()[:zd] - mean) / std
        self.lin["conv1"] = (w.to(dev, _BF16).contiguous(), b.to(dev))

    # ---- building blocks the decoder does not have -----------------------------------------------------------
    def _resample_down(self, p: str, x: Tensor, dims, temporal: bool):
        """Resample downsample2d / downsample3d over the whole sequence (vae2_2.py:101-110, 152-170; vae.py:84-90, 125-139)."""
        T, H, W = dims
        C = x.shape[1]
        a = x.view(T, H, W, C) if C % 64 == 0 else self._act(x, dims, None, False)
        y = self._conv(p + ".resample.1", a, dims, stride_hw=2)
        _, Ho, Wo = ops.conv_out_dims(T, H, W, (1, 3, 3), 1, 2)
        if temporal and T > 1:
            if T < 3:
                raise YumeB200Error("downsample3d needs 1 or >= 3 frames (the reference feeds 1 + 4k)")
            a = y.view(T, Ho, Wo, C) if C % 64 == 0 else self._act(y, (T, Ho, Wo), None, False)
            To = (T - 3) // 2 + 1
            z = self._new((1 + To) * Ho * Wo, C)
            z[:Ho * Wo].copy_(y[:Ho * Wo])                         # frame 0 passes ("Rep" branch, :158-163)
            self._conv(p + ".time_conv", a, (T, Ho, Wo), out=z, out_t_add=1, stride_t=2)
            return z, (1 + To, Ho, Wo)
        return y, (T, Ho, Wo)

    def _down_block(self, i: int, x: Tensor, dims):
        """Down_ResidualBlock (:420-459)."""
        p = f"encoder.downsamples.{i}.downsamples"
        down = i != self.n_down - 1
        t_down = self.t_down[i] if i < len(self.t_down) else False
        x_in, dims_in = x, dims
        for j in range(self.nrb):
            x = self._res_block(f"{p}.{j}", x, dims)
        if down:
            x, dims = self._resample_down(f"{p}.{self.nrb}", x, dims, t_down)
        ops.vae_avgdown_add(x, x_in, dims_in, x_in.shape[1], x.shape[1], 2 if t_down else 1, 2 if down else 1)
        return x, dims

    def _frames(self, video: Tensor) -> Tensor:
        if video.dim() != 4 or video.shape[0] != 3:
            raise YumeB200Error("expected a video [3, T, H, W]")
        keep = 1 + 4 * ((video.shape[1] - 1) // 4)                 # `iter_ = 1 + (t - 1) // 4` chunks of 1, 4, 4, ... (:802-803)
        return video[:, :keep].to(self.device, _F32).contiguous()

    def _head(self, x: Tensor, dims) -> Tensor:
        y = self._conv("encoder.head.2", self._act(x, dims, "encoder.head.0", True), dims)
        w1, b1 = self.lin["conv1"]
        mu = self._new(y.shape[0], w1.shape[0], dtype=_F32)
        ops.gemm(y, w1, b1, mu, ops.YB_EPI_F32)
        out = self._new(self.z_dim, *dims, dtype=_F32)
        ops.nhwc_to_nchw_f32(mu, out.view(self.z_dim, -1))
        return out

    def _middle(self, x: Tensor, dims) -> Tensor:
        x = self._res_block("encoder.middle.0", x, dims)
        x = self._attention("encoder.middle.1", x, dims)
        return self._res_block("encoder.middle.2", x, dims)

    @torch.no_grad()
    def encode(self, video: Tensor) -> Tensor:
        video = self._frames(video)
        _, T, H, W = video.shape
        if H % 16 or W % 16:
            raise YumeB200Error("Wan2.2 VAE encode needs H, W divisible by 16 (patchify 2 x three stride-2 levels)")
        dims = (T, H // 2, W // 2)
        x0 = self._new(dims[0] * dims[1] * dims[2], 64)
        ops.vae_patchify2_bf16(video, x0)
        x = self._conv("encoder.conv1", x0.view(*dims, 64), dims)
        for i in range(self.n_down):
            x, dims = self._down_block(i, x, dims)
        return self._head(self._middle(x, dims), dims)

    def decode(self, z):                                           # the inherited decoder entry point has no weights here
        raise YumeB200Error("this engine holds the encoder side; use Wan22VaeDecoder for decode")


class Wan21VaeEncoder(Wan22VaeEncoder):
    """`WanVAE.encode` (wan/modules/vae.py:515-542, 645-653): f32 [3, T, H, W] -> mu f32 [16, 1 + (T-1)//4, H/8, W/8]. Flat
    `encoder.downsamples` Sequential (:293-306), no AvgDown3D shortcut, RGB straight into `encoder.conv1`."""

    def __init__(self, sd: Dict[str, Tensor], dim: int = 96, z_dim: int = 16, dim_mult: Sequence[int] = (1, 2, 4, 4),
                 num_res_blocks: int = 2, temperal_downsample: Sequence[bool] = (False, True, True),
                 mean: Optional[Tensor] = None, std: Optional[Tensor] = None, device="cuda", **_):
        self.device = torch.device(device)
        self.z_dim = z_dim
        dims = [dim * u for u in [1] + list(dim_mult)]
        self.plan, n = [], 0
        for i in range(len(dim_mult)):
            for _ in range(num_res_blocks):
                self.plan.append((n, "res"))
                n += 1
            if i != len(dim_mult) - 1:
                self.plan.append((n, "downsample3d" if temperal_downsample[i] else "downsample2d"))
                n += 1
        mean = torch.zeros(z_dim) if mean is None else mean
        std = torch.ones(z_dim) if std is None else std
        self._repack_encoder(sd, mean.detach().to(self.device, _F32), std.detach().to(self.device, _F32), dims[-1])

    @torch.no_grad()
    def encode(self, video: Tensor) -> Tensor:
        video = self._frames(video)
        _, T, H, W = video.shape
        if H % 8 or W % 8:
            raise YumeB200Error("Wan2.1 VAE encode needs H, W divisible by 8")
        dims = (T, H, W)
        x0 = self._new(T * H * W, 64)
        ops.nchw_to_nhwc_bf16(video.view(3, -1), x0)
        x = self._conv("encoder.conv1", x0.view(T, H, W, 64), dims)
        for n, kind in self.plan:
            p = f"encoder.downsamples.{n}"
            if kind == "res":
                x = self._res_block(p, x, dims)
            else:
                x, dims = self._resample_down(p, x, dims, kind == "downsample3d")
        return self._head(self._middle(x, dims), dims)


def install_wan22_vae_encoder(vae, device="cuda"):
    """Attach a Wan22VaeEncoder to a live reference `Wan2_2_VAE` wrapper and re-bind its `encode(videos)` (list in / list out,
    a non-list logs the TypeError and returns None: vae2_2.py:1045-1057)."""
    m = vae.model
    sd = dict(m.state_dict())
    mean, inv_std = vae.scale
    dim_mult = list(m.dim_mult)
    eng = Wan22VaeEncoder(sd, dim=sd["encoder.conv1.weight"].shape[0], z_dim=m.z_dim, dim_mult=dim_mult,
                          num_res_blocks=m.num_res_blocks, temperal_downsample=list(m.temperal_downsample),
                          mean=mean.detach().float().cpu(), std=(1.0 / inv_std.detach().float()).cpu(), device=device)
    vae._yb_encoder = eng

    def encode(self, videos, cache=True):
        if not isinstance(videos, list):
            import logging
            logging.info(TypeError("videos should be a list"))
            return None
        return [eng.encode(u) for u in videos]

    vae.encode = types.MethodType(encode, vae)
    return vae


def install_wan21_vae_encoder(vae, device="cuda"):
    """Attach a Wan21VaeEncoder to a live reference `WanVAE` wrapper and re-bind its `encode(videos)` (vae.py:645-653)."""
    m = vae.model
    eng = Wan21VaeEncoder(dict(m.state_dict()), dim=m.dim, z_dim=m.z_dim, dim_mult=list(m.dim_mult),
                          num_res_blocks=m.num_res_blocks, temperal_downsample=list(m.temperal_downsample),
                          mean=vae.mean.detach().float(), std=vae.std.detach().float(), device=device)
    vae._yb_encoder = eng

    def encode(self, videos):
        return [eng.encode(u) for u in videos]

    vae.encode = types.MethodType(encode, vae)
    return vae
