"""H100 ENCODE paths of the two Wan VAEs — SURVEY.md §8(f) "next" row, rank 3: the conditioning / history encodes the samplers
run before the denoise loop (`Wan2_2_VAE.encode`, fastvideo/sample/sample_5b.py:892-893; `WanVAE.encode`,
wan/image2video.py:348-367).

Reference: /root/reference/wan23/modules/vae2_2.py `WanVAE_.encode` (:796-829) and /root/reference/wan/modules/vae.py (:515-542)
encode frame 0 alone and then 4 frames per `Encoder3d.forward` call, threading a feature cache through every `CausalConv3d`.
Unrolled (oracle/wan22vae_enc.py, oracle/wan21vae_enc.py, both pinned to the reference's chunked output) every conv is a causal
conv over the whole frame sequence, so the H100 path is the decoder's design run backwards, on the building blocks of
yume_b200/wan_vae.py: a pass over channels-last bf16
[T, H, W, C] tensors on the wgmma implicit-GEMM conv — one pass when the video fits in device memory, else chunks of 1 + 4a, then 4b
frames carrying the reference's cache state (the decoder's 2-frame conv histories; the last input frame of the stride-2
`time_conv`; AvgDown3D pads in front exactly where its per-call padding does, i.e. only in the first chunk) — with the two strided
`Resample` convs done by the tensor map itself —
  * `Resample(downsample2d)`: ZeroPad2d((0,1,0,1)) + Conv2d(3x3, stride 2) (vae2_2.py:101-104) = `yb_conv3d_causal` with
    `stride_hw = 2`: TMA `elementStrides` sample every second voxel, the pad row/column behind the data is out-of-bounds fill;
  * `Resample(downsample3d)` (:105-110, :158-170): frame 0 bypasses `time_conv`, the rest is CausalConv3d((3,1,1),
    stride (2,1,1), padding 0) over [f0, f1, f2, ...] = `stride_t = 2`, written one output frame behind the copied frame 0;
  * Wan2.2 only: the `AvgDown3D` shortcut of `Down_ResidualBlock` (:320-373, :449-459) is one gather-add, the input `patchify`
    (:284-300) one gather;
  * `conv1` (1x1x1) with the latent normalisation (mu - mean) / std folded into its weights; only the mu half is computed.
No padded or strided copy of any activation.
"""
from __future__ import annotations

import types
from typing import Dict, List, Optional, Sequence

import torch

from . import ops
from ._lib import YumeB200Error
from .wan_vae import _BF16, _F32, Layer, WanVaeEngine, _attn_bytes, _rup

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


def _encoder_tail(c: int, z_dim: int) -> List[Layer]:
    """encoder.middle and encoder.head (+ conv1's mu half): the last layers of both Wan encoders."""
    return [Layer("res", "encoder.middle.0", c, c), Layer("attn", "encoder.middle.1", c), Layer("res", "encoder.middle.2", c, c),
            Layer("head", "encoder.head.2", c, _rup(2 * z_dim, 32) + 2 * _rup(z_dim, 32))]


class WanVaeEncoder(WanVaeEngine):
    """The encode side of both Wan VAEs: f32 [3, T, H, W] -> mu f32 [z_dim, 1 + (T-1)//4, H/SCALE, W/SCALE]. An engine adds its
    layer list, SCALE and `_read` (the chunk's video frames into encoder.conv1's input, or under a row-parallel encode into the
    band buffer of its rows)."""
    SCALE: int

    @property
    def ops(self):
        """This module's op library (see WanVaeEngine)."""
        return ops

    def _repack(self, sd: Dict[str, Tensor], mean: Tensor, std: Tensor) -> None:
        dev = self.device
        sd = self._pack_side(sd, ("encoder.", "conv1."), "conv1", False)
        # conv1 (1x1x1, 2z -> 2z), mu half only (`.chunk(2, dim=1)[0]`, :822), normalisation folded in:
        # (W x + b - mean) / std = (diag(1/std) W) x + (b - mean) / std
        zd = self.z_dim
        W1 = sd["conv1.weight"].detach().float().reshape(2 * zd, 2 * zd)[:zd]
        w = torch.zeros(_rup(zd, 32), _rup(2 * zd, 32), dtype=_F32, device=dev)
        w[:zd, :2 * zd] = W1 / std[:, None]
        b = torch.zeros(_rup(zd, 32), dtype=_F32, device=dev)
        b[:zd] = (sd["conv1.bias"].detach().float()[:zd] - mean) / std
        self.lin["conv1"] = (w.to(dev, _BF16).contiguous(), b.to(dev))

    def _input(self, L: Layer, v: Tensor):
        """encoder.conv1 over its input buffer: carried frames in front, this chunk's frames (patch size L.fs) behind them. Under
        a row-parallel encode the buffer is a band buffer, its rows and both halo rows read straight from the whole video."""
        _, T, H, W = v.shape
        dims = (T, H // L.fs, W // L.fs)
        if self._rows is not None:
            dims = (T, self._band[1] * (dims[1] // self._band[2]), dims[2])
            x0 = self._hist_buf(L.name, *dims, 64, halo=True)
            self._read(v, x0[x0.shape[0] - T:])
        else:
            x0 = self._hist_buf(L.name, *dims, 64)
            self._read(v, x0[x0.shape[0] - T:].view(-1, 64))
        return self._conv(L.name, x0, dims, key=L.name), dims

    def _resample(self, L: Layer, x: Tensor, dims):
        """Resample downsample2d / downsample3d over the frames of this chunk (vae2_2.py:101-110, 152-170; vae.py:84-90,
        125-139). The stride-2 time_conv carries the last frame of its input to the next chunk; frame 0 passes only in the first."""
        p, temporal = L.name, L.ft == 2
        T, H, W = dims
        C = x.shape[1]
        if self._rows is not None:                                 # a band buffer whose row below is the next band's first row
            a = self._act(x, dims, None, False, halo=True, above=False)
        else:
            a = x.view(T, H, W, C) if C % 64 == 0 else self._act(x, dims, None, False)
        _, Ho, Wo = ops.conv_out_dims(T, H, W, (1, 3, 3), 1, 2)
        key = p + ".time_conv"
        if temporal and self._chunk > 0:
            # resample.1 writes behind the carried frame; time_conv reads [carried, 2b new frames] -> b frames
            ybuf = self._hist_buf(key, T, Ho, Wo, C, n=1) if C % 64 == 0 else None
            y = self._conv(p + ".resample.1", a, dims, stride_hw=2, out=None if ybuf is None else ybuf[1:].view(-1, C))
            ain = ybuf if ybuf is not None else self._act(y, (T, Ho, Wo), None, False, key=key, n=1)
            z = self._new((T // 2) * Ho * Wo, C)
            self._conv(p + ".time_conv", ain, (T, Ho, Wo), out=z, stride_t=2, key=key)
            return z, (T // 2, Ho, Wo)
        y = self._conv(p + ".resample.1", a, dims, stride_hw=2)
        if temporal and T > 1:
            if T < 3:
                raise YumeB200Error("downsample3d needs 1 or >= 3 frames (the reference feeds 1 + 4k)")
            a = y.view(T, Ho, Wo, C) if C % 64 == 0 else self._act(y, (T, Ho, Wo), None, False)
            To = (T - 3) // 2 + 1
            z = self._new((1 + To) * Ho * Wo, C)
            z[:Ho * Wo].copy_(y[:Ho * Wo])                         # frame 0 passes ("Rep" branch, :158-163)
            self._conv(p + ".time_conv", a, (T, Ho, Wo), out=z, out_t_add=1, stride_t=2, key=key)
            return z, (1 + To, Ho, Wo)
        if temporal and self._more:                                # frame 0 alone: it is the next chunk's history
            self._keep(key, y.view(T, Ho, Wo, C) if C % 64 == 0 else self._act(y, (T, Ho, Wo), None, False), 1)
        return y, (T, Ho, Wo)

    def _head(self, L: Layer, x: Tensor, dims, out: Tensor) -> None:
        """encoder.head + conv1 (mu half) into `out`, this chunk's latent-frame window of the result."""
        y = self._conv(L.name, self._act(x, dims, "encoder.head.0", True, key=L.name, halo=True), dims, key=L.name)
        w1, b1 = self.lin["conv1"]
        mu = self._new(y.shape[0], w1.shape[0], dtype=_F32)
        ops.gemm(y, w1, b1, mu, ops.YB_EPI_F32)
        if self._rows is not None:                                 # this rank's rows; _stream gathers the others
            r0, hs, _ = self._band
            ops.nhwc_to_nchw_f32_rows(mu, out[:, :, r0:r0 + hs])
        elif self._one_pass:
            ops.nhwc_to_nchw_f32(mu, out.view(self.z_dim, -1))
        else:
            ops.nhwc_to_nchw_f32_win(mu, out)

    def _frames(self, video: Tensor) -> Tensor:
        if video.dim() != 4 or video.shape[0] != 3:
            raise YumeB200Error("expected a video [3, T, H, W]")
        if self._rows is not None:                                 # checked on every rank before the first collective
            if video.shape[2] % self.SCALE or video.shape[3] % self.SCALE:
                raise YumeB200Error(f"Wan VAE encode needs H, W divisible by {self.SCALE}")
            self._set_band(video.shape[2] // self.SCALE)
        keep = 1 + 4 * ((video.shape[1] - 1) // 4)                 # `iter_ = 1 + (t - 1) // 4` chunks of 1, 4, 4, ... (:802-803)
        return video[:, :keep].to(self.device, _F32).contiguous()

    @torch.no_grad()
    def encode(self, video: Tensor) -> Tensor:
        """video f32 [3, T, H, W] -> mu [z_dim, 1 + (T-1)//4, H/s, W/s], in the chunks `plan_chunks` sizes from the free device
        memory. With resume=True a video that extends the last call's video, or its frames before the trailing all-zero
        frames, runs only its new frames (WanVaeEngine._resumed)."""
        v = self._frames(video)
        if self.resume:
            _, T, H, W = v.shape
            return self._resumed(v, v.data_ptr() != video.data_ptr(), self._mu_shape(T, H, W), 4, 1,
                                 lambda n: self.chunk_bytes(n, T, H, W), fork=True)
        return self._encode_chunks(v, self.plan_chunks(*v.shape[1:]))

    def _encode_chunks(self, video: Tensor, lengths: Sequence[int]) -> Tensor:
        """Encode in chunks of `lengths` LATENT frames (a partition of 1 + (T-1)//4): the first chunk reads 1 + 4(n-1) video
        frames, every later one 4n (the reference's frame 0, then 4 frames per call)."""
        video = self._frames(video)
        return self._chunks(video, lengths, self._mu_shape(*video.shape[1:]), 4, 1)

    def _mu_shape(self, T: int, H: int, W: int):
        if H % self.SCALE or W % self.SCALE:
            raise YumeB200Error(f"Wan VAE encode needs H, W divisible by {self.SCALE}")
        return self.z_dim, 1 + (T - 1) // 4, H // self.SCALE, W // self.SCALE

    def _fixed_bytes(self, T: int, H: int, W: int) -> int:
        """mu, and the device copy of the video `encode` makes when it is handed one on another device or not contiguous."""
        return 4 * (self.z_dim * (1 + (T - 1) // 4) * (H // self.SCALE) * (W // self.SCALE) + 3 * T * H * W)

    def _band_bytes(self, n: int, T: int, H: int, W: int) -> int:
        """Upper bound of one rank's device bytes in a row-parallel encode: the largest band in video rows, its halo rows counted
        at every level as two more latent rows, plus the gathered attention input (padded bands, full frames, the attention's
        own buffers and the rows kept), the whole video once, and mu with the padded bands of its all-gather."""
        P, S = self._rows.world, self.SCALE
        Hl, Wl = H // S, W // S
        hb = -(-Hl // P)
        c = next(L for L in self.layers if L.kind == "attn").ci
        gathered = ((P + 2) * n * hb * Wl + n * Hl * Wl) * c * 2 + _attn_bytes(n, Hl * Wl, c)
        band = self._chunk_bytes(n, T, (hb + 2) * S, W) - self._fixed_bytes(T, (hb + 2) * S, W)
        mu = 4 * self.z_dim * (1 + (T - 1) // 4) * Hl * Wl
        return band + gathered + 4 * 3 * T * H * W + (1 + P) * mu

    def plan_chunks(self, T: int, H: int, W: int) -> List[int]:
        """Latent frames per chunk of an encode of T video frames at H x W (see _plan)."""
        return self._plan(1 + (T - 1) // 4, lambda n: self.chunk_bytes(n, T, H, W))


class Wan22VaeEncoder(WanVaeEncoder):
    """`Wan2_2_VAE.encode` for one video: f32 [3, T, H, W] -> mu f32 [z_dim, 1 + (T-1)//4, H/16, W/16]."""
    SCALE = 16                                                     # patchify 2 x three stride-2 levels

    def __init__(self, sd: Dict[str, Tensor], dim: int = 160, z_dim: int = 48, dim_mult: Sequence[int] = (1, 2, 4, 4),
                 num_res_blocks: int = 2, temperal_downsample: Sequence[bool] = (False, True, True),
                 mean: Optional[Tensor] = None, std: Optional[Tensor] = None, device="cuda", precision: str = "bf16",
                 resume: bool = False, **_):
        dims = [dim * u for u in [1] + list(dim_mult)]                               # vae2_2.py:527
        layers = [Layer("in", "encoder.conv1", 64, dims[0], 4, 2)]
        for i in range(len(dim_mult)):                             # Down_ResidualBlock (:420-459)
            p, ci, co = f"encoder.downsamples.{i}.downsamples", dims[i], dims[i + 1]
            down = i != len(dim_mult) - 1
            ft = 2 if i < len(temperal_downsample) and temperal_downsample[i] else 1
            layers.append(Layer("hold", ci=ci))
            layers += [Layer("res", f"{p}.{j}", ci if j == 0 else co, co) for j in range(num_res_blocks)]
            if down:
                layers.append(Layer("down", f"{p}.{num_res_blocks}", co, co, ft, 2))
            layers.append(Layer("avgdown", ci=ci, co=co, ft=ft, fs=2 if down else 1))
        super().__init__(sd, z_dim, layers + _encoder_tail(dims[-1], z_dim), mean, std, device, precision, resume)

    def _read(self, v: Tensor, dst: Tensor) -> None:
        if self._rows is not None:
            ops.vae_patchify2_bf16_rows(v, dst, self._row0(dst.shape[1] - 2))
        elif self._one_pass:
            ops.vae_patchify2_bf16(v, dst)
        else:
            ops.vae_patchify2_bf16_win(v, dst)


class Wan21VaeEncoder(WanVaeEncoder):
    """`WanVAE.encode` (wan/modules/vae.py:515-542, 645-653): f32 [3, T, H, W] -> mu f32 [16, 1 + (T-1)//4, H/8, W/8]. Flat
    `encoder.downsamples` Sequential (:293-306), no AvgDown3D shortcut, RGB straight into `encoder.conv1`."""
    SCALE = 8

    def __init__(self, sd: Dict[str, Tensor], dim: int = 96, z_dim: int = 16, dim_mult: Sequence[int] = (1, 2, 4, 4),
                 num_res_blocks: int = 2, temperal_downsample: Sequence[bool] = (False, True, True),
                 mean: Optional[Tensor] = None, std: Optional[Tensor] = None, device="cuda", precision: str = "bf16",
                 resume: bool = False, **_):
        dims = [dim * u for u in [1] + list(dim_mult)]
        layers, n = [Layer("in", "encoder.conv1", 64, dims[0], 4, 1)], 0
        for i in range(len(dim_mult)):
            ci, co = dims[i], dims[i + 1]
            for _ in range(num_res_blocks):
                layers.append(Layer("res", f"encoder.downsamples.{n}", ci, co))
                n, ci = n + 1, co
            if i != len(dim_mult) - 1:
                layers.append(Layer("down", f"encoder.downsamples.{n}", co, co, 2 if temperal_downsample[i] else 1, 2))
                n += 1
        super().__init__(sd, z_dim, layers + _encoder_tail(dims[-1], z_dim), mean, std, device, precision, resume)

    def _read(self, v: Tensor, dst: Tensor) -> None:
        if self._rows is not None:
            ops.nchw_to_nhwc_bf16_rows(v, dst, self._row0(dst.shape[1] - 2))
        elif self._one_pass:
            ops.nchw_to_nhwc_bf16(v.view(3, -1), dst)
        else:
            ops.nchw_to_nhwc_bf16_win(v, dst)


def install_wan22_vae_encoder(vae, device="cuda", precision: str = "bf16", resume: bool = False):
    """Attach a Wan22VaeEncoder to a live reference `Wan2_2_VAE` wrapper and re-bind its `encode(videos)` (list in / list out,
    a non-list logs the TypeError and returns None: vae2_2.py:1045-1057). precision: "bf16" only (encodes stay bf16). resume:
    keep the last encode's state so that a video extending it encodes only its new frames (WanVaeEngine._resumed)."""
    m = vae.model
    sd = dict(m.state_dict())
    mean, inv_std = vae.scale
    dim_mult = list(m.dim_mult)
    eng = Wan22VaeEncoder(sd, dim=sd["encoder.conv1.weight"].shape[0], z_dim=m.z_dim, dim_mult=dim_mult,
                          num_res_blocks=m.num_res_blocks, temperal_downsample=list(m.temperal_downsample),
                          mean=mean.detach().float().cpu(), std=(1.0 / inv_std.detach().float()).cpu(), device=device,
                          precision=precision, resume=resume)
    vae._yb_encoder = eng

    def encode(self, videos, cache=True):
        if not isinstance(videos, list):
            import logging
            logging.info(TypeError("videos should be a list"))
            return None
        return [eng.encode(u) for u in videos]

    vae.encode = types.MethodType(encode, vae)
    return vae


def install_wan21_vae_encoder(vae, device="cuda", precision: str = "bf16", resume: bool = False):
    """Attach a Wan21VaeEncoder to a live reference `WanVAE` wrapper and re-bind its `encode(videos)` (vae.py:645-653).
    precision: "bf16" only (encodes stay bf16). resume: keep the last encode's state so that a video extending it encodes
    only its new frames (WanVaeEngine._resumed)."""
    m = vae.model
    eng = Wan21VaeEncoder(dict(m.state_dict()), dim=m.dim, z_dim=m.z_dim, dim_mult=list(m.dim_mult),
                          num_res_blocks=m.num_res_blocks, temperal_downsample=list(m.temperal_downsample),
                          mean=vae.mean.detach().float(), std=vae.std.detach().float(), device=device, precision=precision,
                          resume=resume)
    vae._yb_encoder = eng

    def encode(self, videos):
        return [eng.encode(u) for u in videos]

    vae.encode = types.MethodType(encode, vae)
    return vae
