"""H100 decode path of the Wan2.2 VAE (`Wan2_2_VAE.decode`) — the VAE the Yume-5B sampler actually calls
(wan23/textimage2video.py:124; fastvideo/sample/sample_5b.py:1051-1052). SURVEY.md §8(f) "next" row, rank 1.

Reference: /root/reference/wan23/modules/vae2_2.py — `WanVAE_.decode` (:831-860) feeds ONE latent frame at a time through
`Decoder3d` and threads a feature cache through every `CausalConv3d` (:34-44, :216-239, :114-170, :681-737); a Python
loop of T iterations, each launching the whole decoder on a single frame.

H100 redesign: unrolling the cache logic shows every conv is a causal convolution over the whole frame sequence with
zero padding in front (frame 0 skips `time_conv`, `time_conv` never sees frame 0, `DupUp3D` drops its first
factor_t-1 frames — oracle/wan22vae.py states this and is pinned to the reference's chunked output). A decode is therefore a
pass over [T, H, W, C] channels-last bf16 tensors of as many latent frames as fit in device memory (on an 80 GB H100 a 49-frame
704x1280 video fits in one pass, the 81-frame video does not): `decode` splits the latent into chunks the planner sizes from the
free device memory (one chunk whenever the whole sequence fits) and carries the reference's cache state from chunk to chunk —
the last 2 input frames of every 3-tap causal conv, `time_conv`'s input stream from frame 1 on, DupUp3D's first-chunk drop —
so every partition gives the one-pass result. Inside a chunk:
  * every conv (3x3x3, Conv2d 3x3 = (1,3,3), time_conv = (3,1,1)) is the wgmma implicit GEMM `yb_conv3d_causal` with
    `oob_zero_pad`: the causal zero padding is TMA out-of-bounds fill on the UNPADDED activation — no padded copy, no
    feature cache, no per-frame launches;
  * RMS_norm + SiLU (+ nearest-exact 2x upsample) is one gather pass (`yb_vae_rms_act`);
  * `time_conv`'s two channel groups are written straight into interleaved output frames (`out_t_mul/out_t_add`);
  * the ResidualBlock skip add rides in the conv epilogue; the DupUp3D shortcut is one gather-add;
  * the per-frame single-head attention (d = C) is GEMM calls around a softmax kernel (scale folded into Wq, the v bias
    folded through `proj`); `conv2` has the latent de-normalisation z*std + mean folded into its weights.
The building blocks, the chunk driver and the planner are the shared engine base (yume_b200/wan_vae.py); the decode side here
(`WanVaeDecoder`) is shared with the Wan2.1 decoder (yume_b200/vae21.py).
"""
from __future__ import annotations

import math
import types
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import ops
from ._lib import YumeB200Error
from .dit import quantize_weight_fp8
from .wan_vae import _BF16, _F32, Layer, WanVaeEngine, _rup, chunk_lengths  # noqa: F401  (chunk_lengths: re-exported)

Tensor = torch.Tensor


def decoder_param_shapes(dec_dim: int = 256, z_dim: int = 48, dim_mult: Sequence[int] = (1, 2, 4, 4), num_res_blocks: int = 2,
                         temperal_upsample: Sequence[bool] = (True, True, False)) -> Dict[str, tuple]:
    """State-dict keys / shapes of the decode-side modules of `WanVAE_` (conv2 + Decoder3d, vae2_2.py:640-737)."""
    dims = [dec_dim * u for u in [dim_mult[-1]] + list(dim_mult[::-1])]
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
    conv("decoder.conv1", dims[0], z_dim, 3, 3, 3)
    res("decoder.middle.0", dims[0], dims[0])
    s["decoder.middle.1.norm.gamma"] = (dims[0], 1, 1)
    conv("decoder.middle.1.to_qkv", 3 * dims[0], dims[0], 1, 1)
    conv("decoder.middle.1.proj", dims[0], dims[0], 1, 1)
    res("decoder.middle.2", dims[0], dims[0])
    for i in range(len(dim_mult)):
        p, c = f"decoder.upsamples.{i}.upsamples", dims[i]
        for j in range(num_res_blocks + 1):
            res(f"{p}.{j}", c, dims[i + 1])
            c = dims[i + 1]
        if i != len(dim_mult) - 1:
            q = f"{p}.{num_res_blocks + 1}"
            conv(q + ".resample.1", c, c, 3, 3)
            if i < len(temperal_upsample) and temperal_upsample[i]:
                conv(q + ".time_conv", 2 * c, c, 3, 1, 1)
    s["decoder.head.0.gamma"] = (dims[-1], 1, 1, 1)
    conv("decoder.head.2", 12, dims[-1], 3, 3, 3)
    return s


def decoder_front(d0: int) -> List[Layer]:
    """decoder.conv1 and decoder.middle: the first layers of both Wan decoders."""
    return [Layer("in", "decoder.conv1", 64, d0), Layer("res", "decoder.middle.0", d0, d0), Layer("attn", "decoder.middle.1", d0),
            Layer("res", "decoder.middle.2", d0, d0)]


class WanVaeDecoder(WanVaeEngine):
    """The decode side of both Wan VAEs: z [z_dim, T, H, W] -> f32 [3, 1 + (T-1)*s, SCALE*H, SCALE*W] clamped to [-1, 1], s the
    product of the temporal upsamples. An engine adds its layer list, SCALE and `_write` (the head's output into the video)."""
    SCALE: int

    @property
    def ops(self):
        """This module's op library (see WanVaeEngine)."""
        return ops

    def _repack(self, sd: Dict[str, Tensor], mean: Tensor, std: Tensor) -> None:
        dev = self.device
        # decode-side modules only (`conv2`, `decoder.*`); a live WanVAE_ also carries `encoder.*` and `conv1.*`
        sd = self._pack_side(sd, ("decoder.", "conv2."), "conv2", True)
        # conv2 (1x1x1, z -> z) with the latent de-normalisation folded in: conv2(z*std + mean) = (W diag(std)) z + (W mean + b)
        zd = self.z_dim
        W2 = sd["conv2.weight"].detach().float().reshape(zd, zd)
        w = torch.zeros(_rup(zd, 32), 64, dtype=_F32, device=dev)
        w[:zd, :zd] = W2 * std[None, :]
        b = torch.zeros(_rup(zd, 32), dtype=_F32, device=dev)
        b[:zd] = W2 @ mean + sd["conv2.bias"].detach().float()
        self.lin["conv2"] = (w.to(dev, _BF16).contiguous(), b.to(dev))

    def _input(self, L: Layer, z: Tensor):
        """conv2 (latent de-normalisation folded in) and decoder.conv1 on one chunk of the latent (this rank's band of its rows
        under a row-parallel decode)."""
        zd, T, H, W = z.shape
        if self._rows is not None:
            r0, hs, _ = self._band
            z, H = z[:, :, r0:r0 + hs], hs
        N = T * H * W
        zl = self._new(N, 64)
        ops.nchw_to_nhwc_bf16(z.to(self.device, _F32).reshape(zd, N).contiguous(), zl)
        w2, b2 = self.lin["conv2"]
        dims = (T, H, W)
        if self._rows is not None:                               # conv1's band buffer: each frame's rows, then the halo rows
            x0 = self._hist_buf(L.name, T, H, W, 64, zero=True, halo=True)
            h = x0.shape[0] - T
            for t in range(T):
                ops.gemm(zl[t * H * W:(t + 1) * H * W], w2, b2, x0[h + t, 1:H + 1].view(-1, 64)[:, :w2.shape[0]], ops.YB_EPI_BF16)
            self._halo(x0, T)
            return self._conv(L.name, x0, dims, key=L.name), dims
        x0 = self._hist_buf(L.name, T, H, W, 64, zero=True)
        ops.gemm(zl, w2, b2, x0.view(-1, 64)[x0.shape[0] * H * W - N:, :w2.shape[0]], ops.YB_EPI_BF16)
        return self._conv(L.name, x0, dims, key=L.name), dims

    def _resample(self, L: Layer, x: Tensor, dims):
        """Resample upsample2d / upsample3d (vae2_2.py:73-170) over the frames of this chunk."""
        p, t_up = L.name, L.ft == 2
        T, H, W = dims
        N, C = x.shape
        HW = H * W
        if t_up:
            # time_conv's input stream is every frame but frame 0, which bypasses it ("Rep", :118-121): in the first chunk it
            # starts at the chunk's frame 1 (and may be empty), later chunks feed all their frames behind the carried history
            first, key = self._chunk == 0, p + ".time_conv"
            Ts = T - 1 if first else T
            if Ts > 0:
                src = x[HW:] if first else x
                if C % 64:
                    xin = self._act(src, (Ts, H, W), None, False, key=key)
                elif first:
                    xin = src.view(Ts, H, W, C)
                else:
                    xin = self._hist_buf(key, Ts, H, W, C)
                    xin[self.HIST:].view(Ts * HW, C).copy_(src)
                y = self._new((2 * Ts + (1 if first else 0)) * HW, C)
                if first:
                    y[:HW].copy_(x[:HW])
                for g in (0, 1):                                 # group g of stream frame t -> output frame 2t + g (+1 after frame 0)
                    self._conv(f"{p}.time_conv.{g}", xin, (Ts, H, W), out=y, out_t_mul=2, out_t_add=(1 if first else 0) + g,
                               key=key if g == 0 else None)
                x, T = y, y.shape[0] // HW
            else:
                self._keep(key, self._new(0, H, W, _rup(C, 64)))
        a = self._act(x, (T, H, W), None, False, up=2, conv=p + ".resample.1", halo=True)  # nearest-exact 2x, then Conv2d 3x3
        return self._conv(p + ".resample.1", a, (T, 2 * H, 2 * W)), (T, 2 * H, 2 * W)

    def _head(self, L: Layer, x: Tensor, dims, out: Tensor) -> None:
        y = self._conv(L.name, self._act(x, dims, "decoder.head.0", True, key=L.name, halo=True), dims, epilogue=ops.YB_EPI_F32,
                       key=L.name)
        self._write(y, out, dims)

    def _t_scale(self) -> int:
        return math.prod(L.ft for L in self.layers if L.kind == "up")

    def _out_shape(self, T: int, H: int, W: int) -> Tuple[int, int, int, int]:
        return 3, 1 + (T - 1) * self._t_scale(), self.SCALE * H, self.SCALE * W

    @torch.no_grad()
    def decode(self, z: Tensor) -> Tensor:
        """z [z_dim, T, H, W] -> the clamped video (see the class), in the chunks `plan_chunks` sizes from the free device
        memory. With resume=True a latent that extends the last call's latent runs only its new frames (WanVaeEngine._resumed)."""
        if z.dim() != 4 or z.shape[0] != self.z_dim:
            raise YumeB200Error(f"expected a latent [{self.z_dim}, T, H, W]")
        self._set_band(z.shape[2])                               # checked on every rank before the first collective
        if self.resume:
            T, H, W = z.shape[1:]
            src = z.to(self.device, _F32).contiguous()
            return self._resumed(src, src.data_ptr() != z.data_ptr(), self._out_shape(T, H, W), 1, self._t_scale(),
                                 lambda n: self.chunk_bytes(n, T, H, W), fork=False)
        return self._decode_chunks(z, self.plan_chunks(*z.shape[1:]))

    def _decode_chunks(self, z: Tensor, lengths: Sequence[int]) -> Tensor:
        """Decode the latent in chunks of `lengths` latent frames (any partition of T) into one preallocated video."""
        return self._chunks(z, lengths, self._out_shape(*z.shape[1:]), 1, self._t_scale())

    def _fixed_bytes(self, T: int, H: int, W: int) -> int:
        """The whole result, allocated once before the first chunk."""
        return 4 * math.prod(self._out_shape(T, H, W))

    def plan_chunks(self, T: int, H: int, W: int) -> List[int]:
        """Latent frames per chunk of a decode of a T-frame latent at H x W (see _plan)."""
        return self._plan(T, lambda n: self.chunk_bytes(n, T, H, W))


FP8_CONV_SUFFIXES = (".residual.2", ".residual.6", ".resample.1")


def fp8_conv(name: str, cp: int, cout: int) -> bool:
    """The per-conv rule of Wan22VaeDecoder(precision="fp8"): the res-block convs and the Resample Conv2d run on e4m3 operands
    when the padded input width cp and the packed output width cout are multiples of 128 (whole 128-channel scale groups and
    128-wide output tiles). decoder.conv1 (cp 64), the time_convs (their input is a conv output, not a quantising norm pass),
    the 1x1 shortcuts, the mid attention and the head stay bf16."""
    return name.endswith(FP8_CONV_SUFFIXES) and cp % 128 == 0 and cout % 128 == 0


class Wan22VaeDecoder(WanVaeDecoder):
    """`Wan2_2_VAE.decode` (vae2_2.py:1059-1072): z [z_dim, T, H, W] -> f32 [3, 4(T-1)+1, 16H, 16W].
    precision="fp8" runs the convs `fp8_conv` selects on e4m3 operands (include/yume_b200_fp8_vae.h); "bf16" (the default)
    runs every layer in bf16."""
    SCALE = 16                                                   # three 2x spatial upsamples, then unpatchify 2x
    PRECISIONS = ("bf16", "fp8")

    def __init__(self, sd: Dict[str, Tensor], dec_dim: int = 256, z_dim: int = 48, dim_mult: Sequence[int] = (1, 2, 4, 4),
                 num_res_blocks: int = 2, temperal_upsample: Sequence[bool] = (True, True, False),
                 mean: Optional[Tensor] = None, std: Optional[Tensor] = None, device="cuda", precision: str = "bf16",
                 resume: bool = False, **_):
        self.dims = dims = [dec_dim * u for u in [dim_mult[-1]] + list(dim_mult[::-1])]      # vae2_2.py:656
        layers = decoder_front(dims[0])
        for i in range(len(dim_mult)):                           # Up_ResidualBlock (:461-503)
            p, ci, co = f"decoder.upsamples.{i}.upsamples", dims[i], dims[i + 1]
            up = i != len(dim_mult) - 1
            if up:
                layers.append(Layer("hold", ci=ci))
            layers += [Layer("res", f"{p}.{j}", ci if j == 0 else co, co) for j in range(num_res_blocks + 1)]
            if up:
                ft = 2 if i < len(temperal_upsample) and temperal_upsample[i] else 1
                layers += [Layer("up", f"{p}.{num_res_blocks + 1}", co, co, ft, 2), Layer("dupup", ci=ci, co=co, ft=ft, fs=2)]
        layers.append(Layer("head", "decoder.head.2", dims[-1], _rup(12, 32)))
        super().__init__(sd, z_dim, layers, mean, std, device, precision, resume)

    def _repack(self, sd: Dict[str, Tensor], mean: Tensor, std: Tensor) -> None:
        super()._repack(sd, mean, std)
        self.conv8 = {}
        if self.precision != "fp8":
            return
        for name, (w, b, taps) in list(self.conv.items()):
            if fp8_conv(name, w.shape[1] // math.prod(taps), w.shape[0]):
                wq, sw = quantize_weight_fp8(w)                  # per output channel over taps x cp, from the packed bf16 weight
                self.conv8[name] = (wq, sw, b, taps)
                del self.conv[name]                              # no bf16 copy of a converted weight is kept

    def _write(self, y: Tensor, out: Tensor, dims) -> None:
        if self._rows is not None:
            T, hs, W = dims
            r = 2 * self._row0(hs)
            ops.vae_unpatchify2_clamp_rows(y, out[:, :, r:r + 2 * hs], T, hs, W)
        elif self._one_pass:
            ops.vae_unpatchify2_clamp(y, out, *dims)
        else:
            ops.vae_unpatchify2_clamp_win(y, out, *dims)


def install_wan22_vae(vae, device="cuda", precision: str = "bf16", resume: bool = False):
    """Attach a Wan22VaeDecoder to a live reference `Wan2_2_VAE` wrapper and re-bind its `decode(zs)` (same list-in /
    list-out contract and TypeError behaviour as vae2_2.py:1059-1072). precision: see Wan22VaeDecoder. resume: keep the last
    decode's state so that a latent extending it decodes only its new frames (WanVaeEngine._resumed)."""
    m = vae.model
    sd = dict(m.state_dict())
    dims0 = sd["decoder.conv1.weight"].shape[0]
    dim_mult = list(m.dim_mult)
    mean, inv_std = vae.scale
    eng = Wan22VaeDecoder(sd, dec_dim=dims0 // dim_mult[-1], z_dim=m.z_dim, dim_mult=dim_mult,
                          num_res_blocks=m.num_res_blocks, temperal_upsample=m.temperal_upsample,
                          mean=mean.detach().float().cpu(), std=(1.0 / inv_std.detach().float()).cpu(), device=device,
                          precision=precision, resume=resume)
    vae._yb_decoder = eng

    def decode(self, zs):
        if not isinstance(zs, list):
            import logging
            logging.info(TypeError("zs should be a list"))
            return None
        return [eng.decode(u) for u in zs]

    vae.decode = types.MethodType(decode, vae)
    return vae
