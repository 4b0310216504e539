"""The fp8-qdq oracle of `Wan22VaeDecoder(precision="fp8")` — TEST INFRASTRUCTURE ONLY: Wan22VaeOracle with every conv the engine
converts (the res-block convs and the Resample Conv2d whose padded input width and output width are multiples of 128: the
engine's rule, restated here) run on quantised-dequantised operands (include/yume_b200_fp8_vae.h):
  * the weight as the engine packs it (bf16), quantised per output channel over all taps x channels, then dequantised;
  * the conv input rounded to bf16 (what yb_vae_rms_act would store), quantised per voxel and 128-channel group (channels
    padded with zeros to a multiple of 128), then dequantised.
The conv itself stays the fp32 causal conv of the base oracle. Every other layer is Wan22VaeOracle as is."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .fp8 import dequantize_act, quantize_act, quantize_weight
from .wan22vae import Wan22VaeOracle, causal_conv3d

Tensor = torch.Tensor
FP8_CONV_SUFFIXES = (".residual.2", ".residual.6", ".resample.1")


def _rup(v: int, m: int) -> int:
    return (v + m - 1) // m * m


def converted(name: str, ci: int, co: int) -> bool:
    """The engine's per-conv rule (yume_b200.vae22.fp8_conv) in terms of the module's channel counts."""
    return name.endswith(FP8_CONV_SUFFIXES) and _rup(ci, 64) % 128 == 0 and _rup(co, 32) % 128 == 0


def qdq_weight(w: Tensor) -> Tensor:
    """w [co, ci, *k] -> the dequantised e4m3 weight of its bf16 rounding (one scale per output channel)."""
    co = w.shape[0]
    wq, sw = quantize_weight(w.to(torch.bfloat16).float().reshape(co, -1))
    return (wq.float() * sw[:, None]).reshape(w.shape)


def qdq_channels(x: Tensor) -> Tensor:
    """x [1, C, *spatial] -> the dequantised 1x128 e4m3 quantisation of its bf16 rounding, per voxel over the channels."""
    C = x.shape[1]
    v = x[0].movedim(0, -1)
    rows = v.reshape(-1, C).to(torch.bfloat16).float()
    rows = F.pad(rows, (0, _rup(C, 128) - C))
    rows = dequantize_act(*quantize_act(rows))[:, :C]
    return rows.reshape(v.shape).movedim(-1, 0)[None]


class Wan22VaeOracleFp8(Wan22VaeOracle):
    def _fp8(self, p: str) -> bool:
        w = self.sd.get(p + ".weight")
        return w is not None and converted(p, w.shape[1], w.shape[0])

    def _conv(self, p: str, x: Tensor) -> Tensor:
        if not self._fp8(p):
            return super()._conv(p, x)
        return causal_conv3d(qdq_channels(x), qdq_weight(self.sd[p + ".weight"]), self.sd[p + ".bias"])

    def resample(self, p: str, x: Tensor, temporal: bool) -> Tensor:
        """Wan22VaeOracle.resample with the Conv2d on quantised-dequantised operands."""
        q = p + ".resample.1"
        if not self._fp8(q):
            return super().resample(p, x, temporal)
        b, c, t, h, w = x.shape
        if temporal and t > 1:
            y = super()._conv(p + ".time_conv", x[:, :, 1:])
            y = y.reshape(b, 2, c, t - 1, h, w)
            y = torch.stack((y[:, 0], y[:, 1]), 3).reshape(b, c, 2 * (t - 1), h, w)
            x = torch.cat([x[:, :, :1], y], dim=2)
        t = x.shape[2]
        y = x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w)
        y = F.interpolate(y.float(), scale_factor=(2.0, 2.0), mode="nearest-exact")
        y = qdq_channels(y.transpose(0, 1)[None])[0].transpose(0, 1)
        y = F.conv2d(y, qdq_weight(self.sd[q + ".weight"]), self.sd[q + ".bias"], padding=1)
        return y.reshape(b, t, c, 2 * h, 2 * w).permute(0, 2, 1, 3, 4)


__all__ = ["Wan22VaeOracleFp8", "converted", "qdq_weight", "qdq_channels", "FP8_CONV_SUFFIXES"]
