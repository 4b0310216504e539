"""The fp8-qdq oracle: WanOracle with the six block linears that `WanDiT(precision="fp8")` converts (q, k, v, o, cross q, cross o,
ffn.0, ffn.2; q|k|v as one fused matrix quantises per output channel exactly like q, k, v apart) replaced by the same weight and
1x128 activation quantise-dequantise (include/yume_b200_fp8.h), followed by an fp64 linear. Everything else is WanOracle as is.
Also holds the torch twins of the two quantisers, written from the numerics contract alone."""
from __future__ import annotations

from typing import Tuple

import torch

from .wan_dit import WanOracle

Tensor = torch.Tensor
E4M3 = torch.float8_e4m3fn
E4M3_MAX = 448.0
FP8_LINEARS = (".self_attn.q", ".self_attn.k", ".self_attn.v", ".self_attn.o", ".cross_attn.q", ".cross_attn.o", ".ffn.0",
               ".ffn.2")


def quantize_weight(w: Tensor) -> Tuple[Tensor, Tensor]:
    """Per output channel: s_w = amax / 448, Wq = e4m3(clamp(W * (448 / amax), +-448)); zero rows -> s_w = 0, Wq = 0."""
    w = w.float()
    amax = w.abs().amax(dim=1)
    mult = torch.where(amax > 0, E4M3_MAX / amax, torch.zeros_like(amax))
    return (w * mult[:, None]).clamp(-E4M3_MAX, E4M3_MAX).to(E4M3), amax / torch.full_like(amax, E4M3_MAX)


def quantize_act(x: Tensor) -> Tuple[Tensor, Tensor]:
    """1x128 groups of x [M, K] (fp32 values): amax over the group with NaN ignored, inv = 448 / amax, scale = amax / 448, both
    zero when 448 / amax is not finite; q = (x * inv).clamp(-448, 448).to(e4m3). Returns (q [M, K], scale f32 [K / 128, M])."""
    M, K = x.shape
    g = x.float().reshape(M, K // 128, 128)
    a = g.abs()
    amax = torch.where(torch.isnan(a), torch.zeros_like(a), a).amax(dim=-1)
    inv = torch.full_like(amax, E4M3_MAX) / amax
    scale = amax / torch.full_like(amax, E4M3_MAX)     # tensor / tensor: IEEE division (torch divides by a scalar as a product)
    bad = ~torch.isfinite(inv)
    inv = torch.where(bad, torch.zeros_like(inv), inv)
    scale = torch.where(bad, torch.zeros_like(scale), scale)
    q = (g * inv[..., None]).clamp(-E4M3_MAX, E4M3_MAX).to(E4M3)
    return q.reshape(M, K), scale.t().contiguous()


def dequantize_act(q: Tensor, scale: Tensor) -> Tensor:
    """q e4m3 [M, K], scale [K / 128, >= M] -> f32 [M, K]."""
    M, K = q.shape
    return q.float() * scale[:, :M].t().repeat_interleave(128, dim=1)


def qdq_act(x: Tensor) -> Tensor:
    return dequantize_act(*quantize_act(x))


class WanOracleFp8(WanOracle):
    """WanOracle with the converted block linears on fp8-quantised operands (quantise-dequantise, then an fp64 linear)."""

    def _lin(self, name: str, x: Tensor) -> Tensor:
        if not (name.startswith("blocks.") and name.endswith(FP8_LINEARS)):
            return super()._lin(name, x)
        wq, sw = quantize_weight(self.sd[name + ".weight"])
        w = wq.double() * sw.double()[:, None]
        shape = x.shape
        xd = qdq_act(x.reshape(-1, shape[-1])).double()
        y = xd @ w.t()
        b = self.sd.get(name + ".bias")
        if b is not None:
            y = y + b.double()
        return y.float().reshape(*shape[:-1], w.shape[0])


__all__ = ["quantize_weight", "quantize_act", "dequantize_act", "qdq_act", "WanOracleFp8", "E4M3_MAX", "FP8_LINEARS"]
