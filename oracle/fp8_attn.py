"""The fp8-attention oracle: WanOracleFp8 with the self-attention that `WanDiT(precision="fp8_attn")` runs on e4m3 operands
(include/yume_b200_fp8_attn.h) — q and k quantise-dequantised per (token, head) 1x128 group, v per (head, 128-key tile), then
an fp64 softmax attention. Cross-attention and everything else are WanOracleFp8 as is. Also holds the torch twins of the V
quantiser, written from the numerics contract alone.

Left out on purpose: the kernel rounds P = 256 p to e4m3 against its running row maximum, which no whole-row oracle can
reproduce; the tolerances of the tests that compare against this oracle absorb it."""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from .fp8 import E4M3, E4M3_MAX, WanOracleFp8, qdq_act
from .wan_dit import rms_norm, rope_apply

Tensor = torch.Tensor


def vt_pi(f: int) -> int:
    """Key (within its 32-key block) stored at position f of that block of vt8."""
    return 16 * (f // 16) + 2 * ((f % 16) // 4) + 8 * ((f % 4) // 2) + (f % 2)


VT_PERM = torch.tensor([vt_pi(f) for f in range(32)])


def quantize_vt(v: Tensor, heads: int) -> Tuple[Tensor, Tensor]:
    """v [Lk, heads*128] (fp32 values of bf16) -> (vt8 e4m3 [heads, 128, Lkp], s_v f32 [heads, Lkp/128]): per (head, 128-key
    tile) amax (NaN ignored), inv = 448 / amax, s_v = amax / 448, both zero when 448 / amax is not finite; keys >= Lk are zeros;
    within each 32-key block position f holds key pi(f)."""
    Lk = v.shape[0]
    Lkp = (Lk + 127) // 128 * 128
    x = torch.zeros(Lkp, heads * 128, dtype=torch.float32, device=v.device)
    x[:Lk] = v.float()
    t = x.reshape(Lkp // 128, 128, heads, 128).permute(2, 0, 1, 3)           # [h, tile, key, d]
    a = t.abs()
    amax = torch.where(torch.isnan(a), torch.zeros_like(a), a).amax(dim=(-2, -1))   # [h, tile]
    inv = torch.full_like(amax, E4M3_MAX) / amax
    scale = amax / torch.full_like(amax, E4M3_MAX)
    bad = ~torch.isfinite(inv)
    inv = torch.where(bad, torch.zeros_like(inv), inv)
    scale = torch.where(bad, torch.zeros_like(scale), scale)
    q = (t * inv[..., None, None]).clamp(-E4M3_MAX, E4M3_MAX).to(E4M3)      # [h, tile, key, d]
    q = q.reshape(heads, Lkp // 32, 32, 128)[:, :, VT_PERM.to(v.device)]                  # position f <- key pi(f)
    return q.reshape(heads, Lkp, 128).transpose(1, 2).contiguous(), scale.contiguous()


def dequantize_vt(vt8: Tensor, s_v: Tensor, Lk: int) -> Tensor:
    """Inverse layout of quantize_vt: f32 V [Lk, heads*128] of the stored e4m3 values times their tile scales."""
    heads, _, Lkp = vt8.shape
    inv_perm = torch.argsort(VT_PERM).to(vt8.device)
    x = vt8.float().transpose(1, 2).reshape(heads, Lkp // 32, 32, 128)[:, :, inv_perm].reshape(heads, Lkp, 128)
    x = x * s_v.repeat_interleave(128, dim=1)[..., None]
    return x.permute(1, 0, 2).reshape(Lkp, heads * 128)[:Lk]


def qdq_qk(x: Tensor) -> Tensor:
    """q or k [L, heads*128]: the 1x128 quantise-dequantise of yb_quant_rows_fp8 (one group = one head of one token)."""
    return qdq_act(x.float())


def attention_fp64(q: Tensor, k: Tensor, v: Tensor, heads: int, scale: Optional[float] = None) -> Tensor:
    """softmax(q k^T scale) v per head in fp64. q [Lq, heads*128], k / v [Lk, heads*128] -> [Lq, heads*128] fp64."""
    Lq, Lk = q.shape[0], k.shape[0]
    scale = 128 ** -0.5 if scale is None else scale
    qh = q.double().reshape(Lq, heads, 128).transpose(0, 1)
    kh = k.double().reshape(Lk, heads, 128).transpose(0, 1)
    vh = v.double().reshape(Lk, heads, 128).transpose(0, 1)
    p = torch.softmax(qh @ kh.transpose(1, 2) * scale, dim=-1)
    return (p @ vh).transpose(0, 1).reshape(Lq, heads * 128)


def attention_fp8_reference(q: Tensor, k: Tensor, v: Tensor, heads: int) -> Tensor:
    """The fp8 self-attention of bf16 q [Lq, C], k / v [Lk, C] on quantise-dequantised operands, fp64 softmax."""
    vt8, s_v = quantize_vt(v, heads)
    return attention_fp64(qdq_qk(q), qdq_qk(k), dequantize_vt(vt8, s_v, k.shape[0]), heads)


class WanOracleFp8Attn(WanOracleFp8):
    """WanOracleFp8 whose self-attention runs on the fp8-quantised q, k and v of precision="fp8_attn"."""

    def self_attn(self, p: str, x: Tensor, freqs_tok: Tensor, k_len: Optional[int] = None) -> Tensor:
        b, s, n, d = x.shape[0], x.shape[1], self.num_heads, self.d
        q = rms_norm(self._lin(p + ".q", x), self.sd[p + ".norm_q.weight"], self.eps).view(b, s, n, d)
        k = rms_norm(self._lin(p + ".k", x), self.sd[p + ".norm_k.weight"], self.eps).view(b, s, n, d)
        v = self._lin(p + ".v", x).view(b, s, n, d)
        q = torch.stack([rope_apply(q[i], freqs_tok) for i in range(b)])
        k = torch.stack([rope_apply(k[i], freqs_tok) for i in range(b)])
        kl = s if k_len is None else k_len
        outs = []
        for i in range(b):   # the engine's operands are bf16 rows, as flash_attention casts them
            qi, ki, vi = (t[i].reshape(s, n * d).to(torch.bfloat16).float() for t in (q, k, v))
            outs.append(attention_fp8_reference(qi, ki[:kl], vi[:kl], n).to(torch.bfloat16).float())
        return self._lin(p + ".o", torch.stack(outs))


__all__ = ["vt_pi", "VT_PERM", "quantize_vt", "dequantize_vt", "qdq_qk", "attention_fp64", "attention_fp8_reference",
           "WanOracleFp8Attn"]
