"""CPU oracle for the Wan2.2 VAE *decode* path (`Wan2_2_VAE.decode`, what the 5B sampler calls) — TEST INFRASTRUCTURE ONLY.

Restates /root/reference/wan23/modules/vae2_2.py in WHOLE-SEQUENCE form. The reference decodes one latent frame per
call of `Decoder3d.forward` and threads a feature cache through every CausalConv3d (`WanVAE_.decode` :831-860,
`ResidualBlock.forward` :216-239, `Resample.forward` :114-170, `Decoder3d.forward` :681-737). Unrolling that cache
logic gives, for every conv, a causal convolution over the full frame sequence with ZERO padding in front (and zero
spatial padding), with two special cases that come from the first chunk:
  * `Resample(upsample3d)`: frame 0 is not passed through `time_conv` ("Rep" marker, :118-121); `time_conv` runs
    over frames 1.. with zero history (it never sees frame 0; :139-147), each input frame yielding two output frames
    (channel groups [0:C] and [C:2C], :151-154);
  * `DupUp3D(first_chunk=True)` drops the first factor_t - 1 duplicated frames (:416-417).
tests/golden/wan22vae_tiny.pt (tools/make_golden_vae22.py) is produced by the reference's own chunked code; the
whole-sequence restatement below must reproduce it — that equivalence is what the H100 path relies on.
State-dict keys are the reference module tree's (`conv2.*`, `decoder.*`).
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


def causal_conv3d(x: Tensor, w: Tensor, b: Tensor) -> Tensor:
    """CausalConv3d (:17-44) over a whole sequence: zero pad W, H symmetrically, T by 2*pad_t in front only."""
    kt, kh, kw = w.shape[2:]
    x = F.pad(x, (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0))
    return F.conv3d(x, w, b)


def rms_norm(x: Tensor, gamma: Tensor) -> Tensor:
    """RMS_norm (:47-61), channel_first, bias=False: F.normalize over channels * sqrt(C) * gamma."""
    C = x.shape[1]
    return F.normalize(x, dim=1) * (C ** 0.5) * gamma.reshape(1, C, *([1] * (x.dim() - 2)))


class Wan22VaeOracle:
    def __init__(self, sd: Dict[str, Tensor], dec_dim=256, z_dim=48, dim_mult=(1, 2, 4, 4), num_res_blocks=2,
                 temperal_upsample=(True, True, False), mean=None, std=None, **_):
        self.sd, self.z_dim, self.nrb = sd, z_dim, num_res_blocks
        self.dims = [dec_dim * u for u in [dim_mult[-1]] + list(dim_mult[::-1])]     # :656
        self.t_up = list(temperal_upsample)
        self.n_up = len(dim_mult)
        self.mean = torch.zeros(z_dim) if mean is None else mean
        self.std = torch.ones(z_dim) if std is None else std

    def _conv(self, p: str, x: Tensor) -> Tensor:
        return causal_conv3d(x, self.sd[p + ".weight"], self.sd[p + ".bias"])

    def res_block(self, p: str, x: Tensor) -> Tensor:
        """ResidualBlock (:195-239): RMS_norm, SiLU, conv, RMS_norm, SiLU, conv + shortcut."""
        h = self._conv(p + ".shortcut", x) if (p + ".shortcut.weight") in self.sd else x
        y = self._conv(p + ".residual.2", F.silu(rms_norm(x, self.sd[p + ".residual.0.gamma"])))
        y = self._conv(p + ".residual.6", F.silu(rms_norm(y, self.sd[p + ".residual.3.gamma"])))
        return y + h

    def attn_block(self, p: str, x: Tensor) -> Tensor:
        """AttentionBlock (:242-283): per-frame single-head attention over h*w tokens."""
        b, c, t, h, w = x.shape
        y = x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w)
        y = rms_norm(y, self.sd[p + ".norm.gamma"])
        qkv = F.conv2d(y, self.sd[p + ".to_qkv.weight"], self.sd[p + ".to_qkv.bias"])
        q, k, v = qkv.reshape(b * t, 1, c * 3, -1).permute(0, 1, 3, 2).contiguous().chunk(3, dim=-1)
        o = F.scaled_dot_product_attention(q, k, v).squeeze(1).permute(0, 2, 1).reshape(b * t, c, h, w)
        o = F.conv2d(o, self.sd[p + ".proj.weight"], self.sd[p + ".proj.bias"])
        return o.reshape(b, t, c, h, w).permute(0, 2, 1, 3, 4) + x

    def resample(self, p: str, x: Tensor, temporal: bool) -> Tensor:
        """Resample upsample2d / upsample3d (:73-170) over the whole sequence."""
        b, c, t, h, w = x.shape
        if temporal and t > 1:
            y = self._conv(p + ".time_conv", x[:, :, 1:])                    # frames 1.., zero history, never frame 0
            y = y.reshape(b, 2, c, t - 1, h, w)
            y = torch.stack((y[:, 0], y[:, 1]), 3).reshape(b, c, 2 * (t - 1), h, w)
            x = torch.cat([x[:, :, :1], y], dim=2)
        t = x.shape[2]
        y = x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w)
        y = F.interpolate(y.float(), scale_factor=(2.0, 2.0), mode="nearest-exact")
        y = F.conv2d(y, self.sd[p + ".resample.1.weight"], self.sd[p + ".resample.1.bias"], padding=1)
        return y.reshape(b, t, c, 2 * h, 2 * w).permute(0, 2, 1, 3, 4)

    @staticmethod
    def dup_up(x: Tensor, out_c: int, ft: int, fs: int) -> Tensor:
        """DupUp3D (:376-418) applied to the whole sequence == chunk 0 with first_chunk=True followed by the rest."""
        b, in_c, t, h, w = x.shape
        rep = out_c * ft * fs * fs // in_c
        y = x.repeat_interleave(rep, dim=1).view(b, out_c, ft, fs, fs, t, h, w)
        y = y.permute(0, 1, 5, 2, 6, 3, 7, 4).contiguous().view(b, out_c, t * ft, h * fs, w * fs)
        return y[:, :, ft - 1:]

    def up_block(self, i: int, x: Tensor) -> Tensor:
        """Up_ResidualBlock (:461-503)."""
        p = f"decoder.upsamples.{i}"
        up_flag = i != self.n_up - 1
        t_up = self.t_up[i] if i < len(self.t_up) else False
        out_c = self.dims[i + 1]
        main = x
        for j in range(self.nrb + 1):
            main = self.res_block(f"{p}.upsamples.{j}", main)
        if up_flag:
            main = self.resample(f"{p}.upsamples.{self.nrb + 1}", main, t_up)
            return main + self.dup_up(x, out_c, 2 if t_up else 1, 2)
        return main

    @torch.no_grad()
    def decode(self, z: Tensor) -> Tensor:
        """Wan2_2_VAE.decode (:1059-1072) for one latent z [z_dim, T, H, W] -> [3, 4(T-1)+1, 16H, 16W] in [-1, 1]."""
        z = z.unsqueeze(0).float()
        z = z * self.std.view(1, -1, 1, 1, 1) + self.mean.view(1, -1, 1, 1, 1)   # z / (1/std) + mean (:833-838)
        x = self._conv("conv2", z)
        x = self._conv("decoder.conv1", x)
        x = self.res_block("decoder.middle.0", x)
        x = self.attn_block("decoder.middle.1", x)
        x = self.res_block("decoder.middle.2", x)
        for i in range(self.n_up):
            x = self.up_block(i, x)
        x = self._conv("decoder.head.2", F.silu(rms_norm(x, self.sd["decoder.head.0.gamma"])))
        b, c12, f, h, w = x.shape                                            # unpatchify(patch 2) (:305-319)
        x = x.view(b, 3, 2, 2, f, h, w).permute(0, 1, 4, 5, 3, 6, 2).reshape(b, 3, f, h * 2, w * 2)
        return x.float().clamp_(-1, 1).squeeze(0)


# ------------------------------------------------------------------------------------------------------------
def param_shapes(dec_dim=256, z_dim=48, dim_mult=(1, 2, 4, 4), num_res_blocks=2, temperal_upsample=(True, True, False)):
    dims = [dec_dim * u for u in [dim_mult[-1]] + list(dim_mult[::-1])]
    s: Dict[str, tuple] = {"conv2.weight": (z_dim, z_dim, 1, 1, 1), "conv2.bias": (z_dim,),
                           "decoder.conv1.weight": (dims[0], z_dim, 3, 3, 3), "decoder.conv1.bias": (dims[0],)}

    def res(p, ci, co):
        s[p + ".residual.0.gamma"] = (ci, 1, 1, 1)
        s[p + ".residual.2.weight"], s[p + ".residual.2.bias"] = (co, ci, 3, 3, 3), (co,)
        s[p + ".residual.3.gamma"] = (co, 1, 1, 1)
        s[p + ".residual.6.weight"], s[p + ".residual.6.bias"] = (co, co, 3, 3, 3), (co,)
        if ci != co:
            s[p + ".shortcut.weight"], s[p + ".shortcut.bias"] = (co, ci, 1, 1, 1), (co,)

    res("decoder.middle.0", dims[0], dims[0])
    s["decoder.middle.1.norm.gamma"] = (dims[0], 1, 1)
    s["decoder.middle.1.to_qkv.weight"], s["decoder.middle.1.to_qkv.bias"] = (3 * dims[0], dims[0], 1, 1), (3 * dims[0],)
    s["decoder.middle.1.proj.weight"], s["decoder.middle.1.proj.bias"] = (dims[0], dims[0], 1, 1), (dims[0],)
    res("decoder.middle.2", dims[0], dims[0])
    n = len(dim_mult)
    for i, (ci, co) in enumerate(zip(dims[:-1], dims[1:])):
        p = f"decoder.upsamples.{i}.upsamples"
        c = ci
        for j in range(num_res_blocks + 1):
            res(f"{p}.{j}", c, co)
            c = co
        if i != n - 1:
            q = f"{p}.{num_res_blocks + 1}"
            s[q + ".resample.1.weight"], s[q + ".resample.1.bias"] = (co, co, 3, 3), (co,)
            if i < len(temperal_upsample) and temperal_upsample[i]:
                s[q + ".time_conv.weight"], s[q + ".time_conv.bias"] = (2 * co, co, 3, 1, 1), (2 * co,)
    s["decoder.head.0.gamma"] = (dims[-1], 1, 1, 1)
    s["decoder.head.2.weight"], s["decoder.head.2.bias"] = (12, dims[-1], 3, 3, 3), (12,)
    return s


def make_state_dict(seed: int, **cfg) -> Dict[str, Tensor]:
    sd = {}
    for idx, (name, shape) in enumerate(param_shapes(**cfg).items()):
        g = torch.Generator().manual_seed(seed * 6151 + idx)
        t = torch.randn(shape, generator=g)
        if name.endswith(".bias"):
            t = 0.05 * t
        elif name.endswith(".gamma"):
            t = 1.0 + 0.1 * t
        else:
            fan_in = 1
            for d in shape[1:]:
                fan_in *= d
            t = t * (0.8 / fan_in ** 0.5)   # keeps most outputs inside (-1, 1) so the final clamp hides little
        sd[name] = t.to(torch.bfloat16).float()
    return sd
