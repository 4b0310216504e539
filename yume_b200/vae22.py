"""H100 decode path of the Wan2.2 VAE (`Wan2_2_VAE.decode`) — the VAE the Yume-5B sampler actually calls
(wan23/textimage2video.py:124; fastvideo/sample/sample_5b.py:1051-1052). SURVEY.md §8(f) "next" row, rank 1.

Reference: /root/reference/wan23/modules/vae2_2.py — `WanVAE_.decode` (:831-860) feeds ONE latent frame at a time through
`Decoder3d` and threads a feature cache through every `CausalConv3d` (:34-44, :216-239, :114-170, :681-737); a Python
loop of T iterations, each launching the whole decoder on a single frame.

H100 redesign: unrolling the cache logic shows every conv is a causal convolution over the whole frame sequence with
zero padding in front (frame 0 skips `time_conv`, `time_conv` never sees frame 0, `DupUp3D` drops its first
factor_t-1 frames — oracle/wan22vae.py states this and is pinned to the reference's chunked output). The decode is
therefore ONE pass over [T, H, W, C] channels-last bf16 tensors; the whole sequence must fit in device memory (on an 80 GB H100
a 49-frame 704x1280 chunk does, the 81-frame video does not):
  * every conv (3x3x3, Conv2d 3x3 = (1,3,3), time_conv = (3,1,1)) is the wgmma implicit GEMM `yb_conv3d_causal` with
    `oob_zero_pad`: the causal zero padding is TMA out-of-bounds fill on the UNPADDED activation — no padded copy, no
    feature cache, no per-frame launches;
  * RMS_norm + SiLU (+ nearest-exact 2x upsample) is one gather pass (`yb_vae_rms_act`);
  * `time_conv`'s two channel groups are written straight into interleaved output frames (`out_t_mul/out_t_add`);
  * the ResidualBlock skip add rides in the conv epilogue; the DupUp3D shortcut is one gather-add;
  * the per-frame single-head attention (d = C) is GEMM calls around a softmax kernel (scale folded into Wq, the v bias
    folded through `proj`); `conv2` has the latent de-normalisation z*std + mean folded into its weights.
"""
from __future__ import annotations

import types
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import ops
from ._lib import YumeB200Error

Tensor = torch.Tensor
_BF16, _F32 = torch.bfloat16, torch.float32


def _rup(v: int, m: int) -> int:
    return (v + m - 1) // m * m


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


class Wan22VaeDecoder:
    def __init__(self, sd: Dict[str, Tensor], dec_dim: int = 256, z_dim: int = 48, dim_mult: Sequence[int] = (1, 2, 4, 4),
                 num_res_blocks: int = 2, temperal_upsample: Sequence[bool] = (True, True, False),
                 mean: Optional[Tensor] = None, std: Optional[Tensor] = None, device="cuda", **_):
        self.device = torch.device(device)
        self.z_dim, self.nrb = z_dim, num_res_blocks
        self.dims = [dec_dim * u for u in [dim_mult[-1]] + list(dim_mult[::-1])]      # vae2_2.py:656
        self.t_up, self.n_up = list(temperal_upsample), len(dim_mult)
        mean = torch.zeros(z_dim) if mean is None else mean
        std = torch.ones(z_dim) if std is None else std
        self._repack(sd, mean.detach().to(self.device, _F32), std.detach().to(self.device, _F32))

    # ---- weights -------------------------------------------------------------------------------------------
    def _pack_side(self, sd: Dict[str, Tensor], prefixes: Tuple[str, ...], latent_conv: str, attn: str, width: int,
                   split_time_conv: bool) -> Dict[str, Tensor]:
        """Re-pack one side of a `WanVAE_` state dict (decode: `decoder.*` + `conv2`; encode: `encoder.*` + `conv1`): 3-D / 2-D
        convs as [cop, taps*cp] bf16 GEMM weights, 1x1x1 shortcuts as plain matrices, gammas flat, the mid attention with the
        softmax scale folded into q and the v bias folded through `proj`. Returns the fp32 device copy of that side."""
        dev = self.device
        sd = {k: v.detach().to(dev, _F32) for k, v in sd.items() if k.startswith(prefixes)}
        self.conv: Dict[str, Tuple[Tensor, Tensor, tuple]] = {}    # name -> (w bf16 [cop, taps*cp], bias f32 [cop], taps)
        self.lin: Dict[str, Tuple[Tensor, Tensor]] = {}            # 1x1x1 convs as plain GEMM weights
        self.gamma: Dict[str, Tensor] = {}

        def pack_conv(name: str, w: Tensor, b: Tensor) -> None:
            w = w.detach().float()
            if w.dim() == 4:                                        # Conv2d [co, ci, kh, kw] -> taps (1, kh, kw)
                w = w.unsqueeze(2)
            co, ci, kt, kh, kw = w.shape
            cop, cp = _rup(co, 32), _rup(ci, 64)
            wt = torch.zeros(cop, kt * kh * kw, cp, dtype=_F32, device=dev)
            wt[:co, :, :ci] = w.permute(0, 2, 3, 4, 1).reshape(co, kt * kh * kw, ci)
            bp = torch.zeros(cop, dtype=_F32, device=dev)
            bp[:co] = b.detach().float()
            self.conv[name] = (wt.reshape(cop, -1).to(dev, _BF16).contiguous(), bp.to(dev), (kt, kh, kw))

        latent_w = latent_conv + ".weight"
        for k, v in sd.items():
            if k.endswith(".gamma"):
                self.gamma[k[:-6]] = v.detach().to(dev, _F32).reshape(-1).contiguous()
            elif k.endswith(".weight") and v.dim() == 5 and tuple(v.shape[2:]) == (1, 1, 1) and k != latent_w:
                name = k[:-7]                                       # ResidualBlock.shortcut: plain GEMM
                co, ci = v.shape[:2]
                w = torch.zeros(_rup(co, 32), _rup(ci, 8), dtype=_F32, device=dev)
                w[:co, :ci] = v.detach().float().reshape(co, ci)
                b = torch.zeros(_rup(co, 32), dtype=_F32, device=dev)
                b[:co] = sd[name + ".bias"].detach().float()
                self.lin[name] = (w.to(dev, _BF16).contiguous(), b.to(dev))
            elif k.endswith(".time_conv.weight") and split_time_conv:
                name = k[:-7]
                C2 = v.shape[0]
                for g in (0, 1):                                    # the two channel groups become two output frames
                    pack_conv(f"{name}.{g}", v[g * C2 // 2:(g + 1) * C2 // 2], sd[name + ".bias"][g * C2 // 2:(g + 1) * C2 // 2])
            elif k.endswith(".weight") and v.dim() in (4, 5) and "to_qkv" not in k and ".proj." not in k and k != latent_w:
                pack_conv(k[:-7], v, sd[k[:-7] + ".bias"])
        # attention: scale folded into q; v bias folded through proj (softmax rows sum to 1)
        C = width
        Wqkv = sd[attn + ".to_qkv.weight"].detach().float().reshape(3 * C, C)
        bqkv = sd[attn + ".to_qkv.bias"].detach().float()
        Wo = sd[attn + ".proj.weight"].detach().float().reshape(C, C)
        scale = C ** -0.5
        self.att = dict(wq=(Wqkv[:C] * scale).to(dev, _BF16).contiguous(), bq=(bqkv[:C] * scale).to(dev),
                        wk=Wqkv[C:2 * C].to(dev, _BF16).contiguous(), bk=bqkv[C:2 * C].to(dev).contiguous(),
                        wv=Wqkv[2 * C:].to(dev, _BF16).contiguous(),
                        wo=Wo.to(dev, _BF16).contiguous(),
                        bo=(sd[attn + ".proj.bias"].detach().float() + Wo @ bqkv[2 * C:]).to(dev).contiguous())
        return sd

    def _repack(self, sd: Dict[str, Tensor], mean: Tensor, std: Tensor) -> None:
        dev = self.device
        # decode-side modules only (`conv2`, `decoder.*`); a live WanVAE_ also carries `encoder.*` and `conv1.*`
        sd = self._pack_side(sd, ("decoder.", "conv2."), "conv2", "decoder.middle.1", self.dims[0], True)
        # conv2 (1x1x1, z -> z) with the latent de-normalisation folded in: conv2(z*std + mean) = (W diag(std)) z + (W mean + b)
        zd = self.z_dim
        W2 = sd["conv2.weight"].detach().float().reshape(zd, zd)
        w = torch.zeros(_rup(zd, 32), 64, dtype=_F32, device=dev)
        w[:zd, :zd] = W2 * std[None, :]
        b = torch.zeros(_rup(zd, 32), dtype=_F32, device=dev)
        b[:zd] = W2 @ mean + sd["conv2.bias"].detach().float()
        self.lin["conv2"] = (w.to(dev, _BF16).contiguous(), b.to(dev))

    # ---- building blocks -----------------------------------------------------------------------------------
    def _new(self, *shape, dtype=_BF16) -> Tensor:
        return torch.empty(*shape, device=self.device, dtype=dtype)

    def _conv(self, name: str, a: Tensor, dims, epilogue=None, res: Optional[Tensor] = None, out: Optional[Tensor] = None,
              out_t_mul: int = 1, out_t_add: int = 0, stride_t: int = 1, stride_hw: int = 1) -> Tensor:
        """a bf16 [T, H, W, Cp] (unpadded, dense) -> [To*Ho*Wo (or interleaved frames), cop]."""
        w, b, taps = self.conv[name]
        T, H, W = dims
        if epilogue is None:
            epilogue = ops.YB_EPI_RES_BF16 if res is not None else ops.YB_EPI_BF16
        if out is None:
            To, Ho, Wo = ops.conv_out_dims(T, H, W, taps, stride_t, stride_hw)
            out = self._new(To * Ho * Wo, w.shape[0], dtype=_F32 if epilogue == ops.YB_EPI_F32 else _BF16)
        ops.conv3d_causal(a, w, b, out, T, H, W, epilogue, res, taps=taps, oob_zero_pad=True, out_t_mul=out_t_mul,
                          out_t_add=out_t_add, stride_t=stride_t, stride_hw=stride_hw)
        return out

    def _act(self, x: Tensor, dims, gamma: Optional[str], silu: bool, up: int = 1) -> Tensor:
        T, H, W = dims
        out = self._new(T, H * up, W * up, _rup(x.shape[1], 64))
        ops.vae_rms_act(x, dims, out, self.gamma[gamma] if gamma else None, up, silu)
        return out

    def _res_block(self, p: str, x: Tensor, dims) -> Tensor:
        """ResidualBlock (:195-239)."""
        y = self._conv(p + ".residual.2", self._act(x, dims, p + ".residual.0", True), dims)
        res = x
        if (p + ".shortcut") in self.lin:
            w, b = self.lin[p + ".shortcut"]
            res = self._new(x.shape[0], w.shape[0])
            ops.gemm(x, w, b, res, ops.YB_EPI_BF16)
        return self._conv(p + ".residual.6", self._act(y, dims, p + ".residual.3", True), dims, res=res)

    def _attention(self, p: str, x: Tensor, dims) -> Tensor:
        """AttentionBlock (:242-283): per-frame single-head attention over H*W tokens, d = C."""
        T, H, W = dims
        N, C = x.shape
        HW = H * W
        Lf = _rup(HW, 32)                                        # per-frame key count padded for the GEMM tile
        a = self.att
        S, P, o = self._new(HW, Lf, dtype=_F32), self._new(HW, Lf), self._new(N, C)
        if HW % 8:
            # frames whose H*W rows are not 16-byte multiples in the transposed V (tiny latents only): every frame gets its own
            # zero-padded Lf-row slot, so per-frame slices of q, k and v^T start on aligned addresses
            tmp = self._new(T, H, W, C)
            ops.vae_rms_act(x, dims, tmp, self.gamma[p + ".norm"], 1, False)
            hn = torch.zeros(T * Lf + 32, C, device=self.device, dtype=_BF16)
            hn[:T * Lf].view(T, Lf, C)[:, :HW].copy_(tmp.view(T, HW, C))
            q, k, vT = self._new(T * Lf, C), self._new(T * Lf, C), self._new(C, T * Lf + 32)
            ops.gemm(hn[:T * Lf], a["wq"], a["bq"], q, ops.YB_EPI_BF16)
            ops.gemm(hn[:T * Lf], a["wk"], a["bk"], k, ops.YB_EPI_BF16)
            ops.gemm(a["wv"], hn, None, vT, ops.YB_EPI_BF16)
            for f in range(T):
                ops.gemm(q[f * Lf:f * Lf + HW], k[f * Lf:(f + 1) * Lf], None, S, ops.YB_EPI_F32)
                ops.masked_softmax(S, P, HW, HW)
                ops.gemm(P, vT[:, f * Lf:(f + 1) * Lf], None, o[f * HW:(f + 1) * HW], ops.YB_EPI_BF16)
        else:
            Next = _rup(N, 32) + 32
            hn = torch.zeros(Next, C, device=self.device, dtype=_BF16)
            ops.vae_rms_act(x, dims, hn[:N].view(T, H, W, C), self.gamma[p + ".norm"], 1, False)
            q, k = self._new(N, C), torch.zeros(Next, C, device=self.device, dtype=_BF16)
            ops.gemm(hn[:N], a["wq"], a["bq"], q, ops.YB_EPI_BF16)
            ops.gemm(hn[:N], a["wk"], a["bk"], k[:N], ops.YB_EPI_BF16)
            vT = self._new(C, Next)
            ops.gemm(a["wv"], hn, None, vT, ops.YB_EPI_BF16)
            for f in range(T):
                ops.gemm(q[f * HW:(f + 1) * HW], k[f * HW:f * HW + Lf], None, S, ops.YB_EPI_F32)
                ops.masked_softmax(S, P, HW, HW)                 # keys >= HW (padding / next frame) get probability 0
                ops.gemm(P, vT[:, f * HW:f * HW + Lf], None, o[f * HW:(f + 1) * HW], ops.YB_EPI_BF16)
        out = self._new(N, C)
        ops.gemm(o, a["wo"], a["bo"], out, ops.YB_EPI_RES_BF16, res=x)
        return out

    def _resample(self, p: str, x: Tensor, dims, t_up: bool):
        """Resample upsample2d / upsample3d (:73-170) over the whole sequence."""
        T, H, W = dims
        N, C = x.shape
        HW = H * W
        if t_up and T > 1:
            xin = x[HW:].view(T - 1, H, W, C) if C % 64 == 0 else self._act(x[HW:], (T - 1, H, W), None, False)
            y = self._new((2 * T - 1) * HW, C)
            y[:HW].copy_(x[:HW])                                 # frame 0 bypasses time_conv ("Rep", :118-121)
            for g in (0, 1):                                     # group g of input frame t -> output frame 1 + 2(t-1) + g
                self._conv(f"{p}.time_conv.{g}", xin, (T - 1, H, W), out=y, out_t_mul=2, out_t_add=1 + g)
            x, T = y, 2 * T - 1
        a = self._act(x, (T, H, W), None, False, up=2)           # nearest-exact 2x, then Conv2d 3x3 (zero pad 1)
        return self._conv(p + ".resample.1", a, (T, 2 * H, 2 * W)), (T, 2 * H, 2 * W)

    def _up_block(self, i: int, x: Tensor, dims):
        """Up_ResidualBlock (:461-503)."""
        p = f"decoder.upsamples.{i}.upsamples"
        up_flag = i != self.n_up - 1
        t_up = self.t_up[i] if i < len(self.t_up) else False
        x_in, dims_in, ci, co = x, dims, self.dims[i], self.dims[i + 1]
        for j in range(self.nrb + 1):
            x = self._res_block(f"{p}.{j}", x, dims)
        if up_flag:
            x, dims = self._resample(f"{p}.{self.nrb + 1}", x, dims, t_up)
            ops.vae_dupup_add(x, x_in, dims_in, ci, co, 2 if t_up else 1, 2)
        return x, dims

    @torch.no_grad()
    def decode(self, z: Tensor) -> Tensor:
        """z [z_dim, T, H, W] -> f32 [3, 4(T-1)+1, 16H, 16W] clamped to [-1, 1] (Wan2_2_VAE.decode :1059-1072)."""
        if z.dim() != 4 or z.shape[0] != self.z_dim:
            raise YumeB200Error(f"expected a latent [{self.z_dim}, T, H, W]")
        zd, T, H, W = z.shape
        N = T * H * W
        zl = self._new(N, 64)
        ops.nchw_to_nhwc_bf16(z.to(self.device, _F32).reshape(zd, N).contiguous(), zl)
        w2, b2 = self.lin["conv2"]
        x0 = torch.zeros(N, 64, device=self.device, dtype=_BF16)
        ops.gemm(zl, w2, b2, x0[:, :w2.shape[0]], ops.YB_EPI_BF16)
        dims = (T, H, W)
        x = self._conv("decoder.conv1", x0.view(T, H, W, 64), dims)
        x = self._res_block("decoder.middle.0", x, dims)
        x = self._attention("decoder.middle.1", x, dims)
        x = self._res_block("decoder.middle.2", x, dims)
        for i in range(self.n_up):
            x, dims = self._up_block(i, x, dims)
        y = self._conv("decoder.head.2", self._act(x, dims, "decoder.head.0", True), dims, epilogue=ops.YB_EPI_F32)
        out = self._new(3, dims[0], 2 * dims[1], 2 * dims[2], dtype=_F32)
        ops.vae_unpatchify2_clamp(y, out, *dims)
        return out


def install_wan22_vae(vae, device="cuda"):
    """Attach a Wan22VaeDecoder to a live reference `Wan2_2_VAE` wrapper and re-bind its `decode(zs)` (same list-in /
    list-out contract and TypeError behaviour as vae2_2.py:1059-1072)."""
    m = vae.model
    sd = dict(m.state_dict())
    dims0 = sd["decoder.conv1.weight"].shape[0]
    dim_mult = list(m.dim_mult)
    mean, inv_std = vae.scale
    eng = Wan22VaeDecoder(sd, dec_dim=dims0 // dim_mult[-1], z_dim=m.z_dim, dim_mult=dim_mult,
                          num_res_blocks=m.num_res_blocks, temperal_upsample=m.temperal_upsample,
                          mean=mean.detach().float().cpu(), std=(1.0 / inv_std.detach().float()).cpu(), device=device)
    vae._yb_decoder = eng

    def decode(self, zs):
        if not isinstance(zs, list):
            import logging
            logging.info(TypeError("zs should be a list"))
            return None
        return [eng.decode(u) for u in zs]

    vae.decode = types.MethodType(decode, vae)
    return vae
