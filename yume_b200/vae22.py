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
    # chunk-streaming state of the running decode: chunk index, whether another chunk follows, carried conv input frames
    _chunk, _more, _carry = 0, False, None
    HIST = 2                     # carried frames of a 3-tap causal conv (the reference's CACHE_T)
    MEM_MARGIN = 2 << 30         # bytes of free device memory the chunk planner leaves unused

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

    def _hist_buf(self, key: Optional[str], T: int, H: int, W: int, Cp: int, zero: bool = False, n: int = 0) -> Tensor:
        """Input buffer [h + T, H, W, Cp] of a conv whose input stream is `key`: after the first chunk its first h frames (n, or
        HIST when n is 0) are the frames carried from the previous chunk and the producer writes the T new frames behind them."""
        h = (n or self.HIST) if (key is not None and self._chunk > 0) else 0
        buf = torch.zeros(h + T, H, W, Cp, device=self.device, dtype=_BF16) if zero else self._new(h + T, H, W, Cp)
        if h:
            buf[:h].copy_(self._carry[key])
        return buf

    def _keep(self, key: str, frames: Tensor, n: int = 0) -> None:
        """Carry the last n (0: HIST) frames of the input stream `key` into the next chunk (zero frames in front where the stream
        is shorter: the causal zero padding)."""
        if not self._more:
            return
        n = n or self.HIST
        if frames.shape[0] >= n:
            self._carry[key] = frames[frames.shape[0] - n:].clone()
        else:
            c = torch.zeros(n, *frames.shape[1:], device=self.device, dtype=_BF16)
            c[n - frames.shape[0]:].copy_(frames)
            self._carry[key] = c

    def _conv(self, name: str, a: Tensor, dims, epilogue=None, res: Optional[Tensor] = None, out: Optional[Tensor] = None,
              out_t_mul: int = 1, out_t_add: int = 0, stride_t: int = 1, stride_hw: int = 1, key: Optional[str] = None) -> Tensor:
        """a bf16 [h + T, H, W, Cp] (unpadded, dense; h carried frames in front, see _hist_buf) -> [To*Ho*Wo (or interleaved
        frames), cop]. `key`: the input stream whose last frames the next chunk needs."""
        w, b, taps = self.conv[name]
        T, H, W = dims
        h = a.shape[0] - T
        if key is not None:                                      # a stride-2 time_conv carries one frame (vae2_2.py:158-170)
            self._keep(key, a, 1 if stride_t > 1 else self.HIST)
        if epilogue is None:
            epilogue = ops.YB_EPI_RES_BF16 if res is not None else ops.YB_EPI_BF16
        if out is None:
            To, Ho, Wo = ops.conv_out_dims(T, H, W, taps, stride_t, stride_hw)
            out = self._new(To * Ho * Wo, w.shape[0], dtype=_F32 if epilogue == ops.YB_EPI_F32 else _BF16)
        if h:
            ops.conv3d_causal_hist(a, w, b, out, T, H, W, h, epilogue, res, taps=taps, out_t_mul=out_t_mul,
                                   out_t_add=out_t_add, stride_t=stride_t, stride_hw=stride_hw)
        else:
            ops.conv3d_causal(a, w, b, out, T, H, W, epilogue, res, taps=taps, oob_zero_pad=True, out_t_mul=out_t_mul,
                              out_t_add=out_t_add, stride_t=stride_t, stride_hw=stride_hw)
        return out

    def _act(self, x: Tensor, dims, gamma: Optional[str], silu: bool, up: int = 1, key: Optional[str] = None,
             n: int = 0) -> Tensor:
        T, H, W = dims
        out = self._hist_buf(key, T, H * up, W * up, _rup(x.shape[1], 64), n=n)
        ops.vae_rms_act(x, dims, out[out.shape[0] - T:], self.gamma[gamma] if gamma else None, up, silu)
        return out

    def _res_block(self, p: str, x: Tensor, dims) -> Tensor:
        """ResidualBlock (:195-239)."""
        c1, c2 = p + ".residual.2", p + ".residual.6"
        y = self._conv(c1, self._act(x, dims, p + ".residual.0", True, key=c1), dims, key=c1)
        res = x
        if (p + ".shortcut") in self.lin:
            w, b = self.lin[p + ".shortcut"]
            res = self._new(x.shape[0], w.shape[0])
            ops.gemm(x, w, b, res, ops.YB_EPI_BF16)
        return self._conv(c2, self._act(y, dims, p + ".residual.3", True, key=c2), dims, res=res, key=c2)

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
        """Resample upsample2d / upsample3d (:73-170) over the frames of this chunk."""
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
            dupup = ops.vae_dupup_add if self._chunk == 0 else ops.vae_dupup_add_cont     # DupUp3D `first_chunk` (:495-503)
            dupup(x, x_in, dims_in, ci, co, 2 if t_up else 1, 2)
        return x, dims

    # ---- chunk streaming -----------------------------------------------------------------------------------
    def _t_ups(self) -> int:
        return sum(1 for i in range(self.n_up - 1) if i < len(self.t_up) and self.t_up[i])

    def _front(self, z: Tensor):
        """conv2 (latent de-normalisation folded in) and decoder.conv1 on one chunk of the latent."""
        zd, T, H, W = z.shape
        N = T * H * W
        zl = self._new(N, 64)
        ops.nchw_to_nhwc_bf16(z.to(self.device, _F32).reshape(zd, N).contiguous(), zl)
        w2, b2 = self.lin["conv2"]
        x0 = self._hist_buf("decoder.conv1", T, H, W, 64, zero=True)
        ops.gemm(zl, w2, b2, x0.view(-1, 64)[x0.shape[0] * H * W - N:, :w2.shape[0]], ops.YB_EPI_BF16)
        dims = (T, H, W)
        return self._conv("decoder.conv1", x0, dims, key="decoder.conv1"), dims

    def _head(self, x: Tensor, dims) -> Tensor:
        return self._conv("decoder.head.2", self._act(x, dims, "decoder.head.0", True, key="decoder.head.2"), dims,
                          epilogue=ops.YB_EPI_F32, key="decoder.head.2")

    def _decode_chunk(self, z: Tensor, out: Tensor) -> None:
        """Decode one chunk of the latent into `out`, its frame window of the video."""
        x, dims = self._front(z)
        x = self._res_block("decoder.middle.0", x, dims)
        x = self._attention("decoder.middle.1", x, dims)
        x = self._res_block("decoder.middle.2", x, dims)
        for i in range(self.n_up):
            x, dims = self._up_block(i, x, dims)
        y = self._head(x, dims)
        if self._chunk == 0 and not self._more:
            ops.vae_unpatchify2_clamp(y, out, *dims)
        else:
            ops.vae_unpatchify2_clamp_win(y, out, *dims)

    def _out_shape(self, T: int, H: int, W: int) -> Tuple[int, int, int, int]:
        s = 16                                                   # three 2x spatial upsamples, then unpatchify 2x
        return 3, 1 + (T - 1) * (1 << self._t_ups()), s * H, s * W

    @torch.no_grad()
    def decode(self, z: Tensor) -> Tensor:
        """z [z_dim, T, H, W] -> f32 [3, 4(T-1)+1, 16H, 16W] clamped to [-1, 1] (Wan2_2_VAE.decode :1059-1072), in the chunks
        `plan_chunks` sizes from the free device memory."""
        if z.dim() != 4 or z.shape[0] != self.z_dim:
            raise YumeB200Error(f"expected a latent [{self.z_dim}, T, H, W]")
        return self._decode_chunks(z, self.plan_chunks(*z.shape[1:]))

    def _decode_chunks(self, z: Tensor, lengths: Sequence[int]) -> Tensor:
        """Decode the latent in chunks of `lengths` latent frames (any partition of T) into one preallocated video."""
        T, H, W = z.shape[1:]
        if sum(lengths) != T or min(lengths) < 1:
            raise YumeB200Error(f"chunk lengths {list(lengths)} do not partition {T} latent frames")
        out = self._new(*self._out_shape(T, H, W), dtype=_F32)
        s = 1 << self._t_ups()
        t0, f0 = 0, 0
        self._carry = {}
        try:
            for i, n in enumerate(lengths):
                self._chunk, self._more = i, i < len(lengths) - 1
                nf = 1 + (n - 1) * s if i == 0 else n * s
                self._decode_chunk(z[:, t0:t0 + n], out[:, f0:f0 + nf])
                t0, f0 = t0 + n, f0 + nf
        finally:
            self._chunk, self._more, self._carry = 0, False, None
        return out

    # ---- chunk planner -------------------------------------------------------------------------------------
    def _level_plan(self, H: int, W: int) -> List[tuple]:
        """The decoder's layer plan at latent size H x W, frames per chunk frame t_scale: ("in", t_scale, h, w, 64, co),
        ("res", t_scale, h, w, ci, co), ("attn", t_scale, h, w, c, 0), ("up", t_scale, h, w, c, co_of_resample, temporal,
        dupup_in) and ("head", t_scale, h, w, c, f32 output channels)."""
        plan: List[tuple] = [("in", 1, H, W, 64, self.dims[0]), ("res", 1, H, W, self.dims[0], self.dims[0]),
                             ("attn", 1, H, W, self.dims[0], 0), ("res", 1, H, W, self.dims[0], self.dims[0])]
        s, h, w = 1, H, W
        for i in range(self.n_up):
            ci, co = self.dims[i], self.dims[i + 1]
            for j in range(self.nrb + 1):
                plan.append(("res", s, h, w, ci if j == 0 else co, co))
            if i != self.n_up - 1:
                t_up = i < len(self.t_up) and self.t_up[i]
                plan.append(("up", s, h, w, co, co, t_up, ci))
                s, h, w = (2 * s if t_up else s), 2 * h, 2 * w
        plan.append(("head", s, h, w, self.dims[-1], self.conv["decoder.head.2"][0].shape[0]))
        return plan

    def _fixed_bytes(self, T: int, H: int, W: int) -> int:
        """The whole result, allocated once before the first chunk."""
        total = 1
        for d in self._out_shape(T, H, W):
            total *= d
        return 4 * total

    def chunk_bytes(self, n: int, T: int, H: int, W: int) -> int:
        """Upper bound of the device bytes a decode (encode) of T latent (video) frames at H x W allocates on top of the weights
        and its input when its chunks hold n latent frames: the whole result, every carried history, and the largest set of
        activations one step of the layer plan keeps live (every buffer of that step counted as live at once; a chunk after
        the first is counted, it has the most frames at each level)."""
        bf, f4 = 2, 4
        hist = self.HIST
        carries, peak = 0, 0
        for step in self._level_plan(H, W):
            kind, s, h, w, c = step[:5]
            F, vox = n * s, h * w
            cp = _rup(c, 64)
            if kind == "in":                                     # input gather, conv1's input buffer (history in front), conv1 out
                carries += hist * vox * c * bf
                live = (F * vox * c + (F + hist) * vox * c + F * vox * step[5]) * bf
            elif kind == "down":                                 # x, held block input, act, resample.1 out (+1 carried frame),
                vq = (h // 2) * (w // 2)                         # its act, time_conv out
                live = (F * vox * (c + step[6] + cp) + (F + 1) * vq * (c + cp) + F * vq * c) * bf
                if step[5]:
                    carries += vq * cp * bf
            elif kind == "res":                                    # x, the block input a shortcut add holds, y, res, out, two acts
                ci, co = c, step[5]
                carries += hist * vox * (cp + _rup(co, 64)) * bf
                live = F * vox * (2 * ci + 3 * co) * bf + (F + hist) * vox * (cp + _rup(co, 64)) * bf
            elif kind == "attn":
                Lf, Next = _rup(vox, 32), _rup(F * vox, 32) + 32
                live = (F * vox * c * 5 + Next * c * 3 + F * Lf * c * 3) * bf + vox * Lf * (f4 + bf)
            elif kind == "up":
                co, t_up, dup_in = step[5], step[6], step[7]
                F2 = 2 * F if t_up else F
                live = (F * vox * (c + dup_in) + F2 * vox * c) * bf + (F + hist) * vox * cp * bf * (1 if t_up else 0)
                live += F2 * 4 * vox * (cp + _rup(co, 32)) * bf
                if t_up:
                    carries += hist * vox * cp * bf
            else:                                                # head: act, f32 conv output
                live = (F * vox * c + (F + hist) * vox * cp) * bf + F * vox * step[5] * f4
                carries += hist * vox * cp * bf
            peak = max(peak, live)
        return self._fixed_bytes(T, H, W) + carries + peak

    def _plan(self, units: int, nbytes) -> List[int]:
        """Latent frames per chunk: all `units` when they fit (and always off CUDA), else the longest chunks whose `nbytes`
        fit the device's free memory (free + torch's cached, unallocated blocks) minus MEM_MARGIN. The free memory is read
        when the call starts, so other work on the same GPU can make a sequence that would fit alone run in chunks (with the
        same result)."""
        if self.device.type != "cuda":
            return [units]
        free, _ = torch.cuda.mem_get_info(self.device)
        free += torch.cuda.memory_reserved(self.device) - torch.cuda.memory_allocated(self.device)
        return chunk_lengths(units, nbytes, free - self.MEM_MARGIN)

    def plan_chunks(self, T: int, H: int, W: int) -> List[int]:
        """Latent frames per chunk of a decode of a T-frame latent at H x W (see _plan)."""
        return self._plan(T, lambda n: self.chunk_bytes(n, T, H, W))


def chunk_lengths(T: int, nbytes, budget: int) -> List[int]:
    """Partition T latent frames into chunks of the longest length n whose `nbytes(n)` (non-decreasing in n) fits `budget`, the
    last chunk taking the remainder: [T] when the whole sequence fits, chunks of 1 frame when nothing longer does."""
    if nbytes(T) <= budget:
        return [T]
    n = 1
    while n + 1 < T and nbytes(n + 1) <= budget:
        n += 1
    return [n] * (T // n) + ([T % n] if T % n else [])


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
