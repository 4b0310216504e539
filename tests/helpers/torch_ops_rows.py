"""TEST INFRASTRUCTURE: the torch-CPU stand-in of tests/helpers/torch_ops_resume.py extended with the row-band entry points of
include/yume_b200_vae_rows.h (same argument meaning and buffer layouts), for the row-parallel decode run over gloo. Its convs
and GEMMs sum in fp64 before the output rounding, so that a band and the full-height launch give the same values however the
CPU kernels block their sums (the kernels on the GPU sum in one fixed order). Tests monkeypatch it in; the package never
imports it."""
import torch
import torch.nn.functional as F

from helpers import torch_ops, torch_ops_stream
from helpers.torch_ops_resume import *  # noqa: F401,F403  (every stand-in the engines call)


def _conv64(x, w, bias, out, taps, pad, stride, epilogue, res, out_t_mul=1, out_t_add=0):
    """The fp64 convolution of x [T', H', W', Cp] zero padded by `pad` (F.pad order), written as the kernels write it."""
    kt, kh, kw = taps
    Cp, co = x.shape[-1], w.shape[0]
    wt = w.double().view(co, kt, kh, kw, Cp).permute(0, 4, 1, 2, 3)
    xn = F.pad(x.double().permute(3, 0, 1, 2)[None], pad)
    y = F.conv3d(xn, wt, None if bias is None else bias.double(), stride=stride)[0].permute(1, 2, 3, 0)
    To, Ho, Wo = y.shape[:3]
    y = y.reshape(To, Ho * Wo, co)
    if epilogue == torch_ops.YB_EPI_RES_BF16:
        y = y + res.double().view(To, Ho * Wo, co)
    frames = out.view(-1, Ho * Wo, out.shape[-1])
    for t in range(To):
        frames[t * out_t_mul + out_t_add, :, :co] = y[t].to(out.dtype)
    return out


def conv3d_causal(x, w, bias, out, T, H, W, epilogue=torch_ops.YB_EPI_BF16, res=None, taps=(3, 3, 3), oob_zero_pad=False,
                  out_t_mul=1, out_t_add=0, fuse_w=0, cta_pair=None, stride_t=1, stride_hw=1):
    torch_ops_stream.calls.append("conv3d_causal")
    kt, kh, kw = taps
    assert oob_zero_pad and stride_t == 1 and stride_hw == 1 and tuple(x.shape[:3]) == (T, H, W)
    return _conv64(x, w, bias, out, taps, (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0), 1, epilogue, res, out_t_mul, out_t_add)


def conv3d_causal_hist(xbuf, w, bias, out, T, H, W, t_hist, epilogue=torch_ops.YB_EPI_BF16, res=None, taps=(3, 3, 3),
                       out_t_mul=1, out_t_add=0, stride_t=1, stride_hw=1):
    torch_ops_stream.calls.append("conv3d_causal_hist")
    kt, kh, kw = taps
    assert stride_t == 1 and stride_hw == 1 and tuple(xbuf.shape[:3]) == (t_hist + T, H, W) and t_hist == kt - 1
    return _conv64(xbuf, w, bias, out, taps, (kw // 2, kw // 2, kh // 2, kh // 2, 0, 0), 1, epilogue, res, out_t_mul, out_t_add)


def conv3d_rows(xbuf, w, bias, out, T, H, W, t_hist=0, epilogue=torch_ops.YB_EPI_BF16, res=None, taps=(3, 3, 3), full_h=None):
    """yb_conv3d_rows: xbuf [t_hist + T, H + 2, W, Cp] a band buffer; no zero fill in H, W zero padded, time causal or carried."""
    torch_ops_stream.calls.append("conv3d_rows")
    kt, kh, kw = taps
    assert kh == 3 and tuple(xbuf.shape[:3]) == (t_hist + T, H + 2, W) and t_hist in (0, kt - 1) and xbuf.is_contiguous()
    return _conv64(xbuf, w, bias, out, taps, (kw // 2, kw // 2, 0, 0, kt - 1 - t_hist, 0), 1, epilogue, res)


def gemm(a, w, bias, out, epilogue=torch_ops.YB_EPI_BF16, res=None, **_):
    """yb_gemm_bf16 for the VAE's plain layouts (BF16, F32 and RES_BF16 epilogues), summed in fp64."""
    assert epilogue in (torch_ops.YB_EPI_BF16, torch_ops.YB_EPI_F32, torch_ops.YB_EPI_RES_BF16) and not _
    y = a.double() @ w.double().t()
    if bias is not None:
        y = y + bias.double()
    if epilogue == torch_ops.YB_EPI_RES_BF16:
        y = y + res.double()
    out.copy_(y.to(out.dtype))
    return out


def vae_rms_act_rows(x, dims, out, gamma, up=1, silu=True, send=None):
    T, Hs, Ws = dims
    torch_ops_stream.calls.append("vae_rms_act_rows")
    dense = torch.empty(T, Hs * up, Ws * up, out.shape[-1], dtype=out.dtype)
    torch_ops.vae_rms_act(x, dims, dense, gamma, up, silu)
    out[:, 1:Hs * up + 1] = dense
    if send is not None:
        send[0], send[1] = dense[:, 0], dense[:, -1]
    return out


def vae_rows_pack(buf, send):
    send[0], send[1] = buf[:, 1], buf[:, buf.shape[1] - 2]
    return send


def vae_rows_unpack(top, bot, buf):
    buf[:, 0] = 0 if top is None else top
    buf[:, -1] = 0 if bot is None else bot
    return buf


def vae_unpatchify2_clamp_rows(y, out, T, Hs, W):
    torch_ops_stream.calls.append("vae_unpatchify2_clamp_rows")
    v = y[:, :12].view(T, Hs, W, 12).permute(3, 0, 1, 2)[None]
    out.copy_(v.reshape(1, 3, 2, 2, T, Hs, W).permute(0, 1, 4, 5, 3, 6, 2).reshape(3, T, 2 * Hs, 2 * W).clamp(-1, 1))
    return out


def nhwc_to_nchw_f32_rows(x, out, clamp=None):
    torch_ops_stream.calls.append("nhwc_to_nchw_f32_rows")
    Cn, T, h, w = out.shape
    y = x[:, :Cn].t().reshape(Cn, T, h, w)
    out.copy_(y if clamp is None else y.clamp(*clamp))
    return out
