"""TEST INFRASTRUCTURE: the torch-CPU stand-in of tests/helpers/torch_ops.py extended with the chunk-streaming entry points of
include/yume_b200_stream.h (same argument meaning and buffer layouts), plus a launch log so tests can see which forms a decode
issued. Tests monkeypatch it in; the package never imports it."""
import torch
import torch.nn.functional as F

from helpers import torch_ops
from helpers.torch_ops import *  # noqa: F401,F403  (every stand-in the engines call)

calls = []          # names of the stand-in entry points called since the last `calls.clear()`


def _logged(name, fn):
    def wrapper(*a, **k):
        calls.append(name)
        return fn(*a, **k)
    return wrapper


for _name in ("conv3d_causal", "vae_dupup_add", "vae_unpatchify2_clamp", "nhwc_to_nchw_f32", "vae_rms_act"):
    globals()[_name] = _logged(_name, getattr(torch_ops, _name))


def conv3d_causal_hist(xbuf, w, bias, out, T, H, W, t_hist, epilogue=torch_ops.YB_EPI_BF16, res=None, taps=(3, 3, 3),
                       out_t_mul=1, out_t_add=0, stride_t=1, stride_hw=1):
    """yb_conv3d_causal_hist: the carried frames replace the causal zero padding in time; H and W are zero padded."""
    calls.append("conv3d_causal_hist")
    kt, kh, kw = taps
    assert xbuf.shape[0] == t_hist + T and t_hist == (1 if stride_t > 1 else kt - 1) and xbuf.is_contiguous()
    Cp, co = xbuf.shape[-1], w.shape[0]
    wt = w.float().view(co, kt, kh, kw, Cp).permute(0, 4, 1, 2, 3)
    xn = xbuf.float().permute(3, 0, 1, 2)[None]
    xn = F.pad(xn, (0, 1, 0, 1, 0, 0)) if stride_hw > 1 else F.pad(xn, (kw // 2, kw // 2, kh // 2, kh // 2, 0, 0))
    y = F.conv3d(xn, wt, bias, stride=(stride_t, stride_hw, stride_hw))[0].permute(1, 2, 3, 0)
    To, Ho, Wo = y.shape[:3]
    y = y.reshape(To, Ho * Wo, co)
    if epilogue == torch_ops.YB_EPI_RES_BF16:
        y = y + res.float().view(To, Ho * Wo, co)
    frames = out.view(-1, Ho * Wo, out.shape[-1])
    for t in range(To):
        frames[t * out_t_mul + out_t_add, :, :co] = y[t].to(out.dtype)
    return out


def vae_dupup_add_cont(main, x, dims, in_c, out_c, ft, fs):
    """main [ft*T, H*fs, W*fs, out_c] += DupUp3D(x [T, H, W, in_c]), no frame dropped."""
    calls.append("vae_dupup_add_cont")
    T, H, W = dims
    rep = out_c * ft * fs * fs // in_c
    y = x.float().view(T, H, W, in_c).permute(3, 0, 1, 2).repeat_interleave(rep, dim=0).view(out_c, ft, fs, fs, T, H, W)
    up = y.permute(4, 1, 5, 2, 6, 3, 0).reshape(T * ft, H * fs, W * fs, out_c)
    main.copy_((main.float().view(up.shape) + up).reshape(main.shape).to(main.dtype))
    return main


def vae_unpatchify2_clamp_win(y, out, T, H, W):
    calls.append("vae_unpatchify2_clamp_win")
    v = y[:, :12].view(T, H, W, 12).permute(3, 0, 1, 2)[None]
    out.copy_(v.reshape(1, 3, 2, 2, T, H, W).permute(0, 1, 4, 5, 3, 6, 2).reshape(3, T, 2 * H, 2 * W).clamp(-1, 1))
    return out


def nhwc_to_nchw_f32_win(x, out, clamp=None):
    calls.append("nhwc_to_nchw_f32_win")
    Cn, T, h, w = out.shape
    y = x[:, :Cn].t().reshape(Cn, T, h, w)
    out.copy_(y if clamp is None else y.clamp(*clamp))
    return out


def vae_patchify2_bf16_win(video, out):
    calls.append("vae_patchify2_bf16_win")
    return torch_ops.vae_patchify2_bf16(video.contiguous(), out)


def nchw_to_nhwc_bf16_win(x, out):
    calls.append("nchw_to_nhwc_bf16_win")
    return torch_ops.nchw_to_nhwc_bf16(x.reshape(x.shape[0], -1), out)
