"""TEST INFRASTRUCTURE: the torch-CPU stand-in of tests/helpers/torch_ops_rows.py extended with the row-band entry points of
include/yume_b200_vae_rows_enc.h (same argument meaning and buffer layouts) and with strided fp64 twins of the full-height
convs, for the row-parallel ENCODE run over gloo. Like torch_ops_rows every conv sums in fp64 before the output rounding, so a
band and the full-height launch give the same values however the CPU kernels block their sums. `read_frames` records the video
frames each band reader read. Tests monkeypatch it in; the package never imports it."""
import torch

from helpers import torch_ops, torch_ops_stream
from helpers.torch_ops_rows import *  # noqa: F401,F403  (every stand-in the engines call)
from helpers.torch_ops_rows import _conv64

read_frames = []    # frames of the video each band reader read since the last clear()


def _pad_hw(taps, stride_hw):
    """F.pad order (W, W, H, H) of the zero-padded convs: centred for unit stride, one column / row behind for stride 2."""
    _, kh, kw = taps
    return (0, 1, 0, 1) if stride_hw > 1 else (kw // 2, kw // 2, kh // 2, kh // 2)


def conv3d_causal(x, w, bias, out, T, H, W, epilogue=torch_ops.YB_EPI_BF16, res=None, taps=(3, 3, 3), oob_zero_pad=False,
                  out_t_mul=1, out_t_add=0, fuse_w=0, cta_pair=None, stride_t=1, stride_hw=1):
    """yb_conv3d_causal (zero padded, strided forms included), summed in fp64."""
    torch_ops_stream.calls.append("conv3d_causal")
    kt = taps[0]
    assert oob_zero_pad and tuple(x.shape[:3]) == (T, H, W)
    pad = _pad_hw(taps, stride_hw) + ((kt - 1, 0) if stride_t == 1 else (0, 0))
    return _conv64(x, w, bias, out, taps, pad, (stride_t, stride_hw, stride_hw), epilogue, res, out_t_mul, out_t_add)


def conv3d_causal_hist(xbuf, w, bias, out, T, H, W, t_hist, epilogue=torch_ops.YB_EPI_BF16, res=None, taps=(3, 3, 3),
                       out_t_mul=1, out_t_add=0, stride_t=1, stride_hw=1):
    """yb_conv3d_causal_hist: the carried frames replace the causal zero padding in time; summed in fp64."""
    torch_ops_stream.calls.append("conv3d_causal_hist")
    assert tuple(xbuf.shape[:3]) == (t_hist + T, H, W) and t_hist == (1 if stride_t > 1 else taps[0] - 1)
    pad = _pad_hw(taps, stride_hw) + (0, 0)
    return _conv64(xbuf, w, bias, out, taps, pad, (stride_t, stride_hw, stride_hw), epilogue, res, out_t_mul, out_t_add)


def conv3d_rows_down(xbuf, w, bias, out, T, H, W, epilogue=torch_ops.YB_EPI_BF16):
    """yb_conv3d_rows_down: rows 1 .. H + 1 of the band buffer (the last the row below), W zero padded behind, stride 2."""
    torch_ops_stream.calls.append("conv3d_rows_down")
    assert tuple(xbuf.shape[:3]) == (T, H + 2, W) and H % 2 == 0 and xbuf.is_contiguous()
    return _conv64(xbuf[:, 1:], w, bias, out, (1, 3, 3), (0, 1, 0, 0, 0, 0), (1, 2, 2), epilogue, None)


def _band_rows(dense, out, r0):
    """out [T, hs + 2, W, C] = rows r0 - 1 .. r0 + hs of dense [T, H, W, C], zeros outside it."""
    hs, H = out.shape[1] - 2, dense.shape[1]
    out.zero_()
    a, b = max(r0 - 1, 0), min(r0 + hs + 1, H)
    out[:, a - (r0 - 1):b - (r0 - 1)] = dense[:, a:b]
    return out


def vae_patchify2_bf16_rows(video, out, r0):
    torch_ops_stream.calls.append("vae_patchify2_bf16_rows")
    read_frames.append(video.shape[1])
    _, T, H, W = video.shape
    dense = torch.empty(T, H // 2, W // 2, out.shape[-1], dtype=out.dtype)
    torch_ops.vae_patchify2_bf16(video.contiguous(), dense.view(-1, out.shape[-1]))
    return _band_rows(dense, out, r0)


def nchw_to_nhwc_bf16_rows(x, out, r0):
    torch_ops_stream.calls.append("nchw_to_nhwc_bf16_rows")
    read_frames.append(x.shape[1])
    Cn, T, H, W = x.shape
    dense = torch.empty(T, H, W, out.shape[-1], dtype=out.dtype)
    torch_ops.nchw_to_nhwc_bf16(x.reshape(Cn, -1), dense.view(-1, out.shape[-1]))
    return _band_rows(dense, out, r0)
