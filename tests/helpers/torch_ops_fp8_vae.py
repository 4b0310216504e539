"""TEST INFRASTRUCTURE: the chunk-streaming torch-CPU stand-in (tests/helpers/torch_ops_stream.py) extended with the two entry
points of include/yume_b200_fp8_vae.h, written from the header's numerics contract: the activation quantiser is `quantize_act`
(oracle/fp8.py) of the bf16 values vae_rms_act writes, the conv an fp32 conv of the dequantised operands. Monkeypatched into
yume_b200.vae22 by the CPU suite so the precision="fp8" host logic runs without a GPU; never imported by the package."""
import torch
import torch.nn.functional as F

from helpers import torch_ops
from helpers.torch_ops_stream import *  # noqa: F401,F403  (every bf16 and streaming entry point the decoder calls)
from helpers.torch_ops_stream import calls
from oracle.fp8 import dequantize_act, quantize_act

_E4M3 = torch.float8_e4m3fn


def quantize_frames(v: torch.Tensor):
    """bf16 (or its float values) [T, H, W, Cp] -> (e4m3 [T, H, W, Cp], f32 scales [T, Cp/128, H, W]): the activation layout."""
    T, H, W, Cp = v.shape
    q, s = quantize_act(v.float().reshape(-1, Cp))
    return q.view(T, H, W, Cp), s.view(Cp // 128, T, H, W).transpose(0, 1).contiguous()


def dequantize_frames(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    T, H, W, Cp = q.shape
    return dequantize_act(q.reshape(-1, Cp), s.transpose(0, 1).reshape(Cp // 128, -1)).view(T, H, W, Cp)


def vae_rms_act_fp8(x, dims, out, out_scale, gamma, up=1, silu=True):
    calls.append("vae_rms_act_fp8")
    T, Hs, Ws = dims
    v = torch.empty(T, Hs * up, Ws * up, out.shape[-1], dtype=torch.bfloat16)
    torch_ops.vae_rms_act(x, dims, v, gamma, up, silu)
    q, s = quantize_frames(v)
    out.copy_(q)
    out_scale.copy_(s)
    return out


def conv3d_fp8(x, x_scale, w, w_scale, bias, out, T, H, W, t_hist=0, epilogue=torch_ops.YB_EPI_BF16, res=None, taps=(3, 3, 3)):
    calls.append("conv3d_fp8")
    kt, kh, kw = taps
    assert x.shape[0] == t_hist + T and t_hist in (0, kt - 1) and x.is_contiguous() and x_scale.is_contiguous()
    Cp, co = x.shape[-1], w.shape[0]
    xd = dequantize_frames(x, x_scale).permute(3, 0, 1, 2)[None]
    wd = (w.float() * w_scale[:, None]).view(co, kt, kh, kw, Cp).permute(0, 4, 1, 2, 3)
    xd = F.pad(xd, (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1 - t_hist, 0))
    y = F.conv3d(xd, wd, bias)[0].permute(1, 2, 3, 0).reshape(T * H * W, co)
    if epilogue == torch_ops.YB_EPI_RES_BF16:
        y = y + res.float()[:, :co]
    out[:, :co] = y.to(out.dtype)
    return out
