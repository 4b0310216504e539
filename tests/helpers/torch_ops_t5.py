"""TEST INFRASTRUCTURE: helpers.torch_ops plus a torch-CPU stand-in for the umT5 encoder's kernels (yb_t5_attention,
yb_t5_rmsnorm, yb_t5_geglu, include/yume_b200_t5.h) with the kernels' argument meaning and arithmetic (fp32 scores + bias,
masked keys dropped, P rounded to bf16 against an fp32 normaliser, one output rounding), so the CPU suite can drive
yume_b200/t5.py's host logic."""
import torch
import torch.nn.functional as F

from helpers.torch_ops import *  # noqa: F401,F403


def t5_attention(q, k, v, out, B, heads, bias, key_mask=None):
    BL = q.shape[0]
    L, d = BL // B, 64
    f = lambda t: t.float().reshape(B, L, heads, d).transpose(1, 2)          # noqa: E731  [B, heads, L, d]
    s = f(q) @ f(k).transpose(-1, -2)
    idx = torch.arange(L, device=bias.device)[None, :] - torch.arange(L, device=bias.device)[:, None] + L - 1
    s = s + bias[:, idx][None]
    if key_mask is not None:
        s = s.masked_fill(key_mask[:, None, None, :] == 0, float("-inf"))
    p = torch.exp(s - s.amax(dim=-1, keepdim=True))
    o = (p.to(torch.bfloat16).float() @ f(v)) / p.sum(dim=-1, keepdim=True)
    out.copy_(o.transpose(1, 2).reshape(BL, heads * d).to(out.dtype))
    return out


def t5_rmsnorm(x, out, weight, eps=1e-6):
    xf = x.float()
    out.copy_((xf * torch.rsqrt(xf.pow(2).mean(dim=1, keepdim=True) + eps) * weight).to(out.dtype))
    return out


def t5_geglu(ug, out):
    Fd = ug.shape[1] // 2
    out.copy_((ug[:, :Fd].float() * F.gelu(ug[:, Fd:].float(), approximate="tanh")).to(out.dtype))
    return out
