"""TEST INFRASTRUCTURE: torch-CPU stand-ins for the fp8 entry points (include/yume_b200_fp8.h) on top of tests/helpers/torch_ops.py,
written from the header's numerics contract (the quantisers are oracle/fp8.py's twins). Monkeypatched into yume_b200.dit by the
CPU suite so the engine's precision="fp8" host logic runs without a GPU; never imported by the package."""
import torch

from helpers.torch_ops import *  # noqa: F401,F403  (the bf16 entry points the fp8 engine still calls)
from helpers import torch_ops as _t
from oracle.fp8 import dequantize_act, quantize_act
from yume_b200.ops import fp8_scale_ld  # noqa: F401  (host arithmetic the engine asks its ops module for)

YB_EPI_GELU_FP8 = 8


def _store_act(y, out, out_scale):
    q, s = quantize_act(y)
    out.copy_(q)
    out_scale[:, :y.shape[0]] = s
    return out


def gemm_fp8(a, a_scale, w, w_scale, bias, out, epilogue, gate=None, tok_idx=None, out_scale=None):
    """Stand-in of yb_gemm_fp8: the dequantised operands (s_a per row and 1x128 group, s_w per column), fp32 product."""
    M = a.shape[0]
    y = dequantize_act(a, a_scale) @ (w.float() * w_scale[:, None]).t()
    if bias is not None:
        y = y + bias
    if epilogue == YB_EPI_GELU_FP8:
        return _store_act(_t._gelu_tanh(y), out, out_scale)
    if epilogue == _t.YB_EPI_GATE_RES:
        if gate is not None:
            rows = tok_idx.long() if tok_idx is not None else torch.zeros(M, dtype=torch.long)
            y = y * gate[rows]
        out.add_(y)
        return out
    out.copy_(y.to(out.dtype))
    return out


def ln_modulate_fp8(x, out, out_scale, scale, shift, tok_idx=None, weight=None, bias=None, eps=1e-6):
    y = torch.empty(x.shape, dtype=torch.float32)
    _t.ln_modulate(x, y, scale, shift, tok_idx, weight, bias, eps)
    return _store_act(y, out, out_scale)


def quant_rows_fp8(x, out, out_scale):
    return _store_act(x.float(), out, out_scale)
