"""TEST INFRASTRUCTURE: torch-CPU stand-ins for the fp8 self-attention entry points (include/yume_b200_fp8_attn.h) on top of
tests/helpers/torch_ops_fp8.py, written from the header's numerics contract (the V quantiser is oracle/fp8_attn.py's twin).
Monkeypatched into yume_b200.dit by the CPU suite so the engine's precision="fp8_attn" host logic runs without a GPU; never
imported by the package."""
from helpers.torch_ops_fp8 import *  # noqa: F401,F403  (the bf16 and fp8 entry points the engine still calls)
from oracle.fp8 import dequantize_act
from oracle.fp8_attn import attention_fp64, dequantize_vt, quantize_vt
from yume_b200.ops import vt8_keys  # noqa: F401  (host arithmetic the engine asks its ops module for)


def quant_vt_fp8(v, vt8, v_scale, heads):
    q, s = quantize_vt(v.float(), heads)
    vt8.copy_(q)
    v_scale.copy_(s)
    return vt8


def attention_fp8(q8, k8, qk_scale, vt8, v_scale, out, heads, scale=None, split=0):
    """Stand-in of yb_attention_fp8: fp64 attention over the dequantised operands (q scales at rows [0, heads), k scales at
    rows [heads, 2 heads) of qk_scale)."""
    q = dequantize_act(q8, qk_scale[:heads])
    k = dequantize_act(k8, qk_scale[heads:])
    v = dequantize_vt(vt8, v_scale, k8.shape[0])
    out.copy_(attention_fp64(q, k, v, heads, scale).to(out.dtype))
    return out
