"""TEST INFRASTRUCTURE: torch-CPU stand-ins for the fp8 Ulysses entry points (include/yume_b200_fp8_sp.h) on top of
tests/helpers/torch_ops_fp8_attn.py (and through it torch_ops_fp8 / torch_ops), written from the header's contract: each entry point
is a one-GPU fp8 entry point with the exchange's layout, so each twin is the one-GPU twin plus that layout. Monkeypatched into
yume_b200.dit by the CPU suite so the engine's fp8 sequence-parallel host logic runs without a GPU; never imported by the package."""
import torch

from helpers.torch_ops_fp8_attn import *  # noqa: F401,F403  (the bf16, fp8 and fp8-attention entry points the engine still calls)
from helpers import torch_ops as _t
from helpers import torch_ops_fp8 as _t8
from helpers import torch_ops_fp8_attn as _ta


def gather_split(x, split, split_stride, shape):
    """The [M, K] matrix a K-split buffer holds: column k of row m at x.flatten()[(k // split) * split_stride + m * ldx + k % split],
    ldx = x.stride(-2) (yb_quant_rows_fp8_split, yb_gemm_bf16's a_split)."""
    M, K = shape
    ldx = x.stride(-2)
    idx = ((torch.arange(K) // split * split_stride)[None, :] + (torch.arange(M) * ldx)[:, None] +
           (torch.arange(K) % split)[None, :])
    return torch.as_strided(x, (x.numel(),), (1,), x.storage_offset())[idx.flatten()].view(M, K)


def quant_rows_fp8_split(x, out, out_scale, split, split_stride, shape):
    """Stand-in of yb_quant_rows_fp8_split: yb_quant_rows_fp8 of the gathered [M, K] matrix."""
    return _t8.quant_rows_fp8(gather_split(x, split, split_stride, shape), out, out_scale)


def attention_fp8_sp(q8, k8, qk_scale, vt8, v_scale, out_peers, ldo, heads, rank, Lp, scale=None, split=0):
    """Stand-in of yb_attention_fp8_sp: attention_fp8's rows, row g stored into row rank * Lp + g % Lp of out_peers[g // Lp]
    (here the receive buffers themselves, [P, Lp, heads * 128] tensors, in place of their device addresses)."""
    Lq = q8.shape[0]
    rows = torch.empty(Lq, heads * 128, dtype=torch.bfloat16)
    _ta.attention_fp8(q8, k8, qk_scale, vt8, v_scale, rows, heads, scale, split)
    for p, buf in enumerate(out_peers):
        buf.view(-1, Lp, heads * 128)[rank].copy_(rows[p * Lp:(p + 1) * Lp])


def sp_pack_qkv(qkv, wq, wk, rope, rope_len, head_dim, eps, send):
    """Stand-in of yb_sp_pack_qkv: RMSNorm * weight + RoPE on q and on k (the norm over all C columns), v as is, rounded to bf16;
    the columns of owner p's heads into send[p, :L] as q | k | v."""
    L, C3 = qkv.shape
    C = C3 // 3
    P, Lp, W3 = send.shape
    Wh = W3 // 3
    parts = [_t._norm_rope_rows(qkv[:, :C].float(), wq, rope, head_dim, eps, rope_len).to(torch.bfloat16),
             _t._norm_rope_rows(qkv[:, C:2 * C].float(), wk, rope, head_dim, eps, rope_len).to(torch.bfloat16),
             qkv[:, 2 * C:]]
    for p in range(P):
        send[p, :L] = torch.cat([x[:, p * Wh:(p + 1) * Wh] for x in parts], dim=1)
