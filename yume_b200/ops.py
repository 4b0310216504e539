"""Tensor-level wrappers over the C ABI. torch is used only for device memory and the current stream;
every function requires CUDA tensors and calls straight into libyume_b200.so."""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional

import torch

from . import _lib
from ._lib import (YB_ATT_ACCUMULATE, YB_ATT_P_SMEM, YB_EPI_BF16, YB_EPI_F32, YB_EPI_GATE_RES, YB_EPI_GELU_BF16,
                   YB_EPI_GELU_ERF_BF16, YB_EPI_RES_BF16, Conv3dArgs, GemmArgs, YumeB200Error, check)

__all__ = [
    "gemm", "ln_modulate", "rmsnorm_rope", "qk_norm_rope", "flop_count", "attention", "patchify", "unpatchify", "sinusoidal",
    "linear_f32_small", "linear_f32", "umma_probe", "launch_count", "reset_launch_count",
    "YB_EPI_BF16", "YB_EPI_GELU_BF16", "YB_EPI_F32", "YB_EPI_GATE_RES", "YB_EPI_GELU_ERF_BF16", "bcast_add",
    "YB_ATT_P_SMEM", "YB_ATT_ACCUMULATE",
]

_launches = 0
_flops = 0.0        # algorithmic tensor-core FLOPs (2*M*N*K) of the GEMM / conv / attention launches since the last reset


def flop_count() -> float:
    """Algorithmic FLOPs of the tensor-core launches (gemm, conv3d_causal, attention*) since the last reset — bench.py
    derives the tensor-roofline fraction of whole decodes / forwards from it."""
    return _flops


def launch_count() -> int:
    """Number of yume_b200 kernels launched since the last reset (bench.py reports it as gpu_launches)."""
    return _launches


def reset_launch_count() -> None:
    global _launches, _flops
    _launches = 0
    _flops = 0.0


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _need(t: torch.Tensor, dtype, name: str) -> None:
    if not t.is_cuda:
        raise YumeB200Error(f"{name} must be a CUDA tensor (yume_b200 has no CPU path)")
    if t.dtype != dtype:
        raise YumeB200Error(f"{name} must be {dtype}, got {t.dtype}")
    if t.stride(-1) != 1:
        raise YumeB200Error(f"{name} must be contiguous in its last dimension")


def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor, epilogue: int,
         gate: Optional[torch.Tensor] = None, tok_idx: Optional[torch.Tensor] = None, block_n: int = 0,
         n_split: int = 0, split_stride: int = 0, a_split: int = 0, a_split_stride: int = 0,
         shape: Optional[tuple] = None, res: Optional[torch.Tensor] = None, cta_pair: int = 0, split_k: Optional[int] = None) -> torch.Tensor:
    """out = epi(a[M,K] @ w[N,K]^T + bias). a, w bf16 (2-D, row stride arbitrary); see include/yume_b200.h.
    cta_pair: 0 automatic, 1 force the 1-CTA kernel, 2 force the SM-pair kernel (2-CTA cluster, multicast B operand).
    split_k (SM-pair GATE_RES launches): 0 automatic tail split-K, 1 never, 2..12 force that many K segments on the last wave."""
    global _launches, _flops
    _need(a, torch.bfloat16, "a")
    _need(w, torch.bfloat16, "w")
    N, K2 = w.shape
    if shape is not None:          # split layouts: logical (M, K) given explicitly, a / out are the raw buffers
        M, K = shape
    else:
        M, K = a.shape
    if K2 != K:
        raise YumeB200Error(f"gemm K mismatch: {K} vs {K2}")
    want = torch.bfloat16 if epilogue in (YB_EPI_BF16, YB_EPI_GELU_BF16, YB_EPI_GELU_ERF_BF16, YB_EPI_RES_BF16) else torch.float32
    if res is not None:
        _need(res, torch.bfloat16, "res")
    _need(out, want, "out")
    if shape is None and (out.shape[0] != M or out.shape[1] != N):
        raise YumeB200Error(f"gemm out shape {tuple(out.shape)} != ({M}, {N})")
    if bias is not None:
        _need(bias, torch.float32, "bias")
    if gate is not None:
        _need(gate, torch.float32, "gate")
    if tok_idx is not None:
        _need(tok_idx, torch.int32, "tok_idx")
    if split_k is None:
        split_k = GEMM_SPLIT_K
    ws, ws_bytes = None, 0
    if epilogue == YB_EPI_GATE_RES and split_k != 1 and cta_pair != 1:
        # caller-owned workspace of the tail split-K (the library never allocates): a stream-ordered allocation from torch's
        # caching allocator, only for launches the planner actually splits
        ws_bytes = _lib.load().yb_gemm_workspace_bytes(M, N, K, epilogue, cta_pair, split_k)
        if ws_bytes > 0:
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=a.device)
    args = GemmArgs(
        struct_bytes=C.sizeof(GemmArgs), cta_pair=cta_pair, A=a.data_ptr(), B=w.data_ptr(), bias=_ptr(bias), out=out.data_ptr(), gate=_ptr(gate), tok_idx=_ptr(tok_idx),
        lda=a.stride(-2), ldb=w.stride(0), ldo=out.stride(-2), gate_ld=(gate.stride(0) if gate is not None else 0),
        M=M, N=N, K=K, epilogue=epilogue, block_n=block_n, n_split=n_split, split_stride=split_stride,
        a_split=a_split, a_split_stride=a_split_stride, res=_ptr(res),
        res_ld=(res.stride(-2) if res is not None else 0), split_k=split_k, ws=_ptr(ws), ws_bytes=ws_bytes)
    check(_lib.load().yb_gemm_bf16(C.byref(args), _stream()), "yb_gemm_bf16")
    _launches += 1
    _flops += 2.0 * M * N * K
    return out


def ln_modulate(x: torch.Tensor, out: torch.Tensor, scale: Optional[torch.Tensor], shift: Optional[torch.Tensor],
                tok_idx: Optional[torch.Tensor] = None, weight: Optional[torch.Tensor] = None,
                bias: Optional[torch.Tensor] = None, eps: float = 1e-6) -> torch.Tensor:
    """out = LN(x) [* weight + bias] [* (1 + scale[tok]) + shift[tok]]; x f32 [L, C]; out bf16 or f32 [L, C]."""
    global _launches
    _need(x, torch.float32, "x")
    L, Cdim = x.shape
    out_f32 = 1 if out.dtype == torch.float32 else 0
    _need(out, torch.float32 if out_f32 else torch.bfloat16, "out")
    mod_ld = 0
    for name, t in (("scale", scale), ("shift", shift)):
        if t is not None:
            _need(t, torch.float32, name)
            mod_ld = t.stride(0) if t.dim() == 2 else 0
    if scale is not None and shift is not None and scale.dim() == 2 and scale.stride(0) != shift.stride(0):
        raise YumeB200Error("scale and shift must share their row stride")
    check(_lib.load().yb_ln_modulate(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), out_f32, _ptr(scale),
                                     _ptr(shift), mod_ld, _ptr(tok_idx), _ptr(weight), _ptr(bias), L, Cdim, eps,
                                     _stream()), "yb_ln_modulate")
    _launches += 1
    return out


def rmsnorm_rope(qk: torch.Tensor, weight: torch.Tensor, rope: Optional[torch.Tensor], head_dim: int,
                 eps: float = 1e-6, rope_len: Optional[int] = None, pieces: Optional[tuple] = None) -> torch.Tensor:
    """In place on bf16 rows qk [L, C] (row stride arbitrary): RMSNorm over C, * weight, RoPE with rope f32 [L, D/2, 2]."""
    global _launches
    _need(qk, torch.bfloat16, "qk")
    _need(weight, torch.float32, "weight")
    if pieces is not None:         # (L, C, piece_cols, piece_stride): qk is the first piece, rows `qk.stride(0)` apart
        L, Cdim, piece_cols, piece_stride = pieces
    else:
        L, Cdim = qk.shape
        piece_cols, piece_stride = Cdim, 0
    if rope is not None:
        _need(rope, torch.float32, "rope")
        if not rope.is_contiguous() or rope.shape[-1] != 2 or rope.shape[-2] != head_dim // 2:
            raise YumeB200Error("rope must be contiguous f32 [L, D/2, 2]")
        if rope_len is None:
            rope_len = rope.shape[0]
    check(_lib.load().yb_rmsnorm_rope_pieces(qk.data_ptr(), qk.stride(0), piece_cols, piece_stride, weight.data_ptr(),
                                             _ptr(rope), rope_len or 0, L, Cdim, head_dim, eps, _stream()),
          "yb_rmsnorm_rope")
    _launches += 1
    return qk


def qk_norm_rope(q: torch.Tensor, k: torch.Tensor, wq: torch.Tensor, wk: torch.Tensor, rope: Optional[torch.Tensor],
                 head_dim: int, eps: float = 1e-6, rope_len: Optional[int] = None, pieces: Optional[tuple] = None) -> None:
    """RMSNorm(q)*wq, RMSNorm(k)*wk and RoPE on both, in place, ONE launch. q, k: bf16 [L, C] views with the same row
    stride (e.g. two column ranges of the fused qkv buffer). pieces as for rmsnorm_rope."""
    global _launches
    _need(q, torch.bfloat16, "q")
    _need(k, torch.bfloat16, "k")
    _need(wq, torch.float32, "wq")
    _need(wk, torch.float32, "wk")
    if q.stride(0) != k.stride(0):
        raise YumeB200Error("q and k must share their row stride")
    if pieces is not None:
        L, Cdim, piece_cols, piece_stride = pieces
    else:
        if q.shape != k.shape:
            raise YumeB200Error("q and k must have the same shape")
        L, Cdim = q.shape
        piece_cols, piece_stride = Cdim, 0
    if rope is not None:
        _need(rope, torch.float32, "rope")
        if not rope.is_contiguous() or rope.shape[-1] != 2 or rope.shape[-2] != head_dim // 2:
            raise YumeB200Error("rope must be contiguous f32 [L, D/2, 2]")
        if rope_len is None:
            rope_len = rope.shape[0]
    check(_lib.load().yb_qk_norm_rope(q.data_ptr(), k.data_ptr(), q.stride(0), piece_cols, piece_stride, wq.data_ptr(),
                                      wk.data_ptr(), _ptr(rope), rope_len or 0, L, Cdim, head_dim, eps, _stream()),
          "yb_qk_norm_rope")
    _launches += 1


_sm_counts = {}


def _sms(device: torch.device) -> int:
    idx = device.index if device.index is not None else torch.cuda.current_device()
    n = _sm_counts.get(idx)
    if n is None:
        n = _sm_counts[idx] = torch.cuda.get_device_properties(idx).multi_processor_count
    return n


def _attention_ws(Lq: int, Lk: int, heads: int, flags: int, device: torch.device):
    """Caller-owned workspace of the automatic KV tail split (the library never allocates): a fresh stream-ordered
    allocation from torch's caching allocator, only for launches the planner actually splits."""
    nbytes = _lib.load().yb_attention_workspace_bytes(Lq, Lk, heads, _sms(device), flags)
    if nbytes <= 0:
        return None, 0
    return torch.empty(nbytes, dtype=torch.uint8, device=device), nbytes


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, heads: int,
              scale: Optional[float] = None, variant: int = 0, accumulate: bool = False,
              split: int = 0) -> torch.Tensor:
    """softmax(q k^T * scale) v, non-causal. q [Lq, heads*128], k/v [Lk, heads*128] bf16 (row strides arbitrary).
    split: KV split policy (YB_ATT_SPLIT_SHIFT): 0 automatic tail split, 1 never, 2..4 force that many KV segments.
    variant: 0 product kernel (P in registers), 1 debug (P through smem)."""
    global _launches, _flops
    for n, t in (("q", q), ("k", k), ("v", v), ("out", out)):
        _need(t, torch.bfloat16, n)
    Lq, Lk = q.shape[0], k.shape[0]
    if q.shape[1] != heads * 128 or k.shape[1] != heads * 128 or v.shape[1] != heads * 128:
        raise YumeB200Error("attention supports head_dim 128 only")
    if scale is None:
        scale = 1.0 / math.sqrt(128.0)
    flags = (YB_ATT_P_SMEM if variant == 1 else 0) | (YB_ATT_ACCUMULATE if accumulate else 0) | ((split & 7) << 4)
    if variant not in (0, 1):
        raise YumeB200Error("attention variant must be 0 or 1")
    ws, ws_bytes = _attention_ws(Lq, Lk, heads, flags, q.device)
    check(_lib.load().yb_attention_ex(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                                      out.data_ptr(), out.stride(0), Lq, Lk, heads, scale, flags, _ptr(ws), ws_bytes, None,
                                      _stream()), "yb_attention")
    _launches += 1
    _flops += 4.0 * Lq * Lk * heads * 128
    return out


def patchify(x: torch.Tensor, out: torch.Tensor, ph: int, pw: int) -> torch.Tensor:
    """x f32 [Cin, F, H, W] (any strides) -> out bf16 [F*ceil(H/ph)*ceil(W/pw), >= Cin*ph*pw]."""
    global _launches
    if not x.is_cuda or x.dtype != torch.float32:
        raise YumeB200Error("patchify input must be a CUDA float32 tensor")
    _need(out, torch.bfloat16, "out")
    Cin, F, H, W = x.shape
    sc, sf, sh, sw = x.stride()
    check(_lib.load().yb_patchify(x.data_ptr(), sc, sf, sh, sw, out.data_ptr(), out.stride(0), Cin, F, H, W, ph, pw,
                                  _stream()), "yb_patchify")
    _launches += 1
    return out


def unpatchify(y: torch.Tensor, out: torch.Tensor, F: int, Hp: int, Wp: int, ph: int, pw: int) -> torch.Tensor:
    """y f32 [L, ph*pw*Cout] -> out f32 [Cout, F, Hp*ph, Wp*pw] (contiguous)."""
    global _launches
    _need(y, torch.float32, "y")
    _need(out, torch.float32, "out")
    Cout = out.shape[0]
    check(_lib.load().yb_unpatchify(y.data_ptr(), y.stride(0), out.data_ptr(), Cout, F, Hp, Wp, ph, pw, _stream()),
          "yb_unpatchify")
    _launches += 1
    return out


def bcast_add(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """out[r1, r2, :] = a[r1, :] + b[r2, :] (f32, contiguous 2-D inputs)."""
    global _launches
    _need(a, torch.float32, "a")
    _need(b, torch.float32, "b")
    if not (a.is_contiguous() and b.is_contiguous()) or a.shape[1] != b.shape[1]:
        raise YumeB200Error("bcast_add needs contiguous [R, n] operands with equal n")
    out = torch.empty(a.shape[0], b.shape[0], a.shape[1], device=a.device, dtype=torch.float32)
    check(_lib.load().yb_bcast_add(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.shape[0], b.shape[0], a.shape[1],
                                   _stream()), "yb_bcast_add")
    _launches += 1
    return out


def sinusoidal(t: torch.Tensor, dim: int) -> torch.Tensor:
    global _launches
    _need(t, torch.float32, "t")
    out = torch.empty(t.numel(), dim, device=t.device, dtype=torch.float32)
    check(_lib.load().yb_sinusoidal(t.data_ptr(), out.data_ptr(), t.numel(), dim, _stream()), "yb_sinusoidal")
    _launches += 1
    return out


def linear_f32_small(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], silu_in: bool = False) -> torch.Tensor:
    global _launches
    _need(x, torch.float32, "x")
    _need(w, torch.float32, "w")
    M, K = x.shape
    N = w.shape[0]
    if not (x.is_contiguous() and w.is_contiguous()):
        raise YumeB200Error("linear_f32_small needs contiguous operands")
    out = torch.empty(M, N, device=x.device, dtype=torch.float32)
    check(_lib.load().yb_linear_f32_small(x.data_ptr(), w.data_ptr(), _ptr(bias), out.data_ptr(), M, N, K,
                                          1 if silu_in else 0, _stream()), "yb_linear_f32_small")
    _launches += 1
    return out


def linear_f32(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor) -> torch.Tensor:
    global _launches
    _need(x, torch.float32, "x")
    _need(w, torch.float32, "w")
    _need(out, torch.float32, "out")
    M, K = x.shape
    N = w.shape[0]
    if not w.is_contiguous():
        raise YumeB200Error("linear_f32 weight must be contiguous")
    check(_lib.load().yb_linear_f32(x.data_ptr(), x.stride(0), w.data_ptr(), _ptr(bias), out.data_ptr(),
                                    out.stride(0), M, N, K, _stream()), "yb_linear_f32")
    _launches += 1
    return out


def umma_probe(a: torch.Tensor, b: torch.Tensor, mode: int) -> torch.Tensor:
    """wgmma / TMA self-test (tests only). a, b bf16 [128,128] contiguous -> f32 [128,128]."""
    _need(a, torch.bfloat16, "a")
    _need(b, torch.bfloat16, "b")
    d = torch.empty(128, 128, device=a.device, dtype=torch.float32)
    check(_lib.load().yb_umma_probe(a.data_ptr(), b.data_ptr(), d.data_ptr(), mode, _stream()), "yb_umma_probe")
    return d


# ------------------------------------------------------------------------------------------------------------
# VAE decoder ops (hyvideo/vae)
# ------------------------------------------------------------------------------------------------------------
YB_EPI_RES_BF16 = YB_EPI_RES_BF16


# kernel choice of conv3d_causal when the caller does not say (see yb_conv3d_args.cta_pair in include/yume_b200.h)
CONV_CTA_PAIR = 0
GEMM_SPLIT_K = 0     # tail split-K policy of the SM-pair gate+residual GEMM for callers that do not pass one: 0 automatic, 1 never


def conv3d_causal(xpad: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor, T: int, H: int,
                  W: int, epilogue: int = YB_EPI_BF16, res: Optional[torch.Tensor] = None, taps=(3, 3, 3),
                  oob_zero_pad: bool = False, out_t_mul: int = 1, out_t_add: int = 0, fuse_w: int = 0,
                  cta_pair: Optional[int] = None, stride_t: int = 1, stride_hw: int = 1) -> torch.Tensor:
    """Implicit-GEMM causal conv. Default: xpad bf16 [T+2, H+2, W+2, Cp] replicate padded (hyvideo VAE). With
    oob_zero_pad the input is the unpadded [T, H, W, Cp] and the zero padding is TMA out-of-bounds fill (Wan2.2 VAE).
    w bf16 [Cout, kt*kh*kw*Cp]; out rows are output voxels (frame t -> t*out_t_mul + out_t_add). stride_hw / stride_t = 2:
    the Encoder3d Resample convs (see include/yume_b200.h); T, H, W stay the input extents."""
    global _launches, _flops
    _need(xpad, torch.bfloat16, "xpad")
    _need(w, torch.bfloat16, "w")
    Cp = xpad.shape[-1]
    kt, kh, kw = taps
    want = (T, H, W) if oob_zero_pad else (T + kt - 1, H + kh - 1, W + kw - 1)
    if tuple(xpad.shape[:3]) != want or not xpad.is_contiguous() or w.shape[1] != kt * kh * kw * Cp or not w.is_contiguous():
        raise YumeB200Error("conv3d_causal: bad input / weight layout")
    _need(out, torch.float32 if epilogue == YB_EPI_F32 else torch.bfloat16, "out")
    if res is not None:
        _need(res, torch.bfloat16, "res")
    args = Conv3dArgs(struct_bytes=C.sizeof(Conv3dArgs), cta_pair=CONV_CTA_PAIR if cta_pair is None else cta_pair,
                      xpad=xpad.data_ptr(), w=w.data_ptr(), bias=_ptr(bias), out=out.data_ptr(), res=_ptr(res),
                      ldo=out.stride(0), res_ld=(res.stride(0) if res is not None else 0), T=T, H=H, W=W, Cp=Cp,
                      Cout=w.shape[0], epilogue=epilogue, kt=kt, kh=kh, kw=kw, oob_zero_pad=1 if oob_zero_pad else 0,
                      out_t_mul=out_t_mul, out_t_add=out_t_add, fuse_w=fuse_w, stride_t=stride_t, stride_hw=stride_hw)
    check(_lib.load().yb_conv3d_causal(C.byref(args), _stream()), "yb_conv3d_causal")
    _launches += 1
    To, Ho, Wo = conv_out_dims(T, H, W, taps, stride_t, stride_hw)
    _flops += 2.0 * To * Ho * Wo * kt * kh * kw * Cp * w.shape[0]
    return out


def conv_out_dims(T: int, H: int, W: int, taps=(3, 3, 3), stride_t: int = 1, stride_hw: int = 1):
    """Output extents of yb_conv3d_causal: unit stride keeps the extents; the strided forms follow the reference's
    `Resample` (ZeroPad2d((0,1,0,1)) + Conv2d stride 2; unpadded time_conv stride 2)."""
    kt, kh, kw = taps
    To = (T - kt) // stride_t + 1 if stride_t > 1 else T
    Ho, Wo = ((H + 1 - kh) // stride_hw + 1, (W + 1 - kw) // stride_hw + 1) if stride_hw > 1 else (H, W)
    return To, Ho, Wo


def gn_stats(x: torch.Tensor, groups: int) -> torch.Tensor:
    """x bf16 [N, C] -> f64 [G, 2] (sum, sum of squares) per group."""
    global _launches
    _need(x, torch.bfloat16, "x")
    stats = torch.zeros(groups, 2, device=x.device, dtype=torch.float64)
    check(_lib.load().yb_gn_stats(x.data_ptr(), x.stride(0), stats.data_ptr(), x.shape[0], x.shape[1], groups, _stream()),
          "yb_gn_stats")
    _launches += 1
    return stats


def vae_pad_act(x: torch.Tensor, src_dims, out: torch.Tensor, pad: bool, up=(1, 1, 1), stats=None, gamma=None, beta=None,
                groups: int = 32, eps: float = 1e-6, silu: bool = False) -> torch.Tensor:
    """x bf16 [Ts*Hs*Ws, C] -> out bf16 [(T+2p), (H+2p), (W+2p), Cp] (see include/yume_b200.h)."""
    global _launches
    _need(x, torch.bfloat16, "x")
    _need(out, torch.bfloat16, "out")
    Ts, Hs, Ws = src_dims
    if not out.is_contiguous():
        raise YumeB200Error("vae_pad_act output must be contiguous")
    check(_lib.load().yb_vae_pad_act(x.data_ptr(), x.stride(0), Ts, Hs, Ws, x.shape[1], out.data_ptr(), out.shape[-1],
                                     1 if pad else 0, up[0], up[1], up[2], _ptr(stats), _ptr(gamma), _ptr(beta), groups,
                                     eps, 1 if silu else 0, _stream()), "yb_vae_pad_act")
    _launches += 1
    return out


def masked_softmax(S: torch.Tensor, P: torch.Tensor, L: int, hw: int) -> torch.Tensor:
    global _launches
    _need(S, torch.float32, "S")
    _need(P, torch.bfloat16, "P")
    check(_lib.load().yb_masked_softmax(S.data_ptr(), S.stride(0), P.data_ptr(), P.stride(0), L, hw, _stream()),
          "yb_masked_softmax")
    _launches += 1
    return P


def nchw_to_nhwc_bf16(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """x f32 [Cn, N] contiguous -> out bf16 [N, ldo] (extra columns zero)."""
    global _launches
    _need(x, torch.float32, "x")
    _need(out, torch.bfloat16, "out")
    if not (x.is_contiguous() and out.is_contiguous()):
        raise YumeB200Error("nchw_to_nhwc_bf16 needs contiguous tensors")
    check(_lib.load().yb_nchw_to_nhwc_bf16(x.data_ptr(), out.data_ptr(), x.shape[1], x.shape[0], out.shape[1], _stream()),
          "yb_nchw_to_nhwc_bf16")
    _launches += 1
    return out


def nhwc_to_nchw_f32(x: torch.Tensor, out: torch.Tensor, clamp: Optional[tuple] = None) -> torch.Tensor:
    """x f32 [N, ldx] -> out f32 [Cn, N] contiguous (optionally clamped to clamp=(lo, hi))."""
    global _launches
    _need(x, torch.float32, "x")
    _need(out, torch.float32, "out")
    if clamp is not None:
        check(_lib.load().yb_nhwc_to_nchw_f32_clamp(x.data_ptr(), x.stride(0), out.data_ptr(), x.shape[0], out.shape[0],
                                                    float(clamp[0]), float(clamp[1]), _stream()), "yb_nhwc_to_nchw_f32_clamp")
        _launches += 1
        return out
    check(_lib.load().yb_nhwc_to_nchw_f32(x.data_ptr(), x.stride(0), out.data_ptr(), x.shape[0], out.shape[0], _stream()),
          "yb_nhwc_to_nchw_f32")
    _launches += 1
    return out


def vae_assemble_tiles(tiles, th, tw, tlen, tf0, out: torch.Tensor, row_limit: int, blend_extent: int, t_limit: int,
                       t_blend_extent: int) -> torch.Tensor:
    """tiles[ti][i][j]: raw decoded tiles f32 [C, frames, th[i], tw[j]] (contiguous); out f32 [C, F, H, W] (yb_vae_assemble_tiles)."""
    global _launches
    nt, ni, nj = len(tiles), len(tiles[0]), len(tiles[0][0])
    dev = out.device
    flat = [tiles[a][b][c] for a in range(nt) for b in range(ni) for c in range(nj)]
    for t in flat:
        _need(t, torch.float32, "tile")
        if not t.is_contiguous():
            raise YumeB200Error("vae_assemble_tiles needs contiguous tiles")
    table = torch.tensor([t.data_ptr() for t in flat], dtype=torch.int64).to(dev)
    meta = torch.tensor(list(th) + list(tw) + list(tlen) + list(tf0), dtype=torch.int32).to(dev)
    o_th, o_tw, o_tl, o_tf = 0, ni, ni + nj, ni + nj + nt
    _need(out, torch.float32, "out")
    C_, F_, H_, W_ = out.shape
    base = meta.data_ptr()
    check(_lib.load().yb_vae_assemble_tiles(table.data_ptr(), base + 4 * o_th, base + 4 * o_tw, base + 4 * o_tl, base + 4 * o_tf,
                                            nt, ni, nj, C_, F_, H_, W_, row_limit, blend_extent, t_limit, t_blend_extent,
                                            out.data_ptr(), _stream()), "yb_vae_assemble_tiles")
    _launches += 1
    return out


def blend(a: torch.Tensor, b: torch.Tensor, dim: int, extent: int) -> torch.Tensor:
    """In place on b (contiguous f32): cross-fade the first `extent` slices of b along `dim` with the last of a."""
    global _launches
    _need(a, torch.float32, "a")
    _need(b, torch.float32, "b")
    if not (a.is_contiguous() and b.is_contiguous()):
        raise YumeB200Error("blend needs contiguous tiles")
    extent = min(a.shape[dim], b.shape[dim], extent)
    outer = 1
    for d in b.shape[:dim]:
        outer *= d
    inner = 1
    for d in b.shape[dim + 1:]:
        inner *= d
    check(_lib.load().yb_blend(a.data_ptr(), b.data_ptr(), outer, a.shape[dim], b.shape[dim], extent, inner, _stream()),
          "yb_blend")
    _launches += 1
    return b


# ------------------------------------------------------------------------------------------------------------
# Ulysses exchange fused into the kernels (NVLink peer pointers from torch symmetric memory)
# ------------------------------------------------------------------------------------------------------------
def _ptr_array(ptrs):
    arr = (C.c_void_p * len(ptrs))(*[int(p) for p in ptrs])
    return arr


def sp_scatter_qkv(qkv: torch.Tensor, wq: torch.Tensor, wk: torch.Tensor, rope: Optional[torch.Tensor], rope_len: int,
                   head_dim: int, eps: float, peer_ptrs, rank: int, Lp: int) -> None:
    """qkv bf16 [L_local, 3C] -> RMSNorm/RoPE on q,k and scatter q|k|v chunks into the peers' receive buffers."""
    global _launches
    _need(qkv, torch.bfloat16, "qkv")
    L, C3 = qkv.shape
    check(_lib.load().yb_sp_scatter_qkv(qkv.data_ptr(), qkv.stride(0), wq.data_ptr(), wk.data_ptr(), _ptr(rope), rope_len,
                                        L, C3 // 3, head_dim, eps, _ptr_array(peer_ptrs), len(peer_ptrs), rank, Lp,
                                        _stream()), "yb_sp_scatter_qkv")
    _launches += 1


def gemm_sp_qkv(h: torch.Tensor, w_qkv: torch.Tensor, b_qkv: torch.Tensor, peer_ptrs, rank: int, Lp: int,
                sums: torch.Tensor) -> None:
    """Fused q|k|v projection whose epilogue is the Ulysses all-to-all (yb_gemm_sp_qkv). h bf16 [Lp, K]; w_qkv bf16 [3C, K]."""
    global _launches, _flops
    _need(h, torch.bfloat16, "h")
    _need(w_qkv, torch.bfloat16, "w_qkv")
    _need(b_qkv, torch.float32, "b_qkv")
    _need(sums, torch.float32, "sums")
    if not w_qkv.is_contiguous():
        raise YumeB200Error("gemm_sp_qkv weight must be contiguous")
    M, K = h.shape
    C3 = w_qkv.shape[0]
    check(_lib.load().yb_gemm_sp_qkv(h.data_ptr(), h.stride(0), w_qkv.data_ptr(), b_qkv.data_ptr(), M, C3 // 3, K,
                                     _ptr_array(peer_ptrs), len(peer_ptrs), rank, Lp, sums.data_ptr(), _stream()),
          "yb_gemm_sp_qkv")
    _launches += 1
    _flops += 2.0 * M * C3 * K


def sp_bcast_sums(local: torch.Tensor, peer_table_ptrs, rank: int, Lp: int) -> None:
    global _launches
    check(_lib.load().yb_sp_bcast_sums(local.data_ptr(), _ptr_array(peer_table_ptrs), len(peer_table_ptrs), rank, Lp, _stream()),
          "yb_sp_bcast_sums")
    _launches += 1


def sp_post_norm_rope(buf: torch.Tensor, sums: torch.Tensor, wq: torch.Tensor, wk: torch.Tensor, rope: Optional[torch.Tensor],
                      rope_len: int, L: int, Wh: int, Cdim: int, head_dim: int, eps: float) -> None:
    """buf bf16 [>= L rows, 3*Wh] received q|k|v rows in global token order; sums f32 [>= L, 2]; wq / wk f32 [Wh] = this rank's
    slice of the norm weights; rope f32 [>= L, D/2, 2] rows of the GLOBAL tokens."""
    global _launches
    _need(buf, torch.bfloat16, "buf")
    check(_lib.load().yb_sp_post_norm_rope(buf.data_ptr(), sums.data_ptr(), wq.data_ptr(), wk.data_ptr(), _ptr(rope), rope_len, L,
                                           Wh, Cdim, head_dim, eps, _stream()), "yb_sp_post_norm_rope")
    _launches += 1


def attention_sp(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out_peer_ptrs, ldo: int, heads: int, rank: int,
                 Lp: int, scale: Optional[float] = None) -> None:
    global _launches, _flops
    for n, t in (("q", q), ("k", k), ("v", v)):
        _need(t, torch.bfloat16, n)
    if scale is None:
        scale = 1.0 / math.sqrt(128.0)
    flags = 0
    ws, ws_bytes = _attention_ws(q.shape[0], k.shape[0], heads, flags, q.device)
    check(_lib.load().yb_attention_sp(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                                      _ptr_array(out_peer_ptrs), ldo, q.shape[0], k.shape[0], heads, scale,
                                      len(out_peer_ptrs), rank, Lp, flags, _ptr(ws), ws_bytes, _stream()), "yb_attention_sp")
    _launches += 1
    _flops += 4.0 * q.shape[0] * k.shape[0] * heads * 128


def vae_rms_act(x: torch.Tensor, dims, out: torch.Tensor, gamma: Optional[torch.Tensor], up: int = 1, silu: bool = True) -> torch.Tensor:
    """x bf16 [T*Hs*Ws, C] -> out bf16 [T, Hs*up, Ws*up, Cp] (contiguous): RMS_norm*gamma, SiLU, nearest 2x upsample."""
    global _launches
    _need(x, torch.bfloat16, "x")
    _need(out, torch.bfloat16, "out")
    T, Hs, Ws = dims
    if not out.is_contiguous():
        raise YumeB200Error("vae_rms_act output must be contiguous")
    check(_lib.load().yb_vae_rms_act(x.data_ptr(), x.stride(0), out.data_ptr(), _ptr(gamma), T, Hs, Ws, x.shape[1],
                                     out.shape[-1], up, 1 if silu else 0, _stream()), "yb_vae_rms_act")
    _launches += 1
    return out


def vae_dupup_add(main: torch.Tensor, x: torch.Tensor, dims, in_c: int, out_c: int, ft: int, fs: int) -> torch.Tensor:
    global _launches
    _need(main, torch.bfloat16, "main")
    _need(x, torch.bfloat16, "x")
    if not (main.is_contiguous() and x.is_contiguous()):
        raise YumeB200Error("vae_dupup_add needs dense tensors")
    check(_lib.load().yb_vae_dupup_add(main.data_ptr(), x.data_ptr(), dims[0], dims[1], dims[2], in_c, out_c, ft, fs,
                                       _stream()), "yb_vae_dupup_add")
    _launches += 1
    return main


def vae_avgdown_add(main: torch.Tensor, x: torch.Tensor, dims, in_c: int, out_c: int, ft: int, fs: int) -> torch.Tensor:
    """main bf16 [ceil(T/ft), H/fs, W/fs, out_c] += AvgDown3D(x bf16 [T, H, W, in_c]) (dims = the INPUT extents)."""
    global _launches
    _need(main, torch.bfloat16, "main")
    _need(x, torch.bfloat16, "x")
    if not (main.is_contiguous() and x.is_contiguous()) or x.shape[-1] != in_c or main.shape[-1] != out_c:
        raise YumeB200Error("vae_avgdown_add needs dense [.., in_c] / [.., out_c] tensors")
    check(_lib.load().yb_vae_avgdown_add(main.data_ptr(), x.data_ptr(), dims[0], dims[1], dims[2], in_c, out_c, ft, fs,
                                         _stream()), "yb_vae_avgdown_add")
    _launches += 1
    return main


def vae_patchify2_bf16(video: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """video f32 [3, T, H, W] -> out bf16 [T*(H/2)*(W/2), ldo] (12 patch channels, rest zero)."""
    global _launches
    _need(video, torch.float32, "video")
    _need(out, torch.bfloat16, "out")
    if video.dim() != 4 or video.shape[0] != 3 or not video.is_contiguous() or not out.is_contiguous():
        raise YumeB200Error("vae_patchify2_bf16: video must be a contiguous [3, T, H, W]")
    _, T, H, W = video.shape
    check(_lib.load().yb_vae_patchify2_bf16(video.data_ptr(), out.data_ptr(), out.shape[-1], T, H, W, _stream()),
          "yb_vae_patchify2_bf16")
    _launches += 1
    return out


def vae_unpatchify2_clamp(y: torch.Tensor, out: torch.Tensor, T: int, H: int, W: int) -> torch.Tensor:
    global _launches
    _need(y, torch.float32, "y")
    _need(out, torch.float32, "out")
    check(_lib.load().yb_vae_unpatchify2_clamp(y.data_ptr(), y.stride(0), out.data_ptr(), T, H, W, _stream()),
          "yb_vae_unpatchify2_clamp")
    _launches += 1
    return out
