"""CLIP ViT-H/14 image encoder of the 14B I2V path (`CLIPModel.visual`, wan/modules/clip.py:527-542) on the sm_90a kernels.

Per image (~220 launches, all through `ops`):
  resize_bicubic_normalize     F.interpolate(bicubic) + mul_(0.5).add_(0.5) + Normalize, fp32 [3, S, S]
  patchify                     bf16 patch rows [(S/p)^2, 592], columns in Conv2d weight order c*196 + ky*14 + kx
  stream = table; gemm GATE_RES  stream rows 1.. += patches @ W_patch^T; table row 0 = cls + pos[0], rows 1.. = pos
  ln_modulate (affine, f32)    pre_norm
  31 x { ln_modulate -> h bf16; gemm -> q|k|v bf16 (heads padded 80 -> 128); attention; gemm GATE_RES (o-proj);
         ln_modulate -> h; gemm GELU_ERF -> mid bf16; gemm GATE_RES (fc2) }
The residual stream is fp32 (as in the reference under fp16 autocast, where the cat of the fp16 conv output with the bf16
cls row promotes it). The attention kernel has head_dim 128 only: each 80-wide head is padded with 48 zero q/k/v columns
(zero weight rows, zero bias), which add 0*0 to every score, produce P*0 = 0 output columns, and meet zero columns of the
o-projection weight — the result is that of a head_dim-80 kernel with the same accumulation order.
"""
from __future__ import annotations

import contextlib
import math
import types
from typing import Dict, List

import torch
import torch.nn.functional as F

from . import ops

_F32, _BF16 = torch.float32, torch.bfloat16
HEAD_PAD = 128         # head width of the attention kernel


def _k_pad(k: int) -> int:
    return (k + 7) // 8 * 8    # GEMM K % 8 == 0


class ClipVisionEncoder:
    """The vision tower of a reference `VisionTransformer` (pre-norm, gelu, token pool) with `use_31_block=True`: the first
    `layers - 1` blocks run, no post_norm, no head. sd: its state dict (any dtype / device; only what runs is uploaded).
    encode(images) takes the list `CLIPModel.visual` takes and returns fp32 [N, (image_size/patch)^2 + 1, dim]."""

    def __init__(self, sd: Dict[str, torch.Tensor], image_size: int, patch_size: int, dim: int, heads: int, layers: int,
                 mlp_ratio: float, eps: float, mean, std, device="cuda"):
        if image_size % patch_size:
            raise NotImplementedError("image_size must be a multiple of patch_size")
        if dim % heads or dim // heads > HEAD_PAD:
            raise NotImplementedError(f"head_dim {dim}/{heads} is not supported (<= {HEAD_PAD})")
        self.device = torch.device(device)
        self.image_size, self.patch_size, self.dim, self.heads = image_size, patch_size, dim, heads
        self.head_dim = dim // heads
        self.blocks_run = layers - 1                                     # transformer[:-1] (clip.py:295-297)
        self.mlp = int(dim * mlp_ratio)
        self.eps = float(eps)
        self.grid = image_size // patch_size
        self.tokens = self.grid ** 2 + 1
        if tuple(sd["pos_embedding"].shape) != (1, self.tokens, dim):
            raise NotImplementedError("pos_embedding does not match the patch grid (pos_interpolate is not implemented)")
        self.k_patch = 3 * patch_size * patch_size
        self.use_cuda_graph = False
        self._state: Dict[tuple, dict] = {}
        dev = self.device
        f32 = lambda t: t.detach().to(device=dev, dtype=_F32).contiguous()  # noqa: E731
        self.mean = torch.tensor([float(v) for v in mean], dtype=_F32).to(dev)   # T.Normalize's fp32 tensors
        self.std = torch.tensor([float(v) for v in std], dtype=_F32).to(dev)

        w = sd["patch_embedding.weight"].detach().float().reshape(dim, self.k_patch)   # c*p*p + ky*p + kx
        self.w_patch = F.pad(w, (0, _k_pad(self.k_patch) - self.k_patch)).to(device=dev, dtype=_BF16).contiguous()
        cls = sd["cls_embedding"].detach().to(_F32).reshape(1, dim)
        table = sd["pos_embedding"].detach().to(_F32).reshape(self.tokens, dim).clone()
        table[0] = cls[0] + table[0]                                     # cat([cls, x]) + pos, row 0 (clip.py:285,290)
        self.table = table.to(dev).contiguous()
        self.pre_w, self.pre_b = f32(sd["pre_norm.weight"]), f32(sd["pre_norm.bias"])

        H, d, HP = heads, self.head_dim, HEAD_PAD
        self.blocks = []
        for i in range(self.blocks_run):
            p = f"transformer.{i}."
            wqkv = sd[p + "attn.to_qkv.weight"].detach().float().reshape(3, H, d, dim)   # rows (part, head, d)
            bqkv = sd[p + "attn.to_qkv.bias"].detach().float().reshape(3, H, d)
            wqkv = F.pad(wqkv, (0, 0, 0, HP - d)).reshape(3 * H * HP, dim)
            bqkv = F.pad(bqkv, (0, HP - d)).reshape(3 * H * HP)
            wo = sd[p + "attn.proj.weight"].detach().float().reshape(dim, H, d)           # columns (head, d)
            wo = F.pad(wo, (0, HP - d)).reshape(dim, H * HP)
            self.blocks.append(types.SimpleNamespace(
                ln1_w=f32(sd[p + "norm1.weight"]), ln1_b=f32(sd[p + "norm1.bias"]),
                w_qkv=wqkv.to(device=dev, dtype=_BF16).contiguous(), b_qkv=bqkv.to(dev).contiguous(),
                w_o=wo.to(device=dev, dtype=_BF16).contiguous(), b_o=f32(sd[p + "attn.proj.bias"]),
                ln2_w=f32(sd[p + "norm2.weight"]), ln2_b=f32(sd[p + "norm2.bias"]),
                w_fc1=sd[p + "mlp.0.weight"].detach().to(device=dev, dtype=_BF16).contiguous(), b_fc1=f32(sd[p + "mlp.0.bias"]),
                w_fc2=sd[p + "mlp.2.weight"].detach().to(device=dev, dtype=_BF16).contiguous(), b_fc2=f32(sd[p + "mlp.2.bias"])))

    # ---- buffers ------------------------------------------------------------------------------------------------------
    def _buffers(self, shape: tuple) -> dict:
        """Work buffers of one input shape [3, H, W] (the graph of that shape captures their addresses)."""
        st = self._state.get(shape)
        if st is None:
            dev, S, T, HW = self.device, self.image_size, self.tokens, self.heads * HEAD_PAD
            st = dict(img=torch.empty(3, S, S, device=dev, dtype=_F32),
                      # columns k_patch .. K-1 are the K padding of both operands: zeroed here, never written
                      patches=torch.zeros(self.grid ** 2, _k_pad(self.k_patch), device=dev, dtype=_BF16),
                      e=torch.empty(T, self.dim, device=dev, dtype=_F32), x=torch.empty(T, self.dim, device=dev, dtype=_F32),
                      h=torch.empty(T, self.dim, device=dev, dtype=_BF16),
                      qkv=torch.empty(T, 3 * HW, device=dev, dtype=_BF16), att=torch.empty(T, HW, device=dev, dtype=_BF16),
                      mid=torch.empty(T, self.mlp, device=dev, dtype=_BF16))
            self._state[shape] = st
        return st

    # ---- forward ------------------------------------------------------------------------------------------------------
    def _run(self, img: torch.Tensor, st: dict) -> torch.Tensor:
        """img f32 [3, H, W] (any strides) -> st['x'] f32 [tokens, dim]."""
        S, p, HW = self.image_size, self.patch_size, self.heads * HEAD_PAD
        ops.resize_bicubic_normalize(img, st["img"], self.mean, self.std)
        ops.patchify(st["img"].view(3, 1, S, S), st["patches"], p, p)
        e, x, h, qkv, att, mid = st["e"], st["x"], st["h"], st["qkv"], st["att"], st["mid"]
        e.copy_(self.table)
        ops.gemm(st["patches"], self.w_patch, None, e[1:], ops.YB_EPI_GATE_RES)
        ops.ln_modulate(e, x, None, None, weight=self.pre_w, bias=self.pre_b, eps=self.eps)
        scale = 1.0 / math.sqrt(self.head_dim)
        for b in self.blocks:
            ops.ln_modulate(x, h, None, None, weight=b.ln1_w, bias=b.ln1_b, eps=self.eps)
            ops.gemm(h, b.w_qkv, b.b_qkv, qkv, ops.YB_EPI_BF16)
            ops.attention(qkv[:, :HW], qkv[:, HW:2 * HW], qkv[:, 2 * HW:], att, self.heads, scale=scale)
            ops.gemm(att, b.w_o, b.b_o, x, ops.YB_EPI_GATE_RES)
            ops.ln_modulate(x, h, None, None, weight=b.ln2_w, bias=b.ln2_b, eps=self.eps)
            ops.gemm(h, b.w_fc1, b.b_fc1, mid, ops.YB_EPI_GELU_ERF_BF16)
            ops.gemm(mid, b.w_fc2, b.b_fc2, x, ops.YB_EPI_GATE_RES)
        return x

    def _run_graphed(self, img: torch.Tensor, st: dict) -> torch.Tensor:
        """CUDA-graph replay of _run for this input shape: the image is copied into a static buffer, the graph (captured
        after one eager warm-up) replays every launch."""
        g = st.get("graph")
        if g is None:
            st["in"] = torch.empty(img.shape, device=self.device, dtype=_F32)
            st["in"].copy_(img)
            self._run(st["in"], st)                                    # warm-up: first launches, allocator
            torch.cuda.synchronize(self.device)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                self._run(st["in"], st)
            st["graph"] = g = graph
        else:
            st["in"].copy_(img, non_blocking=True)
        g.replay()
        return st["x"]

    def frames(self, videos) -> List[torch.Tensor]:
        """The [3, H, W] images of `videos` in the reference's order: each entry u is a [3, F, H, W] tensor whose F frames
        become F images (`u.transpose(0, 1)` then cat, clip.py:530-536). `videos` is iterated like the reference does."""
        out = []
        for u in videos:
            if u.dim() != 4:
                raise ValueError(f"each image must be a [3, F, H, W] tensor (got {tuple(u.shape)}); "
                                 "F.interpolate would reject it as well")
            if u.shape[0] != 3:
                raise NotImplementedError(f"CLIP images have 3 channels, got {u.shape[0]}")
            if u.dtype != _F32:
                raise NotImplementedError(f"images must be float32 (the reference resizes in their dtype), got {u.dtype}")
            u = u.to(self.device)
            out.extend(u[:, f] for f in range(u.shape[1]))
        return out

    @torch.no_grad()
    def encode(self, videos, interpolation: bool = False) -> torch.Tensor:
        """CLIPModel.visual(videos) without post_norm / head: fp32 [N, tokens, dim], one image after another."""
        if interpolation:
            raise NotImplementedError("interpolation=True (pos_interpolate) is not implemented")
        imgs = self.frames(videos)
        if not imgs:
            raise ValueError("no images")
        out = torch.empty(len(imgs), self.tokens, self.dim, device=self.device, dtype=_F32)
        with torch.cuda.device(self.device) if self.device.type == "cuda" else contextlib.nullcontext():
            for i, img in enumerate(imgs):
                st = self._buffers(tuple(img.shape))
                x = self._run_graphed(img, st) if self.use_cuda_graph else self._run(img, st)
                out[i].copy_(x)
        return out


def _config(clip) -> dict:
    """The VisionTransformer configuration of a live reference CLIPModel; configurations the engine does not implement raise."""
    vis = clip.model.visual
    if vis.pool_type == "attn_pool":
        raise NotImplementedError("pool_type='attn_pool' is not implemented")
    if getattr(vis, "pre_norm", None) is None:
        raise NotImplementedError("VisionTransformer without pre_norm is not implemented")
    for blk in vis.transformer:
        if blk.post_norm:
            raise NotImplementedError("post_norm blocks are not implemented")
        mlp = blk.mlp
        if not isinstance(mlp, torch.nn.Sequential):
            raise NotImplementedError("activation='swi_glu' is not implemented")
        act = mlp[1]
        if not (isinstance(act, torch.nn.GELU) and act.approximate == "none"):
            raise NotImplementedError(f"activation {type(act).__name__} is not implemented (only exact GELU, 'gelu')")
        if blk.causal or blk.attn.causal:
            raise NotImplementedError("causal attention blocks are not implemented")
    norm = clip.transforms.transforms[-1]
    return dict(image_size=int(clip.model.image_size), patch_size=int(vis.patch_size), dim=int(vis.dim),
                heads=int(vis.num_heads), layers=int(vis.num_layers), mlp_ratio=vis.mlp_ratio, eps=float(vis.norm_eps),
                mean=list(norm.mean), std=list(norm.std))


def install_clip(clip, device="cuda") -> ClipVisionEncoder:
    """Re-bind `clip.visual(videos)` of a live reference `CLIPModel` (wan/modules/clip.py:501-542) to the engine. The
    list-in / tensor-out contract is kept; the result has dtype promote_types(clip.dtype, visual weight dtype), fp32 for the
    shipped I2V config (fp16 autocast over bf16 weights). The weights are copied at install time: call it again after
    reloading them."""
    cfg = _config(clip)
    vis = clip.model.visual
    sd = vis.state_dict()
    enc = ClipVisionEncoder(sd, device=device, **cfg)
    out_dtype = torch.promote_types(clip.dtype, next(vis.parameters()).dtype)

    def visual(self, videos, _enc=enc, _dtype=out_dtype):
        return _enc.encode(videos).to(_dtype)

    clip.visual = types.MethodType(visual, clip)
    clip.yume_b200_clip = enc
    return enc
