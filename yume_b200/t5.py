"""umT5-XXL text encoder (`T5Encoder.forward`, wan/modules/t5.py:267-312) on the sm_90a kernels.

Per call, for B prompts of L tokens (about 8 launches per layer, all through `ops`):
  x = table[ids]                  fp32 residual stream [B*L, dim]: torch index_select of the embedding table + an exact upcast
  layers x { t5_rmsnorm -> h bf16; gemm -> q|k|v bf16; t5_attention (bias of this layer, key mask); gemm GATE_RES (o);
             t5_rmsnorm -> h; gemm -> fc1|gate bf16; t5_geglu -> mid bf16; gemm GATE_RES (fc2) }
  t5_rmsnorm (final norm) -> out in the weight dtype
The relative-position bias [heads, 2L-1] of each layer is gathered once per L from the layer's embedding, with the buckets
computed by the reference's own torch expression on the engine's device (relative_position_bucket below): the bucket
boundaries at |j - i| = 16, 32 and 64 sit exactly on a truncation of a float log, so the table follows the device's
evaluation, as the reference does on the device its embedding lives on.
The residual stream and the scores plus bias stay fp32 where the reference (bf16 weights, no autocast) rounds both to bf16.
"""
from __future__ import annotations

import contextlib
import math
import types
from typing import Dict, List

import torch

from . import ops

_F32, _BF16 = torch.float32, torch.bfloat16
HEAD_DIM = 64                                          # yb_t5_attention
RMSNORM_WIDTHS = (128, 256, 512, 768, 1024, 2048, 4096)  # yb_t5_rmsnorm instances


def relative_position_bucket(rel_pos, num_buckets, max_dist):
    """The bidirectional bucket of T5RelativeEmbedding._relative_position_bucket (t5.py:245-264), the same torch expression,
    evaluated on rel_pos's device."""
    num_buckets //= 2
    rel_buckets = (rel_pos > 0).long() * num_buckets
    rel_pos = torch.abs(rel_pos)
    max_exact = num_buckets // 2
    rel_pos_large = max_exact + (torch.log(rel_pos.float() / max_exact) / math.log(max_dist / max_exact) *
                                 (num_buckets - max_exact)).long()
    rel_pos_large = torch.min(rel_pos_large, torch.full_like(rel_pos_large, num_buckets - 1))
    return rel_buckets + torch.where(rel_pos < max_exact, rel_pos, rel_pos_large)


def gemm_block_n(M: int, N: int, sms: int) -> int:
    """N tile of a GEMM launch: 128 when its tiles fill the SMs in less time than 256-wide tiles do, counting a 128-wide
    tile as half a 256-wide one; 0 (the library's automatic choice, 256) otherwise."""
    mt = -(-M // 128)
    waves = lambda bn: -(-(mt * -(-N // bn)) // sms)               # noqa: E731
    return 128 if waves(128) * 128 < waves(256) * 256 else 0


class T5TextEncoder:
    """The encoder of a reference `T5Encoder` (pre-norm blocks, gated-GELU FFN, bidirectional relative-position bias).
    sd: its state dict (any device; bf16 or fp32). __call__(ids, mask) is T5Encoder.forward in eval mode."""

    def __init__(self, sd: Dict[str, torch.Tensor], vocab: int, dim: int, dim_attn: int, dim_ffn: int, num_heads: int,
                 num_layers: int, num_buckets: int, shared_pos: bool, eps: float = 1e-6, max_dist: int = 128,
                 device="cuda"):
        if dim_attn % num_heads or dim_attn // num_heads != HEAD_DIM:
            raise NotImplementedError(f"head_dim {dim_attn}/{num_heads} is not supported (only {HEAD_DIM})")
        if dim not in RMSNORM_WIDTHS:
            raise NotImplementedError(f"dim {dim} is not supported (one of {RMSNORM_WIDTHS})")
        wdt = sd["token_embedding.weight"].dtype
        if wdt == torch.float16:
            raise NotImplementedError("fp16 weights are not implemented (the reference's fp16_clamp is not reproduced)")
        if wdt not in (_BF16, _F32):
            raise NotImplementedError(f"weights of dtype {wdt} are not implemented")
        self.device = torch.device(device)
        self.vocab, self.dim, self.dim_attn, self.dim_ffn = vocab, dim, dim_attn, dim_ffn
        self.heads, self.layers, self.num_buckets, self.shared_pos = num_heads, num_layers, num_buckets, shared_pos
        self.eps, self.max_dist = float(eps), int(max_dist)
        self.out_dtype = wdt
        self._bias: Dict[int, List[torch.Tensor]] = {}
        self._state: Dict[tuple, dict] = {}
        dev = self.device
        f32 = lambda t: t.detach().to(device=dev, dtype=_F32).contiguous()   # noqa: E731
        bf = lambda t: t.detach().to(device=dev, dtype=_BF16).contiguous()   # noqa: E731
        self.table = sd["token_embedding.weight"].detach().to(dev).contiguous()  # gathered in its own dtype, then upcast
        self.norm_w = f32(sd["norm.weight"])
        self.shared_emb = f32(sd["pos_embedding.embedding.weight"]) if shared_pos else None
        self.blocks = []
        for i in range(num_layers):
            p = f"blocks.{i}."
            cat = lambda *names: torch.cat([sd[p + n].detach().to(device=dev, dtype=_BF16) for n in names])  # noqa: E731
            self.blocks.append(types.SimpleNamespace(
                n1=f32(sd[p + "norm1.weight"]), n2=f32(sd[p + "norm2.weight"]),
                w_qkv=cat("attn.q.weight", "attn.k.weight", "attn.v.weight").contiguous(),
                w_o=bf(sd[p + "attn.o.weight"]),
                w_ug=cat("ffn.fc1.weight", "ffn.gate.0.weight").contiguous(),
                w_fc2=bf(sd[p + "ffn.fc2.weight"]),
                emb=None if shared_pos else f32(sd[p + "pos_embedding.embedding.weight"])))

    # ---- per-L tables and buffers -------------------------------------------------------------------------------------
    def buckets(self, L: int) -> torch.Tensor:
        """int64 [2L-1] bucket of relative position j - i = d - (L - 1), computed on the engine's device."""
        rel = torch.arange(2 * L - 1, device=self.device) - (L - 1)
        return relative_position_bucket(rel, self.num_buckets, self.max_dist)

    def bias_tables(self, L: int) -> List[torch.Tensor]:
        """Per layer f32 [heads, 2L-1]: bias of (query i, key j) at column j - i + L - 1 (cached per L)."""
        tabs = self._bias.get(L)
        if tabs is None:
            bk = self.buckets(L)
            gather = lambda emb: emb[bk].t().contiguous()                     # noqa: E731
            if self.shared_pos:
                tabs = [gather(self.shared_emb)] * self.layers
            else:
                tabs = [gather(b.emb) for b in self.blocks]
            self._bias[L] = tabs
        return tabs

    def _buffers(self, B: int, L: int) -> dict:
        st = self._state.get((B, L))
        if st is None:
            dev, M, A, Fd = self.device, B * L, self.dim_attn, self.dim_ffn
            st = dict(x=torch.empty(M, self.dim, device=dev, dtype=_F32), h=torch.empty(M, self.dim, device=dev, dtype=_BF16),
                      qkv=torch.empty(M, 3 * A, device=dev, dtype=_BF16), att=torch.empty(M, A, device=dev, dtype=_BF16),
                      ug=torch.empty(M, 2 * Fd, device=dev, dtype=_BF16), mid=torch.empty(M, Fd, device=dev, dtype=_BF16))
            sms = ops._sms(dev) if dev.type == "cuda" else 132
            st["bn"] = dict(qkv=gemm_block_n(M, 3 * A, sms), o=gemm_block_n(M, self.dim, sms),
                            ug=gemm_block_n(M, 2 * Fd, sms), fc2=gemm_block_n(M, self.dim, sms))
            self._state[(B, L)] = st
        return st

    # ---- input checks -------------------------------------------------------------------------------------------------
    def check_inputs(self, ids: torch.Tensor, mask):
        """Host-side rejection before any launch: ids outside [0, vocab) raise IndexError (as nn.Embedding does on the CPU);
        a mask row without a nonzero entry raises ValueError; a mask that is not [B, L] raises NotImplementedError (3-D) or
        ValueError."""
        if ids.dim() != 2:
            raise ValueError(f"ids must be [B, L], got {tuple(ids.shape)}")
        if ids.dtype not in (torch.int64, torch.int32, torch.int16, torch.uint8, torch.int8):
            raise TypeError(f"ids must be an integer tensor, got {ids.dtype}")
        if ids.numel() == 0:
            raise ValueError("empty ids")
        lo, hi = int(ids.min()), int(ids.max())
        if lo < 0 or hi >= self.vocab:
            raise IndexError(f"index out of range in self: ids span [{lo}, {hi}], vocabulary size {self.vocab}")
        if mask is None:
            return None
        if mask.dim() == 3:
            raise NotImplementedError("3-D attention masks [B, L, L] are not implemented (only key masks [B, L])")
        if tuple(mask.shape) != tuple(ids.shape):
            raise ValueError(f"mask must be [B, L] = {tuple(ids.shape)}, got {tuple(mask.shape)}")
        keep = mask != 0
        empty = ~keep.any(dim=1)
        if bool(empty.any()):
            raise ValueError(f"mask rows {empty.nonzero().flatten().tolist()} have no nonzero entry: every key of them is masked")
        return keep

    # ---- forward ------------------------------------------------------------------------------------------------------
    def _run(self, ids: torch.Tensor, keep, B: int, L: int, out: torch.Tensor) -> torch.Tensor:
        st = self._buffers(B, L)
        x, h, qkv, att, ug, mid, bn = st["x"], st["h"], st["qkv"], st["att"], st["ug"], st["mid"], st["bn"]
        A = self.dim_attn
        x.copy_(self.table.index_select(0, ids.reshape(-1)))
        key_mask = None if keep is None else keep.to(device=self.device, dtype=torch.uint8).contiguous()
        for b, bias in zip(self.blocks, self.bias_tables(L)):
            ops.t5_rmsnorm(x, h, b.n1, self.eps)
            ops.gemm(h, b.w_qkv, None, qkv, ops.YB_EPI_BF16, block_n=bn["qkv"])
            ops.t5_attention(qkv[:, :A], qkv[:, A:2 * A], qkv[:, 2 * A:], att, B, self.heads, bias, key_mask)
            ops.gemm(att, b.w_o, None, x, ops.YB_EPI_GATE_RES, block_n=bn["o"])
            ops.t5_rmsnorm(x, h, b.n2, self.eps)
            ops.gemm(h, b.w_ug, None, ug, ops.YB_EPI_BF16, block_n=bn["ug"])
            ops.t5_geglu(ug, mid)
            ops.gemm(mid, b.w_fc2, None, x, ops.YB_EPI_GATE_RES, block_n=bn["fc2"])
        ops.t5_rmsnorm(x, out, self.norm_w, self.eps)
        return out

    @torch.no_grad()
    def __call__(self, ids: torch.Tensor, mask=None) -> torch.Tensor:
        """T5Encoder.forward(ids, mask): [B, L, dim] in the weight dtype on ids.device, every row (padded queries included)."""
        keep = self.check_inputs(ids, mask)
        B, L = ids.shape
        out = torch.empty(B * L, self.dim, device=self.device, dtype=self.out_dtype)
        with torch.cuda.device(self.device) if self.device.type == "cuda" else contextlib.nullcontext():
            self._run(ids.to(device=self.device, dtype=torch.int64), keep, B, L, out)
        return out.view(B, L, self.dim).to(ids.device)


def _config(model) -> dict:
    """The T5Encoder configuration of a live reference module; configurations the engine does not implement raise."""
    if model.shared_pos:
        rel = [model.pos_embedding]
    else:
        rel = [blk.pos_embedding for blk in model.blocks]
    if any(not r.bidirectional for r in rel):
        raise NotImplementedError("unidirectional position buckets (decoder) are not implemented")
    if len({r.max_dist for r in rel}) != 1:
        raise NotImplementedError("per-layer max_dist values differ")
    eps = {model.norm.eps} | {blk.norm1.eps for blk in model.blocks} | {blk.norm2.eps for blk in model.blocks}
    if len(eps) != 1:
        raise NotImplementedError("the norms use different eps values")
    return dict(vocab=int(model.token_embedding.num_embeddings), dim=int(model.dim), dim_attn=int(model.dim_attn),
                dim_ffn=int(model.dim_ffn), num_heads=int(model.num_heads), num_layers=int(model.num_layers),
                num_buckets=int(model.num_buckets), shared_pos=bool(model.shared_pos), eps=float(eps.pop()),
                max_dist=int(rel[0].max_dist))


def install_t5(text_encoder, device="cuda") -> T5TextEncoder:
    """Re-bind `text_encoder.model.forward` of a live reference `T5EncoderModel` (wan/modules/t5.py:472-513; `.model` is the
    `T5Encoder` its __call__ runs) to the engine. The contract `forward(ids, mask=None) -> [B, L, dim]` is kept: every row, the
    weight dtype, on ids.device. The weights are copied to `device` at install time, so later `.to()` / `.cpu()` calls on the
    module move only the reference's copy; call install_t5 again after reloading weights."""
    model = text_encoder.model
    cfg = _config(model)
    enc = T5TextEncoder(model.state_dict(), device=device, **cfg)

    def forward(self, ids, mask=None, _enc=enc):
        if self.training:
            raise NotImplementedError("T5Encoder in training mode (dropout active) is not implemented: call .eval()")
        return _enc(ids, mask)

    model.forward = types.MethodType(forward, model)
    text_encoder.yume_b200_t5 = enc
    return enc
