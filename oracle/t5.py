"""Functional restatement of the reference's umT5 text encoder: `T5Encoder.forward` (wan/modules/t5.py:267-312) and the blocks
it runs (`T5SelfAttention`, `T5Attention`, `T5FeedForward`, `T5LayerNorm`, `T5RelativeEmbedding`, :53-264), for the
encoder-only configuration `umt5_xxl` builds (:456-469).

`encode(..., dtype=torch.float32)` is the reference's arithmetic in fp32. With `dtype=torch.bfloat16` and bf16 weights it runs
the way the pipelines run the shipped model (`t5_dtype = torch.bfloat16`, no autocast): bf16 linears, bf16 residual stream,
bf16 scores plus bias, the softmax in fp32 rounded back to bf16. Weights of any stored dtype are converted to `dtype` one
layer at a time, so an fp32 run over bf16 weights holds one fp32 layer at a time.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

# the encoder of umt5_xxl (t5.py:456-469) as T5Encoder sees it (encoder_only=True: vocab = vocab_size)
UMT5_XXL = dict(vocab=256384, dim=4096, dim_attn=4096, dim_ffn=10240, num_heads=64, num_layers=24, num_buckets=32,
                shared_pos=False)


def param_shapes(vocab, dim, dim_attn, dim_ffn, num_heads, num_layers, num_buckets, shared_pos):
    """State-dict keys -> shapes of T5Encoder(vocab, dim, dim_attn, dim_ffn, num_heads, num_layers, num_buckets, shared_pos)."""
    shapes = {"token_embedding.weight": (vocab, dim)}
    if shared_pos:
        shapes["pos_embedding.embedding.weight"] = (num_buckets, num_heads)
    for i in range(num_layers):
        p = f"blocks.{i}."
        shapes.update({p + "norm1.weight": (dim,), p + "attn.q.weight": (dim_attn, dim), p + "attn.k.weight": (dim_attn, dim),
                       p + "attn.v.weight": (dim_attn, dim), p + "attn.o.weight": (dim, dim_attn), p + "norm2.weight": (dim,),
                       p + "ffn.gate.0.weight": (dim_ffn, dim), p + "ffn.fc1.weight": (dim_ffn, dim),
                       p + "ffn.fc2.weight": (dim, dim_ffn)})
        if not shared_pos:
            shapes[p + "pos_embedding.embedding.weight"] = (num_buckets, num_heads)
    shapes["norm.weight"] = (dim,)
    return shapes


def _std(key, vocab, dim, dim_attn, dim_ffn, num_heads, num_buckets):
    """The reference's init_weights (t5.py:27-43) per key; norm weights are drawn around 1 instead of set to 1, so that a
    missing norm weight is seen."""
    if key == "token_embedding.weight":
        return 1.0
    if key.endswith("pos_embedding.embedding.weight"):
        return (2 * num_buckets * num_heads) ** -0.5
    if key.endswith("attn.q.weight"):
        return (dim * dim_attn) ** -0.5
    if key.endswith("attn.k.weight") or key.endswith("attn.v.weight"):
        return dim ** -0.5
    if key.endswith("attn.o.weight"):
        return (num_heads * dim_attn) ** -0.5
    if key.endswith("ffn.gate.0.weight") or key.endswith("ffn.fc1.weight"):
        return dim ** -0.5
    if key.endswith("ffn.fc2.weight"):
        return dim_ffn ** -0.5
    return None                                                   # norm weights


def make_state_dict(seed, vocab, dim, dim_attn, dim_ffn, num_heads, num_layers, num_buckets, shared_pos, device="cpu",
                    dtype=torch.float32):
    """Seeded weights of param_shapes(...): N(0, std^2) with the reference's init stds, norm weights 1 + N(0, 0.1^2). Drawn in
    fp32 from a generator on `device` (so the real width can be generated on the GPU), stored as `dtype`."""
    g = torch.Generator(device=device).manual_seed(seed)
    sd = {}
    for k, shp in param_shapes(vocab, dim, dim_attn, dim_ffn, num_heads, num_layers, num_buckets, shared_pos).items():
        t = torch.randn(shp, generator=g, device=device)
        std = _std(k, vocab, dim, dim_attn, dim_ffn, num_heads, num_buckets)
        t = t.mul_(std) if std is not None else t.mul_(0.1).add_(1.0)
        sd[k] = t.to(dtype)
    return sd


def relative_position_bucket(rel_pos, num_buckets, max_dist=128, bidirectional=True):
    """T5RelativeEmbedding._relative_position_bucket (t5.py:245-264), evaluated on rel_pos's device as the reference does."""
    if bidirectional:
        num_buckets //= 2
        rel_buckets = (rel_pos > 0).long() * num_buckets
        rel_pos = torch.abs(rel_pos)
    else:
        rel_buckets = 0
        rel_pos = -torch.min(rel_pos, torch.zeros_like(rel_pos))
    max_exact = num_buckets // 2
    rel_pos_large = max_exact + (torch.log(rel_pos.float() / max_exact) / math.log(max_dist / max_exact) *
                                 (num_buckets - max_exact)).long()
    rel_pos_large = torch.min(rel_pos_large, torch.full_like(rel_pos_large, num_buckets - 1))
    return rel_buckets + torch.where(rel_pos < max_exact, rel_pos, rel_pos_large)


def bucket_table(L, num_buckets, max_dist=128, device="cpu"):
    """[L, L] bucket of (query i, key j): T5RelativeEmbedding.forward(L, L) before the embedding lookup (t5.py:233-243)."""
    rel = torch.arange(L, device=device).unsqueeze(0) - torch.arange(L, device=device).unsqueeze(1)
    return relative_position_bucket(rel, num_buckets, max_dist)


def position_bias(emb, L, max_dist=128):
    """[1, heads, L, L] relative-position bias of embedding weight emb [num_buckets, heads], buckets on emb's device."""
    return emb[bucket_table(L, emb.shape[0], max_dist, emb.device)].permute(2, 0, 1).unsqueeze(0).contiguous()


def rms_norm(x, w, eps):
    """T5LayerNorm.forward (t5.py:61-66): the rsqrt of the fp32 mean square, back to the weight's dtype if it is half."""
    x = x * torch.rsqrt(x.float().pow(2).mean(dim=-1, keepdim=True) + eps)
    if w.dtype in (torch.float16, torch.bfloat16):
        x = x.type_as(w)
    return w * x


def gelu(x):
    """The tanh GELU of t5.py:46-50, in x's dtype."""
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def attention(x, mask, pos_bias, wq, wk, wv, wo, num_heads):
    """T5Attention.forward (t5.py:86-120) for self-attention: no scale, bias + finfo.min at masked keys, softmax in fp32."""
    b, n = x.size(0), num_heads
    c = wq.shape[0] // n
    q = F.linear(x, wq).view(b, -1, n, c)
    k = F.linear(x, wk).view(b, -1, n, c)
    v = F.linear(x, wv).view(b, -1, n, c)
    attn_bias = x.new_zeros(b, n, q.size(1), k.size(1))
    if pos_bias is not None:
        attn_bias += pos_bias
    if mask is not None:
        attn_bias.masked_fill_(mask.view(b, 1, 1, -1) == 0, torch.finfo(x.dtype).min)
    attn = torch.einsum("binc,bjnc->bnij", q, k) + attn_bias
    attn = F.softmax(attn.float(), dim=-1).type_as(attn)
    x = torch.einsum("bnij,bjnc->binc", attn, v)
    return F.linear(x.reshape(b, -1, n * c), wo)


def encode(sd, ids, mask, dim, dim_attn, dim_ffn, num_heads, num_layers, num_buckets, shared_pos, vocab=None, eps=1e-6,
           max_dist=128, dtype=torch.float32):
    """T5Encoder.forward(ids, mask) in eval mode (dropout off): ids [B, L] -> [B, L, dim] in `dtype`. mask [B, L] or None."""
    del dim, dim_attn, dim_ffn, vocab
    L = ids.shape[1]
    x = F.embedding(ids, sd["token_embedding.weight"]).to(dtype)
    shared = position_bias(sd["pos_embedding.embedding.weight"].to(dtype), L, max_dist) if shared_pos else None
    for i in range(num_layers):
        p = f"blocks.{i}."
        w = lambda name: sd[p + name].to(dtype)                                  # noqa: E731  (one layer at a time)
        e = shared if shared_pos else position_bias(w("pos_embedding.embedding.weight"), L, max_dist)
        h = rms_norm(x, w("norm1.weight"), eps)
        x = x + attention(h, mask, e, w("attn.q.weight"), w("attn.k.weight"), w("attn.v.weight"), w("attn.o.weight"),
                          num_heads)
        h = rms_norm(x, w("norm2.weight"), eps)
        x = x + F.linear(F.linear(h, w("ffn.fc1.weight")) * gelu(F.linear(h, w("ffn.gate.0.weight"))), w("ffn.fc2.weight"))
    return rms_norm(x, sd["norm.weight"].to(dtype), eps)
