"""Functional restatement of the reference's CLIP image encoder as the I2V pipeline calls it: `CLIPModel.visual`
(wan/modules/clip.py:527-542) with `use_31_block=True`, for the gelu / pre-norm / token-pool configuration of
`clip_xlm_roberta_vit_h_14` (:471-498).

In fp32 (fp32 state dict, no autocast) this is the arithmetic of the reference's eager code run in fp32. The reference's
`flash_attention` (wan/modules/attention.py:52-60) rounds fp32 q, k, v to bf16 before the kernel and returns the result in the
input dtype; `_attention` below keeps that contract with SDPA. Under `torch.autocast("cuda", torch.float16)` with a bf16 state
dict it runs the way the shipped I2V config does (`clip_dtype = torch.float16`, weights cast to bf16 by
wan/image2video.py:208): fp16 linears / conv, fp32 LayerNorm, an fp32 residual stream, fp16 attention operands.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

MEAN = (0.48145466, 0.4578275, 0.40821073)      # clip.py:457 (OpenAI CLIP)
STD = (0.26862954, 0.26130258, 0.27577711)      # clip.py:458

# the vision tower of clip_xlm_roberta_vit_h_14 (clip.py:475-484, VisionTransformer defaults :211-226)
VIT_H_14 = dict(image_size=224, patch_size=14, dim=1280, heads=16, layers=32, mlp_ratio=4, eps=1e-5)


def param_shapes(image_size, patch_size, dim, heads, layers, mlp_ratio, eps=1e-5, out_dim=1024):
    """State-dict keys -> shapes of VisionTransformer(pool_type='token', pre_norm=True, activation='gelu') (clip.py:246-277)."""
    del heads, eps
    mid = int(dim * mlp_ratio)
    shapes = {"cls_embedding": (1, 1, dim), "pos_embedding": (1, (image_size // patch_size) ** 2 + 1, dim),
              "patch_embedding.weight": (dim, 3, patch_size, patch_size),
              "pre_norm.weight": (dim,), "pre_norm.bias": (dim,)}
    for i in range(layers):
        p = f"transformer.{i}."
        shapes.update({p + "norm1.weight": (dim,), p + "norm1.bias": (dim,),
                       p + "attn.to_qkv.weight": (3 * dim, dim), p + "attn.to_qkv.bias": (3 * dim,),
                       p + "attn.proj.weight": (dim, dim), p + "attn.proj.bias": (dim,),
                       p + "norm2.weight": (dim,), p + "norm2.bias": (dim,),
                       p + "mlp.0.weight": (mid, dim), p + "mlp.0.bias": (mid,),
                       p + "mlp.2.weight": (dim, mid), p + "mlp.2.bias": (dim,)})
    shapes.update({"post_norm.weight": (dim,), "post_norm.bias": (dim,), "head": (dim, out_dim)})
    return shapes


def make_state_dict(seed, image_size, patch_size, dim, heads, layers, mlp_ratio, eps=1e-5, out_dim=1024):
    """Seeded fp32 weights of param_shapes(...): matrices ~ N(0, 1/fan_in), LayerNorm weights 1 + N(0, 0.1^2), biases and
    embeddings ~ N(0, 0.02^2)-ish, so that 30 residual blocks keep the stream at O(1)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in param_shapes(image_size, patch_size, dim, heads, layers, mlp_ratio, eps, out_dim).items():
        if k.endswith("norm1.weight") or k.endswith("norm2.weight") or k.endswith("norm.weight"):
            t = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif k.endswith(".bias"):
            t = 0.02 * torch.randn(shp, generator=g)
        elif k in ("cls_embedding", "pos_embedding", "head"):
            t = dim ** -0.5 * torch.randn(shp, generator=g)          # clip.py:247,255-258
        else:
            fan_in = shp[1] if len(shp) == 2 else shp[1] * shp[2] * shp[3]
            t = fan_in ** -0.5 * torch.randn(shp, generator=g)
        sd[k] = t
    return sd


def preprocess(videos, image_size, mean=MEAN, std=STD):
    """clip.py:529-537: bicubic resize of every [3, F, H, W] entry to image_size^2 (fp32, align_corners=False, no antialias),
    [-1, 1] -> [0, 1], then T.Normalize (sub_(mean).div_(std), mean / std as fp32 tensors)."""
    size = (image_size,) * 2
    x = torch.cat([F.interpolate(u.transpose(0, 1), size=size, mode="bicubic", align_corners=False) for u in videos])
    x = x.mul_(0.5).add_(0.5)
    m = torch.as_tensor(mean, dtype=x.dtype, device=x.device).view(-1, 1, 1)
    s = torch.as_tensor(std, dtype=x.dtype, device=x.device).view(-1, 1, 1)
    return x.sub_(m).div_(s)


def _layer_norm(x, w, b, eps):
    """clip.py:47-51: LayerNorm over x.float(), back to x's dtype."""
    return F.layer_norm(x.float(), (x.shape[-1],), w, b, eps).type_as(x)


def _attention(q, k, v):
    """flash_attention(q, k, v) [B, L, n, d] of wan/modules/attention.py:24-130 (no mask, non-causal, scale 1/sqrt(d)):
    non-half inputs are rounded to bf16 first, the result is returned in the input dtype."""
    out_dtype = q.dtype
    half = lambda t: t if t.dtype in (torch.float16, torch.bfloat16) else t.to(torch.bfloat16)  # noqa: E731
    o = F.scaled_dot_product_attention(half(q).transpose(1, 2), half(k).transpose(1, 2), half(v).transpose(1, 2))
    return o.transpose(1, 2).contiguous().type(out_dtype)


def transformer(sd, x, dim, heads, layers, eps=1e-5):
    """VisionTransformer.forward (clip.py:279-301) from the embeddings on, use_31_block=True: blocks 0 .. layers-2."""
    n, d = heads, dim // heads
    for i in range(layers - 1):                                    # transformer[:-1], clip.py:295-297
        p = f"transformer.{i}."
        h = _layer_norm(x, sd[p + "norm1.weight"], sd[p + "norm1.bias"], eps)
        b, s, c = h.shape
        q, k, v = F.linear(h, sd[p + "attn.to_qkv.weight"], sd[p + "attn.to_qkv.bias"]).view(b, s, 3, n, d).unbind(2)
        a = _attention(q, k, v).reshape(b, s, c)                   # SelfAttention.forward, clip.py:74-92
        x = x + F.linear(a, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
        h = _layer_norm(x, sd[p + "norm2.weight"], sd[p + "norm2.bias"], eps)
        m = F.gelu(F.linear(h, sd[p + "mlp.0.weight"], sd[p + "mlp.0.bias"]))            # nn.GELU(): erf form
        x = x + F.linear(m, sd[p + "mlp.2.weight"], sd[p + "mlp.2.bias"])                 # AttentionBlock, :146-154
    return x


def embed(sd, x, patch_size, eps=1e-5):
    """clip.py:283-292: patch conv (no bias), cls row in front, + pos_embedding, pre_norm."""
    b = x.shape[0]
    x = F.conv2d(x, sd["patch_embedding.weight"], stride=patch_size).flatten(2).permute(0, 2, 1)
    x = torch.cat([sd["cls_embedding"].expand(b, -1, -1), x], dim=1)
    x = x + sd["pos_embedding"]
    return _layer_norm(x, sd["pre_norm.weight"], sd["pre_norm.bias"], eps)


def visual(sd, videos, image_size, patch_size, dim, heads, layers, mlp_ratio=4, eps=1e-5, mean=MEAN, std=STD):
    """CLIPModel.visual(videos): list of [3, F, H, W] fp32 images in [-1, 1] -> [sum F, (image_size/patch)^2 + 1, dim].
    Preprocessing always runs outside autocast in fp32 (the reference enters autocast after it)."""
    del mlp_ratio
    with torch.autocast("cuda", enabled=False):
        x = preprocess(videos, image_size, mean, std)
    return transformer(sd, embed(sd, x, patch_size, eps), dim, heads, layers, eps)
