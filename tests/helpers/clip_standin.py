"""TEST INFRASTRUCTURE: a stand-in for the reference's `CLIPModel` (wan/modules/clip.py:501-542) with the attributes
yume_b200.clip.install_clip reads — `model.image_size`, `model.visual` (a VisionTransformer-shaped module whose state-dict keys
are the reference's), `transforms.transforms[-1]` (Normalize) and `dtype`. Built on the meta device and filled by
`load_state_dict(assign=True)`, so the ViT-H/14 width costs no init."""
import types

import torch
import torch.nn as nn
import torchvision.transforms as T

from oracle import clip as oclip


class QuickGELU(nn.Module):
    def forward(self, x):
        return x * torch.sigmoid(1.702 * x)


class SwiGLU(nn.Module):
    def __init__(self, dim, mid):
        super().__init__()
        self.fc1, self.fc2, self.fc3 = nn.Linear(dim, mid), nn.Linear(dim, mid), nn.Linear(mid, dim)


class _Attn(nn.Module):
    def __init__(self, dim, causal):
        super().__init__()
        self.causal = causal
        self.to_qkv, self.proj = nn.Linear(dim, 3 * dim), nn.Linear(dim, dim)


class _Block(nn.Module):
    def __init__(self, dim, mlp_ratio, activation, post_norm, causal=False):
        super().__init__()
        mid = int(dim * mlp_ratio)
        self.post_norm, self.causal = post_norm, causal
        self.norm1, self.norm2 = nn.LayerNorm(dim), nn.LayerNorm(dim)
        self.attn = _Attn(dim, causal)
        if activation == "swi_glu":
            self.mlp = SwiGLU(dim, mid)
        else:
            act = QuickGELU() if activation == "quick_gelu" else nn.GELU()
            self.mlp = nn.Sequential(nn.Linear(dim, mid), act, nn.Linear(mid, dim), nn.Dropout(0.0))


class _Visual(nn.Module):
    def __init__(self, image_size, patch_size, dim, heads, layers, mlp_ratio, eps, out_dim, activation="gelu",
                 pool_type="token", post_norm=False):
        super().__init__()
        self.image_size, self.patch_size, self.dim, self.mlp_ratio = image_size, patch_size, dim, mlp_ratio
        self.num_heads, self.num_layers, self.pool_type, self.norm_eps = heads, layers, pool_type, eps
        self.patch_embedding = nn.Conv2d(3, dim, patch_size, patch_size, bias=False)
        self.cls_embedding = nn.Parameter(torch.empty(1, 1, dim))
        self.pos_embedding = nn.Parameter(torch.empty(1, (image_size // patch_size) ** 2 + 1, dim))
        self.pre_norm = nn.LayerNorm(dim, eps=eps)
        self.transformer = nn.Sequential(*[_Block(dim, mlp_ratio, activation, post_norm) for _ in range(layers)])
        self.post_norm = nn.LayerNorm(dim, eps=eps)
        self.head = nn.Parameter(torch.empty(dim, out_dim))


def make_clip(sd, cfg, out_dim, dtype=torch.float16, param_dtype=torch.float32, device="cpu", **variant):
    """Stand-in CLIPModel over state dict `sd` (oracle.clip key layout). `variant` passes activation / pool_type / post_norm
    through to the module so unsupported configurations can be built."""
    with torch.device("meta"):
        vis = _Visual(cfg["image_size"], cfg["patch_size"], cfg["dim"], cfg["heads"], cfg["layers"], cfg["mlp_ratio"],
                      cfg["eps"], out_dim, **variant)
    if variant.get("activation") != "swi_glu":
        vis.load_state_dict({k: v.to(device=device, dtype=param_dtype) for k, v in sd.items()}, assign=True)
    model = types.SimpleNamespace(image_size=cfg["image_size"], visual=vis)
    transforms = T.Compose([T.Normalize(mean=list(oclip.MEAN), std=list(oclip.STD))])
    clip = types.SimpleNamespace(model=model, transforms=transforms, dtype=dtype, device=device)
    return clip
