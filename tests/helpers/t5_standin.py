"""TEST INFRASTRUCTURE: a stand-in for the reference's `T5EncoderModel` (wan/modules/t5.py:472-513) whose `.model` mirrors
`T5Encoder` (:267-312): the attributes yume_b200.t5.install_t5 reads (dim, dim_attn, dim_ffn, num_heads, num_layers,
num_buckets, shared_pos, token_embedding, pos_embedding with bidirectional / max_dist, the norms' eps) and the reference's
state-dict keys (tests/test_t5_cpu.py checks them against the layout recorded from the reference's own umt5_xxl). Its forward,
until install_t5 re-binds it, is oracle/t5.py in the weight dtype. Built on the meta device and filled by
`load_state_dict(assign=True)`, so the umT5-XXL width costs no init."""
import types

import torch
import torch.nn as nn

from oracle import t5 as ot5


class _Norm(nn.Module):
    def __init__(self, dim, eps=1e-6):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(dim))


class _RelEmb(nn.Module):
    def __init__(self, num_buckets, num_heads, bidirectional=True, max_dist=128):
        super().__init__()
        self.num_buckets, self.num_heads, self.bidirectional, self.max_dist = num_buckets, num_heads, bidirectional, max_dist
        self.embedding = nn.Embedding(num_buckets, num_heads)


class _Attn(nn.Module):
    def __init__(self, dim, dim_attn, num_heads):
        super().__init__()
        self.dim, self.dim_attn, self.num_heads, self.head_dim = dim, dim_attn, num_heads, dim_attn // num_heads
        self.q, self.k, self.v = (nn.Linear(dim, dim_attn, bias=False) for _ in range(3))
        self.o = nn.Linear(dim_attn, dim, bias=False)


class _FFN(nn.Module):
    def __init__(self, dim, dim_ffn):
        super().__init__()
        self.gate = nn.Sequential(nn.Linear(dim, dim_ffn, bias=False), nn.GELU(approximate="tanh"))
        self.fc1 = nn.Linear(dim, dim_ffn, bias=False)
        self.fc2 = nn.Linear(dim_ffn, dim, bias=False)


class _Block(nn.Module):
    def __init__(self, dim, dim_attn, dim_ffn, num_heads, num_buckets, shared_pos, eps):
        super().__init__()
        self.norm1 = _Norm(dim, eps)
        self.attn = _Attn(dim, dim_attn, num_heads)
        self.norm2 = _Norm(dim, eps)
        self.ffn = _FFN(dim, dim_ffn)
        self.pos_embedding = None if shared_pos else _RelEmb(num_buckets, num_heads)


class T5EncoderStandin(nn.Module):
    def __init__(self, vocab, dim, dim_attn, dim_ffn, num_heads, num_layers, num_buckets, shared_pos, eps=1e-6):
        super().__init__()
        self.dim, self.dim_attn, self.dim_ffn, self.num_heads = dim, dim_attn, dim_ffn, num_heads
        self.num_layers, self.num_buckets, self.shared_pos = num_layers, num_buckets, shared_pos
        self.token_embedding = nn.Embedding(vocab, dim)
        self.pos_embedding = _RelEmb(num_buckets, num_heads) if shared_pos else None
        self.dropout = nn.Dropout(0.1)
        self.blocks = nn.ModuleList([_Block(dim, dim_attn, dim_ffn, num_heads, num_buckets, shared_pos, eps)
                                     for _ in range(num_layers)])
        self.norm = _Norm(dim, eps)

    def forward(self, ids, mask=None):
        sd = self.state_dict()
        cfg = dict(dim=self.dim, dim_attn=self.dim_attn, dim_ffn=self.dim_ffn, num_heads=self.num_heads,
                   num_layers=self.num_layers, num_buckets=self.num_buckets, shared_pos=self.shared_pos)
        return ot5.encode(sd, ids, mask, **cfg, eps=self.norm.eps, dtype=sd["norm.weight"].dtype)


def make_text_encoder(sd, cfg, dtype=torch.bfloat16, text_len=512, device="cpu"):
    """Stand-in T5EncoderModel over state dict `sd` (oracle.t5 key layout), weights cast to `dtype`, in eval mode."""
    with torch.device("meta"):
        model = T5EncoderStandin(**cfg)
    model.load_state_dict({k: v.to(device=device, dtype=dtype) for k, v in sd.items()}, assign=True)
    model.eval().requires_grad_(False)
    return types.SimpleNamespace(model=model, text_len=text_len, dtype=dtype, device=device)
