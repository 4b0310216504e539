"""WanDiT — the H100 denoise-forward engine behind the reference's `WanModel.forward`.

One engine instance owns the re-packed weights of one WanModel (5B `wan23` tree or 14B `wan` tree) and runs the
whole forward through libyume_b200.so. Host code here is orchestration only: shapes, the FramePack segment plan,
RoPE position tables, workspace reuse. Every FLOP and every byte of activation traffic happens in the CUDA
kernels (yume_b200/csrc); there is no PyTorch compute fallback.

Reference semantics followed (file:line in /root/reference):
  forward 5B   wan23/modules/model.py:547-865      forward 14B  wan/modules/model.py:723-1013
  block        wan23/modules/model.py:272-316      block 14B    wan/modules/model.py:444-496
  FramePack    wan23/modules/model.py:588-741      (14B: wan/modules/model.py:768-910)
Numerics: bf16 GEMM/attention inputs with fp32 accumulation, fp32 residual stream / modulation / norms — the
regime the reference runs under torch.autocast(bf16) (SURVEY.md Appendix A).
"""
from __future__ import annotations

import contextlib
import math
from collections import OrderedDict
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import ops
from ._lib import YumeB200Error
from .utils import KernelTimer

Tensor = torch.Tensor
_BF16 = torch.bfloat16
_F32 = torch.float32


def _pad_cols(w: Tensor, mult: int) -> Tensor:
    """Zero-pad the K (last) dimension of a [N, K] matrix to a multiple of `mult` (TMA needs 16-byte row pitch)."""
    k = w.shape[1]
    kp = (k + mult - 1) // mult * mult
    if kp == k:
        return w.contiguous()
    out = w.new_zeros(w.shape[0], kp)
    out[:, :k] = w
    return out


def _pad_rows(w: Tensor, mult: int) -> Tensor:
    n = w.shape[0]
    np_ = (n + mult - 1) // mult * mult
    if np_ == n:
        return w.contiguous()
    out = w.new_zeros(np_, *w.shape[1:])
    out[:n] = w
    return out


@dataclass
class _Segment:
    frames: slice      # frames of the history tensor
    name: str          # embedder (state-dict prefix)
    patch: int         # spatial patch (= 2 * compression)
    pre_2x_f: bool     # apply patch_embedding_2x_f first (deepest history level)


def framepack_plan(hist: int, branch_hist: int) -> List[_Segment]:
    """Which history frames go through which patch embedder, in token order.

    Restates the branch ladder of wan23/modules/model.py:599-718 (identical in wan/modules/model.py:779-898):
    the newest 3 history frames keep full resolution, the next 2 are embedded with 4x4 patches, the next 16 with
    8x8, then 64 with 16x16, then 256 with 32x32, the oldest with 2x_f + 32x32; the very first frame is always kept
    (full resolution up to 86 history frames, 4x4 patches beyond). `branch_hist` is the quantity the reference's
    conditions test (f_num - latent_frame_zero for 5B, f_num - 9 for 14B)."""
    H = hist
    levels = [("patch_embedding", 2), ("patch_embedding_2x", 4), ("patch_embedding_4x", 8),
              ("patch_embedding_8x", 16), ("patch_embedding_16x", 32)]
    if branch_hist <= 6:
        depth = 1
    elif branch_hist <= 22:
        depth = 2
    elif branch_hist <= 86:
        depth = 3
    elif branch_hist <= 342:
        depth = 4
    elif branch_hist <= 1366:
        depth = 5
    else:
        raise UnboundLocalError(
            "freqs_i: the reference has no FramePack branch for more than 1366 history latent frames")
    segs: List[_Segment] = []
    first_level = 0 if depth <= 3 else 1                      # frame 0: 1x up to 86 frames of history, else 2x
    segs.append(_Segment(slice(0, 1), *levels[first_level], False))
    if depth == 1:
        mid = slice(H - 1, H) if H - 2 <= 0 else slice(1, H - 1)
        segs.append(_Segment(mid, *levels[1], False))
        segs.append(_Segment(slice(H - 1, H), *levels[0], False))
        return segs
    # tail windows, newest last: [-3:] 1x, [-5:-3] 2x, [-21:-5] 4x, [-85:-21] 8x, [-341:-85] 16x
    bounds = [3, 5, 21, 85, 341]
    deep = min(depth, 4)                                      # level of the "everything older" segment
    cut = bounds[depth - 1]                                   # frames kept in the finer tail windows
    mid = slice(H - cut, H - cut + 1) if H - (cut + 1) <= 0 else slice(1, H - cut)
    segs.append(_Segment(mid, *levels[deep], depth == 5))
    for lvl in range(depth - 1, 0, -1):                       # coarser -> finer windows
        lo, hi = bounds[lvl], bounds[lvl - 1]
        segs.append(_Segment(slice(H - lo, H - hi), *levels[min(lvl, 4)], False))
    segs.append(_Segment(slice(H - 3, H), *levels[0], False))
    return segs


FP8_MAX = 448.0                                  # largest finite e4m3 value
FP8_WEIGHTS = ("w_qkv", "w_o", "cw_q", "cw_o", "w1", "w2")   # the block linears that precision="fp8" converts
FP8_LN_WIDTHS = (256, 1024, 3072, 5120)          # model widths yb_ln_modulate_fp8 has an instance for
PRECISIONS = ("bf16", "fp8", "fp8_attn")         # WanDiT(precision=): see WanDiT.__init__


def quantize_weight_fp8(w: Tensor) -> Tuple[Tensor, Tensor]:
    """Per-output-channel e4m3 weight (include/yume_b200_fp8.h): s_w[n] = amax_n / 448, Wq = e4m3(clamp(W * 448 / amax_n,
    +-448)); an all-zero row gets s_w = 0 and Wq = 0. w [N, K] any float dtype -> (Wq float8_e4m3fn [N, K], s_w f32 [N])."""
    w = w.float()
    amax = w.abs().amax(dim=1)
    mult = torch.where(amax > 0, FP8_MAX / amax, torch.zeros_like(amax))
    wq = (w * mult[:, None]).clamp(-FP8_MAX, FP8_MAX).to(torch.float8_e4m3fn).contiguous()
    return wq, (amax / torch.full_like(amax, FP8_MAX)).contiguous()   # tensor / tensor: IEEE division, as on every device


def sp_qkv_row_order(dim: int, heads: int, world: int) -> Tensor:
    """Row permutation of the fused [3C, C] q|k|v weight for Ulysses: [peer][part q,k,v][that peer's heads]."""
    wh = (heads // world) * (dim // heads)
    return torch.cat([torch.arange(part * dim + p * wh, part * dim + (p + 1) * wh)
                      for p in range(world) for part in range(3)])


def sp_shard(L: int, world: int, rank: int) -> Tuple[int, int, int]:
    """(rows per rank Lp, first global row, valid rows) of `rank`'s contiguous token shard; L is padded up to
    world*Lp like the reference pads seq_len (wan23/distributed/sequence_parallel.py:120-122)."""
    lp = -(-L // world)
    r0 = rank * lp
    return lp, r0, max(0, min(L, r0 + lp) - r0)


class WanDiT:
    """H100 engine for one WanModel. `variant` is '5b' (wan23 tree) or '14b' (wan tree)."""

    def __init__(self, state_dict: Dict[str, Tensor], variant: str, dim: int, ffn_dim: int, num_heads: int,
                 num_layers: int, in_dim: int, out_dim: int, text_len: int = 512, freq_dim: int = 256,
                 patch_size: Sequence[int] = (1, 2, 2), eps: float = 1e-6, device: str | torch.device = "cuda",
                 precision: str = "bf16"):
        if variant not in ("5b", "14b"):
            raise YumeB200Error("variant must be '5b' or '14b'")
        if precision not in PRECISIONS:
            raise YumeB200Error("precision must be 'bf16', 'fp8' or 'fp8_attn'")
        if precision != "bf16" and (dim % 128 or ffn_dim % 128):
            raise YumeB200Error(f"precision={precision!r} needs dim and ffn_dim divisible by 128 (1x128 scale groups), got {dim}, "
                                f"{ffn_dim}")
        if precision != "bf16" and dim not in FP8_LN_WIDTHS:
            raise YumeB200Error(f"precision={precision!r} runs the fp8 LayerNorm at dim {FP8_LN_WIDTHS} only, got {dim}")
        if tuple(patch_size) != (1, 2, 2):
            raise YumeB200Error("only patch_size (1, 2, 2) is supported (both Yume models use it)")
        if dim % num_heads or dim // num_heads != 128:
            raise YumeB200Error("the attention kernel is built for head_dim 128 (both Yume models)")
        self.variant, self.dim, self.ffn_dim, self.heads, self.layers = variant, dim, ffn_dim, num_heads, num_layers
        self.in_dim, self.out_dim, self.text_len, self.freq_dim, self.eps = in_dim, out_dim, text_len, freq_dim, eps
        self.device = torch.device(device)
        self.head_dim = 128
        # "fp8": the six block linears (q|k|v, o, cross q, cross o, ffn.0, ffn.2) run as e4m3 GEMMs with per-channel weight
        # scales and 1x128 activation scales (include/yume_b200_fp8.h); everything else stays as in "bf16".
        # "fp8_attn": everything "fp8" does, and the self-attention of every block in e4m3 (include/yume_b200_fp8_attn.h)
        self.precision = precision
        self._fp8 = precision != "bf16"
        self._ws: Dict[Tuple, Tensor] = {}
        self._rope_cache: Dict[Tuple, Tensor] = {}
        self.timer = KernelTimer()          # bench.py switches it on to time individual kernels inside a live step
        self.sp_group, self.sp_world, self.sp_rank = None, 1, 0
        self.sp_transport, self._sp_p2p = "auto", None
        # sampler-loop fusion (SURVEY.md §8(f) rank 2), both behind the unchanged forward signature:
        #  context_cache  the embedded context and every block's cross-attention K|V depend only on (context, clip_fea);
        #                 keep them while the caller passes the SAME tensors again (every Euler step of a sampling loop,
        #                 cond / uncond alternating under CFG) instead of recomputing 2 + layers GEMMs per forward
        #  use_cuda_graph replay the fixed-shape step as one CUDA graph (one launch instead of ~460 ctypes calls)
        self.context_cache = True
        self.use_cuda_graph = False
        self._ctx_entries: "OrderedDict[tuple, tuple]" = OrderedDict()
        self._graphs: Dict[tuple, dict] = {}
        self._repack(state_dict)

    # ------------------------------------------------------------------------------------------------------
    # weights
    # ------------------------------------------------------------------------------------------------------
    def _repack(self, sd: Dict[str, Tensor]) -> None:
        dev, C = self.device, self.dim

        def w16(name):
            return sd[name].detach().to(device=dev, dtype=_BF16).contiguous()

        def f32(name):
            return sd[name].detach().to(device=dev, dtype=_F32).contiguous()

        def cat16(names):
            return torch.cat([sd[n].detach().to(device=dev, dtype=_BF16) for n in names], dim=0).contiguous()

        def cat32(names):
            return torch.cat([sd[n].detach().to(device=dev, dtype=_F32) for n in names], dim=0).contiguous()

        def lin(names):   # one of the converted block linears: bf16, or (e4m3, s_w) quantised from the checkpoint's own values
            if self.precision == "bf16":
                return cat16(names)
            return quantize_weight_fp8(cat32(names))

        self.embed: Dict[str, Tuple[Tensor, Tensor]] = {}
        for name in ("patch_embedding", "patch_embedding_2x", "patch_embedding_4x", "patch_embedding_8x",
                     "patch_embedding_16x", "patch_embedding_2x_f"):
            if name + ".weight" in sd:
                w = sd[name + ".weight"].detach().to(device=dev, dtype=_BF16).flatten(1)   # [N, cin*ph*pw]
                b = f32(name + ".bias")
                if name == "patch_embedding_2x_f":                                         # N = in_dim: pad to 32
                    w, b = _pad_rows(w, 32), _pad_rows(b, 32)
                self.embed[name] = (_pad_cols(w, 8), b)
        self.text0 = (w16("text_embedding.0.weight"), f32("text_embedding.0.bias"))
        self.text2 = (w16("text_embedding.2.weight"), f32("text_embedding.2.bias"))
        self.time0 = (f32("time_embedding.0.weight"), f32("time_embedding.0.bias"))
        self.time2 = (f32("time_embedding.2.weight"), f32("time_embedding.2.bias"))
        self.tproj = (f32("time_projection.1.weight"), f32("time_projection.1.bias"))
        self.head_w, self.head_b = f32("head.head.weight"), f32("head.head.bias")
        self.head_mod = f32("head.modulation").reshape(2, C)
        if self.variant == "14b":
            self.img = dict(ln0=(f32("img_emb.proj.0.weight"), f32("img_emb.proj.0.bias")),
                            fc1=(w16("img_emb.proj.1.weight"), f32("img_emb.proj.1.bias")),
                            fc3=(w16("img_emb.proj.3.weight"), f32("img_emb.proj.3.bias")),
                            ln4=(f32("img_emb.proj.4.weight"), f32("img_emb.proj.4.bias")))
        self.blocks = []
        mods = []
        for i in range(self.layers):
            p = f"blocks.{i}"
            sa, ca = p + ".self_attn", p + ".cross_attn"
            blk = dict(
                w_qkv=lin([sa + ".q.weight", sa + ".k.weight", sa + ".v.weight"]),
                b_qkv=cat32([sa + ".q.bias", sa + ".k.bias", sa + ".v.bias"]),
                w_o=lin([sa + ".o.weight"]), b_o=f32(sa + ".o.bias"),
                nq=f32(sa + ".norm_q.weight"), nk=f32(sa + ".norm_k.weight"),
                cw_q=lin([ca + ".q.weight"]), cb_q=f32(ca + ".q.bias"),
                cw_kv=cat16([ca + ".k.weight", ca + ".v.weight"]), cb_kv=cat32([ca + ".k.bias", ca + ".v.bias"]),
                cw_o=lin([ca + ".o.weight"]), cb_o=f32(ca + ".o.bias"),
                cnq=f32(ca + ".norm_q.weight"), cnk=f32(ca + ".norm_k.weight"),
                n3w=f32(p + ".norm3.weight"), n3b=f32(p + ".norm3.bias"),
                w1=lin([p + ".ffn.0.weight"]), b1=f32(p + ".ffn.0.bias"),
                w2=lin([p + ".ffn.2.weight"]), b2=f32(p + ".ffn.2.bias"),
            )
            if self.variant == "14b":
                blk["cw_kv_img"] = cat16([ca + ".k_img.weight", ca + ".v_img.weight"])
                blk["cb_kv_img"] = cat32([ca + ".k_img.bias", ca + ".v_img.bias"])
                blk["cnk_img"] = f32(ca + ".norm_k_img.weight")
            self.blocks.append(blk)
            mods.append(f32(p + ".modulation").reshape(6 * C))
        self.block_mod = torch.stack(mods).contiguous()            # [layers, 6C]
        # cross-attention K/V projections of all blocks as ONE [layers*2C, C] weight: the context is the same for
        # every block, so one GEMM per forward replaces `layers` latency-bound 48-tile GEMMs (model.py:223-224 runs
        # k(context), v(context) inside every block)
        self.cw_kv_all = torch.cat([b.pop("cw_kv") for b in self.blocks], dim=0).contiguous()
        self.cb_kv_all = torch.cat([b.pop("cb_kv") for b in self.blocks], dim=0).contiguous()
        if self.variant == "14b":
            self.cw_kv_img_all = torch.cat([b.pop("cw_kv_img") for b in self.blocks], dim=0).contiguous()
            self.cb_kv_img_all = torch.cat([b.pop("cb_kv_img") for b in self.blocks], dim=0).contiguous()

    def enable_sequence_parallel(self, group, transport: str = "auto") -> None:
        """Shard the token sequence Ulysses-style over `group` (one process per GPU). transport: "p2p" = exchanges
        fused into the kernels over NVLink peer memory (torch symmetric memory) — the q|k|v exchange rides in the RMSNorm+RoPE
        pass, the output exchange in the attention epilogue; "p2p_gemm" = as p2p, but the q|k|v exchange is the EPILOGUE OF THE
        QKV GEMM itself (yb_gemm_sp_qkv: peer stores under the main loop, normalisation finished on the receiver);
        "nccl" = NCCL all_to_all_single; "auto" = p2p when symmetric memory is available. For the NCCL path builds the peer-major fused q|k|v weight:
        rows ordered [peer p][q, k, v][heads p*H/P .. (p+1)*H/P) so that the QKV GEMM's `n_split` epilogue emits
        exactly the chunks the all-to-all sends.
        precision "fp8" / "fp8_attn" run "p2p", "nccl" and "auto" (DESIGN.md §6): the q|k|v GEMM writes the standard [Lp, 3C]
        rows and one norm + RoPE pass scatters them (p2p) or packs them into the NCCL send buffer, so no peer-major weight is built;
        "p2p_gemm" is the bf16 GEMM with the exchange in its epilogue and has no e4m3 form."""
        if transport not in ("auto", "p2p", "p2p_gemm", "nccl"):
            raise YumeB200Error("transport must be auto, p2p, p2p_gemm or nccl")
        import torch.distributed as dist
        if self._fp8:
            if transport == "p2p_gemm":
                raise YumeB200Error(f"transport 'p2p_gemm' fuses the exchange into the bf16 q|k|v GEMM, which has no e4m3 form: "
                                    f"use 'p2p', 'nccl' or 'auto' with precision={self.precision!r}")
            if group is None and not (dist.is_available() and dist.is_initialized()):
                raise YumeB200Error("sequence parallelism needs an initialised torch.distributed process group")
        self.sp_transport, self._sp_p2p = transport, None
        P = dist.get_world_size(group)
        if self.heads % P:
            raise YumeB200Error(f"{self.heads} heads do not divide over {P} ranks")
        self.sp_group, self.sp_world, self.sp_rank = group, P, dist.get_rank(group)
        if P == 1:
            return
        if transport == "nccl":
            self._build_nccl_weights()

    def _build_nccl_weights(self) -> None:
        """Peer-major copies of the fused q|k|v weights: only the bf16 NCCL transport reads them (+6.3 GB at 14B), so they are
        built when that transport is chosen — up front, or when symmetric memory turns out to be unavailable. The fp8 engine
        packs the send buffer from the standard q|k|v rows instead (yb_sp_pack_qkv) and never builds them."""
        if self._fp8 or "w_qkv_sp" in self.blocks[0]:
            return
        idx = sp_qkv_row_order(self.dim, self.heads, self.sp_world).to(self.device)
        for b in self.blocks:
            b["w_qkv_sp"] = b["w_qkv"][idx].contiguous()
            b["b_qkv_sp"] = b["b_qkv"][idx].contiguous()

    @contextlib.contextmanager
    def sequence_parallel_disabled(self):
        """Run forwards on this rank alone (no Ulysses, no collectives) while the block is active — bench.py uses it to
        compare the N-GPU output with the single-GPU output of the SAME engine (`parity_vs_n1`)."""
        saved = (self.sp_world, self.sp_rank)
        self.sp_world, self.sp_rank = 1, 0
        try:
            yield self
        finally:
            self.sp_world, self.sp_rank = saved

    @classmethod
    def from_module(cls, model: torch.nn.Module, variant: str, device="cuda", precision: str = "bf16") -> "WanDiT":
        """Build from a live reference WanModel (or yume_b200.model.WanModel): reads its parameters, never
        modifies the checkpoint format (SURVEY.md §8b 'State-dict')."""
        sd = dict(model.state_dict())
        for name in ("patch_embedding_2x", "patch_embedding_4x", "patch_embedding_8x", "patch_embedding_16x",
                     "patch_embedding_2x_f"):  # attached as plain attributes in the 14B tree (wan/image2video.py:155-159)
            m = getattr(model, name, None)
            if m is not None and name + ".weight" not in sd:
                sd[name + ".weight"], sd[name + ".bias"] = m.weight, m.bias
        return cls(sd, variant, dim=model.dim, ffn_dim=model.ffn_dim, num_heads=model.num_heads,
                   num_layers=model.num_layers, in_dim=model.in_dim, out_dim=model.out_dim, text_len=model.text_len,
                   freq_dim=model.freq_dim, patch_size=model.patch_size, eps=model.eps, device=device, precision=precision)

    # ------------------------------------------------------------------------------------------------------
    # workspace / tables
    # ------------------------------------------------------------------------------------------------------
    def _buf(self, key: str, shape: Tuple[int, ...], dtype) -> Tensor:
        k = (key, tuple(shape), dtype)
        t = self._ws.get(k)
        if t is None:
            for old in [o for o in self._ws if o[0] == key]:   # geometry changed: drop the stale buffer
                del self._ws[old]
                self._graphs.clear()                           # captured graphs hold its address
            t = torch.empty(shape, device=self.device, dtype=dtype)
            self._ws[k] = t
        return t

    def _axis_angles(self, n: int, axis_dim: int) -> Tensor:
        """angles[pos, j] = pos * theta^(-2j/axis_dim) in fp64 (rope_params, model.py:27-35)."""
        inv = 1.0 / torch.pow(10000.0, torch.arange(0, axis_dim, 2, dtype=torch.float64) / axis_dim)
        return torch.outer(torch.arange(n, dtype=torch.float64), inv)

    def _rope_segment(self, f: int, h: int, w: int, f0: int) -> Tensor:
        """fp64 angles [f*h*w, 64] of one regular grid segment with temporal offset f0 (up_fre, model.py:933-940)."""
        d = self.head_dim
        dt, dh = d - 4 * (d // 6), 2 * (d // 6)
        at = self._axis_angles(f0 + f, dt)[f0:]
        ah, aw = self._axis_angles(h, dh), self._axis_angles(w, dh)
        return torch.cat([at.view(f, 1, 1, -1).expand(f, h, w, -1), ah.view(1, h, 1, -1).expand(f, h, w, -1),
                          aw.view(1, 1, w, -1).expand(f, h, w, -1)], dim=-1).reshape(f * h * w, -1)

    def _rope_table(self, segments: Sequence[Tuple[int, int, int, int]]) -> Tensor:
        """(cos, sin) f32 [L, 64, 2] on the device for a token sequence made of grid segments (f, h, w, f0)."""
        key = tuple(segments)
        t = self._rope_cache.get(key)
        if t is None:
            ang = torch.cat([self._rope_segment(*s) for s in segments], dim=0)
            t = torch.stack([ang.cos(), ang.sin()], dim=-1).to(_F32).contiguous().to(self.device)
            if len(self._rope_cache) > 16:
                self._rope_cache.clear()
            self._rope_cache[key] = t
        return t

    # ------------------------------------------------------------------------------------------------------
    # pieces of the forward
    # ------------------------------------------------------------------------------------------------------
    def _embed_tokens(self, u: Tensor, name: str, patch: int, xs: Tensor, row0: int, window: Tuple[int, int]) -> None:
        """Patch-embed u [Cin, f, H, W] (f32, any strides) with Conv3d `name` (kernel == stride == (1,patch,patch)). The
        segment's tokens are global rows [row0, row0 + n); `xs` holds the global rows `window` = [w0, w1) (the whole sequence,
        or this rank's Ulysses shard): only the rows of the segment that fall inside the window are projected — under
        sequence parallelism every rank embeds just its own tokens (the patch gather itself is a cheap index pass)."""
        w, b = self.embed[name]
        cin, f, H, W = u.shape
        if name == "patch_embedding":          # plain Conv3d, no convpadd: odd H / W lose their last row / column
            u = u[:, :, :H // patch * patch, :W // patch * patch]   # (model.py:453-454; convpadd only wraps the 2x..16x embedders)
            cin, f, H, W = u.shape
        hp, wp = -(-H // patch), -(-W // patch)
        n_tok = f * hp * wp
        lo, hi = max(row0, window[0]), min(row0 + n_tok, window[1])
        if lo >= hi:
            return
        a = self._buf("patch_a", (n_tok, w.shape[1]), _BF16)
        if w.shape[1] != cin * patch * patch:
            a.zero_()                                           # K padding columns must be zero
        ops.patchify(u, a, patch, patch)
        ops.gemm(a[lo - row0:hi - row0], w, b, xs[lo - window[0]:hi - window[0]], ops.YB_EPI_F32)

    def _token_stream(self, L: int, n_real: int) -> Tuple[Tensor, Tuple[int, int]]:
        """The fp32 residual stream and the window of global token rows it holds: all L rows on one GPU, this rank's
        contiguous shard of ceil(L / P) rows under Ulysses. Rows that no embedder writes (zero padding tokens of a padded
        grid, rows >= n_real; shard rows past L) are zeroed here."""
        if self.sp_world > 1:
            Lp, r0, n_valid = sp_shard(L, self.sp_world, self.sp_rank)
            xs = self._buf("xs_shard", (Lp, self.dim), _F32)
            filled = max(0, min(n_real, r0 + n_valid) - r0)
            if filled < Lp:
                xs[filled:].zero_()
            return xs, (r0, r0 + n_valid)
        xs = self._buf("xs", (L, self.dim), _F32)
        if n_real < L:
            xs[n_real:].zero_()
        return xs, (0, L)

    def _time_tables(self, t_unique: Tensor):
        """e [U, C], per-block modulation tables [layers, U, 6, C], head table [U, 2, C] (model.py:805-812, 296, 344)."""
        s = ops.sinusoidal(t_unique, self.freq_dim)
        e = ops.linear_f32_small(s, *self.time0)
        e = ops.linear_f32_small(e, *self.time2, silu_in=True)
        e0 = ops.linear_f32_small(e, *self.tproj, silu_in=True)                    # [U, 6C]
        U, C = e.shape[0], self.dim
        mod = ops.bcast_add(self.block_mod, e0).view(self.layers, U, 6, C)
        head = ops.bcast_add(e, self.head_mod).view(U, 2, C)                       # head uses e, not e0 (:344)
        return e, mod, head

    def _context(self, context: Tensor, clip_fea: Optional[Tensor]) -> Tensor:
        """text_embedding on the zero-padded context (+ img_emb for 14B) -> bf16 [text_len (+257), C]
        (model.py:815-821; wan/modules/model.py:939-941)."""
        C = self.dim
        n_img = 257 if self.variant == "14b" else 0
        ctx_in = self._buf("ctx_in", (self.text_len, context.shape[1]), _BF16)
        ctx_in.zero_()
        ctx_in[:context.shape[0]].copy_(context)
        hid = self._buf("ctx_hid", (self.text_len, C), _BF16)
        out = self._buf("ctx_out", (n_img + self.text_len, C), _BF16)
        ops.gemm(ctx_in, self.text0[0], self.text0[1], hid, ops.YB_EPI_GELU_BF16)
        ops.gemm(hid, self.text2[0], self.text2[1], out[n_img:], ops.YB_EPI_BF16)
        if n_img:
            cf = clip_fea.reshape(-1, clip_fea.shape[-1]).to(device=self.device, dtype=_F32).contiguous()
            cd = cf.shape[1]
            a = self._buf("img_a", (n_img, cd), _BF16)
            ops.ln_modulate(cf, a, None, None, None, *self.img["ln0"], eps=1e-5)
            h1 = self._buf("img_h", (n_img, cd), _BF16)
            ops.gemm(a, *self.img["fc1"], h1, ops.YB_EPI_GELU_ERF_BF16)
            h3 = self._buf("img_o", (n_img, C), _F32)
            ops.gemm(h1, *self.img["fc3"], h3, ops.YB_EPI_F32)
            ops.ln_modulate(h3, out[:n_img], None, None, None, *self.img["ln4"], eps=1e-5)
        return out

    def _sp_p2p_state(self, Lp: int):
        """Symmetric-memory receive buffers (both layer parities) and every rank's peer pointers to them. Collective:
        all ranks call it with the same Lp. Returns None (-> NCCL transport) if symmetric memory is unavailable."""
        if self._sp_p2p is not None and self._sp_p2p["Lp"] == Lp:
            return self._sp_p2p
        if self.sp_transport == "nccl":
            return None
        try:
            import torch.distributed._symmetric_memory as symm
            P, Wh = self.sp_world, (self.heads // self.sp_world) * self.head_dim
            n_qkv, n_att = P * Lp * 3 * Wh, P * Lp * Wh
            buf = symm.empty(2 * (n_qkv + n_att), dtype=_BF16, device=self.device)
            hdl = symm.rendezvous(buf, self.sp_group)
            bases = [int(x) for x in hdl.buffer_ptrs]
            off_q = [0, n_qkv]
            off_a = [2 * n_qkv, 2 * n_qkv + n_att]
            sbuf = symm.empty(2 * P * Lp * 2, dtype=_F32, device=self.device)    # [parity][P(src)][Lp][q, k] sums of squares
            shdl = symm.rendezvous(sbuf, self.sp_group)
            sbases = [int(x) for x in shdl.buffer_ptrs]
            self._sp_p2p = dict(
                sums_buf=sbuf, sums_hdl=shdl, sums=[sbuf[o:o + P * Lp * 2].view(P * Lp, 2) for o in (0, P * Lp * 2)],
                sums_ptrs=[[bp + 4 * o for bp in sbases] for o in (0, P * Lp * 2)],
                sums_local=torch.zeros(Lp, 2, device=self.device, dtype=_F32),
                Lp=Lp, buf=buf, hdl=hdl,
                qkv=[buf[o:o + n_qkv].view(P, Lp, 3 * Wh) for o in off_q],
                att=[buf[o:o + n_att].view(P, Lp, Wh) for o in off_a],
                qkv_ptrs=[[bp + 2 * o for bp in bases] for o in off_q],
                att_ptrs=[[bp + 2 * o for bp in bases] for o in off_a])
            ok = True
        except Exception as e:  # transport choice only: the NCCL path below runs the same kernels
            ok, err = False, e
        # the ranks must take the SAME transport: agree on the outcome (a rank that failed alone would otherwise sit in an
        # NCCL all-to-all while its peers wait on a symmetric-memory barrier)
        import torch.distributed as dist
        flag = torch.tensor([1 if ok else 0], device=self.device, dtype=torch.int32)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.sp_group)
        if int(flag.item()) == 0:
            self._sp_p2p = None
            if self.sp_transport in ("p2p", "p2p_gemm"):
                raise YumeB200Error("symmetric memory unavailable on at least one rank" + ("" if ok else f": {err}"))
            import warnings
            warnings.warn("yume_b200: symmetric memory unavailable; Ulysses uses NCCL all-to-all")
            self.sp_transport = "nccl"
            self._build_nccl_weights()
            return None
        return self._sp_p2p

    def _self_attention_sp_p2p(self, i: int, st: dict, b: dict, h: Tensor, xs: Tensor, m: Tensor,
                               tok_idx: Optional[Tensor], rope: Tensor, rope_len: int, L_true: int) -> None:
        """Ulysses with the exchanges fused into the kernels over NVLink peer memory: the RMSNorm+RoPE kernel stores
        q|k|v chunks straight into the owning rank's receive buffer, the attention epilogue stores each output row
        straight into its owner's buffer; two symmetric-memory barriers per block, no NCCL on the data path. Receive
        buffers alternate by layer parity so a fast rank's next-layer writes never land in a buffer a slow rank still
        reads (it cannot be two barriers ahead)."""
        C, D, P = self.dim, self.head_dim, self.sp_world
        Hp = self.heads // P
        Wh = Hp * D
        Lp = xs.shape[0]
        par = i & 1
        T = self.timer
        full = st["qkv"][par].view(P * Lp, 3 * Wh)
        if self.sp_transport == "p2p_gemm":
            # GEMM + all-to-all in one kernel: the projection's epilogue stores every head's columns into its owner's receive
            # buffer and accumulates the per-token sums of squares; the receiver finishes RMSNorm + RoPE after the barrier
            T.begin("gemm_qkv")
            ops.gemm_sp_qkv(h, b["w_qkv"], b["b_qkv"], st["qkv_ptrs"][par], self.sp_rank, Lp, st["sums_local"])
            T.end("gemm_qkv")
            T.begin("sp_scatter_qkv")
            ops.sp_bcast_sums(st["sums_local"], st["sums_ptrs"][par], self.sp_rank, Lp)
            st["hdl"].barrier(channel=0)
            r0w = self.sp_rank * Wh
            rope_g, rope_len_g = self._sp_rope_global
            ops.sp_post_norm_rope(full, st["sums"][par], b["nq"][r0w:r0w + Wh], b["nk"][r0w:r0w + Wh], rope_g, rope_len_g,
                                  P * Lp, Wh, C, D, self.eps)
            T.end("sp_scatter_qkv")
        else:
            qkv = self._buf("qkv", (Lp, 3 * C), _BF16)
            T.begin("gemm_qkv")
            self._linear(h, b["w_qkv"], b["b_qkv"], qkv, ops.YB_EPI_BF16)
            T.end("gemm_qkv")
            T.begin("sp_scatter_qkv")
            ops.sp_scatter_qkv(qkv, b["nq"], b["nk"], rope, rope_len, D, self.eps, st["qkv_ptrs"][par], self.sp_rank, Lp)
            st["hdl"].barrier(channel=0)
            T.end("sp_scatter_qkv")
        T.begin("self_attention")
        if self.precision == "fp8_attn":
            qk8, qk_s, vt8, v_s = self._quant_qkv8(full, L_true, Hp)
            ops.attention_fp8_sp(qk8[:, :Wh], qk8[:L_true, Wh:], qk_s, vt8, v_s, st["att_ptrs"][par], Wh, Hp, self.sp_rank, Lp)
        else:
            ops.attention_sp(full[:, :Wh], full[:L_true, Wh:2 * Wh], full[:L_true, 2 * Wh:], st["att_ptrs"][par], Wh, Hp,
                             self.sp_rank, Lp)
        st["hdl"].barrier(channel=0)
        T.end("self_attention")
        T.begin("gemm_o")
        self._o_proj_sp(st["att"][par], b, xs, m, tok_idx)
        T.end("gemm_o")

    def _o_proj_sp(self, att: Tensor, b: dict, xs: Tensor, m: Tensor, tok_idx: Optional[Tensor]) -> None:
        """The o projection (GATE_RES into this rank's xs) of the exchanged attention output att [P, Lp, heads/P*128], whose
        K-split layout holds row t of the [Lp, C] input as P chunks Lp*Wh apart: the bf16 GEMM reads it through a 3-D map (a_split);
        under fp8 one split quantiser gathers it into the e4m3 pair the fp8 GEMM reads (the one-GPU path's quantiser launch)."""
        P, Lp, Wh = att.shape
        C = self.dim
        if self._fp8:
            a8 = self._act8("att8", Lp, C)
            ops.quant_rows_fp8_split(att, *a8, Wh, Lp * Wh, (Lp, C))
            ops.gemm_fp8(*a8, *b["w_o"], b["b_o"], xs, ops.YB_EPI_GATE_RES, gate=m[:, 2], tok_idx=tok_idx)
            return
        ops.gemm(att, b["w_o"], b["b_o"], xs, ops.YB_EPI_GATE_RES, gate=m[:, 2], tok_idx=tok_idx,
                 a_split=Wh, a_split_stride=Lp * Wh, shape=(Lp, C))

    def _self_attention_sp(self, i: int, b: dict, h: Tensor, xs: Tensor, m: Tensor, tok_idx: Optional[Tensor], rope: Tensor,
                           rope_len: int, L_true: int) -> None:
        """Ulysses self-attention on a token shard (SURVEY.md §8e; design reference wan23/distributed/ulysses.py:9-47,
        sequence_parallel.py:147-176). xs/h hold this rank's Lp tokens. Two all-to-alls per block on the
        head/sequence axis, nothing else is exchanged:
          QKV GEMM -> peer-major [P, Lp, q|k|v of heads/P] (n_split epilogue, no pack kernel)
          RMSNorm (spans all heads) + RoPE on the local tokens, before the exchange
          all-to-all -> [P*Lp tokens, q|k|v of my heads/P] ; attention over all L_true keys for my heads
          all-to-all -> [P, Lp, heads/P*128]; the o-projection reads it through a K-split 3-D TMA map."""
        import torch.distributed as dist
        st = self._sp_p2p_state(xs.shape[0])
        if st is not None:
            return self._self_attention_sp_p2p(i, st, b, h, xs, m, tok_idx, rope, rope_len, L_true)
        C, D, P = self.dim, self.head_dim, self.sp_world
        Hp = self.heads // P
        Wh, W3 = Hp * D, 3 * Hp * D
        Lp = xs.shape[0]
        T = self.timer
        send = self._buf("sp_qkv_send", (P, Lp, W3), _BF16)
        recv = self._buf("sp_qkv_recv", (P, Lp, W3), _BF16)
        if self._fp8:
            # standard [Lp, 3C] rows from the e4m3 GEMM, then yb_sp_scatter_qkv's norm + RoPE with the send buffer as destination
            qkv = self._buf("qkv", (Lp, 3 * C), _BF16)
            T.begin("gemm_qkv")
            self._linear(h, b["w_qkv"], b["b_qkv"], qkv, ops.YB_EPI_BF16)
            T.end("gemm_qkv")
            T.begin("qk_norm_rope")
            ops.sp_pack_qkv(qkv, b["nq"], b["nk"], rope, rope_len, D, self.eps, send)
            T.end("qk_norm_rope")
        else:
            T.begin("gemm_qkv")
            ops.gemm(h, b["w_qkv_sp"], b["b_qkv_sp"], send, ops.YB_EPI_BF16, n_split=W3, split_stride=Lp * W3, shape=(Lp, C))
            T.end("gemm_qkv")
            T.begin("qk_norm_rope")
            ops.qk_norm_rope(send[0], send[0][:, Wh:], b["nq"], b["nk"], rope, D, self.eps, rope_len,
                             pieces=(Lp, C, Wh, Lp * W3))
            T.end("qk_norm_rope")
        T.begin("sp_all_to_all_qkv")
        dist.all_to_all_single(recv, send, group=self.sp_group)
        T.end("sp_all_to_all_qkv")
        full = recv.view(P * Lp, W3)                            # global token order (rank-major shards)
        att_send = self._buf("sp_att_send", (P, Lp, Wh), _BF16)
        att_recv = self._buf("sp_att_recv", (P, Lp, Wh), _BF16)
        T.begin("self_attention")
        self._attention(full, att_send.view(P * Lp, Wh), L_true, Hp)
        T.end("self_attention")
        T.begin("sp_all_to_all_out")
        dist.all_to_all_single(att_recv, att_send, group=self.sp_group)
        T.end("sp_all_to_all_out")
        T.begin("gemm_o")
        self._o_proj_sp(att_recv, b, xs, m, tok_idx)
        T.end("gemm_o")

    def _cross_kv(self, ctx: Tensor, own_storage: bool = False, block: Optional[int] = None):
        """K | V of the embedded context for every block in one GEMM (+ the image branch for 14B), RMSNorm on the K
        halves. Returns per-block (kv_text, kv_img or None) views of [S, 2C]. own_storage: allocate fresh result buffers
        (context-cache entries outlive the call) instead of the shared workspace. block: block `block`'s K | V only, as a
        one-entry list, in workspace buffers of its own (the seams run one block at a time; reusing the forward's buffers
        would evict them and the graphs captured against them)."""
        C, D = self.dim, self.head_dim
        n_img = 257 if self.variant == "14b" else 0
        ctx_txt = ctx[n_img:]
        ids = range(self.layers) if block is None else range(block, block + 1)
        rows = slice(ids[0] * 2 * C, (ids[-1] + 1) * 2 * C)
        tag = "_all" if block is None else "_one"
        alloc = (lambda key, shape: torch.empty(shape, device=self.device, dtype=_BF16)) if own_storage else \
            (lambda key, shape: self._buf(key, shape, _BF16))
        kv_all = alloc("ckv" + tag, (ctx_txt.shape[0], len(ids) * 2 * C))
        ops.gemm(ctx_txt, self.cw_kv_all[rows], self.cb_kv_all[rows], kv_all, ops.YB_EPI_BF16)
        kvi_all = None
        if n_img:
            kvi_all = alloc("ckv_img" + tag, (n_img, len(ids) * 2 * C))
            ops.gemm(ctx[:n_img], self.cw_kv_img_all[rows], self.cb_kv_img_all[rows], kvi_all, ops.YB_EPI_BF16)
        out = []
        for j, i in enumerate(ids):
            b = self.blocks[i]
            kv = kv_all[:, j * 2 * C:(j + 1) * 2 * C]
            ops.rmsnorm_rope(kv[:, :C], b["cnk"], None, D, self.eps)
            kvi = None
            if kvi_all is not None:
                kvi = kvi_all[:, j * 2 * C:(j + 1) * 2 * C]
                ops.rmsnorm_rope(kvi[:, :C], b["cnk_img"], None, D, self.eps)
            out.append((kv, kvi))
        return out

    def _context_kv(self, context: Tensor, clip_fea: Optional[Tensor]):
        """Per-block cross-attention K|V for (context, clip_fea). With `context_cache` the result is kept, keyed on the
        identity AND version counter of the caller's tensors (an in-place edit bumps `_version`; the entry holds references,
        so the addresses cannot be recycled while it lives). Four entries: cond / uncond of two prompts."""
        if not self.context_cache:
            return self._cross_kv(self._context(context.to(device=self.device), clip_fea))
        key = (context.data_ptr(), context._version, tuple(context.shape), context.dtype, str(context.device),
               None if clip_fea is None else (clip_fea.data_ptr(), clip_fea._version, tuple(clip_fea.shape)))
        hit = self._ctx_entries.get(key)
        if hit is not None:
            self._ctx_entries.move_to_end(key)
            return hit[0]
        if torch.cuda.is_current_stream_capturing():           # (the warm-up run before a capture fills the cache)
            return self._cross_kv(self._context(context.to(device=self.device), clip_fea))
        kv = self._cross_kv(self._context(context.to(device=self.device), clip_fea), own_storage=True)
        self._ctx_entries[key] = (kv, context, clip_fea)
        while len(self._ctx_entries) > 4:
            self._ctx_entries.popitem(last=False)
            self._graphs.clear()                               # graphs captured against the evicted K|V buffers
        return kv

    def _block(self, i: int, xs: Tensor, mod: Tensor, tok_idx: Optional[Tensor], rope: Tensor, rope_len: int,
               ctx: List, L_true: Optional[int] = None) -> None:
        """One WanAttentionBlock in place on the fp32 residual stream xs [L, C] (a token shard under Ulysses). mod: the
        modulation tables [layers, U, 6, C]; ctx: every block's cross K|V (_cross_kv); L_true: rows that are self-attention
        keys (default all)."""
        self._block_body(i, xs, mod[i], tok_idx, rope, rope_len, ctx[i], L_true if L_true is not None else xs.shape[0])

    def _block_body(self, i: int, xs: Tensor, m: Tensor, tok_idx: Optional[Tensor], rope: Tensor, rope_len: int, kv,
                    k_len: int) -> None:
        """Block i with its modulation rows m [U, 6, C] (shift_a, scale_a, gate_a, shift_f, scale_f, gate_f) and its cross
        K|V `kv`."""
        b, C, T = self.blocks[i], self.dim, self.timer
        L = xs.shape[0]
        qkv = self._buf("qkv", (L, 3 * C), _BF16)
        att = self._buf("att", (L, C), _BF16)
        T.begin("ln_modulate")
        h = self._norm(xs, m[:, 1], m[:, 0], tok_idx)
        T.end("ln_modulate")
        if self.sp_world > 1:
            self._self_attention_sp(i, b, h, xs, m, tok_idx, rope, rope_len, k_len)
        else:
            self._self_attention(b, h, qkv, att, rope, rope_len, k_len, xs, ops.YB_EPI_GATE_RES, gate=m[:, 2], tok_idx=tok_idx)
        self._cross_and_ffn(b, xs, qkv, att, m, tok_idx, kv)

    def _self_attention(self, b, a, qkv, att, rope, rope_len, k_len, out, epilogue, gate=None, tok_idx=None) -> None:
        """q|k|v projection of the normed input `a`, RMSNorm + RoPE, attention, then the o projection into `out` (GATE_RES on
        the residual stream, or BF16 for the self-attention seam). k_len: rows that are keys. All L on the 5B tree
        (wan23/modules/model.py:846-851); on the 14B regular-grid path the reference passes k_lens = F*H*W, masking the
        zero-padded rows (wan/modules/model.py:311-314, 916)."""
        C, D, T = self.dim, self.head_dim, self.timer
        T.begin("gemm_qkv")
        self._linear(a, b["w_qkv"], b["b_qkv"], qkv, ops.YB_EPI_BF16)
        T.end("gemm_qkv")
        T.begin("qk_norm_rope")
        ops.qk_norm_rope(qkv[:, :C], qkv[:, C:2 * C], b["nq"], b["nk"], rope, D, self.eps, rope_len)
        T.end("qk_norm_rope")
        T.begin("self_attention")
        self._attention(qkv, att, k_len)
        T.end("self_attention")
        T.begin("gemm_o")
        self._linear(self._quant(att, "att8"), b["w_o"], b["b_o"], out, epilogue, gate=gate, tok_idx=tok_idx)
        T.end("gemm_o")

    def _cross_and_ffn(self, b, xs, qkv, att, m, tok_idx, ctx) -> None:
        C, H, D, T = self.dim, self.heads, self.head_dim, self.timer
        # --- cross-attention (no gate, affine norm3) ---
        h = self._norm(xs, None, None, None, b["n3w"], b["n3b"])
        q2 = qkv[:, :C]
        self._linear(h, b["cw_q"], b["cb_q"], q2, ops.YB_EPI_BF16)
        ops.rmsnorm_rope(q2, b["cnq"], None, D, self.eps)
        kv, kvi = ctx                                            # this block's normalised K | V (see _cross_kv)
        T.begin("cross_attention")
        ops.attention(q2, kv[:, :C], kv[:, C:], att, H)
        T.end("cross_attention")
        if kvi is not None:
            ops.attention(q2, kvi[:, :C], kvi[:, C:], att, H, accumulate=True)
        self._linear(self._quant(att, "att8"), b["cw_o"], b["cb_o"], xs, ops.YB_EPI_GATE_RES)
        # --- FFN ---
        h = self._norm(xs, m[:, 4], m[:, 3], tok_idx)
        T.begin("gemm_ffn1")
        hid = self._ffn0(h, b)
        T.end("gemm_ffn1")
        T.begin("gemm_ffn2")
        self._linear(hid, b["w2"], b["b2"], xs, ops.YB_EPI_GATE_RES, gate=m[:, 5], tok_idx=tok_idx)
        T.end("gemm_ffn2")

    # ------------------------------------------------------------------------------------------------------
    # precision: the only places the block code branches on it. Under "fp8" an activation that feeds one of the FP8_WEIGHTS
    # linears is an e4m3 (values, 1x128 scales) pair (include/yume_b200_fp8.h); "fp8_attn" also runs the self-attention in e4m3
    # ------------------------------------------------------------------------------------------------------
    def _act8(self, key: str, rows: int, cols: int) -> Tuple[Tensor, Tensor]:
        """Workspace of one fp8 activation: e4m3 values [rows, cols] and their 1x128 scales f32 [cols / 128, ld >= rows]."""
        return (self._buf(key + "_q", (rows, cols), torch.float8_e4m3fn),
                self._buf(key + "_s", (cols // 128, ops.fp8_scale_ld(rows)), _F32))

    def _norm(self, xs: Tensor, scale, shift, tok_idx, weight=None, bias=None):
        """LayerNorm of xs (affine with weight, bias; modulated with scale, shift) as the next linear's input: bf16 `h`,
        or the e4m3 pair `h8`."""
        L, C = xs.shape
        if self._fp8:
            h8 = self._act8("h8", L, C)
            ops.ln_modulate_fp8(xs, *h8, scale, shift, tok_idx, weight, bias, eps=self.eps)
            return h8
        h = self._buf("h", (L, C), _BF16)
        ops.ln_modulate(xs, h, scale, shift, tok_idx, weight, bias, eps=self.eps)
        return h

    def _quant(self, x: Tensor, key: str):
        """A bf16 activation as the next linear's input: x itself, or x quantised per 1x128 group into the pair `key`."""
        if not self._fp8:
            return x
        x8 = self._act8(key, *x.shape)
        ops.quant_rows_fp8(x, *x8)
        return x8

    def _linear(self, a, w, bias, out, epilogue, gate=None, tok_idx=None) -> None:
        """One of the FP8_WEIGHTS block linears on an input from _norm / _quant / _ffn0."""
        if self._fp8:
            ops.gemm_fp8(*a, *w, bias, out, epilogue, gate=gate, tok_idx=tok_idx)
        else:
            ops.gemm(a, w, bias, out, epilogue, gate=gate, tok_idx=tok_idx)

    def _ffn0(self, h, b: dict):
        """ffn.0 + GELU of the normed input h, as ffn.2's input: bf16 `ffn_hid`, or the e4m3 pair `ffn_hid8` that the GEMM's
        epilogue quantises."""
        if self._fp8:
            hid = self._act8("ffn_hid8", h[0].shape[0], self.ffn_dim)
            ops.gemm_fp8(*h, *b["w1"], b["b1"], hid[0], ops.YB_EPI_GELU_FP8, out_scale=hid[1])
            return hid
        hid = self._buf("ffn_hid", (h.shape[0], self.ffn_dim), _BF16)
        ops.gemm(h, b["w1"], b["b1"], hid, ops.YB_EPI_GELU_BF16)
        return hid

    def _attention(self, qkv: Tensor, att: Tensor, k_len: int, heads: Optional[int] = None) -> None:
        """Self-attention of the normed, roped q|k|v rows over the first k_len rows as keys, into bf16 `att`. "fp8_attn" runs
        it on e4m3 operands (include/yume_b200_fp8_attn.h): q and k are quantised by one launch over the [L, 2C] view (a 1x128
        group is one head of one token: q scales of head h at scale row h, k scales at heads + h), v transposed per (head,
        128-key tile). heads: the heads the rows hold (default all; heads/P on a Ulysses rank's exchanged rows)."""
        H = self.heads if heads is None else heads
        C = H * self.head_dim
        if self.precision != "fp8_attn":
            ops.attention(qkv[:, :C], qkv[:k_len, C:2 * C], qkv[:k_len, 2 * C:], att, H)
            return
        qk8, qk_s, vt8, v_s = self._quant_qkv8(qkv, k_len, H)
        ops.attention_fp8(qk8[:, :C], qk8[:k_len, C:], qk_s, vt8, v_s, att, H)

    def _quant_qkv8(self, qkv: Tensor, k_len: int, H: int):
        """The e4m3 operands of the fp8 attention from bf16 q|k|v rows [L, 3 H 128]: (qk8, qk_s) of the [L, 2 H 128] q|k view, and
        v's first k_len rows transposed (vt8, v_s)."""
        L, C = qkv.shape[0], H * self.head_dim
        Lkp = ops.vt8_keys(k_len)
        qk8, qk_s = self._act8("qk8", L, 2 * C)
        vt8 = self._buf("vt8", (H, 128, Lkp), torch.float8_e4m3fn)
        v_s = self._buf("vt8_s", (H, Lkp // 128), _F32)
        ops.quant_rows_fp8(qkv[:, :2 * C], qk8, qk_s)
        ops.quant_vt_fp8(qkv[:k_len, 2 * C:], vt8, v_s, H)
        return qk8, qk_s, vt8, v_s

    def weight_bytes(self) -> int:
        """Bytes of every weight tensor the engine holds on its device (bench and tests compare the two precisions)."""
        seen, total = set(), 0

        def add(t):
            nonlocal total
            if isinstance(t, Tensor) and t.data_ptr() not in seen:
                seen.add(t.data_ptr())
                total += t.numel() * t.element_size()
            elif isinstance(t, (tuple, list)):
                for u in t:
                    add(u)
            elif isinstance(t, dict):
                for u in t.values():
                    add(u)
        for v in vars(self).values():
            if v is self._ws or v is self._rope_cache or v is self._graphs or v is self._ctx_entries:
                continue
            add(v)
        return total

    def rope_from_reference(self, freqs: Tensor, grid: Optional[Sequence[int]], packed: bool) -> Tuple[Tensor, int]:
        """(cos, sin) table + number of rotated rows from what the reference hands its blocks: on the FramePack path `freqs`
        is the per-token complex table [L, 1, D/2] (model.py:101-105) and is converted as is; on the grid path it is the
        [1024, D/2] axis table and the rows follow from `grid` = (f, h, w) (model.py:54-69) — rebuilt from the same formula."""
        if packed:
            t = torch.view_as_real(freqs.reshape(-1, self.head_dim // 2).to(torch.complex128)).to(_F32).contiguous()
            return t.to(self.device), t.shape[0]
        f, h, w = (int(v) for v in grid)
        t = self._rope_table([(f, h, w, 0)])
        return t, t.shape[0]

    @torch.no_grad()
    def block_forward(self, i: int, x: Tensor, e: Tensor, grid: Optional[Tuple[int, int, int]], context: Tensor,
                      freqs: Optional[Tensor] = None, packed: bool = False, k_len: Optional[int] = None) -> Tensor:
        """Single-block entry (BASELINE.json configs[0]; the `WanAttentionBlock.forward` seam): the arithmetic of one block
        for one sample. x f32 [L, C]; e f32 [L, 6, C] (5B, per token) or [6, C] (14B); context bf16/f32 [S, C] already
        embedded; rope rows from `grid` (regular grid) or the reference's per-token `freqs` (packed); k_len = rows that are
        self-attention keys (seq_lens; default all)."""
        C = self.dim
        with torch.cuda.device(self.device):
            xs = x.to(device=self.device, dtype=_F32).clone().contiguous()
            L = xs.shape[0]
            e = e.to(device=self.device, dtype=_F32)
            if e.dim() == 2:
                e0, tok_idx = e.reshape(1, 6 * C), None
            else:
                e0, tok_idx = e.reshape(L, 6 * C).contiguous(), torch.arange(L, device=self.device, dtype=torch.int32)
            mod = ops.bcast_add(self.block_mod[i:i + 1], e0).view(1, e0.shape[0], 6, C)
            rope, rope_len = self.rope_from_reference(freqs, grid, packed) if (packed or freqs is not None) else \
                (self._rope_table([(grid[0], grid[1], grid[2], 0)]), grid[0] * grid[1] * grid[2])
            kv = self._cross_kv(context.to(device=self.device, dtype=_BF16).contiguous(), block=i)[0]
            with self.sequence_parallel_disabled():           # one sample on this GPU, also under Ulysses
                self._block_body(i, xs, mod[0], tok_idx, rope, min(rope_len, L), kv, L if k_len is None else int(k_len))
        return xs

    @torch.no_grad()
    def self_attention_forward(self, i: int, x: Tensor, grid: Optional[Tuple[int, int, int]], freqs: Optional[Tensor],
                               packed: bool, k_len: Optional[int] = None) -> Tensor:
        """`WanSelfAttention.forward` seam for one sample: x [L, C] (the modulated, normalised input) -> o(attention(...)) as
        bf16 [L, C] — q/k/v projection, RMSNorm(q), RMSNorm(k), RoPE, attention, output projection; no gate, no residual
        (wan23/modules/model.py:178-207)."""
        C = self.dim
        with torch.cuda.device(self.device):
            h = x.to(device=self.device, dtype=_BF16).contiguous()
            L = h.shape[0]
            rope, rope_len = self.rope_from_reference(freqs, grid, packed)
            qkv = self._buf("qkv", (L, 3 * C), _BF16)
            att = self._buf("att", (L, C), _BF16)
            a = self._quant(h, "h8")
            out = torch.empty(L, C, device=self.device, dtype=_BF16)
            self._self_attention(self.blocks[i], a, qkv, att, rope, min(rope_len, L), L if k_len is None else int(k_len), out,
                                 ops.YB_EPI_BF16)
        return out

    # ------------------------------------------------------------------------------------------------------
    # forward
    # ------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, x: Tensor, t: Tensor, context: Tensor, seq_len: int, y: Optional[Tensor] = None,
                clip_fea: Optional[Tensor] = None, latent_frame_zero: Optional[int] = None, packed: bool = True) -> Tensor:
        """One sample. x f32 [C_x, F, H, W] (+ y concatenated on channels), t f32 [1] or [1, L] / [2]-style
        (first = history, last = new), context [S<=text_len, text_dim]. Returns f32 [C_out, F_new, H, W]."""
        with torch.cuda.device(self.device):               # launches take the stream of the ENGINE's device
            if self.use_cuda_graph and self.sp_world == 1 and not self.timer.active:
                # arbitrary per-token t goes through torch.unique (host sync): not capturable
                if self.variant == "14b" or packed or t.numel() == 1:
                    return self._forward_graphed(x, t, context, seq_len, y, clip_fea, latent_frame_zero, packed)
            return self._forward_eager(x, t, context, seq_len, y, clip_fea, latent_frame_zero, packed)

    def _forward_graphed(self, x, t, context, seq_len, y, clip_fea, latent_frame_zero, packed) -> Tensor:
        """CUDA-graph replay of the step: inputs are copied into static device buffers, the graph (captured on first
        use of a geometry, after one eager warm-up run that sizes every workspace buffer) replays all launches, the
        result is copied out of the graph's static output. With the context cache on, the graph contains the step only
        and reads the cached K|V of (context, clip_fea); otherwise the context embedding is part of the graph."""
        dev = self.device
        cached = self.context_cache
        ckey = (context.data_ptr(), context._version, tuple(context.shape),
                None if clip_fea is None else (clip_fea.data_ptr(), clip_fea._version)) if cached else \
            (tuple(context.shape), None if clip_fea is None else tuple(clip_fea.shape))
        key = (tuple(x.shape), None if y is None else tuple(y.shape), t.numel(), int(seq_len), latent_frame_zero,
               bool(packed), cached, ckey)
        g = self._graphs.get(key)
        if g is None:
            st = dict(x=torch.empty(x.shape, device=dev, dtype=_F32), t=torch.empty(t.numel(), device=dev, dtype=_F32),
                      y=None if y is None else torch.empty(y.shape, device=dev, dtype=_F32),
                      ctx=context if cached else torch.empty(context.shape, device=dev, dtype=context.dtype),
                      clip=clip_fea if (cached or clip_fea is None) else torch.empty(clip_fea.shape, device=dev,
                                                                                     dtype=clip_fea.dtype))
            st["x"].copy_(x)
            st["t"].copy_(t.flatten())
            if y is not None:
                st["y"].copy_(y)
            if not cached:
                st["ctx"].copy_(context)
                if clip_fea is not None:
                    st["clip"].copy_(clip_fea)
            args = (st["x"], st["t"], st["ctx"], seq_len, st["y"], st["clip"], latent_frame_zero, packed)
            self._forward_eager(*args)                          # warm-up: allocates workspaces, fills the context cache
            torch.cuda.synchronize(dev)
            graphs_before = self._graphs
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                st["out"] = self._forward_eager(*args)
            st["graph"] = graph
            if self._graphs is graphs_before:                   # (a workspace change during capture would have cleared it)
                self._graphs[key] = st
            g = st
        else:
            g["x"].copy_(x, non_blocking=True)
            g["t"].copy_(t.flatten(), non_blocking=True)
            if y is not None:
                g["y"].copy_(y, non_blocking=True)
            if not cached:
                g["ctx"].copy_(context, non_blocking=True)
                if clip_fea is not None:
                    g["clip"].copy_(clip_fea, non_blocking=True)
        g["graph"].replay()
        return g["out"].clone()

    def _forward_eager(self, x: Tensor, t: Tensor, context: Tensor, seq_len: int, y: Optional[Tensor] = None,
                       clip_fea: Optional[Tensor] = None, latent_frame_zero: Optional[int] = None,
                       packed: bool = True) -> Tensor:
        dev, C = self.device, self.dim
        x = x.to(device=dev, dtype=_F32)
        if y is not None:
            x = torch.cat([x, y.to(device=dev, dtype=_F32)], dim=0)
        if x.shape[0] != self.in_dim:
            raise YumeB200Error(f"input has {x.shape[0]} channels, model expects {self.in_dim}")
        if latent_frame_zero is None:
            latent_frame_zero = 8 if self.variant == "5b" else 9
        cin, Ftot, Hh, Ww = x.shape

        # ---- tokens + rope table -----------------------------------------------------------------------
        if packed:
            hist = Ftot - latent_frame_zero
            if hist < 1:
                raise YumeB200Error("FramePack needs at least one history frame (u1 is empty in the reference)")
            branch_hist = Ftot - (latent_frame_zero if self.variant == "5b" else 9)
            plan = framepack_plan(hist, branch_hist)
            u1, u2 = x[:, :hist], x[:, hist:]
            shapes = []
            for seg in plan:                                   # token counts first (to size the stream)
                f = seg.frames.stop - seg.frames.start
                hh, ww = Hh, Ww
                if seg.pre_2x_f:
                    hh, ww = -(-hh // 4), -(-ww // 4)
                if seg.name == "patch_embedding":              # un-padded embedder floors (see _embed_tokens)
                    shapes.append((f, hh // 2, ww // 2))
                else:
                    shapes.append((f, -(-hh // seg.patch), -(-ww // seg.patch)))
            new_shape = (latent_frame_zero, Hh // 2, Ww // 2)
            L_hist = sum(f * a * b for f, a, b in shapes)
            L = L_hist + new_shape[0] * new_shape[1] * new_shape[2]
            xs, window = self._token_stream(L, L)
            row, f_z, rope_segs = 0, 0, []
            for seg, (f, hp, wp) in zip(plan, shapes):
                src = u1[:, seg.frames]
                if seg.pre_2x_f:                               # model.py:696-698
                    wpre, bpre = self.embed["patch_embedding_2x_f"]
                    f2, h2, w2 = f, -(-Hh // 4), -(-Ww // 4)
                    tmp = self._buf("pre2xf", (f2 * h2 * w2, wpre.shape[0]), _F32)
                    a = self._buf("patch_a", (f2 * h2 * w2, wpre.shape[1]), _BF16)
                    ops.patchify(src, a, 4, 4)
                    ops.gemm(a, wpre, bpre, tmp, ops.YB_EPI_F32)
                    ld = tmp.stride(0)                         # view the token-major result as [Cin, f, h, w]
                    src = torch.as_strided(tmp, (cin, f2, h2, w2), (1, h2 * w2 * ld, w2 * ld, ld))
                n = f * hp * wp
                self._embed_tokens(src, seg.name, seg.patch, xs, row, window)
                rope_segs.append((f, hp, wp, f_z))
                row += n
                f_z += f
            self._embed_tokens(u2, "patch_embedding", 2, xs, row, window)
            rope_segs.append((*new_shape, f_z))
            grid_new, rope_len = new_shape, L
        else:
            grid_new = (Ftot, Hh // 2, Ww // 2)
            L_grid = grid_new[0] * grid_new[1] * grid_new[2]
            if L_grid > seq_len:
                raise AssertionError("seq_lens.max() <= seq_len")   # model.py:755
            L, L_hist = seq_len, 0
            xs, window = self._token_stream(L, L_grid)         # rows >= L_grid: zero padding tokens (model.py:756-759)
            self._embed_tokens(x, "patch_embedding", 2, xs, 0, window)
            rope_segs, rope_len = [(*grid_new, 0)], L_grid
        rope = self._rope_table(rope_segs)

        # ---- timestep tables ---------------------------------------------------------------------------
        t = t.to(device=dev, dtype=_F32).flatten()
        tok_idx = None
        if self.variant == "14b":
            t_unique = t[:1]                                   # per-sample e (wan/modules/model.py:924-928)
        elif packed:
            t_unique = torch.stack([t[0], t[-1]])              # history tokens t[0], new tokens t[-1] (:730-737)
            tok_idx = self._buf("tok_idx", (L,), torch.int32)
            tok_idx[:L_hist] = 0
            tok_idx[L_hist:] = 1
        elif t.numel() == 1:
            t_unique = t
        else:                                                  # arbitrary per-token vector (t2v_dmd, textimage2video.py:629-634)
            if t.numel() != L:
                raise YumeB200Error("per-token t must have seq_len entries")
            t_unique, inv = torch.unique(t, return_inverse=True)
            tok_idx = inv.to(torch.int32).contiguous()
        e_parts, mod_parts, head_parts = [], [], []
        for s in range(0, t_unique.numel(), 16):               # the small-M linear handles 16 rows per launch
            e_, m_, h_ = self._time_tables(t_unique[s:s + 16].contiguous())
            e_parts.append(e_), mod_parts.append(m_), head_parts.append(h_)
        mod = mod_parts[0] if len(mod_parts) == 1 else torch.cat(mod_parts, dim=1).contiguous()
        head_tab = head_parts[0] if len(head_parts) == 1 else torch.cat(head_parts, dim=0).contiguous()

        # ---- context -----------------------------------------------------------------------------------
        ctx = self._context_kv(context, clip_fea)

        # ---- Ulysses: keep only this rank's contiguous token shard --------------------------------------
        # rows that serve as self-attention keys: every row, except on the 14B regular-grid path where the reference
        # masks the zero padding beyond F*H*W (k_lens = seq_lens, wan/modules/model.py:311-314, 916)
        L_true = L_grid if (self.variant == "14b" and not packed) else L
        if self.sp_world > 1:
            import torch.distributed as dist
            Lp, r0, n_valid = sp_shard(L, self.sp_world, self.sp_rank)   # xs already IS this rank's shard (_token_stream)
            if tok_idx is not None:
                ti = self._buf("tok_idx_shard", (Lp,), torch.int32)
                ti.zero_()
                ti[:n_valid].copy_(tok_idx[r0:r0 + n_valid])
                tok_idx = ti
            self._sp_rope_global = (rope, rope_len)              # the p2p_gemm transport rotates on the receiver: global rows
            rope = rope[min(r0, rope.shape[0]):]
            if rope.shape[0] == 0:
                rope = self._rope_table(rope_segs)[:1]
            rope_len = max(0, min(rope_len - r0, Lp))

        # ---- blocks ------------------------------------------------------------------------------------
        for i in range(self.layers):
            self._block(i, xs, mod, tok_idx, rope, rope_len, ctx, L_true)

        # ---- head + unpatchify (fp32, model.py:336-348, 856-890) -----------------------------------------
        Lloc = xs.shape[0]
        hn = self._buf("head_in", (Lloc, C), _F32)
        ops.ln_modulate(xs, hn, head_tab[:, 1], head_tab[:, 0], tok_idx, eps=self.eps)
        yo = self._buf("head_out", (Lloc, 4 * self.out_dim), _F32)
        ops.linear_f32(hn, self.head_w, self.head_b, yo)
        if self.sp_world > 1:                                  # one gather of the head output (gather_forward, :140)
            yo_all = self._buf("head_out_all", (self.sp_world * Lloc, 4 * self.out_dim), _F32)
            dist.all_gather_into_tensor(yo_all, yo, group=self.sp_group)
            yo = yo_all
        out = torch.empty(self.out_dim, grid_new[0], grid_new[1] * 2, grid_new[2] * 2, device=dev, dtype=_F32)
        ops.unpatchify(yo[L_hist:], out, grid_new[0], grid_new[1], grid_new[2], 2, 2)
        return out
