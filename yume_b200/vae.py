"""H100 decode path of the HunyuanVideo causal 3D VAE (`AutoencoderKLCausal3D.decode`, SURVEY.md §8 rows a17-a19).

Reference (file:line in /root/reference/hyvideo/vae):
  autoencoder_kl_causal_3d.py:297-341 decode/_decode, :343-359 blend_v/h/t, :417-463 spatial tiling, :500-531 temporal
  vae.py:131-291 DecoderCausal3D      unet_causal_3d_blocks.py:48-74 CausalConv3d, :129-182 UpsampleCausal3D,
  :348-415 ResnetBlockCausal3D, :615-628 mid block (+ diffusers Attention, pinned diffusers==0.32.0)

Layer table per tile z [16, T, H, W] (upstream 884-16c config, SURVEY.md Appendix C):
  post_quant_conv 1x1x1 16->16 | conv_in 16->512 | mid: resnet, frame-causal 1-head attention (d=512), resnet |
  up0: 3 resnets @512, up (1,2,2)+conv | up1: 3 resnets @512, up (2,2,2)+conv | up2: 3 resnets 512->256, up (2,2,2)+conv |
  up3: 3 resnets 256->128 | GroupNorm, SiLU, conv_out 128->3

H100 mapping: activations are channels-last bf16 [T*H*W, C]. Every 3x3x3 CausalConv3d is an implicit GEMM on the
wgmma kernel (yb_conv3d_causal: 4-D TMA boxes over a replicate-padded buffer, no im2col); GroupNorm-apply + SiLU +
nearest upsample + replicate padding are ONE gather pass that writes that padded buffer (yb_vae_pad_act); the resnet
skip add rides in the conv epilogue (YB_EPI_RES_BF16); the mid-block attention is five GEMM calls around a
frame-causal softmax kernel (no [L, L] mask tensor is ever built; the reference builds it with a Python loop over L).
Tiling / cross-fade follow the reference's order of in-place blends exactly. Status: parity-checked against the
reference-generated fixtures at reduced width (tests/test_gpu_parity.py); full-size performance tuning (conv tile
shapes for the 256x256 level, fusing GroupNorm statistics into the conv epilogue) is next-round work.
"""
from __future__ import annotations

import types
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import ops
from ._lib import YumeB200Error

Tensor = torch.Tensor
_BF16, _F32 = torch.bfloat16, torch.float32

CONFIG_884_16C = dict(in_channels=3, out_channels=3, latent_channels=16, block_out_channels=(128, 256, 512, 512),
                      layers_per_block=2, norm_num_groups=32, act_fn="silu", sample_size=256, sample_tsize=64,
                      scaling_factor=0.476986, time_compression_ratio=4, spatial_compression_ratio=8,
                      mid_block_add_attention=True)


@dataclass
class DecoderOutput:
    sample: Tensor


def _rup(v: int, m: int) -> int:
    return (v + m - 1) // m * m


class HyVaeDecoder:
    """Engine: re-packed decoder weights + the decode orchestration. `sd` uses the reference's state-dict keys."""

    def __init__(self, sd: Dict[str, Tensor], block_out_channels: Sequence[int] = (128, 256, 512, 512),
                 layers_per_block: int = 2, norm_num_groups: int = 32, sample_size: int = 256, sample_tsize: int = 64,
                 time_compression_ratio: int = 4, spatial_compression_ratio: int = 8, latent_channels: int = 16,
                 out_channels: int = 3, device="cuda", **_):
        if time_compression_ratio != 4 or spatial_compression_ratio != 8 or len(block_out_channels) != 4:
            raise YumeB200Error("only the 884 layout (4 blocks, 4x temporal / 8x spatial) is supported")
        self.device = torch.device(device)
        self.boc, self.lpb, self.groups = tuple(block_out_channels), layers_per_block, norm_num_groups
        self.latent_channels, self.out_channels = latent_channels, out_channels
        self.tile_sample_min_tsize = sample_tsize
        self.tile_latent_min_tsize = sample_tsize // time_compression_ratio
        self.tile_sample_min_size = sample_size
        self.tile_latent_min_size = int(sample_size / 8)
        self.tile_overlap_factor = 0.25
        self.use_spatial_tiling = self.use_temporal_tiling = False
        self.up_factors = [(1, 2, 2), (2, 2, 2), (2, 2, 2), None]      # vae.py:176-195 for the 884 layout
        self._repack(sd)

    # ---- weights -------------------------------------------------------------------------------------------
    def _repack(self, sd: Dict[str, Tensor]) -> None:
        dev = self.device
        self.w: Dict[str, Tuple[Tensor, Tensor, int]] = {}     # name -> (weight bf16, bias f32, true Cout)
        self.norm: Dict[str, Tuple[Tensor, Tensor]] = {}
        for k, v in sd.items():
            if k.endswith(".conv.weight") and v.dim() == 5:
                name = k[:-len(".conv.weight")]
                co, ci, kt = v.shape[0], v.shape[1], v.shape[2]
                b = sd[name + ".conv.bias"].detach().to(dev, _F32)
                cop = _rup(co, 32)
                if kt == 3:                                     # [co, ci, kt, kh, kw] -> [co, tap, ci(pad 64)]
                    cp = _rup(ci, 64)
                    wt = torch.zeros(cop, 27, cp, device=dev, dtype=_BF16)
                    wt[:co, :, :ci] = v.detach().to(dev, _BF16).permute(0, 2, 3, 4, 1).reshape(co, 27, ci)
                    wt = wt.reshape(cop, 27 * cp).contiguous()
                else:                                           # 1x1x1 conv_shortcut: plain GEMM weight
                    wt = torch.zeros(cop, _rup(ci, 8), device=dev, dtype=_BF16)
                    wt[:co, :ci] = v.detach().to(dev, _BF16).reshape(co, ci)
                bp = torch.zeros(cop, device=dev, dtype=_F32)
                bp[:co] = b
                self.w[name] = (wt, bp, co)
            elif k.endswith(".weight") and v.dim() == 1:
                name = k[:-len(".weight")]
                self.norm[name] = (v.detach().to(dev, _F32).contiguous(), sd[name + ".bias"].detach().to(dev, _F32).contiguous())
        # post_quant_conv (plain nn.Conv3d 1x1x1): K padded to 64 so its output feeds conv_in's 64-channel padded input
        pq = sd["post_quant_conv.weight"].detach().to(dev, _BF16).reshape(self.latent_channels, self.latent_channels)
        wpq = torch.zeros(32, 64, device=dev, dtype=_BF16)
        wpq[:self.latent_channels, :self.latent_channels] = pq
        bpq = torch.zeros(32, device=dev, dtype=_F32)
        bpq[:self.latent_channels] = sd["post_quant_conv.bias"].detach().to(dev, _F32)
        self.w["post_quant_conv"] = (wpq, bpq, self.latent_channels)
        # mid-block attention: fold 1/sqrt(C) into q, fold the v bias through to_out (softmax rows sum to 1)
        a = "decoder.mid_block.attentions.0"
        C = self.boc[-1]
        f = lambda n: sd[f"{a}.{n}"].detach().to(dev, _F32)  # noqa: E731
        scale = C ** -0.5
        self.att = dict(
            wq=(f("to_q.weight") * scale).to(_BF16).contiguous(), bq=(f("to_q.bias") * scale).contiguous(),
            wk=f("to_k.weight").to(_BF16).contiguous(), bk=f("to_k.bias").contiguous(),
            wv=f("to_v.weight").to(_BF16).contiguous(),
            wo=f("to_out.0.weight").to(_BF16).contiguous(),
            bo=(f("to_out.0.bias") + f("to_out.0.weight") @ f("to_v.bias")).contiguous())

    # ---- building blocks -----------------------------------------------------------------------------------
    def _new(self, *shape, dtype=_BF16) -> Tensor:
        return torch.empty(*shape, device=self.device, dtype=dtype)

    def _conv3(self, name: str, x: Tensor, src_dims, up=(1, 1, 1), norm: Optional[str] = None, silu: bool = False,
               res: Optional[Tensor] = None, out_f32: bool = False):
        """[GroupNorm+SiLU] -> [upsample] -> replicate pad -> 3x3x3 causal conv [+ res]. x bf16 [Ts*Hs*Ws, C]."""
        w, b, co = self.w[name]
        Ts, Hs, Ws = src_dims
        T = 1 + 2 * (Ts - 1) if up[0] == 2 else Ts
        H, W = Hs * up[1], Ws * up[2]
        cp = w.shape[1] // 27
        xpad = self._new(T + 2, H + 2, W + 2, cp)
        if norm is not None:
            g, bt = self.norm[norm]
            ops.vae_pad_act(x, src_dims, xpad, True, up, ops.gn_stats(x, self.groups), g, bt, self.groups, 1e-6, silu)
        else:
            ops.vae_pad_act(x, src_dims, xpad, True, up)
        out = self._new(T * H * W, w.shape[0], dtype=_F32 if out_f32 else _BF16)
        epi = ops.YB_EPI_F32 if out_f32 else (ops.YB_EPI_RES_BF16 if res is not None else ops.YB_EPI_BF16)
        ops.conv3d_causal(xpad, w, b, out, T, H, W, epi, res)
        return out, (T, H, W)

    def _resnet(self, p: str, x: Tensor, dims) -> Tensor:
        """ResnetBlockCausal3D.forward (temb None, no up/down, output_scale_factor 1)."""
        h, _ = self._conv3(p + ".conv1", x, dims, norm=p + ".norm1", silu=True)
        res = x
        if (p + ".conv_shortcut") in self.w:
            w, b, _ = self.w[p + ".conv_shortcut"]
            res = self._new(x.shape[0], w.shape[0])
            ops.gemm(x, w, b, res, ops.YB_EPI_BF16)
        out, _ = self._conv3(p + ".conv2", h, dims, norm=p + ".norm2", silu=True, res=res)
        return out

    def _mid_attention(self, x: Tensor, dims) -> Tensor:
        """Frame-causal single-head attention over all T*H*W tokens (unet_causal_3d_blocks.py:617-626)."""
        T, H, W = dims
        L, C = x.shape
        Lp = _rup(L, 32)
        g, bt = self.norm["decoder.mid_block.attentions.0.group_norm"]
        hn = torch.zeros(Lp, C, device=self.device, dtype=_BF16)
        ops.vae_pad_act(x, dims, hn[:L].view(T, H, W, C), False, (1, 1, 1), ops.gn_stats(x, self.groups), g, bt, self.groups,
                        1e-6, False)
        a = self.att
        q, k = self._new(L, C), self._new(Lp, C)
        ops.gemm(hn[:L], a["wq"], a["bq"], q, ops.YB_EPI_BF16)
        ops.gemm(hn, a["wk"], a["bk"], k, ops.YB_EPI_BF16)
        vT = self._new(C, Lp)                                   # V^T = Wv . hn^T  (its bias is folded into bo)
        ops.gemm(a["wv"], hn, None, vT, ops.YB_EPI_BF16)
        S = self._new(L, Lp, dtype=_F32)
        ops.gemm(q, k, None, S, ops.YB_EPI_F32)
        P = self._new(L, Lp)
        ops.masked_softmax(S, P, L, H * W)
        del S
        o = self._new(L, C)
        ops.gemm(P, vT, None, o, ops.YB_EPI_BF16)
        out = self._new(L, C)
        ops.gemm(o, a["wo"], a["bo"], out, ops.YB_EPI_RES_BF16, res=x)
        return out

    def decode_tile(self, z: Tensor) -> Tensor:
        """post_quant_conv + DecoderCausal3D.forward on one tile z f32 [16, T, H, W] -> f32 [3, 4(T-1)+1, 8H, 8W]."""
        cl, T, H, W = z.shape
        N = T * H * W
        zl = self._new(N, 64)
        ops.nchw_to_nhwc_bf16(z.reshape(cl, N).contiguous(), zl)
        wpq, bpq, _ = self.w["post_quant_conv"]
        x0 = torch.zeros(N, 64, device=self.device, dtype=_BF16)
        ops.gemm(zl, wpq, bpq, x0[:, :32], ops.YB_EPI_BF16)
        dims = (T, H, W)
        x, dims = self._conv3("decoder.conv_in", x0, dims)
        x = self._resnet("decoder.mid_block.resnets.0", x, dims)
        x = self._mid_attention(x, dims)
        x = self._resnet("decoder.mid_block.resnets.1", x, dims)
        for i in range(4):
            for j in range(self.lpb + 1):
                x = self._resnet(f"decoder.up_blocks.{i}.resnets.{j}", x, dims)
            if self.up_factors[i] is not None:
                x, dims = self._conv3(f"decoder.up_blocks.{i}.upsamplers.0.conv", x, dims, up=self.up_factors[i])
        y, dims = self._conv3("decoder.conv_out", x, dims, norm="decoder.conv_norm_out", silu=True, out_f32=True)
        out = self._new(self.out_channels, dims[0] * dims[1] * dims[2], dtype=_F32)
        ops.nhwc_to_nchw_f32(y, out)
        return out.view(1, self.out_channels, *dims)

    # ---- tiling -----------------------------------------------------------------------------------------------
    def enable_tiling(self, use_tiling: bool = True) -> None:
        self.use_spatial_tiling = self.use_temporal_tiling = use_tiling

    def enable_tile_parallel(self, group) -> None:
        """Spread the tiles of a tiled decode over the ranks of `group` (one process per GPU): tiles are independent, so rank r
        decodes tiles r, r + P, ...; every rank then receives the others' raw tiles (one broadcast per tile) and assembles the
        full video. SURVEY.md §8(e): 'VAE decode: tiles are independent -> tile-parallel replicas'
        (fastvideo/models/hunyuan/vae/autoencoder_kl_causal_3d.py:620-741 does the same with an all-gather)."""
        self.tile_group = group

    def tile_plan(self, T: int, H: int, W: int):
        """Windows of the reference's tiled decode for a latent [T, H, W] (autoencoder_kl_causal_3d.py:417-463, 500-531):
        (temporal windows [(t0, len)], row starts/sizes, column starts/sizes, spatially tiled?). Pure host arithmetic."""
        tmin, smin = self.tile_latent_min_tsize, self.tile_latent_min_size
        if self.use_temporal_tiling and T > tmin:
            ov = int(tmin * (1 - self.tile_overlap_factor))
            twin = [(i, min(tmin + 1, T - i)) for i in range(0, T, ov)]
            # a window that decodes to nothing after its first frame is dropped contributes no output (torch.cat of an empty tile)
            twin = [w for k, w in enumerate(twin) if k == 0 or 4 * (w[1] - 1) + 1 - 1 > 0]
        else:
            twin = [(0, T)]
        spatial = self.use_spatial_tiling and (W > smin or H > smin)
        if spatial:
            ov = int(smin * (1 - self.tile_overlap_factor))
            rows = [(i, min(smin, H - i)) for i in range(0, H, ov)]
            cols = [(j, min(smin, W - j)) for j in range(0, W, ov)]
        else:
            rows, cols = [(0, H)], [(0, W)]
        return twin, rows, cols, spatial

    @torch.no_grad()
    def decode(self, z: Tensor) -> Tensor:
        """z [1, 16, T, H, W] -> f32 [1, 3, 4(T-1)+1, 8H, 8W]. Tiled decodes: every tile is decoded RAW (in any order, on any
        rank), then one kernel (`yb_vae_assemble_tiles`) writes the final video, evaluating the reference's in-place
        cross-fade / crop / concatenate sequence per output voxel — no torch.cat, no per-row blend launches."""
        assert len(z.shape) == 5, "The input tensor should have 5 dimensions."      # autoencoder_kl_causal_3d.py:298
        if z.shape[0] != 1:
            return torch.cat([self.decode(zi[None]) for zi in z])                   # use_slicing semantics (:335-337)
        z = z.to(device=self.device, dtype=_F32)
        _, _, T, H, W = z.shape
        twin, rows, cols, spatial = self.tile_plan(T, H, W)
        if len(twin) == 1 and not spatial:
            return self.decode_tile(z[0])
        group = getattr(self, "tile_group", None)
        world, rank = 1, 0
        if group is not None:
            import torch.distributed as dist
            world, rank = dist.get_world_size(group), dist.get_rank(group)
        C = self.out_channels
        tiles, k = [], 0
        for (t0, tl) in twin:
            plane = []
            for (i0, hs) in rows:
                line = []
                for (j0, ws) in cols:
                    shape = (C, 4 * (tl - 1) + 1, 8 * hs, 8 * ws)
                    if k % world == rank:
                        tile = self.decode_tile(z[0, :, t0:t0 + tl, i0:i0 + hs, j0:j0 + ws]).reshape(shape)
                    else:
                        tile = torch.empty(shape, device=self.device, dtype=_F32)
                    line.append(tile)
                    k += 1
                plane.append(line)
            tiles.append(plane)
        if world > 1:                                      # exchange the raw tiles: one broadcast per tile from its owner
            k = 0
            for plane in tiles:
                for line in plane:
                    for tile in line:
                        dist.broadcast(tile, src=dist.get_global_rank(group, k % world), group=group)
                        k += 1
        # temporal layout: tile 0 keeps t_limit + 1 frames, later tiles drop their first frame and keep t_limit (:519-531)
        t_blend = int(self.tile_sample_min_tsize * self.tile_overlap_factor)
        t_limit = self.tile_sample_min_tsize - t_blend
        tlen = [4 * (tl - 1) + 1 - (1 if n > 0 else 0) for n, (_, tl) in enumerate(twin)]
        keep = [min(L, t_limit + (1 if n == 0 else 0)) for n, L in enumerate(tlen)] if len(twin) > 1 else [tlen[0]]
        tf0 = [sum(keep[:n]) for n in range(len(twin))]
        blend = int(self.tile_sample_min_size * self.tile_overlap_factor)
        row_limit = self.tile_sample_min_size - blend
        th, tw = [8 * hs for _, hs in rows], [8 * ws for _, ws in cols]
        Ho = sum(min(row_limit, h) for h in th) if spatial else th[0]
        Wo = sum(min(row_limit, w) for w in tw) if spatial else tw[0]
        out = torch.empty(C, sum(keep), Ho, Wo, device=self.device, dtype=_F32)
        ops.vae_assemble_tiles(tiles, th, tw, tlen, tf0, out, row_limit, blend, t_limit, t_blend)
        return out[None]


def decoder_param_shapes(block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=16,
                         out_channels=3) -> Dict[str, tuple]:
    """State-dict keys / shapes of the decode half of AutoencoderKLCausal3D (vae.py:141-223 module tree)."""
    boc = list(block_out_channels)
    rev = boc[::-1]
    s: Dict[str, tuple] = {"post_quant_conv.weight": (latent_channels, latent_channels, 1, 1, 1),
                           "post_quant_conv.bias": (latent_channels,)}

    def conv(p, ci, co, k=3):
        s[p + ".conv.weight"], s[p + ".conv.bias"] = (co, ci, k, k, k), (co,)

    def norm(p, c):
        s[p + ".weight"], s[p + ".bias"] = (c,), (c,)

    def resnet(p, ci, co):
        norm(p + ".norm1", ci), conv(p + ".conv1", ci, co), norm(p + ".norm2", co), conv(p + ".conv2", co, co)
        if ci != co:
            conv(p + ".conv_shortcut", ci, co, 1)

    c = rev[0]
    conv("decoder.conv_in", latent_channels, c)
    resnet("decoder.mid_block.resnets.0", c, c)
    a = "decoder.mid_block.attentions.0"
    norm(a + ".group_norm", c)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        s[f"{a}.{n}.weight"], s[f"{a}.{n}.bias"] = (c, c), (c,)
    resnet("decoder.mid_block.resnets.1", c, c)
    prev = c
    for i in range(4):
        co = rev[i]
        for j in range(layers_per_block + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else co, co)
        if i < 3:
            conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", co, co)
        prev = co
    norm("decoder.conv_norm_out", boc[0])
    conv("decoder.conv_out", boc[0], out_channels)
    return s


def install_vae(vae, device="cuda"):
    """Attach a HyVaeDecoder to a live reference `AutoencoderKLCausal3D` and re-bind its `decode`
    (same signature and return convention as autoencoder_kl_causal_3d.py:315-341)."""
    cfg = vae.config
    get = (lambda k, d=None: cfg.get(k, d)) if isinstance(cfg, dict) else (lambda k, d=None: getattr(cfg, k, d))
    eng = HyVaeDecoder(dict(vae.state_dict()), block_out_channels=get("block_out_channels"),
                       layers_per_block=get("layers_per_block"), norm_num_groups=get("norm_num_groups", 32),
                       sample_size=get("sample_size"), sample_tsize=get("sample_tsize"),
                       latent_channels=get("latent_channels", 16), out_channels=get("out_channels", 3), device=device)
    vae._yb_decoder = eng

    def decode(self, z, return_dict: bool = True, generator=None):
        eng.use_spatial_tiling, eng.use_temporal_tiling = self.use_spatial_tiling, self.use_temporal_tiling
        dec = eng.decode(z).to(z.dtype)
        if not return_dict:
            return (dec,)
        return DecoderOutput(sample=dec)

    vae.decode = types.MethodType(decode, vae)
    return vae
