"""What the four Wan VAE engines share — `Wan22VaeDecoder` (vae22.py), `Wan21VaeDecoder` (vae21.py) and the two encoders
(vae_enc.py): weight re-packing, the building blocks (causal conv, RMS_norm + SiLU, ResidualBlock, the mid attention), the conv
history carried from chunk to chunk, and the chunk driver and planner. Each engine describes its network once, as a layer list
built from its config: `_run_chunk` walks it to run a chunk and `chunk_bytes` walks it to bound one.
"""
from __future__ import annotations

from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

import torch

from ._lib import YumeB200Error
from .vae_rows import RowGroup

Tensor = torch.Tensor
_BF16, _F32, _E4M3 = torch.bfloat16, torch.float32, torch.float8_e4m3fn


def _rup(v: int, m: int) -> int:
    return (v + m - 1) // m * m


class Layer(NamedTuple):
    """One step of an engine's layer list. `hold` keeps the level's input for the DupUp3D / AvgDown3D shortcut that ends the
    level (`dupup`, `avgdown`)."""
    kind: str               # in | res | attn | hold | up | down | dupup | avgdown | head
    name: str = ""          # module prefix in the state dict
    ci: int = 0             # input channels (hold: those of the held input)
    co: int = 0             # output channels (head: the output columns the planner counts at 4 bytes)
    ft: int = 1             # in: frames per latent frame; up / down / shortcut: time factor
    fs: int = 1             # in: patch size; up / down / shortcut: space factor


def _frames_of(units: int, k: int) -> int:
    """Frames of a stream that hold its first `units` latent frames, k frames per latent frame after frame 0."""
    return 1 + (units - 1) * k if units else 0


class _Kept(NamedTuple):
    """What a resuming engine keeps from its last call (WanVaeEngine._resumed)."""
    src: Tensor                     # its own copy of the input (device, f32)
    out: Tensor                     # the result returned (the caller's tensor; a private copy when `version` is None)
    version: Optional[int]          # out._version when returned: an in-place edit by the caller makes the next call run in full
    snaps: Dict[int, Tuple[int, dict]]   # input frames P -> (latent frames, the carries after them)


class WanVaeEngine:
    """Base of the four engines. An engine builds its layer list from its config and hands it to this constructor; its side
    (decode or encode) supplies `_repack`, the `in`, `up` / `down` and `head` steps (`_input`, `_resample`, `_head`) and `ops`,
    the op library of its own module (which tests replace, module by module, with a CPU stand-in)."""
    # chunk-streaming state of the running call: chunk index, whether another chunk follows, carried conv input frames
    _chunk, _more, _carry = 0, False, None
    HIST = 2                     # carried frames of a 3-tap causal conv (the reference's CACHE_T)
    MEM_MARGIN = 2 << 30         # bytes of free device memory the chunk planner leaves unused
    PRECISIONS = ("bf16",)       # precision= values the engine accepts (Wan22VaeDecoder adds "fp8")
    # precision="fp8": the convs that run on e4m3 operands (Wan22VaeDecoder._repack decides), name -> (Wq e4m3 [cop, taps*cp],
    # s_w f32 [cop], bias f32 [cop], taps). Their input streams are (e4m3 frames, scale frames) pairs, see _hist_buf.
    conv8: Dict[str, Tuple[Tensor, Tensor, Tensor, tuple]] = {}
    _kept: Optional[_Kept] = None   # resume=True: the state kept from the last call
    # row-parallel decode or encode (enable_row_parallel): the RowGroup of the ranks (None: one rank runs everything) and, during a
    # call, the band (r0, rows, H) of the latent's H rows this rank owns. dims are then the band's (T, rows, W), and the input of
    # every conv with kh = 3 is a band buffer with one halo row above and below (include/yume_b200_vae_rows.h).
    _rows = None
    _band: Tuple[int, int, int] = (0, 0, 0)

    def __init__(self, sd: Dict[str, Tensor], z_dim: int, layers: List[Layer], mean: Optional[Tensor], std: Optional[Tensor],
                 device, precision: str = "bf16", resume: bool = False):
        if precision not in self.PRECISIONS:
            raise YumeB200Error(f"{type(self).__name__} supports precision {' or '.join(map(repr, self.PRECISIONS))}, got "
                                f"{precision!r} (the fp8 path is Wan22VaeDecoder's decode only)")
        self.precision = precision
        # resume=True keeps the last call's input, result and carries on the device, so that a call whose input extends the
        # last one runs only its new latent frames (_resumed); False keeps nothing between calls
        self.resume = bool(resume)
        self.device = torch.device(device)
        self.z_dim, self.layers = z_dim, layers
        mean = torch.zeros(z_dim) if mean is None else mean
        std = torch.ones(z_dim) if std is None else std
        self._repack(sd, mean.detach().to(self.device, _F32), std.detach().to(self.device, _F32))

    def enable_row_parallel(self, group=None) -> "WanVaeEngine":
        """Run on the ranks of `group` (torch.distributed; default the world), each rank its band of rows: rank r of P owns
        latent rows [floor(rH/P), floor((r+1)H/P)) and, at every other level, those rows times the level's scale. Every rank
        still passes the whole input and gets the whole result (a decode's clamped video, an encode's mu), equal bit for bit to
        the one-GPU call: the convs read one halo row of each neighbouring band (exchanged after every norm pass), the mid
        attention runs on the gathered full frames, and one all-gather at the end of a call assembles the result. A group of one
        rank keeps the one-GPU path. Call it on every rank; every later call is then a collective of the group. It drops the
        state a resuming engine keeps (reset()). Raises YumeB200Error without an initialised process group or with
        precision="fp8"."""
        if self.precision == "fp8":
            raise YumeB200Error("enable_row_parallel: the fp8 decode has no row-parallel form; use precision='bf16'")
        rows = RowGroup(group)
        self._rows = rows if rows.world > 1 else None
        self.reset()                                             # kept carries would belong to another band
        return self

    def _set_band(self, H: int) -> None:
        """Under a row-parallel call on H latent rows: this rank's band, or YumeB200Error (raised on every rank, before the first
        collective) when there are fewer rows than ranks."""
        if self._rows is None:
            return
        P = self._rows.world
        if H < P:
            raise YumeB200Error(f"a row-parallel {type(self).__name__} on {P} ranks needs at least {P} latent rows, got {H}")
        r0, r1 = self._rows.band(H)
        self._band = (r0, r1 - r0, H)

    def _row0(self, rows: int) -> int:
        """First row of this rank's band at a level whose band has `rows` rows."""
        r0, hs, _ = self._band
        return r0 * (rows // hs)

    # ---- weights -------------------------------------------------------------------------------------------
    def _pack_side(self, sd: Dict[str, Tensor], prefixes: Tuple[str, ...], latent_conv: str,
                   split_time_conv: bool) -> Dict[str, Tensor]:
        """Re-pack one side of a `WanVAE_` state dict (decode: `decoder.*` + `conv2`; encode: `encoder.*` + `conv1`): 3-D / 2-D
        convs as [cop, taps*cp] bf16 GEMM weights, 1x1x1 shortcuts as plain matrices, gammas flat, the mid attention with the
        softmax scale folded into q and the v bias folded through `proj`. Returns the fp32 device copy of that side."""
        dev = self.device
        sd = {k: v.detach().to(dev, _F32) for k, v in sd.items() if k.startswith(prefixes)}
        self.conv: Dict[str, Tuple[Tensor, Tensor, tuple]] = {}    # name -> (w bf16 [cop, taps*cp], bias f32 [cop], taps)
        self.lin: Dict[str, Tuple[Tensor, Tensor]] = {}            # 1x1x1 convs as plain GEMM weights
        self.gamma: Dict[str, Tensor] = {}

        def pack_conv(name: str, w: Tensor, b: Tensor) -> None:
            w = w.detach().float()
            if w.dim() == 4:                                        # Conv2d [co, ci, kh, kw] -> taps (1, kh, kw)
                w = w.unsqueeze(2)
            co, ci, kt, kh, kw = w.shape
            cop, cp = _rup(co, 32), _rup(ci, 64)
            wt = torch.zeros(cop, kt * kh * kw, cp, dtype=_F32, device=dev)
            wt[:co, :, :ci] = w.permute(0, 2, 3, 4, 1).reshape(co, kt * kh * kw, ci)
            bp = torch.zeros(cop, dtype=_F32, device=dev)
            bp[:co] = b.detach().float()
            self.conv[name] = (wt.reshape(cop, -1).to(dev, _BF16).contiguous(), bp.to(dev), (kt, kh, kw))

        latent_w = latent_conv + ".weight"
        for k, v in sd.items():
            if k.endswith(".gamma"):
                self.gamma[k[:-6]] = v.detach().to(dev, _F32).reshape(-1).contiguous()
            elif k.endswith(".weight") and v.dim() == 5 and tuple(v.shape[2:]) == (1, 1, 1) and k != latent_w:
                name = k[:-7]                                       # ResidualBlock.shortcut: plain GEMM
                co, ci = v.shape[:2]
                w = torch.zeros(_rup(co, 32), _rup(ci, 8), dtype=_F32, device=dev)
                w[:co, :ci] = v.detach().float().reshape(co, ci)
                b = torch.zeros(_rup(co, 32), dtype=_F32, device=dev)
                b[:co] = sd[name + ".bias"].detach().float()
                self.lin[name] = (w.to(dev, _BF16).contiguous(), b.to(dev))
            elif k.endswith(".time_conv.weight") and split_time_conv:
                name = k[:-7]
                C2 = v.shape[0]
                for g in (0, 1):                                    # the two channel groups become two output frames
                    pack_conv(f"{name}.{g}", v[g * C2 // 2:(g + 1) * C2 // 2], sd[name + ".bias"][g * C2 // 2:(g + 1) * C2 // 2])
            elif k.endswith(".weight") and v.dim() in (4, 5) and "to_qkv" not in k and ".proj." not in k and k != latent_w:
                pack_conv(k[:-7], v, sd[k[:-7] + ".bias"])
        # attention: scale folded into q; v bias folded through proj (softmax rows sum to 1)
        attn = next(L for L in self.layers if L.kind == "attn")
        C, p = attn.ci, attn.name
        Wqkv = sd[p + ".to_qkv.weight"].detach().float().reshape(3 * C, C)
        bqkv = sd[p + ".to_qkv.bias"].detach().float()
        Wo = sd[p + ".proj.weight"].detach().float().reshape(C, C)
        scale = C ** -0.5
        self.att = dict(wq=(Wqkv[:C] * scale).to(dev, _BF16).contiguous(), bq=(bqkv[:C] * scale).to(dev),
                        wk=Wqkv[C:2 * C].to(dev, _BF16).contiguous(), bk=bqkv[C:2 * C].to(dev).contiguous(),
                        wv=Wqkv[2 * C:].to(dev, _BF16).contiguous(),
                        wo=Wo.to(dev, _BF16).contiguous(),
                        bo=(sd[p + ".proj.bias"].detach().float() + Wo @ bqkv[2 * C:]).to(dev).contiguous())
        return sd

    # ---- building blocks -----------------------------------------------------------------------------------
    def _new(self, *shape, dtype=_BF16) -> Tensor:
        return torch.empty(*shape, device=self.device, dtype=dtype)

    @property
    def _one_pass(self) -> bool:
        """The running chunk is the whole sequence: it issues the one-pass launches."""
        return self._chunk == 0 and not self._more

    def _hist_buf(self, key: Optional[str], T: int, H: int, W: int, Cp: int, zero: bool = False, n: int = 0, fp8: bool = False,
                  halo: bool = False):
        """Input buffer [h + T, H, W, Cp] of a conv whose input stream is `key`: after the first chunk its first h frames (n, or
        HIST when n is 0) are the frames carried from the previous chunk and the producer writes the T new frames behind them.
        fp8: the pair (e4m3 [h + T, H, W, Cp], f32 scales [h + T, Cp / 128, H, W]) of an e4m3 conv's input, frames carried alike.
        halo: a band buffer [h + T, H + 2, W, Cp] (carried frames with their halo rows)."""
        h = (n or self.HIST) if (key is not None and self._chunk > 0) else 0
        H = H + 2 if halo else H
        if fp8:
            buf = (self._new(h + T, H, W, Cp, dtype=_E4M3), self._new(h + T, Cp // 128, H, W, dtype=_F32))
            if h:
                for b, c in zip(buf, self._carry[key]):
                    b[:h].copy_(c)
            return buf
        buf = torch.zeros(h + T, H, W, Cp, device=self.device, dtype=_BF16) if zero else self._new(h + T, H, W, Cp)
        if h:
            buf[:h].copy_(self._carry[key])
        return buf

    def _keep(self, key: str, frames, n: int = 0) -> None:
        """Carry the last n (0: HIST) frames of the input stream `key` into the next chunk (zero frames in front where the stream
        is shorter: the causal zero padding; for an e4m3 stream, zero values with zero scales)."""
        if not self._more:
            return
        n = n or self.HIST

        def last(f: Tensor) -> Tensor:
            if f.shape[0] >= n:
                return f[f.shape[0] - n:].clone()
            c = torch.zeros(n, *f.shape[1:], device=self.device, dtype=f.dtype)
            c[n - f.shape[0]:].copy_(f)
            return c
        self._carry[key] = tuple(last(f) for f in frames) if isinstance(frames, tuple) else last(frames)

    def _conv(self, name: str, a, dims, epilogue=None, res: Optional[Tensor] = None, out: Optional[Tensor] = None,
              out_t_mul: int = 1, out_t_add: int = 0, stride_t: int = 1, stride_hw: int = 1, key: Optional[str] = None) -> Tensor:
        """a bf16 [h + T, H, W, Cp] (unpadded, dense; h carried frames in front, see _hist_buf) -> [To*Ho*Wo (or interleaved
        frames), cop]. `key`: the input stream whose last frames the next chunk needs. An e4m3 conv (conv8) takes the pair
        _hist_buf(fp8=True) made and writes bf16 rows."""
        ops = self.ops
        T, H, W = dims
        if key is not None:                                      # a stride-2 time_conv carries one frame (vae2_2.py:158-170)
            self._keep(key, a, 1 if stride_t > 1 else self.HIST)
        if epilogue is None:
            epilogue = ops.YB_EPI_RES_BF16 if res is not None else ops.YB_EPI_BF16
        if isinstance(a, tuple):
            w8, sw, b, taps = self.conv8[name]
            if out is None:
                out = self._new(T * H * W, w8.shape[0])
            ops.conv3d_fp8(a[0], a[1], w8, sw, b, out, T, H, W, a[0].shape[0] - T, epilogue, res, taps=taps)
            return out
        w, b, taps = self.conv[name]
        h = a.shape[0] - T
        if out is None:
            To, Ho, Wo = ops.conv_out_dims(T, H, W, taps, stride_t, stride_hw)
            out = self._new(To * Ho * Wo, w.shape[0], dtype=_F32 if epilogue == ops.YB_EPI_F32 else _BF16)
        if self._rows is not None and a.shape[1] == H + 2 and stride_hw > 1:    # a band's Resample downsample2d
            ops.conv3d_rows_down(a, w, b, out, T, H, W, epilogue)
        elif self._rows is not None and a.shape[1] == H + 2:     # a band buffer (_act with halo): the row-halo conv
            ops.conv3d_rows(a, w, b, out, T, H, W, h, epilogue, res, taps=taps, full_h=self._band[2] * (H // self._band[1]))
        elif h:
            ops.conv3d_causal_hist(a, w, b, out, T, H, W, h, epilogue, res, taps=taps, out_t_mul=out_t_mul,
                                   out_t_add=out_t_add, stride_t=stride_t, stride_hw=stride_hw)
        else:
            ops.conv3d_causal(a, w, b, out, T, H, W, epilogue, res, taps=taps, oob_zero_pad=True, out_t_mul=out_t_mul,
                              out_t_add=out_t_add, stride_t=stride_t, stride_hw=stride_hw)
        return out

    def _act(self, x: Tensor, dims, gamma: Optional[str], silu: bool, up: int = 1, key: Optional[str] = None,
             n: int = 0, conv: Optional[str] = None, halo: bool = False, above: bool = True):
        """The input buffer of the conv `conv` (see _hist_buf): RMS_norm * gamma, SiLU, 2x upsample of x; an e4m3 pair when that
        conv is one of conv8. halo (a conv with kh = 3) under a row-parallel call: a band buffer whose halo rows of the T new
        frames come from the neighbouring ranks (above=False: only the row below, for the stride-2 Resample conv)."""
        ops = self.ops
        T, H, W = dims
        g = self.gamma[gamma] if gamma else None
        if halo and self._rows is not None:
            out = self._hist_buf(key, T, H * up, W * up, _rup(x.shape[1], 64), n=n, halo=True)
            send = self._new(2, T, W * up, out.shape[-1])
            ops.vae_rms_act_rows(x, dims, out[out.shape[0] - T:], g, up, silu, send=send)
            self._halo(out, T, send, above)
            return out
        if conv in self.conv8:
            q, s = self._hist_buf(key, T, H * up, W * up, _rup(x.shape[1], 64), n=n, fp8=True)
            ops.vae_rms_act_fp8(x, dims, q[q.shape[0] - T:], s[s.shape[0] - T:], g, up, silu)
            return q, s
        out = self._hist_buf(key, T, H * up, W * up, _rup(x.shape[1], 64), n=n)
        ops.vae_rms_act(x, dims, out[out.shape[0] - T:], g, up, silu)
        return out

    def _halo(self, buf: Tensor, T: int, send: Optional[Tensor] = None, above: bool = True) -> None:
        """Fill the halo rows of the T new frames of the band buffer `buf` from the neighbouring ranks (zeros at the image's
        edge). send [2, T, W, Cp]: the band's top and bottom rows of those frames, packed from `buf` when not given. above=False
        fills only the row below (the row above is then zeros)."""
        new = buf[buf.shape[0] - T:]
        if send is None:
            send = self._new(2, T, *buf.shape[2:])
            self.ops.vae_rows_pack(new, send)
        top, bot = self._rows.exchange(send) if above else (None, self._rows.from_below(send))
        self.ops.vae_rows_unpack(top, bot, new)

    def _attention_rows(self, p: str, x: Tensor, dims) -> Tensor:
        """The mid attention of a row-parallel decode: every rank gathers the full frames, runs `_attention` on them (the same
        launches as one rank) and keeps its own rows."""
        T, hs, W = dims
        r0, _, H = self._band
        C = x.shape[1]
        full = torch.cat(self._rows.gather(x.view(T, hs, W, C), 1, self._rows.sizes(H)), 1)
        y = self._attention(p, full.view(T * H * W, C), (T, H, W))
        return y.view(T, H, W, C)[:, r0:r0 + hs].reshape(T * hs * W, C)

    def _res_block(self, p: str, x: Tensor, dims) -> Tensor:
        """ResidualBlock (vae2_2.py:195-239)."""
        ops = self.ops
        c1, c2 = p + ".residual.2", p + ".residual.6"
        y = self._conv(c1, self._act(x, dims, p + ".residual.0", True, key=c1, conv=c1, halo=True), dims, key=c1)
        res = x
        if (p + ".shortcut") in self.lin:
            w, b = self.lin[p + ".shortcut"]
            res = self._new(x.shape[0], w.shape[0])
            ops.gemm(x, w, b, res, ops.YB_EPI_BF16)
        return self._conv(c2, self._act(y, dims, p + ".residual.3", True, key=c2, conv=c2, halo=True), dims, res=res, key=c2)

    def _attention(self, p: str, x: Tensor, dims) -> Tensor:
        """AttentionBlock (vae2_2.py:242-283): per-frame single-head attention over H*W tokens, d = C."""
        ops = self.ops
        T, H, W = dims
        N, C = x.shape
        HW = H * W
        Lf = _rup(HW, 32)                                        # per-frame key count padded for the GEMM tile
        a = self.att
        S, P, o = self._new(HW, Lf, dtype=_F32), self._new(HW, Lf), self._new(N, C)
        if HW % 8:
            # frames whose H*W rows are not 16-byte multiples in the transposed V (tiny latents only): every frame gets its own
            # zero-padded Lf-row slot, so per-frame slices of q, k and v^T start on aligned addresses
            tmp = self._new(T, H, W, C)
            ops.vae_rms_act(x, dims, tmp, self.gamma[p + ".norm"], 1, False)
            hn = torch.zeros(T * Lf + 32, C, device=self.device, dtype=_BF16)
            hn[:T * Lf].view(T, Lf, C)[:, :HW].copy_(tmp.view(T, HW, C))
            q, k, vT = self._new(T * Lf, C), self._new(T * Lf, C), self._new(C, T * Lf + 32)
            ops.gemm(hn[:T * Lf], a["wq"], a["bq"], q, ops.YB_EPI_BF16)
            ops.gemm(hn[:T * Lf], a["wk"], a["bk"], k, ops.YB_EPI_BF16)
            ops.gemm(a["wv"], hn, None, vT, ops.YB_EPI_BF16)
            for f in range(T):
                ops.gemm(q[f * Lf:f * Lf + HW], k[f * Lf:(f + 1) * Lf], None, S, ops.YB_EPI_F32)
                ops.masked_softmax(S, P, HW, HW)
                ops.gemm(P, vT[:, f * Lf:(f + 1) * Lf], None, o[f * HW:(f + 1) * HW], ops.YB_EPI_BF16)
        else:
            Next = _rup(N, 32) + 32
            hn = torch.zeros(Next, C, device=self.device, dtype=_BF16)
            ops.vae_rms_act(x, dims, hn[:N].view(T, H, W, C), self.gamma[p + ".norm"], 1, False)
            q, k = self._new(N, C), torch.zeros(Next, C, device=self.device, dtype=_BF16)
            ops.gemm(hn[:N], a["wq"], a["bq"], q, ops.YB_EPI_BF16)
            ops.gemm(hn[:N], a["wk"], a["bk"], k[:N], ops.YB_EPI_BF16)
            vT = self._new(C, Next)
            ops.gemm(a["wv"], hn, None, vT, ops.YB_EPI_BF16)
            for f in range(T):
                ops.gemm(q[f * HW:(f + 1) * HW], k[f * HW:f * HW + Lf], None, S, ops.YB_EPI_F32)
                ops.masked_softmax(S, P, HW, HW)                 # keys >= HW (padding / next frame) get probability 0
                ops.gemm(P, vT[:, f * HW:f * HW + Lf], None, o[f * HW:(f + 1) * HW], ops.YB_EPI_BF16)
        out = self._new(N, C)
        ops.gemm(o, a["wo"], a["bo"], out, ops.YB_EPI_RES_BF16, res=x)
        return out

    # ---- chunk streaming -----------------------------------------------------------------------------------
    def _run_chunk(self, src: Tensor, out: Tensor) -> None:
        """Run one chunk of the input, `src`, through the layer list into `out`, its frame window of the result."""
        ops = self.ops
        for L in self.layers:
            if L.kind == "in":
                x, dims = self._input(L, src)
            elif L.kind == "res":
                x = self._res_block(L.name, x, dims)
            elif L.kind == "attn":
                x = self._attention(L.name, x, dims) if self._rows is None else self._attention_rows(L.name, x, dims)
            elif L.kind == "hold":
                held, held_dims = x, dims
            elif L.kind in ("up", "down"):
                x, dims = self._resample(L, x, dims)
            elif L.kind == "dupup":                              # DupUp3D drops frames in the first chunk only (:495-503)
                dupup = ops.vae_dupup_add if self._chunk == 0 else ops.vae_dupup_add_cont
                dupup(x, held, held_dims, L.ci, L.co, L.ft, L.fs)
                held = None
            elif L.kind == "avgdown":
                ops.vae_avgdown_add(x, held, held_dims, held.shape[1], x.shape[1], L.ft, L.fs)
                held = None
            else:
                self._head(L, x, dims, out)

    def _chunks(self, src: Tensor, lengths: Sequence[int], out_shape, k_in: int, k_out: int) -> Tensor:
        """Run `src` in chunks of `lengths` latent frames into one preallocated f32 result of `out_shape`. A chunk of n latent
        frames reads n * k_in frames of `src` and writes n * k_out frames of the result, the first chunk k - 1 fewer of each
        (frame 0 stands alone)."""
        units = 1 + (src.shape[1] - 1) // k_in
        if sum(lengths) != units or min(lengths) < 1:
            raise YumeB200Error(f"chunk lengths {list(lengths)} do not partition {units} latent frames")
        out = self._new(*out_shape, dtype=_F32)
        self._stream(src, out, lengths, k_in, k_out)
        return out

    def _stream(self, src: Tensor, out: Tensor, lengths: Sequence[int], k_in: int, k_out: int, u0: int = 0,
                carry: Optional[dict] = None, keep: bool = False, snap: int = -1):
        """Run latent frames u0 .. u0 + sum(lengths) of `src` in chunks of `lengths` into their frame windows of `out`. u0 > 0
        continues a stream whose carries at latent frame u0 are `carry`: every chunk is then a chunk after the first. keep: the
        last chunk carries as if another followed (a resuming engine). Returns the carries at the end (keep) and those after
        latent frame `snap` (when a chunk ends there), each a dict the running stream no longer writes into. A row-parallel call
        then all-gathers the bands of the frames it wrote."""
        t_in, t_out = _frames_of(u0, k_in), _frames_of(u0, k_out)
        t0 = t_out
        self._carry = {} if carry is None else dict(carry)
        at_snap = None
        try:
            for i, n in enumerate(lengths):
                self._chunk, self._more = i + (1 if u0 else 0), keep or i < len(lengths) - 1
                n_in, n_out = (n * k_in, n * k_out) if self._chunk else (1 + (n - 1) * k_in, 1 + (n - 1) * k_out)
                self._run_chunk(src[:, t_in:t_in + n_in], out[:, t_out:t_out + n_out])
                t_in, t_out, u0 = t_in + n_in, t_out + n_out, u0 + n
                if u0 == snap:
                    at_snap = dict(self._carry)                  # _keep replaces carries, never writes into one
            res = (dict(self._carry) if keep else None), at_snap
        finally:
            self._chunk, self._more, self._carry = 0, False, None
        if self._rows is not None and t0 < out.shape[1]:
            self._gather_rows(out, t0)
        return res

    def _gather_rows(self, out: Tensor, t0: int) -> None:
        """All-gather the row bands of frames t0 .. of the result `out` [C, F, S * H, ...], S its rows per latent row (a decoder's
        SCALE, 1 for an encoder's mu): every rank wrote its own band, and ends with every band."""
        r0, hs, H = self._band
        S = out.shape[2] // H
        sizes = [S * h for h in self._rows.sizes(H)]
        row = 0
        for r, b in enumerate(self._rows.gather(out[:, t0:, r0 * S:(r0 + hs) * S], 2, sizes)):
            if r != self._rows.rank:
                out[:, t0:, row:row + sizes[r]].copy_(b)
            row += sizes[r]

    # ---- resuming across calls -----------------------------------------------------------------------------
    def retained_bytes(self) -> int:
        """Device bytes a resuming engine holds between calls: its copy of the last input, the result it returned (a reference:
        shared with the caller while the caller keeps it) and the carried conv frames of every snapshot. 0 when nothing is
        kept (resume=False, before the first call, after reset())."""
        k = self._kept
        if k is None:
            return 0
        seen, total = set(), 0
        tensors = [k.src, k.out] + [t for _, c in k.snaps.values() for v in c.values()
                                    for t in (v if isinstance(v, tuple) else (v,))]
        for t in tensors:
            if t.data_ptr() not in seen:
                seen.add(t.data_ptr())
                total += t.numel() * t.element_size()
        return total

    def reset(self) -> None:
        """Drop the state a resuming engine keeps between calls: the next call runs in full."""
        self._kept = None

    def _resumed(self, src: Tensor, owned: bool, out_shape, k_in: int, k_out: int, nbytes, fork: bool) -> Tensor:
        """A call of a resuming engine on `src` (on the device, f32, contiguous; `owned`: not the caller's tensor). When the kept
        input of the last call and `src` agree bit for bit on the first P frames, P a snapshot of the kept state, only the
        latent frames after P run, as later chunks of the kept stream; the result's first frames are the kept result's.
        Snapshots: the end of the input, and for an encoder (`fork`) also the start of its trailing all-zero frames when that
        is a latent-frame boundary. Anything else runs in full. Either way the state of this call replaces the kept one."""
        kept, self._kept = self._kept, None                      # dropped if this call fails
        units = 1 + (src.shape[1] - 1) // k_in
        comparable = (kept is not None and kept.src.shape[0] == src.shape[0] and kept.src.shape[2:] == src.shape[2:]
                      and (kept.version is None or kept.out._version == kept.version))
        match = torch.empty(2, dtype=torch.int32, device=self.device)
        self.ops.vae_frame_match(kept.src if comparable else None, src, match)
        first, zero = match.tolist()                             # the one synchronisation a resuming call adds
        if self._rows is not None:                               # every rank resumes from the same snapshot and forks alike
            first = self._rows.min_int(first if comparable else 0)
            if fork:
                zero = self._rows.min_int(zero)
        snaps = kept.snaps if comparable else {}
        P = max((p for p in snaps if p <= first), default=0)
        u0, carry = snaps[P] if P else (0, None)
        fu = 1 + (zero - 1) // k_in if fork and zero > 0 and (zero - 1) % k_in == 0 and zero < src.shape[1] else -1
        if u0 < fu:                                              # the stream passes the fork: a chunk ends there
            lengths = self._plan(fu - u0, nbytes) + self._plan(units - fu, nbytes)
        else:
            lengths = self._plan(units - u0, nbytes) if units > u0 else []
        out = self._new(*out_shape, dtype=_F32)
        if u0:
            n = _frames_of(u0, k_out)
            out[:, :n].copy_(kept.out[:, :n])
        kept = None
        end, at_fork = self._stream(src, out, lengths, k_in, k_out, u0, carry, keep=True, snap=fu)
        new_snaps = {src.shape[1]: (units, end)}
        if at_fork is not None:
            new_snaps[zero] = (fu, at_fork)
        elif fu > 0 and zero in snaps and zero <= first:         # the fork lies in the resumed prefix: still valid
            new_snaps[zero] = snaps[zero]
        version = None if out.is_inference() else out._version
        self._kept = _Kept(src if owned else src.clone(), out if version is not None else out.clone(), version, new_snaps)
        return out

    # ---- chunk planner -------------------------------------------------------------------------------------
    def chunk_bytes(self, n: int, T: int, H: int, W: int) -> int:
        """`_chunk_bytes`, or under a row-parallel decode the bound of one rank (`_band_bytes`)."""
        return self._chunk_bytes(n, T, H, W) if self._rows is None else self._band_bytes(n, T, H, W)

    def _band_bytes(self, n: int, T: int, H: int, W: int) -> int:
        """Upper bound of one rank's device bytes in a row-parallel decode: the largest band, its halo rows counted at every level
        as two more latent rows, plus the gathered attention input (padded bands, full frames, the attention's own buffers and
        the rows kept), and the whole video with the padded bands of its all-gather."""
        P = self._rows.world
        hb = -(-H // P)
        attn = next(L for L in self.layers if L.kind == "attn")
        s = next(L for L in self.layers if L.kind == "in").ft
        F, c = n * s, attn.ci
        gathered = ((P + 2) * F * hb * W + F * H * W) * c * 2 + _attn_bytes(F, H * W, c)
        return self._chunk_bytes(n, T, hb + 2, W) + gathered + (1 + P) * self._fixed_bytes(T, H, W)

    def _chunk_bytes(self, n: int, T: int, H: int, W: int) -> int:
        """Upper bound of the device bytes a decode (encode) of T latent (video) frames at H x W allocates on top of the weights
        and its input when its chunks hold n latent frames: the whole result, every carried history, and the largest set of
        activations one step of the layer list keeps live (every buffer of that step counted as live at once; a chunk after
        the first is counted, it has the most frames at each level). The shortcut steps add no bytes of their own: `up` and
        `down` count the held level input."""
        bf, f4 = 2, 4
        hist = self.HIST
        carries, peak, held = 0, 0, 0
        for L in self.layers:
            if L.kind == "in":                                   # frames per latent frame, input size
                s, h, w = L.ft, H // L.fs, W // L.fs
            F, vox = n * s, h * w
            c, co = L.ci, L.co
            cp = _rup(c, 64)
            live = 0
            if L.kind == "in":                                   # input gather, conv1's input buffer (history in front), its out
                carries += hist * vox * c * bf
                live = (F * vox * c + (F + hist) * vox * c + F * vox * co) * bf
            elif L.kind == "hold":
                held = c
            elif L.kind == "down":                               # x, held block input, act, resample.1 out (+1 carried frame),
                vq = (h // 2) * (w // 2)                         # its act, time_conv out
                live = (F * vox * (c + held + cp) + (F + 1) * vq * (c + cp) + F * vq * c) * bf
                if L.ft == 2:
                    carries += vq * cp * bf
                s, h, w = s // L.ft, h // L.fs, w // L.fs
            elif L.kind == "res":                                # x, the block input a shortcut add holds, y, res, out, two acts
                carries += hist * vox * (cp + _rup(co, 64)) * bf
                live = F * vox * (2 * c + 3 * co) * bf + (F + hist) * vox * (cp + _rup(co, 64)) * bf
            elif L.kind == "attn":
                live = _attn_bytes(F, vox, c)
            elif L.kind == "up":
                t_up = L.ft == 2
                F2 = 2 * F if t_up else F
                live = (F * vox * (c + held) + F2 * vox * c) * bf + (F + hist) * vox * cp * bf * (1 if t_up else 0)
                live += F2 * 4 * vox * (cp + _rup(co, 32)) * bf
                if t_up:
                    carries += hist * vox * cp * bf
                s, h, w = s * L.ft, h * L.fs, w * L.fs
            elif L.kind in ("dupup", "avgdown"):
                held = 0
            elif L.kind == "head":                               # act, f32 conv output
                live = (F * vox * c + (F + hist) * vox * cp) * bf + F * vox * co * f4
                carries += hist * vox * cp * bf
            peak = max(peak, live)
        return self._fixed_bytes(T, H, W) + carries + peak

    def _plan(self, units: int, nbytes) -> List[int]:
        """Latent frames per chunk: all `units` when they fit (and always off CUDA), else the longest chunks whose `nbytes`
        fit the device's free memory (free + torch's cached, unallocated blocks) minus MEM_MARGIN. The free memory is read
        when the call starts, so other work on the same GPU can make a sequence that would fit alone run in chunks (with the
        same result). A row-parallel decode plans with the smallest budget of its ranks, so that all run the same chunks."""
        free = self._free_bytes()
        budget = _UNBOUNDED if free is None else free - self.MEM_MARGIN
        if self._rows is not None:
            budget = self._rows.min_int(budget)
        return [units] if budget == _UNBOUNDED else chunk_lengths(units, nbytes, budget)

    def _free_bytes(self) -> Optional[int]:
        """Free device memory the planner may use (free + torch's cached, unallocated blocks); None off CUDA."""
        if self.device.type != "cuda":
            return None
        free, _ = torch.cuda.mem_get_info(self.device)
        return free + torch.cuda.memory_reserved(self.device) - torch.cuda.memory_allocated(self.device)


_UNBOUNDED = 1 << 62                # the planner's budget off CUDA: everything in one chunk


def _attn_bytes(F: int, vox: int, c: int) -> int:
    """Bytes the mid attention (`_attention`) allocates for F frames of vox tokens and c channels."""
    Lf, Next = _rup(vox, 32), _rup(F * vox, 32) + 32
    return (F * vox * c * 5 + Next * c * 3 + F * Lf * c * 3) * 2 + vox * Lf * (4 + 2)


def chunk_lengths(T: int, nbytes, budget: int) -> List[int]:
    """Partition T latent frames into chunks of the longest length n whose `nbytes(n)` (non-decreasing in n) fits `budget`, the
    last chunk taking the remainder: [T] when the whole sequence fits, chunks of 1 frame when nothing longer does."""
    if nbytes(T) <= budget:
        return [T]
    n = 1
    while n + 1 < T and nbytes(n + 1) <= budget:
        n += 1
    return [n] * (T // n) + ([T % n] if T % n else [])
