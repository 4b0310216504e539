"""TEST INFRASTRUCTURE: the four Wan VAE engines checked launch by launch.

A SPEC states the launches of one chunk of Wan22VaeDecoder (bf16 and precision="fp8"), Wan21VaeDecoder, Wan22VaeEncoder and
Wan21VaeEncoder independently of yume_b200/wan_vae.py and its engines: from the whole-sequence oracles (oracle/wan22vae.py,
wan21vae.py, wan22vae_enc.py, wan21vae_enc.py, wan22vae_fp8.py) and the reference module tree their state-dict keys name. Given
the chunk index, whether more chunks follow, its latent frames and H x W, it lists the chunk's stages in launch order, each with
its ops entry and the source of every operand:
  * an earlier stage's output, or a named row / column / frame range of it (the decoder's time_conv stream without frame 0,
    the encoder's frame 0 that bypasses time_conv, the per-frame key / value slices of the mid attention);
  * a weight the spec packs from the state-dict keys itself ([cop, taps*cp] convs, conv2 with std / mean folded in, the conv1 mu
    half, q scaled, the v bias folded through proj, e4m3 weights by oracle.fp8.quantize_weight), a gamma by its key;
  * for the history rows of a conv's input buffer, the last n frames of the same stream in the previous chunks (zero frames
    where the stream is shorter): 2 for a 3-tap conv, 1 for the stride-2 time_conv, e4m3 value / scale pairs on the fp8 path.
    The checker keeps these carries itself, from the operands it has verified, and on a resumed call starts from the carries
    it recorded at the latent frame the call resumes from;
  * the input's frame window, and for a writer the result's frame window.

A CHECKER (dit_dataflow.Checker, whose Src / Stage / operand comparison it reuses) stands in front of the `ops` of vae22, vae21
and vae_enc. Every chunk of `_run_chunk` is one region; inside it each launch must be the spec's next stage, each operand
torch.equal to its source (view shape, frame count, t_hist, scale frames), and each output within the kernel's contract bound
(the conv references of test_gpu_kernel_contract_ext, conv_fp8_reference / conv_fp8_bound, rms_act_bound, softmax_bound,
avgdown_ref, the gemm bounds); quantisers and layout kernels bit for bit; a windowed writer leaves every frame of the result
outside its window untouched. An entry the spec does not know fails; helpers and constants (conv_out_dims, YB_*) pass.
Large launches are sampled (output voxels for the convs, rows for the GEMMs and the softmax); stage snapshots are dropped
after their last reader."""
from __future__ import annotations

import contextlib
import inspect
import math
from dataclasses import dataclass
from typing import Dict, List

import torch
import test_gpu_kernel_contract as KC
import test_gpu_kernel_contract_ext as KE
import test_gpu_kernel_contract_fp8_vae as KV
import test_gpu_kernel_contract_prod as KP
from helpers import dit_dataflow as DF
from helpers.dit_dataflow import NONE, Src, Stage, V
from oracle.fp8 import quantize_act, quantize_weight
from oracle.wan21vae import Wan21VaeOracle
from oracle.wan21vae_enc import Wan21VaeEncodeOracle
from oracle.wan22vae import Wan22VaeOracle
from oracle.wan22vae_enc import Wan22VaeEncodeOracle, patchify2
from oracle.wan22vae_fp8 import converted
from yume_b200 import ops as _real_ops

ENTRIES = ("gemm", "conv3d_causal", "conv3d_causal_hist", "conv3d_fp8", "vae_rms_act", "vae_rms_act_fp8", "masked_softmax",
           "vae_dupup_add", "vae_dupup_add_cont", "vae_avgdown_add", "nchw_to_nhwc_bf16", "nchw_to_nhwc_bf16_win",
           "nhwc_to_nchw_f32", "nhwc_to_nchw_f32_win", "vae_patchify2_bf16", "vae_patchify2_bf16_win", "vae_unpatchify2_clamp",
           "vae_unpatchify2_clamp_win")
OUTSIDE = ("vae_frame_match",)      # launched by a resuming call before its chunks; its contract is test_gpu_vae_resume's
SIGS = {e: inspect.signature(getattr(_real_ops, e)) for e in ENTRIES}
EPI = dict(BF16=0, F32=2, RES_BF16=5)    # include/yume_b200.h
HIST = 2                            # carried frames of a 3-tap causal conv
FULL = 4096                         # launches with at most this many output voxels / rows are checked everywhere
U32 = KC.U32
_BF, _F32, _E4M3 = torch.bfloat16, torch.float32, torch.float8_e4m3fn


def _rup(v, m):
    return (v + m - 1) // m * m


def frames_of(units, k):
    """Frames of a stream that hold its first `units` latent frames, k per latent frame after frame 0."""
    return 1 + (units - 1) * k if units else 0


# ------------------------------------------------------------------------------------------------------------
# sources
# ------------------------------------------------------------------------------------------------------------
def R(stage, part="", rows=None, cols=None, fn=None, label=None):
    """Stage output `part`, rows [r0, r1) and columns [c0, c1) of it, then fn."""
    rs = slice(*rows) if rows is not None else slice(None)
    cs = slice(*cols) if cols is not None else slice(None)
    lab = label or (f"{stage}{'.' + part if part else ''}" + (f"[{rows[0]}:{rows[1]}]" if rows else "") +
                    (f"[:, {cols[0]}:{cols[1]}]" if cols else ""))
    f = fn or (lambda t: t)
    return Src(lab, lambda ck: f(ck.snap[stage][part][rs, cs]), "tensor", (stage,))


def MAP(src, fn, label):
    return Src(label, lambda ck: fn(src.get(ck)), src.kind, src.reads)


def JOIN(srcs, fn, label):
    return Src(label, lambda ck: fn([s.get(ck) for s in srcs]), "tensor", sum((s.reads for s in srcs), ()))


def W(label, value):
    s = Src(label, lambda ck: value)
    s.value = value
    return s


def HISTCAT(stream, n, new, shape, dtype, part=None):
    """The input buffer of a conv after the first chunk: the carried last n frames of `stream`, then the new frames."""
    def get(ck):
        return torch.cat([ck.hist(stream, n, shape, dtype, part), new.get(ck)], 0)
    what = {None: "", 0: " values", 1: " scales"}[part]
    return Src(f"hist({stream}{what}, {n}) + {new.label}", get, "tensor", new.reads)


def WIN(label, fn):
    """The result tensor of the running call (or a frame window of it): the operand must be that very view."""
    return Src(label, lambda ck: fn(ck.env["out"]), "window")


def SHAPE(shape):
    """An output buffer: only its view shape is the spec's."""
    return Src(f"a buffer of shape {tuple(shape)}", lambda ck: tuple(shape), "shape")


def SRC_FRAMES(label, fn):
    return Src(label, lambda ck: fn(ck.env["src"]))


# ------------------------------------------------------------------------------------------------------------
# the checker
# ------------------------------------------------------------------------------------------------------------
class _Proxy:
    """Stands for `ops` in vae22 / vae21 / vae_enc: the known entries go through the checker, constants and helpers pass, any
    other launching entry fails."""

    def __init__(self, ck):
        self._ck = ck
        for e in ENTRIES + OUTSIDE:
            if hasattr(ck.base, e):
                setattr(self, e, self._wrap(e))

    def _wrap(self, entry):
        def call(*a, **k):
            return self._ck.launch(entry, a, k)
        return call

    def __getattr__(self, name):
        v = getattr(self._ck.base, name)
        if callable(v) and not name.startswith("YB_") and name != "conv_out_dims":
            def unknown(*a, **k):
                raise AssertionError(f"{self._ck.tag}: the engine launched ops.{name}, an entry the spec does not know")
            return unknown
        return v


@dataclass
class Chunk:
    index: int              # 0: the first chunk of a stream (no history); > 0: a chunk after the first
    more: bool              # another chunk follows (or a resuming call carries as if one did)
    n: int                  # latent frames
    t_in: int               # first input frame
    n_in: int
    t_out: int              # first result frame
    n_out: int
    u_end: int              # latent frames done after this chunk


class Checker(DF.Checker):
    def __init__(self, base, spec, tag, keep_snaps=False):
        super().__init__(base, tag)
        self.spec, self.proxy = spec, _Proxy(self)
        self.carry: Dict[str, object] = {}       # stream -> carried frames (tensor, or (e4m3, scales)) the running chunk reads
        self.next_carry: Dict[str, object] = {}
        self.snaps: Dict[int, dict] = {}         # latent frames -> the carries after them (resume sessions)
        self.keep_snaps = keep_snaps
        self.queue: List[Chunk] = []
        self.chunks_run = 0

    # ---- what the test expects the engine to run ---------------------------------------------------------------
    def expect(self, lengths, u0=0, resume=False):
        """The chunks of the next call: latent lengths `lengths` from latent frame u0 (u0 > 0: resumed from the carries
        recorded there); `resume`: every chunk carries as if another followed."""
        k_in, k_out = self.spec.k_in, self.spec.k_out
        t_in, t_out, u = frames_of(u0, k_in), frames_of(u0, k_out), u0
        for i, n in enumerate(lengths):
            idx = i + (1 if u0 else 0)
            n_in, n_out = (n * k_in, n * k_out) if idx else (frames_of(n, k_in), frames_of(n, k_out))
            self.queue.append(Chunk(idx, resume or i < len(lengths) - 1, n, t_in, n_in, t_out, n_out, u + n))
            t_in, t_out, u = t_in + n_in, t_out + n_out, u + n
        self._start_u = u0

    def begin_stream(self, src, out):
        self.env["src"], self.env["out"] = src, out
        u0 = getattr(self, "_start_u", 0)
        self.carry = dict(self.snaps[u0]) if u0 else {}

    # ---- carries ---------------------------------------------------------------------------------------------------
    def hist(self, stream, n, shape, dtype, part=None):
        c = self.carry.get(stream)
        if c is None:
            return torch.zeros(n, *shape, dtype=dtype, device=self.spec.dev)
        c = c if part is None else c[part]
        if c.shape[0] != n:
            raise AssertionError(f"{self.tag}: spec carry of {stream} holds {c.shape[0]} frames, a reader wants {n}")
        return c

    def keep(self, stream, n, frames):
        def last(f):
            if f.shape[0] >= n:
                return f[f.shape[0] - n:].clone()
            z = torch.zeros(n, *f.shape[1:], dtype=f.dtype, device=f.device)
            z[n - f.shape[0]:] = f
            return z
        self.next_carry[stream] = tuple(last(f) for f in frames) if isinstance(frames, tuple) else last(frames)

    # ---- one chunk -------------------------------------------------------------------------------------------------
    @contextlib.contextmanager
    def chunk(self):
        if not self.queue:
            raise AssertionError(f"{self.tag}: the engine ran a chunk the spec does not expect")
        c = self.queue.pop(0)
        self.cur = c
        self.program, self.phases, self.snap = [], {}, {}
        self.add_phase("chunk", self.spec.chunk(c))
        self.next_carry = {}
        tag = self.tag
        self.tag = f"{tag} chunk {self.chunks_run} (latent frames {c.u_end - c.n}..{c.u_end - 1})"
        try:
            with self.region("chunk"):
                yield
        finally:
            self.tag = tag
        self.carry = {**self.carry, **self.next_carry}
        if self.keep_snaps:
            self.snaps[c.u_end] = dict(self.carry)
        self.snap = {}
        self.chunks_run += 1

    def launch(self, entry, a, k):
        fn = getattr(self.base, entry)
        if entry in OUTSIDE:
            if self.phase is not None:
                raise AssertionError(f"{self.tag}: {entry} launched inside a chunk")
            return fn(*a, **k)
        if self.phase is None:
            raise AssertionError(f"{self.tag}: {entry} launched outside a chunk")
        if self.pos >= self.stop:
            raise AssertionError(f"{self.tag}: launch {self.pos + 1} ({entry}) is beyond the spec's {self.stop} stages")
        st = self.program[self.pos]
        if entry != st.entry:
            raise AssertionError(f"{self.tag}: stage '{st.name}' operand 'entry': the engine launched {entry}, the spec's "
                                 f"entry is {st.entry}")
        b = SIGS[entry].bind(*a, **k)
        b.apply_defaults()
        args = b.arguments
        inp = {}
        for p, src in st.inputs.items():
            try:
                inp[p] = src.get(self)
            except (RuntimeError, IndexError) as e:
                raise AssertionError(f"{self.tag}: stage '{st.name}' operand '{p}': {src.label} cannot be formed from the "
                                     f"outputs the engine made: {e}") from e
            if src.kind == "shape":
                if not isinstance(args[p], torch.Tensor) or tuple(args[p].shape) != inp[p]:
                    raise AssertionError(f"{self.tag}: stage '{st.name}' operand '{p}' is not {src.label}: shape "
                                         f"{tuple(getattr(args[p], 'shape', ()))}")
            elif src.kind == "window":
                _same_view(self.tag, st.name, p, args[p], inp[p], src)
            else:
                DF._same(self.tag, st.name, p, args[p], inp[p], src)
        pre = self.env["out"].clone() if getattr(st, "window", None) else None
        out = fn(*a, **k)
        if self.base is _real_ops:
            torch.cuda.synchronize()
        for stream, n, f in getattr(st, "keeps", ()):
            self.keep(stream, n, f(args, inp))
        if self.last_read.get(st.name, -1) > self.pos:
            self.snap[st.name] = {part: f(args).clone() for part, f in st.outputs.items()}
        if st.check is not None:
            self.worst[entry] = max(self.worst.get(entry, 0.0), st.check(self, st, args, inp))
        if pre is not None:
            _outside_window(self, st, pre)
        del inp, pre
        for name in [n for n in self.snap if self.last_read.get(n, -1) <= self.pos]:
            del self.snap[name]
        self.pos += 1
        return out


def _same_view(tag, stage, param, got, want, src):
    if not isinstance(got, torch.Tensor) or got.data_ptr() != want.data_ptr() or got.shape != want.shape or \
            got.stride() != want.stride():
        what = "not a tensor" if not isinstance(got, torch.Tensor) else \
            f"view at element offset {(got.data_ptr() - want.data_ptr()) // max(1, got.element_size())}, shape " \
            f"{tuple(got.shape)} stride {got.stride()}; the spec's is shape {tuple(want.shape)} stride {want.stride()}"
        raise AssertionError(f"{tag}: stage '{stage}' operand '{param}' is not {src.label}: {what}")


def _outside_window(ck, st, pre):
    """Every frame of the result outside the chunk's window keeps its bits."""
    c, out = ck.cur, ck.env["out"]
    iv = {4: torch.int32, 2: torch.int16}[out.element_size()]
    a, b = out.view(iv), pre.view(iv)
    for sl in (slice(0, c.t_out), slice(c.t_out + c.n_out, None)):
        d = a[:, sl] != b[:, sl]
        if bool(d.any()):
            raise AssertionError(f"{ck.tag}: stage '{st.name}' operand 'out': {int(d.sum())} elements of the result outside "
                                 f"frames [{c.t_out}, {c.t_out + c.n_out}) changed")


def _stage(name, entry, inputs, outputs, check, keeps=(), window=False):
    st = Stage(name, entry, inputs, outputs, check)
    st.keeps, st.window = keeps, window
    return st


# ------------------------------------------------------------------------------------------------------------
# output checks
# ------------------------------------------------------------------------------------------------------------
def _gen(*key):
    return KP._cpu_gen("vae_dataflow", *key)


def _sample(n, key):
    if n <= FULL:
        return torch.arange(n)
    g = _gen(n, key)
    return torch.unique(torch.cat([torch.randint(0, n, (FULL,), generator=g), torch.tensor([0, n - 1])]))


def check_gemm(ck, st, a, inp):
    """gemm_epilogue_ref over gemm_ref_rows_cols: every row of a small launch, else 2 full rows per 128-row band and 2 full
    columns per 64-column band (gemm_sample)."""
    A, B, bias, epi, res = inp["a"], inp["w"], inp["bias"], inp["epilogue"], inp["res"]
    M, N = A.shape[0], B.shape[0]
    key = (ck.tag, st.name)
    rows, cols = DF._rows(M, key).to(A.device), DF._cols(N, key).to(A.device)
    (accR, FR), (accC, FC) = KP.gemm_ref_rows_cols(A, B, rows, cols)
    out = a["out"]
    worst = 0.0
    allr = torch.arange(M, device=A.device)
    for rr, cc, acc, Fb in ((rows, None, accR, FR), (allr, cols, accC, FC)):
        if acc.numel() == 0:
            continue
        pick = (lambda t: t[rr]) if cc is None else (lambda t: t[:, cc])
        b = None if bias is None else (bias.double() if cc is None else bias.double()[cc])[None].expand_as(acc)
        r = None if res is None else pick(res).double()
        ref, bound = KP.gemm_epilogue_ref(epi, acc, Fb, bias=b, res=r)
        worst = max(worst, DF._ratio(pick(out), ref, bound, f"{ck.tag}: stage '{st.name}' output"))
    return worst


def _conv_geom(buf_frames, T, H, W, taps, stride_t, stride_hw):
    kt, kh, kw = taps
    To = T if stride_t == 1 else (buf_frames - kt) // stride_t + 1
    Ho, Wo = (H, W) if stride_hw == 1 else ((H + 1 - kh) // stride_hw + 1, (W + 1 - kw) // stride_hw + 1)
    return To, Ho, Wo


def conv_ref_at(buf, w, vox, dims_out, T, H, W, taps, stride_t, stride_hw):
    """fp64 (acc, F = 2*K*u32*conv(|x|, |w|)) of the zero-padded causal conv at output voxels `vox` (linear in dims_out): the
    buffer's h = frames - T leading frames replace the causal zero padding (unit stride in time), the stride-2 time_conv reads
    its buffer unpadded, the stride-2 Conv2d pads one zero row / column behind (the references of
    test_gpu_kernel_contract_ext._conv_ref, gathered per voxel)."""
    kt, kh, kw = taps
    nb, _, _, Cp = buf.shape
    To, Ho, Wo = dims_out
    t, rem = vox // (Ho * Wo), vox % (Ho * Wo)
    ho, wo = rem // Wo, rem % Wo
    dt, dh, dw = torch.meshgrid(torch.arange(kt), torch.arange(kh), torch.arange(kw), indexing="ij")
    dt, dh, dw = dt.flatten()[None], dh.flatten()[None], dw.flatten()[None]
    pt = 0 if stride_t > 1 else (kt - 1) - (nb - T)
    ph, pw = (kh // 2, kw // 2) if stride_hw == 1 else (0, 0)
    ti = t[:, None] * stride_t + dt - pt
    hi = ho[:, None] * stride_hw + dh - ph
    wi = wo[:, None] * stride_hw + dw - pw
    ok = (ti >= 0) & (ti < nb) & (hi >= 0) & (hi < H) & (wi >= 0) & (wi < W)
    idx = torch.where(ok, (ti * H + hi) * W + wi, torch.zeros_like(ti)).to(buf.device)
    xv = buf.reshape(-1, Cp)[idx].double() * ok.to(buf.device)[..., None]
    xv = xv.reshape(len(vox), -1)
    wd = w.double()
    K = wd.shape[1]
    return xv @ wd.t(), 2.0 * K * U32 * (xv.abs() @ wd.abs().t())


def check_conv(ck, st, a, inp):
    buf = inp["xbuf"] if "xbuf" in inp else inp["xpad"]
    w, bias, epi, res, taps = inp["w"], inp["bias"], inp["epilogue"], inp["res"], inp["taps"]
    T, H, W = inp["T"], inp["H"], inp["W"]
    st_t, st_hw = inp["stride_t"], inp["stride_hw"]
    dims = _conv_geom(buf.shape[0], T, H, W, taps, st_t, st_hw)
    To, Ho, Wo = dims
    out = a["out"]
    frames = out.reshape(-1, Ho * Wo, out.shape[-1])
    cop = w.shape[0]
    vox = _sample(To * Ho * Wo, (ck.tag, st.name))
    worst = 0.0
    for i in range(0, len(vox), 512):
        v = vox[i:i + 512]
        acc, Fb = conv_ref_at(buf, w, v, dims, T, H, W, taps, st_t, st_hw)
        vd = v.to(buf.device)
        r = None if res is None else res.reshape(-1, res.shape[-1])[vd, :cop].double()
        ref, bound = KP.gemm_epilogue_ref(epi, acc, Fb, bias=bias.double()[None].expand_as(acc), res=r)
        t, p = vd // (Ho * Wo), vd % (Ho * Wo)
        got = frames[t * inp["out_t_mul"] + inp["out_t_add"], p, :cop]
        worst = max(worst, DF._ratio(got, ref, bound, f"{ck.tag}: stage '{st.name}' output"))
    return worst


def check_conv8(ck, st, a, inp):
    q, s, w8, sw, bias, res, taps = inp["x"], inp["x_scale"], inp["w"], inp["w_scale"], inp["bias"], inp["res"], inp["taps"]
    T, H, W, th = inp["T"], inp["H"], inp["W"], inp["t_hist"]
    Cp = q.shape[-1]
    cop = w8.shape[0]
    wd = (w8.double() * sw.double()[:, None]).view(cop, -1, Cp)
    vox = _sample(T * H * W, (ck.tag, st.name))
    worst = 0.0
    for i in range(0, len(vox), 1024):
        v = vox[i:i + 1024]
        t, rem = v // (H * W), v % (H * W)
        ref, sabs = KV.conv_fp8_reference(q, s, wd, bias, res, t, rem // W, rem % W, T, th, taps)
        bound = KV.conv_fp8_bound(sabs, math.prod(taps) * Cp // 128, 2.0 ** -8, ref)
        worst = max(worst, DF._ratio(a["out"][v.to(q.device), :cop], ref, bound, f"{ck.tag}: stage '{st.name}' output"))
    return worst


def _rms_check(ck, st, x, dims, out, gamma, up, silu, what):
    """out [T, Hs*up, Ws*up, Cp] against rms_act_bound of x [N, C] (+ bf16 rounding) at sampled source voxels, pad columns
    exactly 0; gamma None without SiLU is a copy and must be bit-exact."""
    T, Hs, Ws = dims
    N, C = x.shape
    Cp = out.shape[-1]
    o = out.reshape(T, Hs, up, Ws, up, Cp).permute(0, 1, 3, 2, 4, 5).reshape(N, up * up, Cp)
    vox = _sample(N, (ck.tag, st.name)).to(x.device)
    got = o[vox]
    if bool((got[..., C:] != 0).any()):
        raise AssertionError(f"{ck.tag}: stage '{st.name}' {what}: channel padding not zero")
    if gamma is None and not silu:
        if not torch.equal(got[..., :C], x[vox][:, None].expand(-1, up * up, -1)):
            raise AssertionError(f"{ck.tag}: stage '{st.name}' {what}: the copy is not bit-exact")
        return 0.0
    nch, G = KE.rms_instance(C, Cp)
    y, f32 = KE.rms_act_bound(x[vox].double(), gamma, C, nch, G, silu)
    y, f32 = y[:, None].expand(-1, up * up, -1), f32[:, None].expand(-1, up * up, -1)
    return DF._ratio(got[..., :C], y, KC.bf16_out_bound(y, f32), f"{ck.tag}: stage '{st.name}' {what}")


def check_rms(ck, st, a, inp):
    return _rms_check(ck, st, inp["x"], inp["dims"], a["out"], inp["gamma"], inp["up"], inp["silu"], "output")


def quantize_frames(v):
    """bf16 [T, H, W, Cp] -> (e4m3 [T, H, W, Cp], f32 scales [T, Cp/128, H, W]), quantize_act per voxel and 128-channel group."""
    T, H, W, Cp = v.shape
    q, s = quantize_act(v.float().reshape(-1, Cp))
    return q.view(T, H, W, Cp), s.view(Cp // 128, T, H, W).transpose(0, 1).contiguous()


def check_rms8(ck, st, a, inp):
    """The bf16 values vae_rms_act writes for the same arguments within the vae_rms_act bound, and the e4m3 pair
    bit-identical to quantize_act of them (the contract of yb_vae_rms_act_fp8)."""
    out = a["out"]
    tmp = torch.empty(out.shape, dtype=_BF, device=out.device)
    ck.base.vae_rms_act(inp["x"], inp["dims"], tmp, inp["gamma"], inp["up"], inp["silu"])
    if ck.base is _real_ops:
        torch.cuda.synchronize()
    worst = _rms_check(ck, st, inp["x"], inp["dims"], tmp, inp["gamma"], inp["up"], inp["silu"], "bf16 values")
    q, s = quantize_frames(tmp)
    del tmp
    if not (torch.equal(out.view(torch.uint8), q.view(torch.uint8)) and torch.equal(a["out_scale"], s)):
        raise AssertionError(f"{ck.tag}: stage '{st.name}' output: {int((out.view(torch.uint8) != q.view(torch.uint8)).sum())} "
                             f"e4m3 bytes / {int((a['out_scale'] != s).sum())} scales differ from the twin")
    return worst


def check_softmax(ck, st, a, inp):
    S, L, hw = inp["S"], inp["L"], inp["hw"]
    rows = DF._rows(S.shape[0], (ck.tag, st.name)).to(S.device)
    p, f32, keep = KE.softmax_bound(S[rows], L, hw)
    P = a["P"][rows]
    if not bool((P[~keep] == 0).all()):
        raise AssertionError(f"{ck.tag}: stage '{st.name}' output: a masked entry is not exactly 0")
    return DF._ratio(P, p, KC.bf16_out_bound(p, f32), f"{ck.tag}: stage '{st.name}' output")


def _dupup(x, dims, in_c, out_c, ft, fs, drop):
    """DupUp3D (oracle/wan22vae.py Wan22VaeOracle.dup_up) of x [T*H*W, in_c] as [To, H*fs, W*fs, out_c]; drop: the first
    chunk's ft - 1 leading frames are dropped, a later chunk keeps every frame."""
    T, H, W = dims
    xn = x.float().view(T, H, W, in_c).permute(3, 0, 1, 2)[None]
    rep = out_c * ft * fs * fs // in_c
    y = xn.repeat_interleave(rep, dim=1).view(1, out_c, ft, fs, fs, T, H, W)
    y = y.permute(0, 1, 5, 2, 6, 3, 7, 4).reshape(out_c, T * ft, H * fs, W * fs)
    return (y[:, ft - 1:] if drop else y).permute(1, 2, 3, 0)


def check_dupup(drop):
    def check(ck, st, a, inp):
        main = inp["main"]
        up = _dupup(inp["x"], inp["dims"], inp["in_c"], inp["out_c"], inp["ft"], inp["fs"], drop)
        want = (main.float().view(up.shape) + up).reshape(main.shape).to(_BF)
        d = a["main"] != want
        if bool(d.any()):
            raise AssertionError(f"{ck.tag}: stage '{st.name}' output: {int(d.sum())} of {d.numel()} elements differ from "
                                 f"main + DupUp3D(x)")
        return 0.0
    return check


def check_avgdown(ck, st, a, inp):
    in_c, out_c, ft, fs = inp["in_c"], inp["out_c"], inp["ft"], inp["fs"]
    G = in_c * ft * fs * fs // out_c
    mean, absmean = KE.avgdown_ref(inp["x"], inp["dims"], in_c, out_c, ft, fs)
    ref = inp["main"].double().view(mean.shape) + mean
    bound = KC.bf16_out_bound(ref, (G - 1) * U32 * absmean + U32 * ref.abs())
    return DF._ratio(a["main"].view(mean.shape), ref, bound, f"{ck.tag}: stage '{st.name}' output")


def _exact(ck, st, got, want):
    if got.shape != want.shape or not torch.equal(got, want.to(got.device)):
        n = int((got != want.to(got.device)).sum()) if got.shape == want.shape else -1
        raise AssertionError(f"{ck.tag}: stage '{st.name}' output: {n} elements differ from the layout twin")
    return 0.0


def check_nchw_to_nhwc(ck, st, a, inp):
    x, out = inp["x"], a["out"]
    want = torch.zeros(out.shape, dtype=_BF, device=out.device)
    want[:, :x.shape[0]] = x.reshape(x.shape[0], -1).t().to(_BF)
    return _exact(ck, st, out, want)


def check_patchify(ck, st, a, inp):
    v, out = inp["video"], a["out"]
    p = patchify2(v[None])[0]
    want = torch.zeros(out.shape, dtype=_BF, device=out.device)
    want[:, :12] = p.permute(1, 2, 3, 0).reshape(-1, 12).to(_BF)
    return _exact(ck, st, out, want)


def check_unpatchify(ck, st, a, inp):
    y, T, H, W = inp["y"], inp["T"], inp["H"], inp["W"]
    v = y[:, :12].reshape(T, H, W, 12).permute(3, 0, 1, 2)[None]                 # oracle/wan22vae.py decode: unpatchify
    want = v.reshape(1, 3, 2, 2, T, H, W).permute(0, 1, 4, 5, 3, 6, 2).reshape(3, T, 2 * H, 2 * W).clamp(-1, 1)
    return _exact(ck, st, a["out"], want)


def check_nhwc_to_nchw(ck, st, a, inp):
    x, out, clamp = inp["x"], a["out"], inp["clamp"]
    Cn = out.shape[0]
    want = x[:, :Cn].t().reshape(out.shape)
    if clamp is not None:
        want = want.clamp(*clamp)
    return _exact(ck, st, out, want)


# ------------------------------------------------------------------------------------------------------------
# the spec
# ------------------------------------------------------------------------------------------------------------
_GEMM_REST = dict(gate=NONE, tok_idx=NONE, block_n=V(0), n_split=V(0), split_stride=V(0), a_split=V(0), a_split_stride=V(0),
                  shape=NONE, cta_pair=V(0), split_k=NONE)


class Spec:
    """The launches of one chunk of a Wan VAE engine, written from its oracle. kind: wan22_dec | wan21_dec | wan22_enc |
    wan21_enc; precision "fp8" (wan22_dec only) runs the convs oracle.wan22vae_fp8.converted selects on e4m3 operands."""

    def __init__(self, kind, sd, cfg, mean, std, dev, precision="bf16"):
        self.kind, self.dev, self.fp8 = kind, torch.device(dev), precision == "fp8"
        self.dec = kind.endswith("dec")
        oracle = {"wan22_dec": Wan22VaeOracle, "wan21_dec": Wan21VaeOracle, "wan22_enc": Wan22VaeEncodeOracle,
                  "wan21_enc": Wan21VaeEncodeOracle}[kind]
        self.orc = oracle(sd, mean=mean, std=std, **cfg)
        self.sd = {k: v.detach().to(self.dev, _F32) for k, v in sd.items()}
        self.zd = self.orc.z_dim
        self.mean = (torch.zeros(self.zd) if mean is None else mean).detach().to(self.dev, _F32)
        self.std = (torch.ones(self.zd) if std is None else std).detach().to(self.dev, _F32)
        self.k_in, self.k_out = (1, 4) if self.dec else (4, 1)
        self.fs_in = 2 if kind == "wan22_enc" else 1
        self._w = {}

    # ---- weights, packed from the state-dict keys ------------------------------------------------------------------
    def conv_w(self, name):
        """name -> (w, bias, taps, fp8): w bf16 [rup(co, 32), taps * rup(ci, 64)] (taps-major, channels minor; a Conv2d is
        taps (1, kh, kw)), or the (e4m3, s_w) pair of it; the decoder's time_conv.g is output group g of time_conv."""
        if name not in self._w:
            base, g = name, None
            if name.endswith((".time_conv.0", ".time_conv.1")):
                base, g = name[:-2], int(name[-1])
            w, b = self.sd[base + ".weight"], self.sd[base + ".bias"]
            if g is not None:
                c2 = w.shape[0] // 2
                w, b = w[g * c2:(g + 1) * c2], b[g * c2:(g + 1) * c2]
            if w.dim() == 4:
                w = w.unsqueeze(2)
            co, ci, kt, kh, kw = w.shape
            cop, cp = _rup(co, 32), _rup(ci, 64)
            wt = torch.zeros(cop, kt * kh * kw, cp, dtype=_F32, device=self.dev)
            wt[:co, :, :ci] = w.permute(0, 2, 3, 4, 1).reshape(co, kt * kh * kw, ci)
            bp = torch.zeros(cop, dtype=_F32, device=self.dev)
            bp[:co] = b
            wb = wt.reshape(cop, -1).to(_BF).contiguous()
            fp8 = self.fp8 and g is None and converted(base, ci, co)
            if fp8:
                q, s = quantize_weight(wb.float())
                wsrc = (W(f"e4m3 {name}.weight", q), W(f"s_w of {name}.weight", s))
            else:
                wsrc = W(f"bf16 {name}.weight [cop, taps*cp]", wb)
            self._w[name] = (wsrc, W(f"{name}.bias", bp), (kt, kh, kw), fp8)
        return self._w[name]

    def lin(self, name):
        """A 1x1x1 shortcut as a plain GEMM weight [rup(co, 32), rup(ci, 8)] and its bias."""
        w = self.sd[name + ".weight"]
        co, ci = w.shape[:2]
        wp = torch.zeros(_rup(co, 32), _rup(ci, 8), dtype=_F32, device=self.dev)
        wp[:co, :ci] = w.reshape(co, ci)
        bp = torch.zeros(_rup(co, 32), dtype=_F32, device=self.dev)
        bp[:co] = self.sd[name + ".bias"]
        return W(f"bf16 {name}.weight", wp.to(_BF).contiguous()), W(f"{name}.bias", bp)

    def gamma(self, key):
        return W(key, self.sd[key].reshape(-1).contiguous())

    def attn_w(self, p, C):
        """to_qkv split, the softmax scale C^-0.5 folded into q, the v bias folded through proj (softmax rows sum to 1)."""
        Wqkv = self.sd[p + ".to_qkv.weight"].reshape(3 * C, C)
        bqkv = self.sd[p + ".to_qkv.bias"]
        Wo = self.sd[p + ".proj.weight"].reshape(C, C)
        sc = C ** -0.5
        return dict(wq=W(f"{p} q weight * C^-0.5", (Wqkv[:C] * sc).to(_BF).contiguous()),
                    bq=W(f"{p} q bias * C^-0.5", bqkv[:C] * sc),
                    wk=W(f"{p} k weight", Wqkv[C:2 * C].to(_BF).contiguous()), bk=W(f"{p} k bias", bqkv[C:2 * C].contiguous()),
                    wv=W(f"{p} v weight", Wqkv[2 * C:].to(_BF).contiguous()),
                    wo=W(f"{p}.proj.weight", Wo.to(_BF).contiguous()),
                    bo=W(f"{p}.proj.bias + proj.weight @ v bias", (self.sd[p + ".proj.bias"] + Wo @ bqkv[2 * C:]).contiguous()))

    def conv2_w(self):
        """conv2 (z -> z) with the latent de-normalisation z*std + mean folded in: (W diag(std)) z + (W mean + b)."""
        zd = self.zd
        W2 = self.sd["conv2.weight"].reshape(zd, zd)
        w = torch.zeros(_rup(zd, 32), 64, dtype=_F32, device=self.dev)
        w[:zd, :zd] = W2 * self.std[None, :]
        b = torch.zeros(_rup(zd, 32), dtype=_F32, device=self.dev)
        b[:zd] = W2 @ self.mean + self.sd["conv2.bias"]
        return W("conv2.weight * std", w.to(_BF).contiguous()), W("conv2.weight @ mean + conv2.bias", b)

    def conv1_w(self):
        """conv1's mu half with the latent normalisation (mu - mean) / std folded in."""
        zd = self.zd
        W1 = self.sd["conv1.weight"].reshape(2 * zd, 2 * zd)[:zd]
        w = torch.zeros(_rup(zd, 32), _rup(2 * zd, 32), dtype=_F32, device=self.dev)
        w[:zd, :2 * zd] = W1 / self.std[:, None]
        b = torch.zeros(_rup(zd, 32), dtype=_F32, device=self.dev)
        b[:zd] = (self.sd["conv1.bias"][:zd] - self.mean) / self.std
        return W("conv1.weight[:z] / std", w.to(_BF).contiguous()), W("(conv1.bias[:z] - mean) / std", b)

    # ---- one chunk -----------------------------------------------------------------------------------------------
    def chunk(self, c: Chunk):
        return _Build(self, c).run()


class _Build:
    def __init__(self, sp: Spec, c: Chunk):
        self.sp, self.c, self.st = sp, c, []

    def add(self, *a, **k):
        self.st.append(_stage(*a, **k))

    # ---- building blocks -------------------------------------------------------------------------------------------
    def gemm(self, name, a, w, bias, epi, res=None):
        self.add(name, "gemm", dict(a=a, w=w, bias=bias if bias is not None else NONE, epilogue=V(epi),
                                    res=res if res is not None else NONE, **_GEMM_REST),
                 {"": lambda x: x["out"]}, check_gemm)
        return R(name)

    def act(self, name, x, dims, c, gamma, silu, conv=None, up=1):
        """RMS_norm * gamma, SiLU, 2x upsample of x [N, rup(c, 32)] into the new frames of a conv input buffer; the e4m3 pair when
        that conv runs on e4m3 operands."""
        ins = dict(x=x, dims=V(tuple(dims)), gamma=self.sp.gamma(gamma + ".gamma") if gamma else NONE, up=V(up),
                   silu=V(silu))
        if conv is not None and self.sp.conv_w(conv)[3]:
            self.add(name, "vae_rms_act_fp8", ins, {"q": lambda a: a["out"], "s": lambda a: a["out_scale"]}, check_rms8)
            return (R(name, "q"), R(name, "s"))
        self.add(name, "vae_rms_act", ins, {"": lambda a: a["out"]}, check_rms)
        return R(name)

    def conv(self, name, new, dims, Cp, stream=None, epi=EPI["BF16"], res=None, out_t_mul=1, out_t_add=0, stride_t=1,
             stride_hw=1, outputs=None, keep_out=None, carry=True):
        """A causal conv over the buffer [h + T, H, W, Cp]: h = 0 in the first chunk (or without a stream), else the carried
        last h frames of `stream` (1 for the stride-2 time_conv, else 2), then the new frames `new`. carry: this launch is the
        one after which the stream's last frames are carried (time_conv's second group reads the same buffer)."""
        w, bias, taps, fp8 = self.sp.conv_w(name)
        T, H, W = dims
        n = 1 if stride_t > 1 else HIST
        h = n if (stream is not None and self.c.index > 0) else 0
        keeps = []
        if fp8:
            q, s = new
            if h:
                q = HISTCAT(stream, h, q, (H, W, Cp), _E4M3, part=0)
                s = HISTCAT(stream, h, s, (Cp // 128, H, W), _F32, part=1)
            ins = dict(x=q, x_scale=s, w=w[0], w_scale=w[1], bias=bias, T=V(T), H=V(H), W=V(W), t_hist=V(h), epilogue=V(epi),
                       res=res if res is not None else NONE, taps=V(taps), out=SHAPE((T * H * W, w[0].value.shape[0])))
            if stream is not None and carry:
                keeps.append((stream, n, lambda a, inp: (inp["x"], inp["x_scale"])))
            self.add(name, "conv3d_fp8", ins, outputs or {"": lambda a: a["out"]}, check_conv8, keeps)
            return R(name)
        ins = dict(w=w, bias=bias, T=V(T), H=V(H), W=V(W), epilogue=V(epi), res=res if res is not None else NONE, taps=V(taps),
                   out_t_mul=V(out_t_mul), out_t_add=V(out_t_add), stride_t=V(stride_t), stride_hw=V(stride_hw))
        if out_t_mul == 1 and out_t_add == 0:
            To, Ho, Wo = _conv_geom(h + T, T, H, W, taps, stride_t, stride_hw)
            ins["out"] = SHAPE((To * Ho * Wo, w.value.shape[0]))
        if h:
            ins.update(xbuf=HISTCAT(stream, h, new, (H, W, Cp), _BF), t_hist=V(h))
            entry, p = "conv3d_causal_hist", "xbuf"
        else:
            ins.update(xpad=new, oob_zero_pad=V(True), fuse_w=V(0), cta_pair=NONE)
            entry, p = "conv3d_causal", "xpad"
        if stream is not None and carry:
            keeps.append((stream, n, lambda a, inp: inp[p]))
        if keep_out is not None:
            keeps.append(keep_out)
        self.add(name, entry, ins, outputs or {"": lambda a: a["out"]}, check_conv, keeps)
        return R(name)

    def res_block(self, p, x, dims, ci, co):
        """ResidualBlock: RMS_norm, SiLU, conv, RMS_norm, SiLU, conv + shortcut (oracle res_block)."""
        T, H, W = dims
        c1, c2 = p + ".residual.2", p + ".residual.6"
        cp1, cp2 = _rup(ci, 64), _rup(co, 64)
        a1 = self.act(p + ".residual.0", x, dims, ci, p + ".residual.0", True, conv=c1)
        y = self.conv(c1, a1, dims, cp1, stream=c1)
        res = x
        if p + ".shortcut.weight" in self.sp.sd:
            res = self.gemm(p + ".shortcut", x, *self.sp.lin(p + ".shortcut"), EPI["BF16"])
        a2 = self.act(p + ".residual.3", y, dims, co, p + ".residual.3", True, conv=c2)
        return self.conv(c2, a2, dims, cp2, stream=c2, epi=EPI["RES_BF16"], res=res)

    def attention(self, p, x, dims, C):
        """AttentionBlock: per-frame single-head attention over the frame's H*W tokens (oracle attn_block). Every frame's keys
        and values are an Lf = rup(H*W, 32)-row slice; rows past the frame's H*W get probability 0. With H*W a multiple of 8 the
        slices run over the dense rows (the next frame's keys, then zero rows past the last frame); else each frame has its own
        zero-filled Lf-row slot, whose padding rows carry only the q / k biases."""
        T, H, W = dims
        HW, N = H * W, T * H * W
        Lf = _rup(HW, 32)
        a = self.sp.attn_w(p, C)
        self.act(p + ".norm", x, dims, C, p + ".norm", False)
        if HW % 8:
            def slots(t, extra=0):
                z = torch.zeros(T * Lf + extra, C, dtype=_BF, device=t.device)
                z[:T * Lf].view(T, Lf, C)[:, :HW] = t.reshape(T, HW, C)
                return z
            hn = MAP(R(p + ".norm"), slots, f"{p}.norm in per-frame {Lf}-row slots")
            hnv = MAP(R(p + ".norm"), lambda t: slots(t, 32), f"{p}.norm in per-frame {Lf}-row slots + 32 zero rows")
            q = self.gemm(p + ".q", hn, a["wq"], a["bq"], EPI["BF16"])
            k = self.gemm(p + ".k", hn, a["wk"], a["bk"], EPI["BF16"])
            self.gemm(p + ".vT", a["wv"], hnv, None, EPI["BF16"])
            qf = lambda f: R(p + ".q", rows=(f * Lf, f * Lf + HW))                     # noqa: E731
            kf = lambda f: R(p + ".k", rows=(f * Lf, (f + 1) * Lf))                    # noqa: E731
            vf = lambda f: R(p + ".vT", cols=(f * Lf, (f + 1) * Lf))                   # noqa: E731
        else:
            Next = _rup(N, 32) + 32
            hn = MAP(R(p + ".norm"), lambda t: t.reshape(N, C), f"{p}.norm rows")

            def padded(t):
                z = torch.zeros(Next, C, dtype=_BF, device=t.device)
                z[:N] = t.reshape(N, C)
                return z
            q = self.gemm(p + ".q", hn, a["wq"], a["bq"], EPI["BF16"])
            self.gemm(p + ".k", hn, a["wk"], a["bk"], EPI["BF16"])
            self.gemm(p + ".vT", a["wv"], MAP(R(p + ".norm"), padded, f"{p}.norm rows + {Next - N} zero rows"), None,
                      EPI["BF16"])

            def kf(f):
                def get(t):
                    z = torch.zeros(Lf, C, dtype=_BF, device=t.device)
                    r1 = min(N, f * HW + Lf)
                    z[:r1 - f * HW] = t[f * HW:r1]
                    return z
                return MAP(R(p + ".k"), get, f"{p}.k rows [{f * HW}:{f * HW + Lf}] (zero past row {N})")
            qf = lambda f: R(p + ".q", rows=(f * HW, (f + 1) * HW))                    # noqa: E731

            def vf(f):
                def get(t):
                    return t[:, f * HW:f * HW + Lf]
                return MAP(R(p + ".vT"), get, f"{p}.vT columns [{f * HW}:{f * HW + Lf}]")
        for f in range(T):
            fp = f"{p}.frame{f}"
            self.gemm(fp + ".S", qf(f), kf(f), None, EPI["F32"])
            self.add(fp + ".softmax", "masked_softmax", dict(S=R(fp + ".S"), L=V(HW), hw=V(HW)), {"": lambda x: x["P"]},
                     check_softmax)
            self.gemm(fp + ".PV", R(fp + ".softmax"), vf(f), None, EPI["BF16"])
        o = JOIN([R(f"{p}.frame{f}.PV") for f in range(T)], lambda ts: torch.cat(ts, 0), f"{p} PV rows of every frame")
        return self.gemm(p + ".proj", o, a["wo"], a["bo"], EPI["RES_BF16"], res=x)

    # ---- decoder ---------------------------------------------------------------------------------------------------
    def dec_input(self, dims):
        """conv2 (latent de-normalisation folded in) into decoder.conv1's buffer, then decoder.conv1."""
        T, H, W = dims
        c, zd = self.c, self.sp.zd
        N = T * H * W
        zin = SRC_FRAMES(f"latent frames [{c.t_in}:{c.t_in + c.n_in}]",
                         lambda s: s[:, c.t_in:c.t_in + c.n_in].float().reshape(zd, N))
        self.add("in", "nchw_to_nhwc_bf16", dict(x=zin), {"": lambda a: a["out"]}, check_nchw_to_nhwc)
        self.gemm("conv2", R("in"), *self.sp.conv2_w(), EPI["BF16"])

        def rows(t):
            z = torch.zeros(N, 64, dtype=_BF, device=t.device)
            z[:, :t.shape[1]] = t
            return z.view(T, H, W, 64)
        x0 = MAP(R("conv2"), rows, "conv2 rows (zero columns to 64)")
        return self.conv("decoder.conv1", x0, dims, 64, stream="decoder.conv1")

    def up(self, p, x, dims, ci, co, t_up):
        """Resample upsample2d / upsample3d (oracle resample): frame 0 bypasses time_conv, whose stream is every later frame
        (in the first chunk from the chunk's frame 1, possibly none); the two output channel groups of stream frame t are
        frames 2t + g (+1 behind frame 0); then nearest-exact 2x and the Conv2d 3x3."""
        T, H, W = dims
        HW = H * W
        C = _rup(ci, 32)
        if t_up:
            first, stream = self.c.index == 0, p + ".time_conv"
            Ts = T - 1 if first else T
            if Ts > 0:
                new = MAP(x, lambda t: t[HW:] if first else t, f"{x.label} frames {'1..' if first else 'all'}")
                if C % 64:
                    new = self.act(stream + ".in", new, (Ts, H, W), ci, None, False)
                else:
                    new = MAP(new, lambda t: t.reshape(Ts, H, W, C), new.label)
                lead = 1 if first else 0
                for g in (0, 1):
                    self.conv(f"{stream}.{g}", new, (Ts, H, W), _rup(ci, 64), stream=stream, carry=g == 0,
                              out_t_mul=2, out_t_add=lead + g,
                              outputs={"": lambda a, g=g, lead=lead: a["out"].reshape(-1, HW, a["out"].shape[-1])[lead + g::2]})

                def assemble(ts, first=first):
                    y0, g0, g1 = ts
                    y = torch.stack((g0, g1), 1).reshape(2 * Ts * HW, -1)
                    return torch.cat([y0[:HW], y], 0) if first else y
                x = JOIN([x, R(stream + ".0"), R(stream + ".1")], assemble,
                         f"{'frame 0 of ' + x.label + ', ' if first else ''}time_conv groups 0 / 1 interleaved")
                T = 2 * Ts + (1 if first else 0)
        a = self.act(p + ".resample.1.in", x, (T, H, W), ci, None, False, conv=p + ".resample.1", up=2)
        return self.conv(p + ".resample.1", a, (T, 2 * H, 2 * W), _rup(ci, 64)), (T, 2 * H, 2 * W)

    def dupup(self, name, main, held, held_dims, ci, co, ft, fs):
        first = self.c.index == 0
        entry = "vae_dupup_add" if first else "vae_dupup_add_cont"
        self.add(name, entry, dict(main=main, x=held, dims=V(tuple(held_dims)), in_c=V(ci), out_c=V(co), ft=V(ft), fs=V(fs)),
                 {"": lambda a: a["main"]}, check_dupup(first))
        return R(name)

    def dec_head(self, x, dims, c_last):
        T, H, W = dims
        c = self.c
        a = self.act("decoder.head.0", x, dims, c_last, "decoder.head.0", True, conv="decoder.head.2")
        y = self.conv("decoder.head.2", a, dims, _rup(c_last, 64), stream="decoder.head.2", epi=EPI["F32"])
        one = c.index == 0 and not c.more
        if self.sp.kind == "wan22_dec":
            out = WIN("the result" if one else f"result frames [{c.t_out}:{c.t_out + c.n_out}]",
                      (lambda o: o) if one else (lambda o: o[:, c.t_out:c.t_out + c.n_out]))
            self.add("write", "vae_unpatchify2_clamp" if one else "vae_unpatchify2_clamp_win",
                     dict(y=y, out=out, T=V(T), H=V(H), W=V(W)), {}, check_unpatchify, window=True)
        else:
            out = WIN("the result as [3, frames*h*w]" if one else f"result frames [{c.t_out}:{c.t_out + c.n_out}]",
                      (lambda o: o.view(3, -1)) if one else (lambda o: o[:, c.t_out:c.t_out + c.n_out]))
            self.add("write", "nhwc_to_nchw_f32" if one else "nhwc_to_nchw_f32_win", dict(x=y, out=out, clamp=V((-1.0, 1.0))),
                     {}, check_nhwc_to_nchw, window=True)

    def decoder(self):
        orc, c = self.sp.orc, self.c
        _, _, H, W = self.sp.src_shape
        dims = (c.n, H, W)
        x = self.dec_input(dims)
        d0 = (orc.dims if self.sp.kind == "wan22_dec" else [orc.plan[0][2]])[0]
        x = self.res_block("decoder.middle.0", x, dims, d0, d0)
        x = self.attention("decoder.middle.1", x, dims, d0)
        x = self.res_block("decoder.middle.2", x, dims, d0, d0)
        if self.sp.kind == "wan22_dec":
            for i in range(orc.n_up):
                p = f"decoder.upsamples.{i}.upsamples"
                ci, co = orc.dims[i], orc.dims[i + 1]
                held, held_dims = x, dims
                c_in = ci
                for j in range(orc.nrb + 1):
                    x = self.res_block(f"{p}.{j}", x, dims, c_in, co)
                    c_in = co
                if i != orc.n_up - 1:
                    t_up = orc.t_up[i] if i < len(orc.t_up) else False
                    x, dims = self.up(f"{p}.{orc.nrb + 1}", x, dims, co, co, t_up)
                    x = self.dupup(f"decoder.upsamples.{i}.shortcut", x, held, held_dims, ci, co, 2 if t_up else 1, 2)
            c_last = orc.dims[-1]
        else:
            for n, kind, ci, co in orc.plan:
                p = f"decoder.upsamples.{n}"
                if kind == "res":
                    x = self.res_block(p, x, dims, ci, co)
                    c_last = co
                else:
                    x, dims = self.up(p, x, dims, ci, co, kind == "upsample3d")
        self.dec_head(x, dims, c_last)

    # ---- encoder ---------------------------------------------------------------------------------------------------
    def enc_input(self):
        c, fs = self.c, self.sp.fs_in
        _, _, H, W = self.sp.src_shape
        dims = (c.n_in, H // fs, W // fs)
        one = c.index == 0 and not c.more
        frames = SRC_FRAMES(f"video frames [{c.t_in}:{c.t_in + c.n_in}]", lambda s: s[:, c.t_in:c.t_in + c.n_in])
        if self.sp.kind == "wan22_enc":
            self.add("in", "vae_patchify2_bf16" if one else "vae_patchify2_bf16_win", dict(video=frames),
                     {"": lambda a: a["out"]}, check_patchify)
        else:
            x = MAP(frames, lambda v: v.reshape(3, -1), frames.label + " as [3, frames*H*W]") if one else frames
            self.add("in", "nchw_to_nhwc_bf16" if one else "nchw_to_nhwc_bf16_win", dict(x=x), {"": lambda a: a["out"]},
                     check_nchw_to_nhwc)
        x0 = MAP(R("in"), lambda t: t.reshape(*dims, 64), "in")
        return self.conv("encoder.conv1", x0, dims, 64, stream="encoder.conv1"), dims

    def down(self, p, x, dims, C, temporal):
        """Resample downsample2d / downsample3d (oracle resample_down): Conv2d 3x3 stride 2 behind ZeroPad2d((0,1,0,1)); then
        frame 0 passes and time_conv (3,1,1) stride 2, unpadded, runs over the whole resampled stream, whose last frame the next
        chunk carries (in the first chunk of one frame, that frame alone)."""
        T, H, W = dims
        Cc = _rup(C, 32)
        Ho, Wo = (H + 1 - 3) // 2 + 1, (W + 1 - 3) // 2 + 1
        stream = p + ".time_conv"
        if Cc % 64:
            a = self.act(p + ".resample.1.in", x, dims, C, None, False)
        else:
            a = MAP(x, lambda t: t.reshape(T, H, W, Cc), x.label)
        frames = lambda t: t.reshape(T, Ho, Wo, -1)                                    # noqa: E731
        if temporal and self.c.index > 0:
            y = self.conv(p + ".resample.1", a, dims, _rup(C, 64), stride_hw=2)
            tin = self.act(stream + ".in", y, (T, Ho, Wo), C, None, False) if Cc % 64 else MAP(y, frames, y.label)
            z = self.conv(stream, tin, (T, Ho, Wo), _rup(C, 64), stream=stream, stride_t=2)
            return z, (T // 2, Ho, Wo)
        one_frame_carry = temporal and T == 1 and self.c.more
        keep = (stream, 1, lambda a_, inp: a_["out"].reshape(T, Ho, Wo, -1)) if one_frame_carry and not Cc % 64 else None
        y = self.conv(p + ".resample.1", a, dims, _rup(C, 64), stride_hw=2, keep_out=keep)
        if temporal and T > 1:
            tin = self.act(stream + ".in", y, (T, Ho, Wo), C, None, False) if Cc % 64 else MAP(y, frames, y.label)
            To = (T - 3) // 2 + 1
            self.conv(stream, tin, (T, Ho, Wo), _rup(C, 64), stream=stream, stride_t=2, out_t_add=1,
                      outputs={"": lambda a_: a_["out"].reshape(-1, Ho * Wo, a_["out"].shape[-1])[1:]})
            x = JOIN([y, R(stream)], lambda ts: torch.cat([ts[0][:Ho * Wo], ts[1].reshape(-1, ts[1].shape[-1])], 0),
                     f"frame 0 of {p}.resample.1, then {stream}")
            return x, (1 + To, Ho, Wo)
        if one_frame_carry and Cc % 64:
            self.act(stream + ".in", y, (T, Ho, Wo), C, None, False)
            self.st[-1].keeps = [(stream, 1, lambda a_, inp: a_["out"])]
        return y, (T, Ho, Wo)

    def avgdown(self, name, main, held, held_dims, ci, co, ft, fs):
        self.add(name, "vae_avgdown_add", dict(main=main, x=held, dims=V(tuple(held_dims)), in_c=V(ci), out_c=V(co), ft=V(ft),
                                               fs=V(fs)), {"": lambda a: a["main"]}, check_avgdown)
        return R(name)

    def encoder(self):
        orc, c, zd = self.sp.orc, self.c, self.sp.zd
        x, dims = self.enc_input()
        if self.sp.kind == "wan22_enc":
            for i in range(orc.n):
                p = f"encoder.downsamples.{i}.downsamples"
                ci, co = orc.dims[i], orc.dims[i + 1]
                down = i != orc.n - 1
                t_down = orc.t_down[i] if i < len(orc.t_down) else False
                held, held_dims, c_in = x, dims, ci
                for j in range(orc.nrb):
                    x = self.res_block(f"{p}.{j}", x, dims, c_in, co)
                    c_in = co
                if down:
                    x, dims = self.down(f"{p}.{orc.nrb}", x, dims, co, t_down)
                x = self.avgdown(f"encoder.downsamples.{i}.shortcut", x, held, held_dims, ci, co, 2 if t_down else 1,
                                 2 if down else 1)
            d = orc.dims[-1]
        else:
            for n, kind, ci, co in orc.plan:
                p = f"encoder.downsamples.{n}"
                if kind == "res":
                    x = self.res_block(p, x, dims, ci, co)
                else:
                    x, dims = self.down(p, x, dims, co, kind == "downsample3d")
                d = co
        x = self.res_block("encoder.middle.0", x, dims, d, d)
        x = self.attention("encoder.middle.1", x, dims, d)
        x = self.res_block("encoder.middle.2", x, dims, d, d)
        a = self.act("encoder.head.0", x, dims, d, "encoder.head.0", True, conv="encoder.head.2")
        y = self.conv("encoder.head.2", a, dims, _rup(d, 64), stream="encoder.head.2")
        mu = self.gemm("conv1", y, *self.sp.conv1_w(), EPI["F32"])
        one = c.index == 0 and not c.more
        out = WIN("the result as [z, frames*h*w]" if one else f"result frames [{c.t_out}:{c.t_out + c.n_out}]",
                  (lambda o: o.view(zd, -1)) if one else (lambda o: o[:, c.t_out:c.t_out + c.n_out]))
        self.add("write", "nhwc_to_nchw_f32" if one else "nhwc_to_nchw_f32_win", dict(x=mu, out=out, clamp=NONE), {},
                 check_nhwc_to_nchw, window=True)

    def run(self):
        if self.sp.dec:
            self.decoder()
        else:
            self.encoder()
        return self.st


# ------------------------------------------------------------------------------------------------------------
# running a call
# ------------------------------------------------------------------------------------------------------------
def install(mp, modules, eng, spec, tag, keep_snaps=False):
    """Put a checker between `eng` and the ops of `modules` (vae22, vae21, vae_enc): every `_run_chunk` becomes one chunk
    region of the spec, `_stream` hands the checker the input and the result. Returns the checker; ck.expect(...) states the
    chunks of each following call."""
    base = modules[0].ops
    ck = Checker(base, spec, tag, keep_snaps)
    for m in modules:
        mp.setattr(m, "ops", ck.proxy)
    real_stream, real_chunk = eng._stream, eng._run_chunk

    def stream(src, out, *a, **k):
        spec.src_shape = tuple(src.shape)
        ck.begin_stream(src, out)
        return real_stream(src, out, *a, **k)

    def run_chunk(src, out):
        with ck.chunk():
            return real_chunk(src, out)
    mp.setattr(eng, "_stream", stream)
    mp.setattr(eng, "_run_chunk", run_chunk)
    return ck


def finish(ck):
    if ck.queue:
        raise AssertionError(f"{ck.tag}: {len(ck.queue)} expected chunk(s) never ran")
