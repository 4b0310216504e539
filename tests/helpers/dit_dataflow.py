"""TEST INFRASTRUCTURE: the WanDiT forward checked launch by launch.

A SPEC states the dataflow of one forward independently of yume_b200/dit.py, from the reference's WanModel.forward
(wan23/modules/model.py:547-865, wan/modules/model.py:723-1013, as oracle/wan_dit.py restates it): an ordered list of stages in
six phases (embed: the FramePack segments of WanOracle._segments or the grid, each a patchify + GEMM; time: the sinusoid, the
time MLP and projection, the block and head tables, per 16-row chunk; context: the text MLP and the 14B image MLP; cross_kv; one
WanAttentionBlock; head: the modulated LayerNorm, the head linear, unpatchify of the new frames). Each stage names its ops entry,
where every operand must come from (an earlier stage's output, a weight rebuilt from the reference's state-dict keys, the
forward's own inputs in the reference's token layout, a modulation row with its token index, RoPE rows from
oracle.wan_dit.grid_freqs, the first k_len rows) and which per-element bound its output must meet. At the first block's entry the
whole residual stream must equal the embed GEMMs' outputs row for row in the reference's token order, with exact zeros on the
padding rows, and each token's index must point at the table row of its own timestep.

A CHECKER sits between the engine and its ops module (`dit.ops`). Outside a checked region it only passes launches through;
inside one it takes the next stage for every launch and checks
  order    the entry is the stage's, and the region makes exactly the spec's number of launches;
  inputs   every operand is torch.equal to the source the stage names (view shape, row count, scale table included);
  output   right after the launch, against an fp64 recomputation from those inputs within the kernel's contract bound
           (tests/test_gpu_kernel_contract*.py: gemm_epilogue_ref / gemm_bounds, _ln_ref, _rr_ref, attention_bound_prod,
           the fp8 gemm_bound, attention_fp8_bound, sinusoidal_ref, linear_f32_small_ref, linear_f32_ref; the fp8
           quantisers bit-identical to their twins in oracle/fp8*.py; patchify, unpatchify and bcast_add bit-identical to the
           torch stand-ins' reshapes and the fp32 add).
Only the snapshots a later stage (or the block-entry check) reads are kept, and each is dropped after its last reader, so
production L fits. Large launches are sampled like the production contract (gemm_sample rows and columns, attention_sample
rows). The geometry comes from WanOracle._segments, the convpadd shapes and grid_freqs, never from the oracle's CPU pack (its
real-width conv3d is far too slow at production sizes).

The same spec and checker run on the H100 (tests/test_gpu_dit_dataflow.py) and over the torch stand-ins at tiny width on the
CPU (tests/test_dit_dataflow_cpu.py), where wiring defects are patched into the engine and must be caught."""
from __future__ import annotations

import contextlib
import inspect
import math
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional

import torch

import test_gpu_kernel_contract as KC
import test_gpu_kernel_contract_ext as KE
import test_gpu_kernel_contract_fp8 as K8
import test_gpu_kernel_contract_fp8_attn as KA
import test_gpu_kernel_contract_prod as KP
from helpers import torch_ops as TO
from oracle import synth
from oracle.fp8 import dequantize_act, quantize_act, quantize_weight
from oracle.fp8_attn import dequantize_vt, quantize_vt
from oracle.wan_dit import WanOracle, grid_freqs
from yume_b200 import ops as _real_ops

D = 128                       # head_dim of both trees
EPS = 1e-6
ENTRIES = ("gemm", "gemm_fp8", "ln_modulate", "ln_modulate_fp8", "qk_norm_rope", "rmsnorm_rope", "quant_rows_fp8",
           "quant_vt_fp8", "attention", "attention_fp8", "patchify", "sinusoidal", "linear_f32_small", "bcast_add", "linear_f32",
           "unpatchify")
SIGS = {e: inspect.signature(getattr(_real_ops, e)) for e in ENTRIES}
EPI = dict(BF16=0, GELU=1, F32=2, GATE_RES=3, GELU_ERF=4, GELU_FP8=8)     # include/yume_b200.h, include/yume_b200_fp8.h
IMG_EPS = 1e-5                # MLPProj's LayerNorms (nn.LayerNorm default, wan/modules/model.py:533-537)
T_CHUNK = 16                  # timestep rows per time-table launch chain (yb_linear_f32_small's M limit)
FULL_ROWS = 1024              # launches with at most this many rows are checked on every row, larger ones sampled


# ------------------------------------------------------------------------------------------------------------
# sources
# ------------------------------------------------------------------------------------------------------------
@dataclass
class Src:
    """Where an operand must come from. get(ck) -> the expected value; kind: 'tensor' (torch.equal), 'scale' (a 1x128 scale
    table: equal on the source's columns, the table at least that long), 'rope' (rows equal to within one f32 ulp of values
    <= 1: the oracle's complex polar and the engine's cos / sin round the same fp64 angle), 'value' (== / is None)."""
    label: str
    get: Callable
    kind: str = "tensor"
    reads: tuple = ()          # stage names whose snapshots this source reads


def S(stage, part="", rows=None, cols=None, kind="tensor", fn=None, what=""):
    """Stage `stage`'s output (part `part`), rows [:rows] (or [lo:hi] for a pair), columns [c0:c1], then `fn` (a view)."""
    rows = None if rows is None else (rows if isinstance(rows, tuple) else (0, rows))
    rs = slice(None) if rows is None else slice(*rows)
    cs = slice(None) if cols is None else slice(*cols)
    label = f"{stage}{'.' + part if part else ''}" + \
        (f"[{rows[0] or ''}:{'' if rows[1] is None else rows[1]}]" if rows is not None else "") + \
        (f"[:, {cols[0]}:{cols[1]}]" if cols is not None else "") + (f" {what}" if what else "")
    f = fn or (lambda t: t)
    return Src(label, lambda ck: f(ck.snap[stage][part][rs, cs]), kind, (stage,))


def CAT(*srcs):
    return Src("cat(" + ", ".join(s.label for s in srcs) + ")", lambda ck: torch.cat([s.get(ck) for s in srcs], dim=1),
               "tensor", sum((s.reads for s in srcs), ()))


def T(label, value, kind="tensor"):
    return Src(label, lambda ck: value, kind)


def E(label, key, fn=lambda t: t):
    """A tensor of the run that exists only once it starts (the block's input rows, the embedded context, the modulation rows)."""
    return Src(label, lambda ck: fn(ck.env[key]))


def V(value):
    return Src(repr(value), lambda ck: value, "value")


NONE = V(None)


@dataclass
class Stage:
    name: str
    entry: str
    inputs: Dict[str, Src]
    outputs: Dict[str, Callable]          # part -> fn(bound args) -> tensor kept as the stage's output
    check: Optional[Callable] = None      # fn(checker, stage, args, inp) -> worst |err| / bound


# ------------------------------------------------------------------------------------------------------------
# the checker
# ------------------------------------------------------------------------------------------------------------
class _Proxy:
    """Stands for the ops module inside dit.py: the ten block entries go through the checker, everything else is the module's."""

    def __init__(self, ck):
        self._ck = ck
        for e in ENTRIES:
            if hasattr(ck.base, e):
                setattr(self, e, self._wrap(e))

    def _wrap(self, entry):
        def call(*a, **k):
            return self._ck.launch(entry, a, k)
        return call

    def __getattr__(self, name):
        return getattr(self._ck.base, name)


class Checker:
    def __init__(self, base, tag, att_plan=None):
        self.base, self.tag = base, tag
        self.att_plan = att_plan or (lambda Lq, Lk, H, flags: 1)   # KV segments of an attention launch (1 on the CPU)
        self.snap: Dict[str, Dict[str, torch.Tensor]] = {}
        self.program: List[Stage] = []
        self.phases: Dict[str, range] = {}
        self.pos, self.stop, self.phase = 0, 0, None
        self.worst: Dict[str, float] = {}
        self.stream = None                  # the residual stream the last pass-through GATE_RES launch wrote
        self.env: Dict[str, torch.Tensor] = {}   # what the run hands the block: x_in (and for the seams ctx, mod)
        self.pinned: set = set()            # stages whose snapshots the block-entry check reads (kept until unpin)
        self.entered: List[str] = []        # phases in the order they were opened
        self.proxy = _Proxy(self)

    # ---- program -----------------------------------------------------------------------------------------------
    def add_phase(self, name, stages):
        start = len(self.program)
        self.program += stages
        self.phases[name] = range(start, len(self.program))
        self.last_read = {}
        for j, st in enumerate(self.program):
            for src in st.inputs.values():
                for r in src.reads:
                    self.last_read[r] = j

    def enter(self, phase):
        """Close the open phase (it must have made all its launches) and open `phase`: launches from here on are its stages."""
        self.leave()
        rg = self.phases[phase]
        self.phase, self.pos, self.stop = phase, rg.start, rg.stop
        self.entered.append(phase)

    def leave(self):
        """Close the open phase, if any: it must have made exactly the spec's number of launches."""
        if self.phase is None:
            return
        phase, rg, ended = self.phase, self.phases[self.phase], self.pos
        self.phase = None
        if ended != rg.stop:
            raise AssertionError(f"{self.tag}: {phase} made {ended - rg.start} launches, the spec has {len(rg)}: stage "
                                 f"'{self.program[ended].name}' ({self.program[ended].entry}) never ran")

    @contextlib.contextmanager
    def region(self, phase):
        """Launches inside are the stages of `phase`, exactly as many as it has."""
        assert self.phase is None, f"{self.tag}: region {phase} opened inside {self.phase}"
        self.enter(phase)
        try:
            yield
        except BaseException:
            self.phase = None
            raise
        self.leave()

    def unpin(self):
        for name in self.pinned:
            self.snap.pop(name, None)
        self.pinned = set()

    # ---- one launch ----------------------------------------------------------------------------------------------
    def launch(self, entry, a, k):
        fn = getattr(self.base, entry)
        if self.phase is None:
            out = fn(*a, **k)
            args = SIGS[entry].bind(*a, **k).arguments
            if entry in ("gemm", "gemm_fp8") and args.get("epilogue") == EPI["GATE_RES"]:
                self.stream = args["out"]
            return out
        if self.pos >= self.stop:
            raise AssertionError(f"{self.tag}: {self.phase}: launch {self.pos - self.phases[self.phase].start + 1} ({entry}) "
                                 f"is beyond the spec's {len(self.phases[self.phase])} stages")
        st = self.program[self.pos]
        if entry != st.entry:
            raise AssertionError(f"{self.tag}: stage '{st.name}' expects a {st.entry} launch, the engine made {entry}")
        b = SIGS[entry].bind(*a, **k)
        b.apply_defaults()
        args = b.arguments
        inp = {}
        for p, src in st.inputs.items():
            inp[p] = src.get(self)
            _same(self.tag, st.name, p, args[p], inp[p], src)
        out = fn(*a, **k)
        if self.base is _real_ops:
            torch.cuda.synchronize()
        args["ret"] = out                   # the entries that allocate their output (sinusoidal, linear_f32_small, bcast_add)
        keep = (st.name in self.last_read and self.last_read[st.name] > self.pos) or st.name in self.pinned
        if keep:
            self.snap[st.name] = {part: f(args).clone() for part, f in st.outputs.items()}
        if st.check is not None:
            w = st.check(self, st, args, inp)
            self.worst[st.name] = max(self.worst.get(st.name, 0.0), w)
        del inp
        for name in [n for n in self.snap if self.last_read.get(n, -1) <= self.pos and n not in self.pinned]:
            del self.snap[name]
        self.pos += 1
        return out

    def report(self):
        return ", ".join(f"{n} {w:.3f}" for n, w in self.worst.items())


def _same(tag, stage, param, got, want, src):
    def fail(why):
        raise AssertionError(f"{tag}: stage '{stage}' operand '{param}' is not {src.label}: {why}")
    if src.kind == "value":
        if want is None:
            if got is not None:
                fail("got a tensor / value where the spec has none")
        elif isinstance(want, float):
            if got is None or not math.isclose(got, want, rel_tol=1e-12):
                fail(f"{got} != {want}")
        elif isinstance(got, torch.Tensor) or got != want:
            fail(f"{got} != {want}")
        return
    if not isinstance(got, torch.Tensor):
        fail(f"got {got!r}")
    want = want.to(got.device)
    if src.kind == "scale":
        if got.dim() != 2 or got.shape[0] != want.shape[0] or got.shape[1] < want.shape[1]:
            fail(f"scale table {tuple(got.shape)} for {tuple(want.shape)}")
        got = got[:, :want.shape[1]]
    elif src.kind == "rope":
        if got.shape[0] < want.shape[0] or got.shape[1:] != want.shape[1:]:
            fail(f"table {tuple(got.shape)} for {tuple(want.shape)} rows")
        d = (got[:want.shape[0]].double() - want.double()).abs().max() if want.numel() else 0.0
        if float(d) > 2.0 ** -23:
            fail(f"rows differ by up to {float(d):.3g}")
        return
    if got.shape != want.shape:
        fail(f"shape {tuple(got.shape)}, the spec's is {tuple(want.shape)}")
    if got.dtype != want.dtype:
        fail(f"dtype {got.dtype}, the spec's is {want.dtype}")
    if not torch.equal(got, want):
        n = int((got != want).sum()) if got.dtype != torch.float8_e4m3fn else \
            int((got.view(torch.uint8) != want.view(torch.uint8)).sum())
        fail(f"{n} of {got.numel()} elements differ")


# ------------------------------------------------------------------------------------------------------------
# output checks (contract bounds; fp64 on the device of the operands)
# ------------------------------------------------------------------------------------------------------------
def _rows(M, key):
    return torch.arange(M) if M <= FULL_ROWS else KP.gemm_sample(M, 1, key)[0]


def _cols(N, key):
    return torch.arange(0) if N <= FULL_ROWS else KP.gemm_sample(1, N, key)[1]


def _ratio(got, ref, bound, what):
    err = (got.double() - ref).abs()
    r = torch.where(bound > 0, err / bound, torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    r = torch.where(torch.isnan(err), torch.full_like(err, math.inf), r)
    worst = float(r.max()) if r.numel() else 0.0
    if not worst <= 1.0:
        i = tuple(int(v) for v in torch.unravel_index(r.argmax().cpu(), r.shape))
        raise AssertionError(f"{what}: {int((r > 1).sum())} of {r.numel()} elements out of bound; worst at {i}: got "
                             f"{float(got[i]):.6g} ref {float(ref[i]):.6g} bound {float(bound[i]):.3g} (|err|/bound {worst:.3g})")
    return worst


def _mod_rows(t, tok, rows):
    """Rows `rows` of a [U, C] modulation table under token index `tok` (None: one row for every token) as fp64 [R, C]."""
    if t is None:
        return None
    t = t if t.dim() == 2 else t[None]
    idx = tok[rows.to(tok.device)].long() if tok is not None else torch.zeros(len(rows), dtype=torch.long, device=t.device)
    return t.double()[idx]


def _shape(ck, st, param, t, want):
    if tuple(t.shape) != tuple(want):
        raise AssertionError(f"{ck.tag}: stage '{st.name}' operand '{param}' has shape {tuple(t.shape)}, the spec's is "
                             f"{tuple(want)}")


def check_ln(ck, st, a, inp):
    """_ln_ref on every row, into bf16 (bf16_out_bound) or f32 (the head)."""
    x, out, tok = inp["x"], a["out"], inp["tok_idx"]
    L, C = x.shape
    _shape(ck, st, "out", out, (L, C))
    worst = 0.0
    for r0 in range(0, L, 4096):
        rows = torch.arange(r0, min(L, r0 + 4096), device=x.device)
        y, f32 = KC._ln_ref(x[rows], C, inp["eps"], inp["weight"], inp["bias"], _mod_rows(inp["scale"], tok, rows),
                            _mod_rows(inp["shift"], tok, rows))
        bound = f32 if out.dtype == torch.float32 else KC.bf16_out_bound(y, f32)
        worst = max(worst, _ratio(out[rows], y, bound, f"{ck.tag}: stage '{st.name}' output"))
    return worst


def check_ln8(ck, st, a, inp):
    """The f32 LayerNorm the quantiser reads (ln_modulate into f32) within _ln_ref, and the e4m3 pair bit-identical to the twin of
    it (the contract of yb_ln_modulate_fp8, tests/test_gpu_kernel_contract_fp8.py)."""
    x, tok = inp["x"], inp["tok_idx"]
    L, C = x.shape
    y32 = torch.empty(L, C, dtype=torch.float32, device=x.device)
    ck.base.ln_modulate(x, y32, inp["scale"], inp["shift"], tok, inp["weight"], inp["bias"], eps=EPS)
    worst = 0.0
    for r0 in range(0, L, 4096):
        rows = torch.arange(r0, min(L, r0 + 4096), device=x.device)
        y, f32 = KC._ln_ref(x[rows], C, EPS, inp["weight"], inp["bias"], _mod_rows(inp["scale"], tok, rows),
                            _mod_rows(inp["shift"], tok, rows))
        worst = max(worst, _ratio(y32[rows], y, f32, f"{ck.tag}: stage '{st.name}' f32 LayerNorm"))
    _twin(ck, st, a["out"], a["out_scale"][:, :L], *quantize_act(y32))
    return worst


def _twin(ck, st, q, s, tq, ts):
    tq, ts = tq.to(q.device), ts.to(s.device)
    if not (torch.equal(q.view(torch.uint8), tq.to(q.device).view(torch.uint8)) and torch.equal(s, ts.to(s.device))):
        raise AssertionError(f"{ck.tag}: stage '{st.name}' output: {int((q.view(torch.uint8) != tq.view(torch.uint8)).sum())} "
                             f"e4m3 bytes / {int((s != ts).sum())} scales differ from the twin")


def check_q8(ck, st, a, inp):
    M = inp["x"].shape[0]
    _twin(ck, st, a["out"], a["out_scale"][:, :M], *quantize_act(inp["x"].float()))
    return 0.0


def check_vt8(ck, st, a, inp):
    _twin(ck, st, a["vt8"], a["v_scale"], *quantize_vt(inp["v"].float(), inp["heads"]))
    return 0.0


def check_rr(ck, st, a, inp):
    """_rr_ref on every operand the launch normalises in place (q and k, or qk)."""
    worst = 0.0
    pairs = [("q", "wq"), ("k", "wk")] if "q" in inp else [("qk", "weight")]
    for p, w in pairs:
        x, out = inp[p], a[p]
        L = x.shape[0]
        rope, rlen = inp["rope"], inp.get("rope_len") or 0
        for r0 in range(0, L, 8192):
            r1 = min(L, r0 + 8192)
            rp = None if rope is None else rope[r0:].to(x.device)
            y, bound = KC._rr_ref(x[r0:r1], inp[w].to(x.device), rp, max(0, min(rlen - r0, r1 - r0)), D)
            worst = max(worst, _ratio(out[r0:r1], y, bound, f"{ck.tag}: stage '{st.name}' output {p}"))
    return worst


def _gate_rows(inp, rows, N, dev):
    g = inp.get("gate")
    if g is None:
        return torch.ones(len(rows), N, dtype=torch.float64, device=dev)
    return _mod_rows(g, inp.get("tok_idx"), rows)


def check_gemm(ck, st, a, inp):
    """gemm_epilogue_ref over gemm_ref_rows_cols: every row of a small launch, else 2 full rows per 128-row band and 2 full columns
    per 64-column band (gemm_sample)."""
    A, B, bias, epi = inp["a"], inp["w"], inp["bias"], inp["epilogue"]
    M, N = A.shape[0], B.shape[0]
    out = a["out"]
    _shape(ck, st, "out", out, (M, N))
    rows, cols = _rows(M, (ck.tag, st.name)).to(A.device), _cols(N, (ck.tag, st.name)).to(A.device)
    (accR, FR), (accC, FC) = KP.gemm_ref_rows_cols(A, B, rows, cols)
    worst = 0.0
    allr = torch.arange(M, device=A.device)
    for rr, cc, acc, Fb in ((rows, None, accR, FR), (allr, cols, accC, FC)):
        if acc.numel() == 0:
            continue
        pick = (lambda t: t[rr]) if cc is None else (lambda t: t[:, cc])
        b = None if bias is None else (bias.double() if cc is None else bias.double()[cc])[None].expand_as(acc)
        x0 = g = None
        if epi == EPI["GATE_RES"]:
            x0 = pick(inp["out"]).double()
            g = _gate_rows(inp, rr, N, A.device)
            g = g if cc is None else g[:, cc]
        ref, bound = KP.gemm_epilogue_ref(epi, acc, Fb, bias=b, x0=x0, gate=g)
        worst = max(worst, _ratio(pick(out), ref, bound, f"{ck.tag}: stage '{st.name}' output"))
    return worst


def check_gemm8(ck, st, a, inp):
    """The fp8 gemm_bound over the dequantised operands, on full rows (every row of a small launch, else gemm_sample's rows)."""
    M, K = inp["a"].shape
    N = inp["w"].shape[0]
    epi = inp["epilogue"]
    rows = _rows(M, (ck.tag, st.name)).to(inp["a"].device)
    wd = inp["w"].double() * inp["w_scale"].double()[:, None]
    ad = dequantize_act(inp["a"][rows], inp["a_scale"][:, rows]).double()
    ref = ad @ wd.t()
    if inp["bias"] is not None:
        ref = ref + inp["bias"].double()
    out_ulp = {EPI["BF16"]: 2.0 ** -8, EPI["F32"]: 2.0 ** -24, EPI["GATE_RES"]: 2.0 ** -24, EPI["GELU_FP8"]: 0.0}[epi]
    bound = K8.gemm_bound(ad.abs(), wd.abs(), K, out_ulp, ref)
    what = f"{ck.tag}: stage '{st.name}' output"
    if epi == EPI["GELU_FP8"]:
        sc = a["out_scale"][:, rows]
        gref, bound = K8.gelu_fp8_bound(ref, bound, sc.t().repeat_interleave(128, dim=1).double())
        return _ratio(dequantize_act(a["out"][rows], sc), gref, bound, what)
    if epi == EPI["GATE_RES"]:
        gt = _gate_rows(inp, rows, N, ad.device)
        ref = inp["out"][rows].double() + ref * gt
        bound = bound * gt.abs() + 2.0 ** -24 * ref.abs()
    return _ratio(a["out"][rows], ref, bound, what)


def _exact(ck, st, got, want, what="output"):
    if got.shape != want.shape or not torch.equal(got, want.to(got.device)):
        n = int((got != want.to(got.device)).sum()) if got.shape == want.shape else got.numel()
        raise AssertionError(f"{ck.tag}: stage '{st.name}' {what}: {n} of {got.numel()} elements differ from the spec's "
                             f"{tuple(want.shape)} (bit-exact entry)")
    return 0.0


def check_patchify(ck, st, a, inp):
    """Columns [0, Cin*ph*pw) bit-identical to the stand-in's reshape (zero fill past H, W: convpadd); the K padding columns the
    GEMM also reads must be zero."""
    x, out, ph, pw = inp["x"], a["out"], inp["ph"], inp["pw"]
    Cin, Fr, H, W = x.shape
    n, kc = Fr * -(-H // ph) * -(-W // pw), Cin * ph * pw
    if out.shape[0] != n or out.shape[1] < kc:
        raise AssertionError(f"{ck.tag}: stage '{st.name}' operand 'out' is {tuple(out.shape)} for {n} tokens of {kc} columns")
    _exact(ck, st, out[:, :kc], TO.patchify(x, torch.empty(n, kc, dtype=torch.bfloat16, device=x.device), ph, pw))
    return _exact(ck, st, out[:, kc:], torch.zeros_like(out[:, kc:]), "K padding columns")


def check_sin(ck, st, a, inp):
    ref, bound = KE.sinusoidal_ref(inp["t"], inp["dim"])
    _shape(ck, st, "out", a["ret"], ref.shape)
    return _ratio(a["ret"], ref, bound, f"{ck.tag}: stage '{st.name}' output")


def check_lfs(ck, st, a, inp):
    ref, bound = KE.linear_f32_small_ref(inp["x"], inp["w"], inp["bias"], inp["silu_in"])
    _shape(ck, st, "out", a["ret"], ref.shape)
    return _ratio(a["ret"], ref, bound, f"{ck.tag}: stage '{st.name}' output")


def check_bcast(ck, st, a, inp):
    return _exact(ck, st, a["ret"], inp["a"][:, None] + inp["b"][None])


def check_lin32(ck, st, a, inp):
    """linear_f32_ref on every row of a small launch, else on gemm_sample's rows."""
    x, out = inp["x"], a["out"]
    M, N = x.shape[0], inp["w"].shape[0]
    _shape(ck, st, "out", out, (M, N))
    rows = _rows(M, (ck.tag, st.name)).to(x.device)
    ref, bound = KE.linear_f32_ref(x[rows], inp["w"], inp["bias"])
    return _ratio(out[rows], ref, bound, f"{ck.tag}: stage '{st.name}' output")


def check_unpatchify(ck, st, a, inp):
    out, y = a["out"], inp["y"]
    Fr, Hp, Wp, ph, pw = (inp[p] for p in ("F", "Hp", "Wp", "ph", "pw"))
    _shape(ck, st, "out", out, (y.shape[1] // (ph * pw), Fr, Hp * ph, Wp * pw))
    return _exact(ck, st, out, TO.unpatchify(y, torch.empty(out.shape, device=y.device), Fr, Hp, Wp, ph, pw))


def _att_rows(Lq, H, key):
    return [torch.arange(Lq)] * H if Lq <= FULL_ROWS else KP.attention_sample(Lq, H, key)


def check_att(ck, st, a, inp):
    """attention_bound_prod per head on all query rows of a small launch, else attention_sample's; accumulate adds the bf16
    rounding of the result and of the sum (test_gpu_kernel_contract.test_attention_split_and_accumulate)."""
    q, k, v, H = inp["q"], inp["k"], inp["v"], inp["heads"]
    Lq, Lk = q.shape[0], k.shape[0]
    acc = inp["accumulate"]
    ns = ck.att_plan(Lq, Lk, H, 2 if acc else 0)
    nkv = -(-Lk // 128)
    scale = 1 / math.sqrt(D)
    worst = 0.0
    for h, rows in enumerate(_att_rows(Lq, H, (ck.tag, st.name))):
        sl = slice(h * D, (h + 1) * D)
        kh, vh = k[:, sl].double(), v[:, sl].double()
        rows = rows.to(q.device)
        for c0 in range(0, len(rows), 1024):
            rc = rows[c0:c0 + 1024]
            ref, bound = KP.attention_bound_prod(q[rc, sl].double(), kh, vh, scale, nkv, ns)
            if acc:
                fill = inp["out"][rc, sl].double()
                bound = bound + KC.U16 * ref.abs() + KC.U16 * (ref + fill).abs()
                ref = ref + fill
            worst = max(worst, _ratio(a["out"][rc, sl], ref, bound, f"{ck.tag}: stage '{st.name}' output head {h}"))
    return worst


def check_att8(ck, st, a, inp):
    H = inp["heads"]
    Lq, Lk = inp["q8"].shape[0], inp["k8"].shape[0]
    qd = dequantize_act(inp["q8"], inp["qk_scale"][:H])
    kd = dequantize_act(inp["k8"], inp["qk_scale"][H:])
    vd = dequantize_vt(inp["vt8"], inp["v_scale"], Lk)
    ns = ck.att_plan(Lq, Lk, H, 0)
    nkv = -(-Lk // 128)
    worst = 0.0
    for h, rows in enumerate(_att_rows(Lq, H, (ck.tag, st.name))):
        sl = slice(h * D, (h + 1) * D)
        kh, vh = kd[:, sl].double(), vd[:, sl].double()
        rows = rows.to(qd.device)
        for c0 in range(0, len(rows), 1024):
            rc = rows[c0:c0 + 1024]
            ref, bound = KA.attention_fp8_bound(qd[rc, sl].double(), kh, vh, 1 / math.sqrt(D), nkv, ns)
            worst = max(worst, _ratio(a["out"][rc, sl], ref, bound, f"{ck.tag}: stage '{st.name}' output head {h}"))
    return worst


# ------------------------------------------------------------------------------------------------------------
# the spec
# ------------------------------------------------------------------------------------------------------------
@dataclass
class Geometry:
    """What the spec needs to know about one block run, all of it derived outside dit.py."""
    variant: str
    precision: str
    C: int
    H: int
    k_len: int                      # rows that are self-attention keys
    rope: torch.Tensor              # (cos, sin) f32 [R, 64, 2] of the rotated rows (rope_rows of grid_freqs)
    tok: Optional[torch.Tensor]     # int32 [L]: the modulation row of every token, or None (one row for all)
    kv_col: int = 0                 # position of the block among the blocks of the cross K|V GEMM
    layout: Optional["Layout"] = None   # the whole forward (None: a seam, whose context and modulation rows the caller hands in)


@dataclass
class Segment:
    """One patch-embedded piece of the token sequence: frames [f0, f1) of the input, the embedder and its patch, whether
    patch_embedding_2x_f runs first, and the token grid (f, h, w) it yields at rows [row0, row0 + f*h*w)."""
    f0: int
    f1: int
    name: str
    patch: int
    pre_2x_f: bool
    crop: bool                      # plain Conv3d (patch_embedding): odd H / W lose their last row / column; else convpadd
    grid: tuple
    row0: int

    @property
    def n(self):
        return math.prod(self.grid)


@dataclass
class Layout:
    """The reference's token layout of one forward (from WanOracle._segments, convpadd shapes and grid_freqs) and its inputs on
    the device."""
    x: torch.Tensor                 # f32 [in_dim, F, H, W] (y concatenated on 14B)
    segs: List[Segment]
    L: int                          # rows of the residual stream (seq_len on the grid path)
    n_real: int                     # rows the embedders write; the rest are zero padding tokens
    L_hist: int                     # history tokens in front of the new frames' grid
    grid: tuple                     # token grid of the new frames
    t_rows: List[float]             # the timestep of each table row, in row order
    context: torch.Tensor           # [S, text_dim] as the caller passed it
    clip: Optional[torch.Tensor]    # [257, clip_dim] (14B)
    layers: int = 0

    @property
    def t_chunks(self):
        return [min(T_CHUNK, len(self.t_rows) - s) for s in range(0, len(self.t_rows), T_CHUNK)]


def _w(sd, names, dev):
    return torch.cat([sd[n] for n in names], dim=0).to(device=dev, dtype=torch.bfloat16).contiguous()


def _b(sd, names, dev):
    return torch.cat([sd[n] for n in names], dim=0).to(device=dev, dtype=torch.float32).contiguous()


class Weights:
    """Block weights rebuilt from the reference's state-dict keys: bf16, or the (e4m3, s_w) pair of oracle.fp8.quantize_weight."""

    def __init__(self, sd, precision, dev):
        self.sd, self.fp8, self.dev = sd, precision != "bf16", dev

    def lin(self, i, names):
        ws = [f"blocks.{i}.{n}.weight" for n in names]
        label = "|".join(ws)
        if not self.fp8:
            return T(f"bf16 {label}", _w(self.sd, ws, self.dev)), None
        q, s = quantize_weight(torch.cat([self.sd[n] for n in ws], 0).to(self.dev))
        return T(f"e4m3 {label}", q), T(f"s_w of {label}", s.contiguous())

    def bias(self, i, names):
        return T(f"blocks.{i}.{'|'.join(names)} bias", _b(self.sd, [f"blocks.{i}.{n}.bias" for n in names], self.dev))

    def vec(self, i, name):
        return T(f"blocks.{i}.{name}", self.sd[f"blocks.{i}.{name}"].to(device=self.dev, dtype=torch.float32).reshape(-1))

    def kv(self, ids, img):
        k, v = ("k_img", "v_img") if img else ("k", "v")
        names = [f"blocks.{i}.cross_attn.{p}" for i in ids for p in (k, v)]
        return (T(f"bf16 cross {k}|{v} weights of blocks {list(ids)}", _w(self.sd, [n + ".weight" for n in names], self.dev)),
                T(f"cross {k}|{v} biases of blocks {list(ids)}", _b(self.sd, [n + ".bias" for n in names], self.dev)))


def _tok(geo):
    return T("token index", geo.tok) if geo.tok is not None else NONE


def _gemm_stage(name, geo, a, w, bias, epi, out_src=None, gate=None, tok=False):
    """A block linear: bf16 gemm, or gemm_fp8 on an (e4m3, scales) input `a` = (values Src, scales Src)."""
    ins = dict(bias=bias, epilogue=V(epi), gate=gate if gate is not None else NONE, tok_idx=_tok(geo) if tok else NONE)
    if out_src is not None:
        ins["out"] = out_src
    if geo.precision != "bf16":
        ins.update(a=a[0], a_scale=a[1], w=w[0], w_scale=w[1])
        outs = {"": lambda x: x["out"]}
        if epi == EPI["GELU_FP8"]:
            outs = {"q": lambda x: x["out"], "s": lambda x: x["out_scale"][:, :x["a"].shape[0]]}
        else:
            ins["out_scale"] = NONE
        return Stage(name, "gemm_fp8", ins, outs, check_gemm8)
    ins.update(a=a, w=w[0], n_split=V(0), a_split=V(0), shape=NONE, res=NONE)
    return Stage(name, "gemm", ins, {"": lambda x: x["out"]}, check_gemm)


def _norm_stage(name, geo, x, scale=None, shift=None, w=None, b=None):
    ins = dict(x=x, scale=scale or NONE, shift=shift or NONE, tok_idx=_tok(geo) if scale is not None else NONE,
               weight=w or NONE, bias=b or NONE, eps=V(EPS))
    if geo.precision == "bf16":
        return Stage(name, "ln_modulate", ins, {"": lambda a: a["out"]}, check_ln)
    return Stage(name, "ln_modulate_fp8", ins, {"q": lambda a: a["out"], "s": lambda a: a["out_scale"][:, :a["x"].shape[0]]},
                 check_ln8)


def _act(stage, geo):
    """How a linear reads stage `stage`'s output: the bf16 rows, or its (e4m3, scales) pair."""
    if geo.precision == "bf16":
        return S(stage)
    return (S(stage, "q"), S(stage, "s", kind="scale"))


def _quant_stage(name, x):
    return Stage(name, "quant_rows_fp8", dict(x=x), {"q": lambda a: a["out"], "s": lambda a: a["out_scale"][:, :a["x"].shape[0]]},
                 check_q8)


def _table(lay, kind, j, i=None):
    """Row j of the block-i modulation table (kind 'mod', [U, 6, C] rows) or of the head table (kind 'head', [U, 2, C]): the
    time phase's bcast_add outputs of every 16-row chunk, concatenated along the timestep rows."""
    names = [f"time[{c}].{kind}" for c in range(len(lay.t_chunks))]

    def get(ck):
        parts = []
        for n, u in zip(names, lay.t_chunks):
            t = ck.snap[n][""]
            parts.append(t.view(lay.layers, u, 6, -1)[i] if kind == "mod" else t.view(u, 2, -1))
        return torch.cat(parts, 0)[:, j]
    return Src(f"{kind} table row {j}" + (f" of block {i}" if i is not None else "") + f" ({'|'.join(names)})", get, "tensor",
               tuple(names))


def _mod(j, geo=None, i=None):
    names = ("shift_a", "scale_a", "gate_a", "shift_f", "scale_f", "gate_f")
    if geo is not None and geo.layout is not None:
        return _table(geo.layout, "mod", j, i)
    return E(f"modulation row {j} ({names[j]})", "mod", lambda m: m[:, j])


X_IN = E("the block's input rows", "x_in")


def self_attention_stages(geo, wt, i, a_in, out_src, epi, gate=None, tok=False):
    """q|k|v projection of `a_in`, RMSNorm(q), RMSNorm(k), RoPE, attention over the first k_len rows, o projection
    (model.py:178-207)."""
    C, H, kl = geo.C, geo.H, geo.k_len
    qkv = ["self_attn.q", "self_attn.k", "self_attn.v"]
    st = [_gemm_stage("qkv", geo, a_in, wt.lin(i, qkv), wt.bias(i, qkv), EPI["BF16"])]
    st.append(Stage("qk_rope", "qk_norm_rope",
                    dict(q=S("qkv", cols=(0, C)), k=S("qkv", cols=(C, 2 * C)), wq=wt.vec(i, "self_attn.norm_q.weight"),
                         wk=wt.vec(i, "self_attn.norm_k.weight"), rope=T("RoPE rows of grid_freqs", geo.rope, "rope"),
                         rope_len=V(geo.rope.shape[0]), head_dim=V(D), eps=V(EPS), pieces=NONE),
                    {"q": lambda a: a["q"], "k": lambda a: a["k"]}, check_rr))
    if geo.precision == "fp8_attn":
        st.append(_quant_stage("qk_q8", CAT(S("qk_rope", "q"), S("qk_rope", "k"))))
        st.append(Stage("v_t8", "quant_vt_fp8", dict(v=S("qkv", rows=kl, cols=(2 * C, 3 * C)), heads=V(H)),
                        {"vt": lambda a: a["vt8"], "s": lambda a: a["v_scale"]}, check_vt8))
        st.append(Stage("self_att", "attention_fp8",
                        dict(q8=S("qk_q8", "q", cols=(0, C)), k8=S("qk_q8", "q", rows=kl, cols=(C, 2 * C)),
                             qk_scale=S("qk_q8", "s", kind="scale"), vt8=S("v_t8", "vt"), v_scale=S("v_t8", "s"), heads=V(H),
                             scale=NONE, split=V(0)),
                        {"": lambda a: a["out"]}, check_att8))
    else:
        st.append(Stage("self_att", "attention",
                        dict(q=S("qk_rope", "q"), k=S("qk_rope", "k", rows=kl), v=S("qkv", rows=kl, cols=(2 * C, 3 * C)),
                             heads=V(H), scale=NONE, variant=V(0), accumulate=V(False), split=V(0)),
                        {"": lambda a: a["out"]}, check_att))
    att = "self_att"
    if geo.precision != "bf16":
        st.append(_quant_stage("att_q8", S("self_att")))
        att = "att_q8"
    st.append(_gemm_stage("o", geo, _act(att, geo), wt.lin(i, ["self_attn.o"]), wt.bias(i, ["self_attn.o"]), epi,
                          out_src=out_src, gate=gate, tok=tok))
    return st


def block_stages(geo, wt, i):
    """WanAttentionBlock.forward of block i (5B model.py:272-316, 14B wan/modules/model.py:444-496): x += o(attn(norm1)) * gate_a;
    x += cross(norm3(x)); x += ffn(norm2(x)) * gate_f."""
    C, H = geo.C, geo.H
    kc = geo.kv_col * 2 * C
    st = [_norm_stage("norm1", geo, X_IN, _mod(1, geo, i), _mod(0, geo, i))]
    st += self_attention_stages(geo, wt, i, _act("norm1", geo), X_IN, EPI["GATE_RES"], gate=_mod(2, geo, i), tok=True)
    st.append(_norm_stage("norm3", geo, S("o"), w=wt.vec(i, "norm3.weight"), b=wt.vec(i, "norm3.bias")))
    st.append(_gemm_stage("cross_q", geo, _act("norm3", geo), wt.lin(i, ["cross_attn.q"]), wt.bias(i, ["cross_attn.q"]),
                          EPI["BF16"]))
    st.append(Stage("cross_q_norm", "rmsnorm_rope", dict(qk=S("cross_q"), weight=wt.vec(i, "cross_attn.norm_q.weight"),
                                                           rope=NONE, head_dim=V(D), eps=V(EPS), pieces=NONE),
                    {"": lambda a: a["qk"]}, check_rr))
    st.append(Stage("cross_att", "attention",
                    dict(q=S("cross_q_norm"), k=S(f"k_norm[{i}]"), v=S("ckv", cols=(kc + C, kc + 2 * C)), heads=V(H),
                         scale=NONE, variant=V(0), accumulate=V(False), split=V(0)),
                    {"": lambda a: a["out"]}, check_att))
    att = "cross_att"
    if geo.variant == "14b":              # o = text attention + image attention (wan/modules/model.py:380-388)
        st.append(Stage("img_att", "attention",
                        dict(q=S("cross_q_norm"), k=S(f"k_img_norm[{i}]"), v=S("ckv_img", cols=(kc + C, kc + 2 * C)),
                             out=S("cross_att"), heads=V(H), scale=NONE, variant=V(0), accumulate=V(True), split=V(0)),
                        {"": lambda a: a["out"]}, check_att))
        att = "img_att"
    if geo.precision != "bf16":
        st.append(_quant_stage("cross_q8", S(att)))
        att = "cross_q8"
    st.append(_gemm_stage("cross_o", geo, _act(att, geo), wt.lin(i, ["cross_attn.o"]), wt.bias(i, ["cross_attn.o"]),
                          EPI["GATE_RES"], out_src=S("o")))
    st.append(_norm_stage("norm2", geo, S("cross_o"), _mod(4, geo, i), _mod(3, geo, i)))
    st.append(_gemm_stage("ffn0", geo, _act("norm2", geo), wt.lin(i, ["ffn.0"]), wt.bias(i, ["ffn.0"]),
                          EPI["GELU"] if geo.precision == "bf16" else EPI["GELU_FP8"]))
    st.append(_gemm_stage("ffn2", geo, _act("ffn0", geo), wt.lin(i, ["ffn.2"]), wt.bias(i, ["ffn.2"]), EPI["GATE_RES"],
                          out_src=S("cross_o"), gate=_mod(5, geo, i), tok=True))
    return st


def cross_kv_stages(geo, wt, ids):
    """K | V of the embedded context for blocks `ids` as one GEMM over their weights (+ the image rows for 14B), then RMSNorm on
    each block's K half in place (model.py:223-224, wan/modules/model.py:377-378); V stays the GEMM's columns."""
    C = geo.C
    n_img = 257 if geo.variant == "14b" else 0
    g = dict(epilogue=V(EPI["BF16"]), gate=NONE, tok_idx=NONE, n_split=V(0), a_split=V(0), shape=NONE, res=NONE)
    w, b = wt.kv(ids, False)
    fwd = geo.layout is not None          # the context phase's outputs, else the context the seam's caller hands in
    txt = S("text2") if fwd else E("context text rows", "ctx", lambda c: c[n_img:])
    st = [Stage("ckv", "gemm", dict(a=txt, w=w, bias=b, **g), {"": lambda a: a["out"]}, check_gemm)]
    if n_img:
        w, b = wt.kv(ids, True)
        img = S("img_ln4") if fwd else E("context image rows", "ctx", lambda c: c[:n_img])
        st.append(Stage("ckv_img", "gemm", dict(a=img, w=w, bias=b, **g), {"": lambda a: a["out"]}, check_gemm))
    for j, i in enumerate(ids):
        cols = (j * 2 * C, j * 2 * C + C)
        rr = dict(rope=NONE, head_dim=V(D), eps=V(EPS), pieces=NONE)
        st.append(Stage(f"k_norm[{i}]", "rmsnorm_rope", dict(qk=S("ckv", cols=cols), weight=wt.vec(i, "cross_attn.norm_k.weight"),
                                                               **rr), {"": lambda a: a["qk"]}, check_rr))
        if n_img:
            st.append(Stage(f"k_img_norm[{i}]", "rmsnorm_rope",
                            dict(qk=S("ckv_img", cols=cols), weight=wt.vec(i, "cross_attn.norm_k_img.weight"), **rr),
                            {"": lambda a: a["qk"]}, check_rr))
    return st


def _gemm16(name, a, w, bias, epi):
    """A bf16 GEMM outside the block (embedders, text and image MLPs): no gate, no split layout."""
    ins = dict(a=a, w=w, bias=bias, epilogue=V(epi), gate=NONE, tok_idx=NONE, n_split=V(0), a_split=V(0), shape=NONE, res=NONE)
    return Stage(name, "gemm", ins, {"": lambda x: x["out"]}, check_gemm)


def _sd16(sd, name, dev, pad_k=1, pad_n=1):
    """Weight `name` [N, ...] flattened to [N, K] bf16, K zero-padded to a multiple of pad_k (the 16-byte row pitch TMA needs)
    and N to a multiple of pad_n; its bias f32, zero-padded alike."""
    w = sd[name + ".weight"].flatten(1).to(device=dev, dtype=torch.bfloat16)
    b = sd[name + ".bias"].to(device=dev, dtype=torch.float32)
    N, K = w.shape
    Np, Kp = -(-N // pad_n) * pad_n, -(-K // pad_k) * pad_k
    wp = torch.zeros(Np, Kp, dtype=torch.bfloat16, device=dev)
    wp[:N, :K] = w
    bp = torch.zeros(Np, dtype=torch.float32, device=dev)
    bp[:N] = b
    lab = f"{name}" + (f" (K padded to {Kp})" if Kp != K else "") + (f" (N padded to {Np})" if Np != N else "")
    return T(f"bf16 {lab}.weight", wp), T(f"{lab}.bias", bp)


def _sd32(sd, name, dev, shape=None):
    t = sd[name].to(device=dev, dtype=torch.float32)
    return T(name, (t.reshape(shape) if shape else t).contiguous())


def _patchify_stage(name, x, patch):
    return Stage(name, "patchify", dict(x=x, ph=V(patch), pw=V(patch)), {"": lambda a: a["out"]}, check_patchify)


def embed_stages(lay, sd, dev):
    """One patchify + GEMM (EPI_F32 into the segment's rows of the stream) per segment in token order (model.py:599-729); the
    deepest FramePack level runs patchify(4x4) + the patch_embedding_2x_f GEMM (N = in_dim padded to 32) in front, and its
    embedder reads that GEMM's output as [in_dim, f, ceil(H/4), ceil(W/4)]. The grid path is one segment."""
    cin = lay.x.shape[0]
    st = []
    for k, sg in enumerate(lay.segs):
        fr = f"frames [{sg.f0}:{sg.f1}]"
        if sg.pre_2x_f:
            H, W = lay.x.shape[2:]
            h2, w2, f = -(-H // 4), -(-W // 4), sg.f1 - sg.f0
            st.append(_patchify_stage(f"embed[{k}].2x_f.patchify",
                                      Src(f"x[:, {sg.f0}:{sg.f1}]", lambda ck, sg=sg: lay.x[:, sg.f0:sg.f1]), 4))
            st.append(_gemm16(f"embed[{k}].2x_f", S(f"embed[{k}].2x_f.patchify"),
                              *_sd16(sd, "patch_embedding_2x_f", dev, 8, 32), EPI["F32"]))
            x = S(f"embed[{k}].2x_f", fn=lambda t, f=f, h2=h2, w2=w2: t[:, :cin].t().reshape(cin, f, h2, w2),
                  what=f"[:, :{cin}] as [{cin}, {f}, {h2}, {w2}]")
        else:
            hh, ww = (sg.grid[1] * sg.patch, sg.grid[2] * sg.patch) if sg.crop else lay.x.shape[2:]
            x = Src(f"x[:, {sg.f0}:{sg.f1}, :{hh}, :{ww}]", lambda ck, sg=sg, hh=hh, ww=ww: lay.x[:, sg.f0:sg.f1, :hh, :ww])
        st.append(_patchify_stage(f"embed[{k}].patchify", x, sg.patch))
        st.append(_gemm16(f"embed[{k}]", S(f"embed[{k}].patchify"), *_sd16(sd, sg.name, dev, 8), EPI["F32"]))
    return st


def time_stages(lay, sd, dev, C):
    """Per chunk of at most 16 table rows (model.py:805-812, 296, 344): sinusoid(t) -> time_embedding.0 -> SiLU ->
    time_embedding.2 = e -> SiLU -> time_projection.1 = e0; block table = blocks.*.modulation + e0, head table = e +
    head.modulation."""
    mods = T("blocks.*.modulation [layers, 6C]", torch.stack([sd[f"blocks.{i}.modulation"].reshape(-1) for i in range(lay.layers)])
             .to(device=dev, dtype=torch.float32).contiguous())
    st = []
    for c, s0 in enumerate(range(0, len(lay.t_rows), T_CHUNK)):
        rows = lay.t_rows[s0:s0 + T_CHUNK]
        p = f"time[{c}]"
        lin = lambda name, x, w, silu: Stage(  # noqa: E731
            name, "linear_f32_small", dict(x=x, w=_sd32(sd, w + ".weight", dev), bias=_sd32(sd, w + ".bias", dev), silu_in=V(silu)),
            {"": lambda a: a["ret"]}, check_lfs)
        st.append(Stage(f"{p}.sinusoidal", "sinusoidal",
                        dict(t=T(f"timesteps {rows}", torch.tensor(rows, dtype=torch.float32, device=dev)), dim=V(sd[
                            "time_embedding.0.weight"].shape[1])), {"": lambda a: a["ret"]}, check_sin))
        st.append(lin(f"{p}.emb0", S(f"{p}.sinusoidal"), "time_embedding.0", False))
        st.append(lin(f"{p}.emb2", S(f"{p}.emb0"), "time_embedding.2", True))
        st.append(lin(f"{p}.proj", S(f"{p}.emb2"), "time_projection.1", True))
        st.append(Stage(f"{p}.mod", "bcast_add", dict(a=mods, b=S(f"{p}.proj")), {"": lambda a: a["ret"]}, check_bcast))
        st.append(Stage(f"{p}.head", "bcast_add", dict(a=S(f"{p}.emb2"), b=_sd32(sd, "head.modulation", dev, (2, C))),
                        {"": lambda a: a["ret"]}, check_bcast))
    return st


def context_stages(lay, sd, dev, variant, text_len):
    """text_embedding on the context zero-padded to text_len rows: Linear, GELU(tanh), Linear (model.py:815-821); on 14B the
    MLPProj of the CLIP features: LayerNorm (eps 1e-5), Linear, GELU(erf), Linear, LayerNorm (wan/modules/model.py:529-541)."""
    ctx = lay.context.to(device=dev, dtype=torch.bfloat16)
    pad = torch.cat([ctx, ctx.new_zeros(text_len - ctx.shape[0], ctx.shape[1])])
    st = [_gemm16("text0", T(f"context ({ctx.shape[0]} rows) zero-padded to {text_len} rows", pad),
                  *_sd16(sd, "text_embedding.0", dev), EPI["GELU"]),
          _gemm16("text2", S("text0"), *_sd16(sd, "text_embedding.2", dev), EPI["BF16"])]
    if variant == "14b":
        def ln(name, x, key):
            return Stage(name, "ln_modulate", dict(x=x, scale=NONE, shift=NONE, tok_idx=NONE, weight=_sd32(sd, key + ".weight", dev),
                                                   bias=_sd32(sd, key + ".bias", dev), eps=V(IMG_EPS)),
                         {"": lambda a: a["out"]}, check_ln)
        st.append(ln("img_ln0", T("clip_fea rows (f32)", lay.clip.to(device=dev, dtype=torch.float32).contiguous()),
                     "img_emb.proj.0"))
        st.append(_gemm16("img_fc1", S("img_ln0"), *_sd16(sd, "img_emb.proj.1", dev), EPI["GELU_ERF"]))
        st.append(_gemm16("img_fc3", S("img_fc1"), *_sd16(sd, "img_emb.proj.3", dev), EPI["F32"]))
        st.append(ln("img_ln4", S("img_fc3"), "img_emb.proj.4"))
    return st


def head_stages(geo, sd, dev):
    """Head.forward (model.py:336-348; wan/modules/model.py:516-526): LayerNorm * (1 + head row 1) + head row 0 of every token's
    timestep (built from e, not e0), head.head into f32, then unpatchify of rows [L_hist:] over the new frames' grid
    (model.py:867-890). The input is the last block's final GATE_RES output."""
    lay = geo.layout
    f, h, w = lay.grid
    return [Stage("head_ln", "ln_modulate", dict(x=S("ffn2"), scale=_table(lay, "head", 1), shift=_table(lay, "head", 0),
                                                 tok_idx=_tok(geo), weight=NONE, bias=NONE, eps=V(EPS)),
                  {"": lambda a: a["out"]}, check_ln),
            Stage("head_lin", "linear_f32", dict(x=S("head_ln"), w=_sd32(sd, "head.head.weight", dev),
                                                 bias=_sd32(sd, "head.head.bias", dev)), {"": lambda a: a["out"]}, check_lin32),
            Stage("unpatchify", "unpatchify", dict(y=S("head_lin", rows=(lay.L_hist, None)), F=V(f), Hp=V(h), Wp=V(w), ph=V(2),
                                                   pw=V(2)), {}, check_unpatchify)]


# ------------------------------------------------------------------------------------------------------------
# running a cell
# ------------------------------------------------------------------------------------------------------------
def rope_rows(freqs):
    """(cos, sin) f32 [R, 64, 2] of the reference's complex per-token multipliers [R, 1, 64]."""
    return torch.view_as_real(freqs.reshape(freqs.shape[0], -1).to(torch.complex128)).float().contiguous()


def install(mp, dit_module, eng, sd, geo, i, tag, kv_ids, seam="block", att_plan=None, target_call=None):
    """A checker for one seam call: block_forward (seam 'block': the one-block cross K|V launches of kv_ids, then block i) or
    self_attention_forward. The caller hands in ck.env's 'x_in', 'ctx' and 'mod'."""
    ck = Checker(dit_module.ops, tag, att_plan)
    dev = geo.rope.device
    wt = Weights(sd, geo.precision, dev)
    if seam == "self_attention":
        fp8 = geo.precision != "bf16"
        stages = [_quant_stage("in_q8", X_IN)] if fp8 else []
        ck.add_phase("self_attention", stages + self_attention_stages(geo, wt, i, _act("in_q8", geo) if fp8 else X_IN, None,
                                                                      EPI["BF16"]))
    else:
        ck.add_phase("cross_kv", cross_kv_stages(geo, wt, kv_ids))
        ck.add_phase("block", block_stages(geo, wt, i))
    mp.setattr(dit_module, "ops", ck.proxy)
    real_kv, real_body, real_sa = eng._cross_kv, eng._block_body, eng.self_attention_forward
    calls = {"body": 0}

    def cross_kv(*a, **k):
        with ck.region("cross_kv"):
            return real_kv(*a, **k)

    def body(j, xs, *a, **k):
        n = calls["body"]
        calls["body"] += 1
        if n != (i if target_call is None else target_call):
            return real_body(j, xs, *a, **k)
        with ck.region("block"):
            return real_body(j, xs, *a, **k)

    def self_attention(*a, **k):
        with ck.region("self_attention"):
            return real_sa(*a, **k)
    if seam == "self_attention":
        mp.setattr(eng, "self_attention_forward", self_attention)
    else:
        mp.setattr(eng, "_cross_kv", cross_kv)
        mp.setattr(eng, "_block_body", body)
    return ck


PHASES = ("embed", "time", "context", "cross_kv", "block", "head")


def check_stream(ck, lay, xs, tok):
    """The residual stream and the token index the first block receives: rows [row0, row0 + n) of every segment equal to that
    segment's embed GEMM output, the rows past n_real exact zeros; tok_idx the geometry's (every token -> its timestep's row)."""
    what = "block 0 input"
    if tuple(xs.shape) != (lay.L, xs.shape[1]):
        raise AssertionError(f"{ck.tag}: stage '{what}' operand 'xs' has {xs.shape[0]} rows, the spec's stream {lay.L}")
    for k, sg in enumerate(lay.segs):
        _same(ck.tag, what, "xs", xs[sg.row0:sg.row0 + sg.n], ck.snap[f"embed[{k}]"][""],
              Src(f"embed[{k}] (the {sg.name} GEMM) at rows [{sg.row0}:{sg.row0 + sg.n}]", None))
    _same(ck.tag, what, "xs", xs[lay.n_real:], torch.zeros_like(xs[lay.n_real:]),
          Src(f"zero padding tokens at rows [{lay.n_real}:{lay.L}]", None))
    _same(ck.tag, what, "tok_idx", tok, ck.geo.tok, T("each token's timestep row", ck.geo.tok) if ck.geo.tok is not None else NONE)
    ck.unpin()


def install_forward(mp, dit_module, eng, sd, geo, i, tag, att_plan=None):
    """Put a checker for the whole forward between `eng` and its ops module: every launch from the token stream to unpatchify
    is the spec's, except those of the blocks other than i (which pass through; block i must be the last, so that the head
    reads its output). The phases open as the engine reaches them: embed at _token_stream, time at the first _time_tables,
    context at _context, cross_kv around _cross_kv, block around the i-th _block_body, head after the last; the forward must
    have entered all six in that order."""
    lay = geo.layout
    assert i == lay.layers - 1, "the head reads the checked block's output: check the last block"
    ck = Checker(dit_module.ops, tag, att_plan)
    ck.geo = geo
    dev = geo.rope.device
    wt = Weights(sd, geo.precision, dev)
    ck.add_phase("embed", embed_stages(lay, sd, dev))
    ck.add_phase("time", time_stages(lay, sd, dev, geo.C))
    ck.add_phase("context", context_stages(lay, sd, dev, geo.variant, eng.text_len))
    ck.add_phase("cross_kv", cross_kv_stages(geo, wt, list(range(lay.layers))))
    ck.add_phase("block", block_stages(geo, wt, i))
    ck.add_phase("head", head_stages(geo, sd, dev))
    ck.pinned = {f"embed[{k}]" for k in range(len(lay.segs))}
    mp.setattr(dit_module, "ops", ck.proxy)
    real = {n: getattr(eng, n) for n in ("_token_stream", "_time_tables", "_context", "_cross_kv", "_block_body",
                                         "_forward_eager")}
    calls = {"body": 0}

    def token_stream(*a, **k):
        out = real["_token_stream"](*a, **k)
        ck.enter("embed")
        return out

    def tables(*a, **k):
        if ck.phase != "time":
            ck.enter("time")
        return real["_time_tables"](*a, **k)

    def context(*a, **k):
        ck.enter("context")
        return real["_context"](*a, **k)

    def cross_kv(*a, **k):
        ck.enter("cross_kv")
        out = real["_cross_kv"](*a, **k)
        ck.leave()
        return out

    def body(j, xs, m, tok, *a, **k):
        n = calls["body"]
        calls["body"] += 1
        if n == 0:
            ck.leave()
            check_stream(ck, lay, xs, tok)
        if n == i:
            ck.env["x_in"] = ck.stream.clone() if n else xs.clone()
            with ck.region("block"):
                out = real["_block_body"](j, xs, m, tok, *a, **k)
        else:
            out = real["_block_body"](j, xs, m, tok, *a, **k)
        if n == lay.layers - 1:
            ck.enter("head")
        return out

    def forward(*a, **k):
        out = real["_forward_eager"](*a, **k)
        ck.leave()
        if tuple(ck.entered) != PHASES:
            raise AssertionError(f"{ck.tag}: the forward ran the phases {ck.entered}, the spec's are {list(PHASES)}")
        return out
    for n, f in (("_token_stream", token_stream), ("_time_tables", tables), ("_context", context), ("_cross_kv", cross_kv),
                 ("_block_body", body), ("_forward_eager", forward)):
        mp.setattr(eng, n, f)
    return ck


# ------------------------------------------------------------------------------------------------------------
# paths: the inputs of one forward and the geometry the spec derives from them (oracle.wan_dit, not dit.py)
# ------------------------------------------------------------------------------------------------------------
def path_inputs(cfg, path, frames, H, W, lfz=None, pad=0, seed=0, ctx_len=24, t=None):
    """Forward arguments of a path: '5b_grid' (scalar t, seq_len = L_grid + pad: padding rows are keys on the 5B tree; `t` a
    per-frame list gives a per-token t over seq_len = L_grid), '5b_framepack' (history t[0], new frames t[-1]), '14b_framepack'
    (image branch), '14b_grid_padded' (seq_len = L_grid + pad: padding rows are not keys)."""
    inp = synth.make_inputs(cfg, seed, frames, H, W, ctx_len)
    packed = "framepack" in path
    L_grid = frames * (H // 2) * (W // 2)
    if t is not None:
        assert not packed and pad == 0 and len(t) == frames
        tt = torch.tensor(t, dtype=torch.float32).repeat_interleave(L_grid // frames)
    else:
        tt = torch.tensor([700.0]) if not (packed and cfg["variant"] == "5b") else torch.tensor([0.0, 900.0])
    args = dict(x=inp["x"], t=tt, context=inp["context"], seq_len=L_grid + pad, packed=packed, latent_frame_zero=lfz)
    if cfg["variant"] == "14b":
        args.update(y=inp["y"], clip_fea=inp["clip_fea"])
    return args


def warm_inputs(cfg, path, frames, H, W, lfz=None, pad=0, seed=0, t=None):
    """What an earlier forward on the same engine leaves in the reused workspaces: a prompt of text_len rows and, on a padded
    grid, the largest grid that fits the same seq_len (so the padding rows of the checked run hold non-zero tokens)."""
    if "framepack" in path or pad == 0:
        return path_inputs(cfg, path, frames, H, W, lfz, pad, seed + 1, ctx_len=cfg["text_len"], t=t)
    seq_len = frames * (H // 2) * (W // 2) + pad
    best = max(((f * h * w, f, h, w) for f in range(1, 2 * frames + 1) for h in range(H // 2, H + 1)
                for w in range(W // 2, W + 1) if f * h * w <= seq_len), key=lambda c: c[0])
    _, f, h, w = best
    args = path_inputs(cfg, path, f, 2 * h, 2 * w, lfz, 0, seed + 1, ctx_len=cfg["text_len"])
    args["seq_len"] = seq_len
    return args


def path_geometry(cfg, sd, precision, args, dev, layers=None):
    """Geometry of a forward from the reference's own token layout (WanOracle._segments, the convpadd and plain-Conv3d shapes,
    grid_freqs): the segments and their rows, k_len, RoPE rows, timestep rows and each token's row."""
    orc = WanOracle(sd, **synth.oracle_kwargs(cfg))
    x = args["x"] if args.get("y") is None else torch.cat([args["x"], args["y"]], 0)
    five = cfg["variant"] == "5b"
    _, Ft, Hh, Ww = x.shape
    segs, freqs, row = [], [], 0

    def add(f0, f1, name, pre, padm, fz):
        nonlocal row
        p = sd[name + ".weight"].shape[-1]
        h, w = (-(-Hh // 4), -(-Ww // 4)) if pre else (Hh, Ww)
        g = (f1 - f0, -(-h // p), -(-w // p)) if padm else (f1 - f0, h // p, w // p)
        segs.append(Segment(f0, f1, name, p, pre, not padm, g, row))
        freqs.append(grid_freqs(orc.tables, *g, fz))
        row += segs[-1].n
        return fz + g[0]
    if args["packed"]:
        lfz = args["latent_frame_zero"] or (8 if five else 9)
        hist = Ft - lfz
        fz = 0
        for sl, name, padm, pre in orc._segments(hist, Ft - (lfz if five else 9)):
            fr = range(hist)[sl]
            fz = add(fr.start, fr.stop, name, pre, padm, fz)
        L_hist = row
        add(hist, Ft, "patch_embedding", False, 0, fz)
        L = n_real = k_len = row
    else:
        add(0, Ft, "patch_embedding", False, 0, 0)
        L_hist, n_real, L = 0, row, args["seq_len"]
        k_len = L if five else n_real
    t = args["t"].flatten().float()
    tok = None
    if not five:
        t_rows = [float(t[0])]
    elif args["packed"]:
        t_rows = [float(t[0]), float(t[-1])]
        tok = torch.cat([torch.zeros(L_hist), torch.ones(L - L_hist)]).to(torch.int32)
    elif t.numel() == 1:
        t_rows = [float(t[0])]
    else:
        vals = sorted(set(t.tolist()))
        t_rows = vals
        tok = torch.searchsorted(torch.tensor(vals, dtype=torch.float32), t).to(torch.int32)
    clip = args.get("clip_fea")
    lay = Layout(x.float().to(dev), segs, L, n_real, L_hist, segs[-1].grid, t_rows, args["context"],
                 None if clip is None else clip.reshape(-1, clip.shape[-1]), layers or cfg["num_layers"])
    geo = Geometry(cfg["variant"], precision, cfg["dim"], cfg["num_heads"], k_len, rope_rows(torch.cat(freqs)).to(dev),
                   None if tok is None else tok.to(dev), layout=lay)
    return geo


def engine_forward(eng, args):
    return eng.forward(args["x"], args["t"], args["context"], args["seq_len"], y=args.get("y"), clip_fea=args.get("clip_fea"),
                       latent_frame_zero=args["latent_frame_zero"], packed=args["packed"])


def oracle_forward(orc, cfg, args):
    kw = dict(seq_len=args["seq_len"], latent_frame_zero=args["latent_frame_zero"])
    if cfg["variant"] == "5b":
        t = args["t"] if args["packed"] or args["t"].numel() == 1 else args["t"].view(1, -1)   # per-token t: [B, seq_len]
        return orc.forward([args["x"]], t, [args["context"]], flag=args["packed"], **kw)
    return orc.forward([args["x"]], args["t"], [args["context"]], y=[args["y"]], clip_fea=args["clip_fea"],
                       rand_num_img=0.5 if args["packed"] else 0.1, **kw)


def run_path(mp, dit_module, eng, sd, cfg, precision, args, i, tag, att_plan=None, warm=None):
    """The engine's forward checked launch by launch with block i (the last) in full; `warm`: the arguments of an unchecked
    forward run first on the same engine, whose leftovers the checked run must not read. Returns the checker."""
    if warm is not None:
        engine_forward(eng, warm)
    geo = path_geometry(cfg, sd, precision, args, eng.device, eng.layers)
    geo.kv_col = i
    ck = install_forward(mp, dit_module, eng, sd, geo, i, tag, att_plan=att_plan)
    engine_forward(eng, args)
    return ck


def run_block_seam(mp, dit_module, eng, sd, cfg, precision, i, L, tag, att_plan=None, seed=3):
    """block_forward(i) on the packed-freqs path (per-token e on the 5B tree, one e row on the 14B tree), with its one-block
    cross K|V launches checked."""
    dev = eng.device
    C = cfg["dim"]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(L, C, generator=g)
    e = 0.5 * torch.randn(L, 6, C, generator=g) if cfg["variant"] == "5b" else 0.5 * torch.randn(6, C, generator=g)
    ctx = torch.randn(cfg["text_len"] + (257 if cfg["variant"] == "14b" else 0), C, generator=g)
    hw = L // 2
    freqs = grid_freqs(WanOracle(sd, **synth.oracle_kwargs(cfg)).tables, 2, 1, hw, f0=3)
    geo = Geometry(cfg["variant"], precision, C, cfg["num_heads"], L, rope_rows(freqs).to(dev),
                   torch.arange(L, dtype=torch.int32, device=dev) if cfg["variant"] == "5b" else None, kv_col=0)
    ck = install(mp, dit_module, eng, sd, geo, i, tag, [i], att_plan=att_plan, target_call=0)
    ck.env.update(x_in=x.to(dev), ctx=ctx.to(device=dev, dtype=torch.bfloat16),
                  mod=(sd[f"blocks.{i}.modulation"].reshape(1, 6 * C) + e.reshape(-1, 6 * C)).view(-1, 6, C).to(dev))
    eng.block_forward(i, x, e, None, ctx, freqs=freqs, packed=True)
    return ck


def run_self_attention_seam(mp, dit_module, eng, sd, cfg, precision, i, L, tag, att_plan=None, seed=4):
    dev = eng.device
    C = cfg["dim"]
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(L, C, generator=g).to(torch.bfloat16)
    freqs = grid_freqs(WanOracle(sd, **synth.oracle_kwargs(cfg)).tables, 2, 1, L // 2, f0=5)
    geo = Geometry(cfg["variant"], precision, C, cfg["num_heads"], L, rope_rows(freqs).to(dev), None)
    ck = install(mp, dit_module, eng, sd, geo, i, tag, None, seam="self_attention", att_plan=att_plan)
    ck.env["x_in"] = h.to(dev)
    eng.self_attention_forward(i, h, None, freqs, True)
    return ck
