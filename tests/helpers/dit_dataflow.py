"""TEST INFRASTRUCTURE: the WanDiT block checked launch by launch.

A SPEC states the dataflow of one Wan block (and of the cross-attention K|V launches in front of it) independently of
yume_b200/dit.py, from the reference's WanAttentionBlock (wan23/modules/model.py:272-316, wan/modules/model.py:444-496, as
oracle/wan_dit.py restates it): an ordered list of stages, each naming its ops entry, where every operand must come from (an
earlier stage's output, a weight rebuilt from the reference's state-dict keys, a modulation row with its token index, RoPE rows
from oracle.wan_dit.grid_freqs, the first k_len rows) and which per-element bound its output must meet.

A CHECKER sits between the engine and its ops module (`dit.ops`). Outside a checked region it only passes launches through;
inside one it takes the next stage for every launch and checks
  order    the entry is the stage's, and the region makes exactly the spec's number of launches;
  inputs   every operand is torch.equal to the source the stage names (view shape, row count, scale table included);
  output   right after the launch, against an fp64 recomputation from those inputs within the kernel's contract bound
           (tests/test_gpu_kernel_contract*.py: gemm_epilogue_ref / gemm_bounds, _ln_ref, _rr_ref, attention_bound_prod,
           the fp8 gemm_bound, attention_fp8_bound; the fp8 quantisers bit-identical to their twins in oracle/fp8*.py).
Only the snapshots a later stage reads are kept, and each is dropped after its last reader, so production L fits. Large
launches are sampled like the production contract (gemm_sample rows and columns, attention_sample rows).

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
import test_gpu_kernel_contract_fp8 as K8
import test_gpu_kernel_contract_fp8_attn as KA
import test_gpu_kernel_contract_prod as KP
from oracle import synth
from oracle.fp8 import dequantize_act, quantize_act, quantize_weight
from oracle.fp8_attn import dequantize_vt, quantize_vt
from oracle.wan_dit import WanOracle, grid_freqs
from yume_b200 import ops as _real_ops

D = 128                       # head_dim of both trees
EPS = 1e-6
ENTRIES = ("gemm", "gemm_fp8", "ln_modulate", "ln_modulate_fp8", "qk_norm_rope", "rmsnorm_rope", "quant_rows_fp8",
           "quant_vt_fp8", "attention", "attention_fp8")
SIGS = {e: inspect.signature(getattr(_real_ops, e)) for e in ENTRIES}
EPI = dict(BF16=0, GELU=1, F32=2, GATE_RES=3, GELU_FP8=8)     # include/yume_b200.h, include/yume_b200_fp8.h
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


def S(stage, part="", rows=None, cols=None, kind="tensor"):
    rs = slice(None) if rows is None else slice(0, rows)
    cs = slice(None) if cols is None else slice(*cols)
    label = f"{stage}{'.' + part if part else ''}" + (f"[:{rows}]" if rows is not None else "") + \
        (f"[:, {cols[0]}:{cols[1]}]" if cols is not None else "")
    return Src(label, lambda ck: ck.snap[stage][part][rs, cs], kind, (stage,))


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
        self.env: Dict[str, torch.Tensor] = {}   # what the run hands the block: x_in, ctx, mod (filled by Cell's wrappers)
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

    @contextlib.contextmanager
    def region(self, phase):
        """Launches inside are the stages of `phase`, exactly as many as it has."""
        rg = self.phases[phase]
        assert self.phase is None, f"{self.tag}: region {phase} opened inside {self.phase}"
        self.phase, self.pos, self.stop = phase, rg.start, rg.stop
        try:
            yield
        finally:
            ended, self.phase = self.pos, None
        if ended != rg.stop:
            raise AssertionError(f"{self.tag}: {phase} made {ended - rg.start} launches, the spec has {len(rg)}: stage "
                                 f"'{self.program[ended].name}' ({self.program[ended].entry}) never ran")

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
        keep = st.name in self.last_read and self.last_read[st.name] > self.pos
        if keep:
            self.snap[st.name] = {part: f(args).clone() for part, f in st.outputs.items()}
        if st.check is not None:
            w = st.check(self, st, args, inp)
            self.worst[st.name] = max(self.worst.get(st.name, 0.0), w)
        del inp
        for name in [n for n in self.snap if self.last_read.get(n, -1) <= self.pos]:
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


def check_ln(ck, st, a, inp):
    x, out, tok = inp["x"], a["out"], inp["tok_idx"]
    L, C = x.shape
    worst = 0.0
    for r0 in range(0, L, 4096):
        rows = torch.arange(r0, min(L, r0 + 4096), device=x.device)
        y, f32 = KC._ln_ref(x[rows], C, EPS, inp["weight"], inp["bias"], _mod_rows(inp["scale"], tok, rows),
                            _mod_rows(inp["shift"], tok, rows))
        worst = max(worst, _ratio(out[rows], y, KC.bf16_out_bound(y, f32), f"{ck.tag}: stage '{st.name}' output"))
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
    rows, cols = _rows(M, (ck.tag, st.name)).to(A.device), _cols(N, (ck.tag, st.name)).to(A.device)
    (accR, FR), (accC, FC) = KP.gemm_ref_rows_cols(A, B, rows, cols)
    out = a["out"]
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


def _mod(j):
    names = ("shift_a", "scale_a", "gate_a", "shift_f", "scale_f", "gate_f")
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
    st = [_norm_stage("norm1", geo, X_IN, _mod(1), _mod(0))]
    st += self_attention_stages(geo, wt, i, _act("norm1", geo), X_IN, EPI["GATE_RES"], gate=_mod(2), tok=True)
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
    st.append(_norm_stage("norm2", geo, S("cross_o"), _mod(4), _mod(3)))
    st.append(_gemm_stage("ffn0", geo, _act("norm2", geo), wt.lin(i, ["ffn.0"]), wt.bias(i, ["ffn.0"]),
                          EPI["GELU"] if geo.precision == "bf16" else EPI["GELU_FP8"]))
    st.append(_gemm_stage("ffn2", geo, _act("ffn0", geo), wt.lin(i, ["ffn.2"]), wt.bias(i, ["ffn.2"]), EPI["GATE_RES"],
                          out_src=S("cross_o"), gate=_mod(5), tok=True))
    return st


def cross_kv_stages(geo, wt, ids):
    """K | V of the embedded context for blocks `ids` as one GEMM over their weights (+ the image rows for 14B), then RMSNorm on
    each block's K half in place (model.py:223-224, wan/modules/model.py:377-378); V stays the GEMM's columns."""
    C = geo.C
    n_img = 257 if geo.variant == "14b" else 0
    g = dict(epilogue=V(EPI["BF16"]), gate=NONE, tok_idx=NONE, n_split=V(0), a_split=V(0), shape=NONE, res=NONE)
    w, b = wt.kv(ids, False)
    st = [Stage("ckv", "gemm", dict(a=E("context text rows", "ctx", lambda c: c[n_img:]), w=w, bias=b, **g),
                {"": lambda a: a["out"]}, check_gemm)]
    if n_img:
        w, b = wt.kv(ids, True)
        st.append(Stage("ckv_img", "gemm", dict(a=E("context image rows", "ctx", lambda c: c[:n_img]), w=w, bias=b, **g),
                        {"": lambda a: a["out"]}, check_gemm))
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


# ------------------------------------------------------------------------------------------------------------
# running a cell
# ------------------------------------------------------------------------------------------------------------
def rope_rows(freqs):
    """(cos, sin) f32 [R, 64, 2] of the reference's complex per-token multipliers [R, 1, 64]."""
    return torch.view_as_real(freqs.reshape(freqs.shape[0], -1).to(torch.complex128)).float().contiguous()


def install(mp, dit_module, eng, sd, geo, i, tag, kv_ids, seam="block", att_plan=None, target_call=None):
    """Put a checker for block i (and the cross K|V launches of blocks kv_ids, unless seam == 'self_attention') between `eng` and
    its ops module. The engine then runs unchanged: _context / _time_tables hand the checker the embedded context and the
    modulation table, _cross_kv is the cross K|V region, the `target_call`-th _block_body call (default: the one for block i)
    the block region. Returns the checker; ck.env takes 'x_in' (and for seams 'ctx', 'mod') from the caller where the engine
    does not produce them."""
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
    real_context, real_tables, real_kv = eng._context, eng._time_tables, eng._cross_kv
    real_body, real_sa = eng._block_body, eng.self_attention_forward
    calls = {"body": 0}

    def context(*a, **k):
        out = real_context(*a, **k)
        ck.env["ctx"] = out.clone()
        return out

    def tables(*a, **k):
        e, mod, head = real_tables(*a, **k)
        ck.env["mod_table"] = mod.clone()
        ck.env["mod"] = ck.env["mod_table"][i]
        return e, mod, head

    def cross_kv(*a, **k):
        with ck.region("cross_kv"):
            return real_kv(*a, **k)

    def body(j, xs, *a, **k):
        n = calls["body"]
        calls["body"] += 1
        if n != (i if target_call is None else target_call):
            return real_body(j, xs, *a, **k)
        if "x_in" not in ck.env:
            ck.env["x_in"] = ck.stream.clone()
        with ck.region("block"):
            return real_body(j, xs, *a, **k)

    def self_attention(*a, **k):
        with ck.region("self_attention"):
            return real_sa(*a, **k)
    mp.setattr(eng, "_context", context)
    mp.setattr(eng, "_time_tables", tables)
    if seam == "self_attention":
        mp.setattr(eng, "self_attention_forward", self_attention)
    else:
        mp.setattr(eng, "_cross_kv", cross_kv)
        mp.setattr(eng, "_block_body", body)
    return ck


def check_modulation_rows(ck, sd, cfg, i, t_rows):
    """Row u of the engine's modulation table for block i is blocks.i.modulation + time_projection(t_rows[u]) (the reference's
    e0, model.py:805-812, recomputed by the oracle): pins which timestep each row stands for, so that a token index pointing at
    a row is a statement about the token's timestep."""
    orc = WanOracle(sd, **synth.oracle_kwargs(cfg))
    _, e0 = orc.time_embed(torch.tensor(t_rows, dtype=torch.float32))
    want = sd[f"blocks.{i}.modulation"].reshape(1, 6, -1).double() + e0.double().view(len(t_rows), 6, -1)
    got = ck.env["mod_table"][i].double().cpu()
    assert got.shape == want.shape, f"{ck.tag}: modulation table rows {tuple(got.shape)}, want {tuple(want.shape)}"
    err = float((got - want).abs().max() / want.abs().max())
    assert err < 1e-3, f"{ck.tag}: modulation row order: rows differ from the timesteps {t_rows} by {err:.2e}"


# ------------------------------------------------------------------------------------------------------------
# paths: the inputs of one forward and the geometry the spec derives from them (oracle.wan_dit, not dit.py)
# ------------------------------------------------------------------------------------------------------------
def path_inputs(cfg, path, frames, H, W, lfz=None, pad=0, seed=0):
    """Forward arguments of a path: '5b_grid' (scalar t, seq_len = L_grid + pad: padding rows are keys on the 5B tree),
    '5b_framepack' (history t[0], new frames t[-1]), '14b_framepack' (image branch), '14b_grid_padded' (seq_len = L_grid + pad:
    padding rows are not keys)."""
    inp = synth.make_inputs(cfg, seed, frames, H, W, 24)
    packed = "framepack" in path
    L_grid = frames * (H // 2) * (W // 2)
    args = dict(x=inp["x"], t=torch.tensor([700.0]) if not (packed and cfg["variant"] == "5b") else torch.tensor([0.0, 900.0]),
                context=inp["context"], seq_len=L_grid + pad, packed=packed, latent_frame_zero=lfz)
    if cfg["variant"] == "14b":
        args.update(y=inp["y"], clip_fea=inp["clip_fea"])
    return args


def path_geometry(cfg, sd, precision, args, dev):
    """Geometry of a forward from the oracle's own token layout: k_len, RoPE rows, token index, modulation timesteps."""
    orc = WanOracle(sd, **synth.oracle_kwargs(cfg))
    x = args["x"] if args.get("y") is None else torch.cat([args["x"], args["y"]], 0)
    five = cfg["variant"] == "5b"
    if args["packed"]:
        lfz = args["latent_frame_zero"] or (8 if five else 9)
        tok, freqs, n_hist, _ = orc.pack(x.float(), lfz)
        L, k_len = tok.shape[1], tok.shape[1]
        tok_idx = torch.cat([torch.zeros(n_hist), torch.ones(L - n_hist)]).to(torch.int32) if five else None
        t_rows = [float(args["t"][0]), float(args["t"][-1])] if five else [float(args["t"][0])]
    else:
        f, h, w = x.shape[1], x.shape[2] // 2, x.shape[3] // 2
        freqs = grid_freqs(orc.tables, f, h, w)
        L = args["seq_len"]
        k_len = L if five else f * h * w
        tok_idx, t_rows = None, [float(args["t"][0])]
    geo = Geometry(cfg["variant"], precision, cfg["dim"], cfg["num_heads"], k_len, rope_rows(freqs).to(dev),
                   None if tok_idx is None else tok_idx.to(dev))
    return geo, L, t_rows


def engine_forward(eng, args):
    return eng.forward(args["x"], args["t"], args["context"], args["seq_len"], y=args.get("y"), clip_fea=args.get("clip_fea"),
                       latent_frame_zero=args["latent_frame_zero"], packed=args["packed"])


def oracle_forward(orc, cfg, args):
    kw = dict(seq_len=args["seq_len"], latent_frame_zero=args["latent_frame_zero"])
    if cfg["variant"] == "5b":
        return orc.forward([args["x"]], args["t"], [args["context"]], flag=args["packed"], **kw)
    return orc.forward([args["x"]], args["t"], [args["context"]], y=[args["y"]], clip_fea=args["clip_fea"],
                       rand_num_img=0.5 if args["packed"] else 0.1, **kw)


def run_path(mp, dit_module, eng, sd, cfg, precision, args, i, tag, att_plan=None):
    """The engine's forward with block i and the all-layer cross K|V launches checked. Returns the checker."""
    dev = eng.device
    geo, L, t_rows = path_geometry(cfg, sd, precision, args, dev)
    geo.kv_col = i
    ck = install(mp, dit_module, eng, sd, geo, i, tag, list(range(eng.layers)), att_plan=att_plan)
    engine_forward(eng, args)
    check_modulation_rows(ck, sd, cfg, i, t_rows)
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
