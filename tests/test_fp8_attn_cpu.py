"""precision="fp8_attn" without a GPU: the V quantiser twin against the numerics contract (include/yume_b200_fp8_attn.h), the
engine's fp8_attn host logic over the torch stand-ins (tests/helpers/torch_ops_fp8_attn.py) against the fp8-attention oracle, the
public switches and rejections, the entry-point guard of the new header, and the GPU contract's attention bound against a
tile-by-tile model of the kernel and realistic defects."""
import contextlib
import math
from pathlib import Path

import pytest
import torch

import test_gpu_kernel_contract_fp8_attn as KA
from helpers import torch_ops_fp8_attn
from oracle import synth
from oracle.fp8 import quantize_act
from oracle.fp8_attn import VT_PERM, WanOracleFp8Attn, dequantize_vt, quantize_vt, vt_pi
from test_fp8_cpu import CASES, _forward, _mirror_kwargs, _oracle, _truncate
from test_kernel_contract_cpu import _entry_problems
from yume_b200 import dit
from yume_b200._lib import YumeB200Error

HEADER = Path(__file__).resolve().parents[1] / "include" / "yume_b200_fp8_attn.h"
E4M3 = torch.float8_e4m3fn


# ------------------------------------------------------------------------------------------------------------
# the V quantiser twin
# ------------------------------------------------------------------------------------------------------------
def test_key_permutation_is_a_bijection_within_each_32_key_block():
    assert sorted(vt_pi(f) for f in range(32)) == list(range(32))
    assert VT_PERM.tolist() == [vt_pi(f) for f in range(32)]
    # thread t = lane % 4 of the A fragment holds positions 4t..4t+3 and 16+4t..16+4t+3; its accumulator holds keys
    # 8g + 2t + {0, 1}: the positions of every thread map onto its own accumulator columns
    for t in range(4):
        mine = {8 * g + 2 * t + e for g in range(4) for e in range(2)}
        assert {vt_pi(f) for f in [*range(4 * t, 4 * t + 4), *range(16 + 4 * t, 16 + 4 * t + 4)]} == mine


def test_vt_twin_layout_scales_and_partial_tile():
    g = torch.Generator().manual_seed(0)
    Lk, H = 300, 2
    v = torch.randn(Lk, H * 128, generator=g).to(torch.bfloat16).float()
    vt8, sv = quantize_vt(v, H)
    assert vt8.shape == (H, 128, 384) and vt8.dtype == E4M3 and sv.shape == (H, 3)
    for h in range(H):
        for j in range(3):
            blk = v[j * 128:min(Lk, j * 128 + 128), h * 128:(h + 1) * 128]
            assert sv[h, j] == blk.abs().max() / torch.tensor(448.0)
    # vt8[h, d, 32 b + f] = q(V[32 b + pi(f), h 128 + d])
    key = 32 * 5 + vt_pi(13)
    want = (v[key, 128 + 7] * (torch.tensor(448.0) / (sv[1, key // 128] * 448))).clamp(-448, 448)
    assert abs(float(vt8[1, 7, 32 * 5 + 13].float()) - float(want)) <= abs(float(want)) * 2 ** -4 + 1e-6
    assert (vt8[:, :, 320:].float() == 0).all(), "keys >= Lk are stored as zeros"
    back = dequantize_vt(vt8, sv, Lk)
    sc = sv.repeat_interleave(128, dim=1)[:, :Lk].t().repeat_interleave(128, dim=1)
    assert ((back - v).abs() <= torch.maximum(v.abs() * 2 ** -4, sc * 2 ** -10) * (1 + 1e-6)).all()


def test_vt_twin_zero_tiny_and_nan_blocks():
    g = torch.Generator().manual_seed(1)
    v = torch.randn(384, 256, generator=g)
    v[:128, :128] = 0.0                               # zero block
    v[128:256, :128] = 1e-38                          # 448 / amax overflows: zeros with scale 0
    v[300, 200] = float("nan")                        # NaN stays NaN and takes no part in the block maximum
    vt8, sv = quantize_vt(v, 2)
    assert sv[0, 0] == 0 and sv[0, 1] == 0 and (vt8[0, :, :256].float() == 0).all()
    blk = v[256:384, 128:256].clone()
    blk[300 - 256, 200 - 128] = 0.0
    assert sv[1, 2] == blk.abs().max() / torch.tensor(448.0)
    nan = torch.isnan(vt8.float())
    assert int(nan.sum()) == 1 and bool(nan[1, 200 - 128].any())


# ------------------------------------------------------------------------------------------------------------
# the engine's fp8_attn host logic
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def cpu_engine(monkeypatch):
    monkeypatch.setattr(dit, "ops", torch_ops_fp8_attn)
    monkeypatch.setattr(torch.cuda, "device", lambda *_a, **_k: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)

    def make(cfg, sd, precision="fp8_attn"):
        kw = synth.oracle_kwargs(cfg)
        variant = kw.pop("variant")
        return dit.WanDiT(sd, variant, device="cpu", precision=precision, **kw)
    return make


# measured worst over CASES: engine over the stand-ins vs the fp8-attention oracle 1.64e-2 (the fp8 engine's 1.54e-2 plus the
# bf16 roundings of q|k|v and the attention output, which move e4m3 roundings); vs the reference's bf16 forward 2.7e-2
QDQ_BAR = 3e-2
REF_BAR = 5e-2
# one self-attention of 128 tokens alone (the seam test): measured 3.30e-2. With q, k and v all in e4m3, a last-bit difference
# between the engine's and the oracle's bf16 q|k|v moves whole e4m3 steps, and no later layer averages them out
SEAM_BAR = 5e-2


@pytest.mark.parametrize("fname,case", CASES)
def test_fp8_attn_host_logic_matches_the_oracle(cpu_engine, golden_dir, fname, case):
    g = torch.load(golden_dir / fname, weights_only=False)
    cfg, c = g["cfg"], g["cases"][case]
    sd = synth.make_state_dict(cfg, g["seed_w"])
    inp = synth.make_inputs(cfg, c["seed"], c["frames"], c["H"], c["W"], c["ctx_len"])
    eng = cpu_engine(cfg, sd)
    got = _forward(eng, cfg, c, inp)
    want = _oracle(WanOracleFp8Attn(sd, **synth.oracle_kwargs(cfg)), cfg, c, inp)
    rel = float((got - want).norm() / want.norm())
    ref = float((got - c["out"]).norm() / c["out"].norm())
    print(f"{fname}:{case}: vs fp8-attention oracle {rel:.2e}, vs reference bf16 forward {ref:.2e}")
    assert rel < QDQ_BAR
    assert ref < REF_BAR


def test_fp8_attn_rejections(cpu_engine):
    sd = synth.make_state_dict(synth.CFG_5B_TINY, 0)
    with pytest.raises(YumeB200Error, match="divisible by 128"):
        cpu_engine(dict(synth.CFG_5B_TINY, ffn_dim=500), sd)
    with pytest.raises(YumeB200Error, match="divisible by 128"):
        cpu_engine(dict(synth.CFG_5B_TINY, dim=200), sd)
    cfg = dict(synth.CFG_5B_TINY, dim=1536, num_heads=12)
    with pytest.raises(YumeB200Error, match="fp8 LayerNorm"):
        cpu_engine(cfg, synth.make_state_dict(cfg, 0))
    eng = cpu_engine(synth.CFG_5B_TINY, sd)
    with pytest.raises(YumeB200Error, match="sequence parallel"):
        eng.enable_sequence_parallel(None)


def test_public_switches_and_the_self_attention_seam(cpu_engine, golden_dir):
    """install(model, precision="fp8_attn") through both of its paths, the mirrors' .install(precision=), and the
    WanSelfAttention seam against the fp8-attention oracle's self-attention."""
    import yume_b200
    from oracle.wan_dit import grid_freqs
    from yume_b200.model import WanModel5B, install
    g = torch.load(golden_dir / "wan23_tiny.pt", weights_only=False)
    cfg = g["cfg"]
    sd = synth.make_state_dict(cfg, g["seed_w"])

    def fp8_attn(m):
        eng = m._yb_engine
        return eng.precision == "fp8_attn" and all(b[k][0].dtype == E4M3 for b in eng.blocks for k in dit.FP8_WEIGHTS)
    with torch.device("meta"):
        mirror = WanModel5B(model_type="ti2v", **_mirror_kwargs(cfg))
    m = mirror.install("cpu", state_dict=sd, precision="fp8_attn")
    assert fp8_attn(m)
    loaded = WanModel5B(model_type="ti2v", **_mirror_kwargs(cfg))
    loaded.load_state_dict({k: v for k, v in sd.items() if k in loaded.state_dict()})
    assert fp8_attn(install(loaded, device="cpu", precision="fp8_attn"))

    calls = []
    real = torch_ops_fp8_attn.attention_fp8

    def spy(*a, **k):
        calls.append(a[0].shape)
        return real(*a, **k)
    m = yume_b200.install_seams(m)
    orc = WanOracleFp8Attn(sd, **synth.oracle_kwargs(cfg))
    gen = torch.Generator().manual_seed(5)
    L, C = 2 * 8 * 8, cfg["dim"]
    h = torch.randn(1, L, C, generator=gen).to(torch.bfloat16).float()
    fr = grid_freqs(orc.tables, 2, 8, 8, f0=3)
    want = orc.self_attn("blocks.0.self_attn", h, fr)[0]
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(torch_ops_fp8_attn, "attention_fp8", spy)
        got = m.blocks[0].self_attn(h, torch.tensor([L]), None, fr, None, None, None, True)[0]
    assert calls, "the self-attention seam did not run the fp8 attention"
    rel = float((got.float() - want).norm() / want.norm())
    print(f"fp8_attn self-attention seam vs fp8-attention oracle {rel:.2e}")
    assert got.dtype == torch.bfloat16 and rel < SEAM_BAR


# ------------------------------------------------------------------------------------------------------------
# C-ABI guards over include/yume_b200_fp8_attn.h
# ------------------------------------------------------------------------------------------------------------
def test_fp8_attn_header_symbols_are_bound():
    import re
    from yume_b200 import _lib
    declared = set(re.findall(r"^\s*(?:int|long long)\s+(yb_\w+)\s*\(", HEADER.read_text(), flags=re.M))
    assert declared == set(_lib.FP8_ATTN_SIGNATURES) == {"yb_quant_vt_fp8", "yb_attention_fp8"}
    others = (set(_lib.SIGNATURES) | set(_lib.CLIP_SIGNATURES) | set(_lib.T5_SIGNATURES) | set(_lib.STREAM_SIGNATURES)
              | set(_lib.FP8_SIGNATURES))
    assert not declared & others


def test_every_fp8_attn_entry_point_has_a_contract_test():
    assert _entry_problems(HEADER, modules=(KA,)) == []


def test_fp8_attn_entry_point_guard_notices_a_missing_test(monkeypatch):
    covers = dict(KA.COVERS)
    del covers["yb_quant_vt_fp8"]
    monkeypatch.setattr(KA, "COVERS", covers)
    assert _entry_problems(HEADER, modules=(KA,)) == ["entry point without a contract test: yb_quant_vt_fp8"]


# ------------------------------------------------------------------------------------------------------------
# the GPU contract's attention bound against a tile-by-tile model of the kernel
# ------------------------------------------------------------------------------------------------------------
LOG2E = 1.4426950408889634
R, LK = 16, 145 * 128 - 37          # 16 query rows over the 5B-like 145 KV tiles, the last one partial


def _bound_operands(same_v_scale=False):
    """q, k, v of one head (q doubled so that the softmax is not flat). same_v_scale: a flat softmax over positive V whose
    128-key tiles all have the same amax, so that one V scale is valid for every tile and the whole sum can live in one
    accumulator (the no-promotion defect; a positive sum is where its truncations add up)."""
    g = torch.Generator().manual_seed(11)
    q = torch.randn(R, 128, generator=g) * (0.1 if same_v_scale else 2)
    k = torch.randn(LK, 128, generator=g)
    k[LK - 1] = q[0] * 2                               # the last valid key dominates row 0 (an off-by-one mask must show)
    v = torch.randn(LK, 128, generator=g)
    if same_v_scale:
        v = v.abs().clamp(max=3.5)
        v[::128, 0] = 4.0
    k_other = torch.randn(LK, 128, generator=g) * 3    # a neighbouring head's keys, for its k scales
    q8, sq = quantize_act(q.to(torch.bfloat16).float())
    kk = torch.cat([k, k_other], dim=1).to(torch.bfloat16).float()
    k8, sk = quantize_act(kk)                          # scale rows: this head, the neighbour head
    vt8, sv = quantize_vt(v.to(torch.bfloat16).float(), 1)
    return q8.double(), sq[0].double(), k8[:, :128].double(), sk.double(), vt8, sv[0].double()


def _kernel_model(q8, sq, k8, sk, vt8, sv, scale, defect=None):
    """The kernel per 128-key tile in fp64: S in four k32 steps, each truncated to ACC_BITS; s = S s_k; mask; online softmax in
    the log2 domain; P8 = e4m3(256 p) against the running max; O_tile in four truncated k32 steps over the stored (permuted) key
    order; promotion O = O alpha + O_tile s_v / 256; out = O / l."""
    bits = KA.ACC_BITS
    nkv = -(-LK // 128)
    v_pos = vt8[0].t().double()                        # [Lkp, 128] in stored position order
    perm = torch.arange(nkv * 128).reshape(-1, 32)[:, VT_PERM].flatten()    # position -> key
    if defect == "wrong_permutation":
        perm = torch.arange(nkv * 128)
    k_scale = sk[1] if defect == "neighbour_head_scale" else sk[0]
    rq = sq * scale * LOG2E
    m = torch.full((R,), -math.inf, dtype=torch.float64)
    l = torch.zeros(R, dtype=torch.float64)
    o = torch.zeros(R, 128, dtype=torch.float64)
    k8p = torch.cat([k8, torch.zeros(nkv * 128 - LK, 128, dtype=torch.float64)])
    ks = torch.cat([k_scale, torch.zeros(nkv * 128 - LK, dtype=torch.float64)])
    last = LK - 1 if defect == "mask_off_by_one" else LK   # the defect drops the last valid key
    for j in range(nkv):
        keys = torch.arange(j * 128, j * 128 + 128)
        s = torch.zeros(R, 128, dtype=torch.float64)
        for c in range(0, 128, 32):
            s = _truncate(s + q8[:, c:c + 32] @ k8p[keys, c:c + 32].t(), bits)
        x = s * ks[keys] * rq[:, None]
        x[:, keys >= last] = -math.inf
        mn = torch.maximum(m, x.amax(dim=1))
        al = torch.exp2(m - mn)
        m = mn
        pe = torch.exp2(x - m[:, None])                # p against the running max
        l = l * al + pe.sum(dim=1)
        p8 = (256 * pe).float().to(torch.float8_e4m3fn).double()
        if defect == "no_promotion":                   # O stays in the tensor-core accumulator across tiles
            o = o * al[:, None]
            for c in range(0, 128, 32):
                pos = torch.arange(j * 128 + c, j * 128 + c + 32)
                o = _truncate(o + p8[:, perm[pos] - j * 128] @ v_pos[pos], bits)
            continue
        ot = torch.zeros(R, 128, dtype=torch.float64)
        for c in range(0, 128, 32):
            pos = torch.arange(j * 128 + c, j * 128 + c + 32)
            ot = _truncate(ot + p8[:, perm[pos] - j * 128] @ v_pos[pos], bits)
        f = 1.0 if defect == "no_s_v" else float(sv[j])
        f = f if defect == "no_1_256" else f / 256
        o = o * al[:, None] + ot * f
    if defect == "no_promotion":
        o = o * float(sv[0]) / 256
    return (o / l[:, None]).float().to(torch.bfloat16).double()


@pytest.mark.parametrize("defect", [None, "no_s_v", "no_1_256", "wrong_permutation", "no_promotion", "mask_off_by_one",
                                    "neighbour_head_scale"])
def test_attention_bound_accepts_the_kernel_model_and_rejects_defects(defect):
    q8, sq, k8, sk, vt8, sv = _bound_operands(same_v_scale=defect == "no_promotion")
    scale = 1 / math.sqrt(128.0)
    qd, kd = q8 * sq[:, None], k8 * sk[0][:, None]
    vd = dequantize_vt(vt8, sv[None].float(), LK).double()
    ref, bound = KA.attention_fp8_bound(qd, kd, vd, scale, -(-LK // 128))
    got = _kernel_model(q8, sq, k8, sk, vt8, sv, scale, defect)
    ratio = float(((got - ref).abs() / bound).max())
    print(f"{defect}: worst |err|/bound {ratio:.3f}")
    if defect is None:
        assert ratio <= 1.0
    else:
        assert ratio > 1.0, f"{defect} passes the bound (worst ratio {ratio:.3f})"
