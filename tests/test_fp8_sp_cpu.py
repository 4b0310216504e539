"""The fp8 Ulysses entry points (include/yume_b200_fp8_sp.h) without a GPU: their torch twins (tests/helpers/torch_ops_fp8_sp.py)
against the fp8 contracts they restate, the header's symbols and its entry-point guard, and the engine's public rules for fp8 under
sequence parallelism that need no process group."""
import contextlib
import re
from pathlib import Path

import pytest
import torch

import test_gpu_kernel_contract_fp8_sp as KS
from helpers import torch_ops, torch_ops_fp8_sp
from oracle import synth
from oracle.fp8 import quantize_act
from test_kernel_contract_cpu import _entry_problems
from yume_b200 import dit
from yume_b200._lib import YumeB200Error

HEADER = Path(__file__).resolve().parents[1] / "include" / "yume_b200_fp8_sp.h"
E4M3 = torch.float8_e4m3fn


def _split_buffer(x, P):
    """[Lp, C] -> the exchange buffer [P, Lp, C / P] that holds it K-split."""
    Lp, C = x.shape
    return x.view(Lp, P, C // P).permute(1, 0, 2).contiguous()


@pytest.mark.parametrize("P,Wh", [(2, 512), (4, 256), (8, 128)])
def test_split_quantiser_twin_equals_the_gathered_quantiser(P, Wh):
    g = torch.Generator().manual_seed(P)
    Lp, C = 37, P * Wh
    x = (torch.randn(Lp, C, generator=g) * torch.exp(torch.randn(1, C, generator=g))).to(torch.bfloat16)
    x[0, :128] = 0.0                                   # zero group (scale 0)
    x[1, Wh - 128:Wh] = 1e-38                          # 448 / amax overflows: zeros with scale 0, at a chunk's last group
    x[2, Wh] = float("nan")                            # NaN stays NaN, first column of the second chunk
    x[3, Wh - 1] = 1e4                                 # a group edge: the last column of a chunk sets its group's scale
    att = _split_buffer(x, P)
    q = torch.empty(Lp, C, dtype=E4M3)
    s = torch.full((C // 128, 40), float("nan"))
    torch_ops_fp8_sp.quant_rows_fp8_split(att, q, s, Wh, Lp * Wh, (Lp, C))
    tq, ts = quantize_act(x.float())
    nan = torch.isnan(tq.float())
    assert torch.equal(torch.isnan(q.float()), nan) and int(nan.sum()) == 1
    assert torch.equal(q.view(torch.uint8)[~nan], tq.view(torch.uint8)[~nan])
    assert torch.equal(s[:, :Lp], ts)
    assert float(s[0, 0]) == 0.0 and float(s[(Wh - 128) // 128, 1]) == 0.0
    assert s[(Wh - 1) // 128, 3] == x[3, Wh - 1].float() / torch.tensor(448.0)


def test_gather_reads_the_layout_the_bf16_gemm_reads():
    """gather_split is the a_split layout of the bf16 GEMM's stand-in: the same [M, K] matrix."""
    g = torch.Generator().manual_seed(3)
    P, Lp, Wh = 4, 9, 256
    att = torch.randn(P, Lp, Wh, generator=g).to(torch.bfloat16)
    w = torch.eye(P * Wh).to(torch.bfloat16)
    via_gemm = torch.empty(Lp, P * Wh)
    torch_ops.gemm(att, w, None, via_gemm, torch_ops.YB_EPI_F32, a_split=Wh, a_split_stride=Lp * Wh, shape=(Lp, P * Wh))
    assert torch.equal(torch_ops_fp8_sp.gather_split(att, Wh, Lp * Wh, (Lp, P * Wh)).float(), via_gemm)


def test_pack_twin_writes_the_send_buffer_layout():
    """send[p, t] = q | k | v of owner p's heads, each normalised over ALL C columns (not over the Wh columns it holds), as the
    bf16 path's n_split layout plus qk_norm_rope over the pieces gives it."""
    g = torch.Generator().manual_seed(4)
    P, Lp, C, D = 4, 11, 1024, 128
    Wh = C // P
    qkv = (torch.randn(Lp, 3 * C, generator=g) * 2).to(torch.bfloat16)
    wq, wk = 1 + 0.3 * torch.randn(C, generator=g), 1 + 0.3 * torch.randn(C, generator=g)
    ang = torch.rand(Lp, D // 2, generator=g) * 6.3
    rope = torch.stack([ang.cos(), ang.sin()], dim=-1)
    send = torch.full((P, Lp, 3 * Wh), float("nan")).to(torch.bfloat16)
    torch_ops_fp8_sp.sp_pack_qkv(qkv, wq, wk, rope, Lp - 3, D, 1e-6, send)
    ref = qkv.view(Lp, 3, P, Wh).permute(2, 0, 1, 3).reshape(P, Lp, 3 * Wh).clone()
    torch_ops.qk_norm_rope(ref[0], ref[0][:, Wh:], wq, wk, rope, D, 1e-6, Lp - 3, pieces=(Lp, C, Wh, Lp * 3 * Wh))
    assert torch.equal(send.view(torch.int16), ref.view(torch.int16))
    assert torch.equal(send[1, :, 2 * Wh:], qkv[:, 2 * C + Wh:2 * C + 2 * Wh]), "v is copied, not normalised"
    q0 = qkv[:, :C].float()
    rstd = torch.rsqrt(q0.pow(2).mean(dim=1, keepdim=True) + 1e-6)
    last = (q0[Lp - 1:, Wh:2 * Wh] * rstd[Lp - 1:] * wq[Wh:2 * Wh]).to(torch.bfloat16)   # row >= rope_len: not rotated
    assert torch.equal(send[1, Lp - 1:, :Wh], last)


def test_attention_sp_twin_stores_rows_into_their_owners_slots():
    g = torch.Generator().manual_seed(5)
    P, Lp, H = 3, 40, 2
    W = H * 128
    x = torch.randn(P * Lp, 3 * W, generator=g).to(torch.bfloat16)
    qk8, qk_s = quantize_act(x[:, :2 * W].float())
    from oracle.fp8_attn import quantize_vt
    vt8, v_s = quantize_vt(x[:, 2 * W:].float(), H)
    want = torch.empty(P * Lp, W, dtype=torch.bfloat16)
    torch_ops_fp8_sp.attention_fp8(qk8[:, :W], qk8[:, W:], qk_s, vt8, v_s, want, H)
    rank = 1
    bufs = [torch.full((P, Lp, W), float("nan")).to(torch.bfloat16) for _ in range(P)]
    torch_ops_fp8_sp.attention_fp8_sp(qk8[:, :W], qk8[:, W:], qk_s, vt8, v_s, bufs, W, H, rank, Lp)
    for p in range(P):
        assert torch.equal(bufs[p][rank], want[p * Lp:(p + 1) * Lp])
        assert bool(torch.isnan(bufs[p][[r for r in range(P) if r != rank]].float()).all())


def test_fp8_engine_sequence_parallel_rules(monkeypatch):
    """No process group: the fp8 engine says what is missing (a bf16 engine behaves as it always did). p2p_gemm is refused with its
    reason before any group is consulted; an unknown transport keeps its message."""
    monkeypatch.setattr(dit, "ops", torch_ops_fp8_sp)
    monkeypatch.setattr(torch.cuda, "device", lambda *_a, **_k: contextlib.nullcontext())
    kw = synth.oracle_kwargs(synth.CFG_5B_TINY)
    variant = kw.pop("variant")
    sd = synth.make_state_dict(synth.CFG_5B_TINY, 0)
    for precision in ("fp8", "fp8_attn"):
        eng = dit.WanDiT(sd, variant, device="cpu", precision=precision, **kw)
        with pytest.raises(YumeB200Error, match="sequence parallelism needs an initialised torch.distributed process group"):
            eng.enable_sequence_parallel(None)
        with pytest.raises(YumeB200Error, match="p2p_gemm.*e4m3"):
            eng.enable_sequence_parallel(None, transport="p2p_gemm")
        with pytest.raises(YumeB200Error, match="transport must be"):
            eng.enable_sequence_parallel(None, transport="ring")
        assert eng.sp_world == 1 and eng.sp_group is None


# ------------------------------------------------------------------------------------------------------------
# C-ABI guards over include/yume_b200_fp8_sp.h
# ------------------------------------------------------------------------------------------------------------
def test_fp8_sp_header_symbols_are_bound():
    from yume_b200 import _lib
    declared = set(re.findall(r"^\s*(?:int|long long)\s+(yb_\w+)\s*\(", HEADER.read_text(), flags=re.M))
    assert declared == set(_lib.FP8_SP_SIGNATURES) == {"yb_quant_rows_fp8_split", "yb_attention_fp8_sp", "yb_sp_pack_qkv"}
    others = (set(_lib.SIGNATURES) | set(_lib.CLIP_SIGNATURES) | set(_lib.T5_SIGNATURES) | set(_lib.STREAM_SIGNATURES)
              | set(_lib.FP8_SIGNATURES) | set(_lib.FP8_ATTN_SIGNATURES) | set(_lib.FP8_VAE_SIGNATURES)
              | set(_lib.RESUME_SIGNATURES))
    assert not declared & others


def test_every_fp8_sp_entry_point_has_a_contract_test():
    assert _entry_problems(HEADER, modules=(KS,)) == []


def test_fp8_sp_entry_point_guard_notices_a_missing_test(monkeypatch):
    covers = dict(KS.COVERS)
    del covers["yb_sp_pack_qkv"]
    monkeypatch.setattr(KS, "COVERS", covers)
    assert _entry_problems(HEADER, modules=(KS,)) == ["entry point without a contract test: yb_sp_pack_qkv"]
