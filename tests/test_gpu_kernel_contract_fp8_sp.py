"""Per-element contract of the fp8 Ulysses entry points (include/yume_b200_fp8_sp.h) on one H100, every rank of a P-GPU run
emulated on the one device (as tests/test_gpu_kernel_contract_prod.py does for yb_attention_sp), at the production per-rank shapes:
5B (L = 18 480) and 14B chunk (L = 21 930) at P = 2 / 4 / 8, the 14B grid (L = 42 840) at P = 8, and the k_lens form (seq_len 43 008
over 42 840 keys) at P = 8.

- yb_attention_fp8_sp: the P receive buffers (NaN-poisoned, guard-banded), assembled into global order, are bit-identical to
  yb_attention_fp8 on the same operands; after each emulated rank's launch only that rank's slot of every receiver has been written.
  Rank 0's rows are also held to `attention_fp8_bound` on the sampled rows. Forced KV splits 2 / 3 / 4 run the combine's peer scatter.
- yb_quant_rows_fp8_split: bit-identical to yb_quant_rows_fp8 of the gathered [Lp, C] matrix, with zero, tiny and NaN groups.
- yb_sp_pack_qkv: the send buffer equals, element for element, the one the bf16 NCCL path makes from the same bf16 q|k|v rows (the
  n_split GEMM's peer-major layout, then yb_qk_norm_rope over the pieces)."""
import ctypes as C
import math

import pytest
import torch

gpu = pytest.mark.gpu
E4M3 = torch.float8_e4m3fn

COVERS = {
    "yb_attention_fp8_sp": ["test_attention_fp8_sp_bit_identical_to_attention_fp8", "test_attention_fp8_sp_rejects_bad_arguments"],
    "yb_quant_rows_fp8_split": ["test_quant_rows_fp8_split_bit_identical_to_gathered"],
    "yb_sp_pack_qkv": ["test_sp_pack_qkv_equals_the_bf16_send_buffer"],
}

# (id, model width C, P, Lp, heads per rank, keys): the per-rank shapes of the production geometries
SP_SHAPES = [
    ("5b.sp2", 3072, 2, 9240, 12, 18480), ("5b.sp4", 3072, 4, 4620, 6, 18480), ("5b.sp8", 3072, 8, 2310, 3, 18480),
    ("14b_chunk.sp2", 5120, 2, 10965, 20, 21930), ("14b_chunk.sp4", 5120, 4, 5483, 10, 21930),
    ("14b_chunk.sp8", 5120, 8, 2742, 5, 21930),
    ("14b_grid.sp8", 5120, 8, 5355, 5, 42840),
    ("14b_grid_seq_len_43008.sp8", 5120, 8, 5376, 5, 42840),
]
ATT_ROWS = [dict(id=i, C=c, P=p, Lp=lp, heads=h, Lk=lk, split=0) for i, c, p, lp, h, lk in SP_SHAPES] + \
    [dict(id=f"5b.sp8.split{ns}", C=3072, P=8, Lp=2310, heads=3, Lk=18480, split=ns) for ns in (2, 3, 4)]
QUANT_ROWS = [dict(id=i, C=c, P=p, Lp=lp) for i, c, p, lp, _h, _lk in SP_SHAPES if "seq_len" not in i]
PACK_ROWS = QUANT_ROWS


def _lib():
    import yume_b200
    from yume_b200 import _lib as L
    yume_b200.load()
    return L.load()


@gpu
@pytest.mark.parametrize("rid", [r["id"] for r in ATT_ROWS])
def test_attention_fp8_sp_bit_identical_to_attention_fp8(rid):
    import test_gpu_kernel_contract as KC
    from oracle.fp8 import dequantize_act
    from oracle.fp8_attn import dequantize_vt
    from test_gpu_kernel_contract_fp8_attn import _operands, attention_fp8_bound
    from test_gpu_kernel_contract_prod import Lean, attention_sample
    from yume_b200 import ops
    lib = _lib()
    row = next(r for r in ATT_ROWS if r["id"] == rid)
    P, Lp, H, Lk, split = row["P"], row["Lp"], row["heads"], row["Lk"], row["split"]
    Lq, Wh = P * Lp, H * 128
    scale = 1 / math.sqrt(128.0)
    plan = (C.c_int * 4)()
    assert lib.yb_attention_plan(Lq, Lk, H, torch.cuda.get_device_properties(0).multi_processor_count, (split & 7) << 4, plan) == 0
    if split:
        assert plan[2] == split and plan[1] > 0, f"split {split} was not planned: {tuple(plan)}"
    tag = f"attention_fp8_sp {rid} P{P} Lp{Lp} Lq{Lq} Lk{Lk} h{H} tail{plan[1]} ns{plan[2]}"
    recv = [Lean(P * Lp, Wh, torch.bfloat16) for _ in range(P)]
    ptrs = [b.view.data_ptr() for b in recv]
    for r in range(P):
        buf, qk8, qk_s, vt8, v_s = _operands(Lq, Lk, H, (rid, r))   # rank r's gathered q|k|v of its heads, quantised
        del buf
        want = torch.empty(Lq, Wh, dtype=torch.bfloat16, device="cuda")
        ops.attention_fp8(qk8[:, :Wh], qk8[:Lk, Wh:], qk_s, vt8, v_s, want, H, scale=scale, split=split)
        ops.attention_fp8_sp(qk8[:, :Wh], qk8[:Lk, Wh:], qk_s, vt8, v_s, ptrs, Wh, H, r, Lp, scale=scale, split=split)
        torch.cuda.synchronize()
        for p in range(P):
            slots = recv[p].view.view(P, Lp, Wh)
            got = slots[r]
            assert not bool(torch.isnan(got).any()), f"{tag}: receiver {p} slot {r} not fully written"
            assert torch.equal(got.view(torch.int16), want[p * Lp:(p + 1) * Lp].view(torch.int16)), \
                f"{tag}: receiver {p} slot {r} differs from yb_attention_fp8 rows {p * Lp}..{(p + 1) * Lp}"
            if r + 1 < P:
                assert bool(torch.isnan(slots[r + 1:]).all()), f"{tag}: rank {r} wrote outside its slot of receiver {p}"
        if r == 0:                                                    # the bound, on rank 0's rows
            qd = dequantize_act(qk8[:, :Wh], qk_s[:H])
            kd = dequantize_act(qk8[:Lk, Wh:], qk_s[H:])
            vd = dequantize_vt(vt8, v_s, Lk)
            samples = attention_sample(Lq, H, ("fp8_sp", rid))
            worst = 0.0
            for h in range(H):
                sl = slice(h * 128, (h + 1) * 128)
                r_idx = samples[h].to("cuda")
                for c0 in range(0, len(r_idx), 1024):
                    rc = r_idx[c0:c0 + 1024]
                    ref, bound = attention_fp8_bound(qd[rc, sl].double(), kd[:, sl].double(), vd[:, sl].double(), scale,
                                                     -(-Lk // 128), plan[2])
                    worst = max(worst, float(((want[rc, sl].double() - ref).abs() / bound).max()))
            KC.WORST[f"fp8_sp.{rid}"] = max(KC.WORST.get(f"fp8_sp.{rid}", 0.0), worst)
            print(f"[contract] {tag}: worst |err|/bound {worst:.3f}")
            assert worst <= 1.0, f"{tag}: worst |err|/bound {worst:.3f}"
        del qk8, qk_s, vt8, v_s, want
    for p in range(P):
        recv[p].check(f"{tag} receiver {p}")


@gpu
def test_attention_fp8_sp_rejects_bad_arguments():
    lib = _lib()
    H, P, Lp = 2, 2, 128
    Lq = Lk = P * Lp
    W = H * 128
    q8 = torch.zeros(Lq, W, dtype=E4M3, device="cuda")
    sc = torch.zeros(2 * H, Lq, device="cuda")
    vt8 = torch.zeros(H, 128, Lk, dtype=E4M3, device="cuda")
    vs = torch.zeros(H, Lk // 128, device="cuda")
    bufs = [torch.zeros(Lq, W, dtype=torch.bfloat16, device="cuda") for _ in range(P)]
    s = torch.cuda.current_stream().cuda_stream

    def call(world=P, rank=0, lp=Lp, lq=Lq, lk=Lk, flags=0, ptrs=None):
        ptrs = ptrs if ptrs is not None else [b.data_ptr() for b in bufs]
        arr = (C.c_void_p * len(ptrs))(*ptrs)
        return lib.yb_attention_fp8_sp(q8.data_ptr(), W, q8.data_ptr(), W, sc.data_ptr(), Lq, vt8.data_ptr(), vs.data_ptr(), arr, W,
                                       lq, lk, H, 0.088, world, rank, lp, flags, None, 0, s)
    assert call() == 0
    assert call(world=1, ptrs=[bufs[0].data_ptr()]) == -1       # one rank is not a Ulysses launch
    assert call(rank=2) == -1
    assert call(lq=Lq - 128, lk=Lq - 128) == -1                  # Lq must be world * Lp
    assert call(lk=Lq + 1) == -1                                 # more keys than gathered rows
    assert call(flags=2) == -1                                   # no accumulate form
    assert call(ptrs=[bufs[0].data_ptr(), 0]) == -1              # a missing peer
    assert call(ptrs=[bufs[0].data_ptr(), bufs[1].data_ptr() + 2]) == -3
    torch.cuda.synchronize()


def _special_groups(x):
    """x [Lp, C] bf16: a zero group, a group whose 448 / amax overflows, a NaN element; on chunk edges of the K split."""
    x[0, :128] = 0.0
    x[1, 128:256] = 1e-38
    x[2, 300] = float("nan")
    x[3, -128:] = 0.0
    return x


@gpu
@pytest.mark.parametrize("rid", [r["id"] for r in QUANT_ROWS] + ["edges"])
def test_quant_rows_fp8_split_bit_identical_to_gathered(rid):
    from test_gpu_kernel_contract_prod import _cuda_gen, _rand
    from yume_b200 import ops
    row = dict(C=1024, P=4, Lp=77) if rid == "edges" else next(r for r in QUANT_ROWS if r["id"] == rid)
    Cd, P, Lp = row["C"], row["P"], row["Lp"]
    Wh = Cd // P
    g = _cuda_gen(("fp8_sp.quant", rid))
    att = _rand(g, P * Lp, Wh, 3.0).view(P, Lp, Wh)              # the exchange buffer [P, Lp, Wh]
    att.mul_(torch.exp(torch.randn(P, 1, Wh, device="cuda", generator=g)).to(torch.bfloat16))
    gathered = att.permute(1, 0, 2).reshape(Lp, Cd).contiguous()
    gathered = _special_groups(gathered)
    att.copy_(gathered.view(Lp, P, Wh).permute(1, 0, 2))
    backing = torch.full((Lp + 32, Cd), 0x5A, dtype=torch.uint8, device="cuda")   # 16 guard rows above and below
    backing[16:16 + Lp] = 0x7F                                                     # e4m3 NaN: every element must be written
    q = backing[16:16 + Lp].view(E4M3)
    s = torch.full((Cd // 128, ops.fp8_scale_ld(Lp)), float("nan"), device="cuda")
    ops.quant_rows_fp8_split(att, q, s, Wh, Lp * Wh, (Lp, Cd))
    tq = torch.empty(Lp, Cd, dtype=E4M3, device="cuda")
    ts = torch.full_like(s, float("nan"))
    ops.quant_rows_fp8(gathered, tq, ts)
    torch.cuda.synchronize()
    assert bool((backing[:16] == 0x5A).all()) and bool((backing[16 + Lp:] == 0x5A).all()), f"{rid}: guard rows changed"
    assert torch.equal(q.view(torch.uint8), tq.view(torch.uint8)), \
        f"{rid}: {int((q.view(torch.uint8) != tq.view(torch.uint8)).sum())} bytes differ from the gathered quantiser"
    assert torch.equal(s[:, :Lp], ts[:, :Lp])
    if rid == "edges":
        assert float(s[0, 0]) == 0.0 and float(s[1, 1]) == 0.0 and bool(torch.isnan(q[2, 300].float()))


@gpu
@pytest.mark.parametrize("rid", [r["id"] for r in PACK_ROWS])
def test_sp_pack_qkv_equals_the_bf16_send_buffer(rid):
    from test_gpu_kernel_contract_prod import Lean, _cuda_gen, _rand
    from yume_b200 import ops
    row = next(r for r in PACK_ROWS if r["id"] == rid)
    Cd, P, Lp = row["C"], row["P"], row["Lp"]
    Wh, D, eps = Cd // P, 128, 1e-6
    W3 = 3 * Wh
    g = _cuda_gen(("fp8_sp.pack", rid))
    qkv = _rand(g, Lp, 3 * Cd, 2.0)
    nq, nk = (1 + 0.3 * torch.randn(Cd, device="cuda", generator=g) for _ in range(2))
    ang = torch.rand(Lp, D // 2, device="cuda", generator=g) * 6.3
    rope = torch.stack([ang.cos(), ang.sin()], dim=-1).contiguous()
    rope_len = Lp - 37                                           # the last rows of a padded shard are not rotated
    # the bf16 NCCL path: the n_split GEMM stores column part*C + p*Wh + j of a row at send[p, row, part*Wh + j], then
    # yb_qk_norm_rope normalises q and k over the Wh-column pieces
    ref = torch.empty(P, Lp, W3, dtype=torch.bfloat16, device="cuda")
    ref.copy_(qkv.view(Lp, 3, P, Wh).permute(2, 0, 1, 3).reshape(P, Lp, W3))
    ops.qk_norm_rope(ref[0], ref[0][:, Wh:], nq, nk, rope, D, eps, rope_len, pieces=(Lp, Cd, Wh, Lp * W3))
    send = Lean(P * Lp, W3, torch.bfloat16)
    ops.sp_pack_qkv(qkv, nq, nk, rope, rope_len, D, eps, send.view.view(P, Lp, W3))
    torch.cuda.synchronize()
    send.check(f"sp_pack_qkv {rid}")
    got = send.view.view(P, Lp, W3)
    diff = got.view(torch.int16) != ref.view(torch.int16)
    assert not bool(diff.any()), f"sp_pack_qkv {rid}: {int(diff.sum())} elements differ from the bf16 path, first at " \
        f"{tuple(int(v) for v in diff.nonzero()[0])}"
