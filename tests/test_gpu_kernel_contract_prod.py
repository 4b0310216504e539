"""Per-element kernel contract at production shapes (`-m gpu`): the GEMM, attention and conv launches the engines make, at the
sizes they make them, so that the kernels' cross-tile control flow runs as it does in production — a persistent GEMM CTA walking
~13 tiles (5B) to ~45 (14B grid) through the group-N raster with the TMA / mbarrier ring phase carried from tile to tile, the
all-layer cross K|V GEMM's raster of hundreds of N tiles on 4 M tiles, attention's K/V ring wrapping ~60 times over 145 to 335
KV tiles with one online-softmax rescale per tile, the automatic tail split of the 5B and 14B-chunk self-attention, and the
conv's 4-D TMA boxes over full-size VAE frames.

PROD_TABLE holds one row per distinct launch (entry, shape, epilogue, flags, the configuration it comes from);
test_table_covers_the_engines_launches runs the engines with recording wrappers around yume_b200.ops and fails on a launch
without a row. tests/test_kernel_contract_cpu.py checks on the CPU that every row is multi-wave (>= 3 tiles per CTA; >= 100 KV
tiles for self-attention) unless it exists for its raster shape, that 5B and 14B self-attention rows take the tail split, and
that the sample sets below hit every output tile, conv box and (head, unit) of each row's plan.

Same rules as tests/test_gpu_kernel_contract.py, whose machinery this file imports, with one deliberate gap: the fp64 reference
is SAMPLED. Coverage of every element comes from the poison check (the output starts as NaN, or for in-place GATE_RES the same
operands run once more under the F32 epilogue into a NaN buffer, and afterwards every element must be finite; the guard rows /
columns around it must keep their bits), and coverage of every tile from the sample rule:
  GEMM       for every 128-row band 2 full rows (one seeded, plus the band's last valid row), for every 64-column band 2 full
             columns (likewise): every tile of any block_n and of the 256-row SM-pair tiles holds sampled elements;
  conv       2 output voxels of every (TT, TH, TW) box of the launch's plan (one seeded, plus the box's last valid voxel), all
             Cout columns;
  attention  4 query rows of every 128-row query tile of every (head, 256-row unit) (3 seeded, plus the tile's last valid
             row), plus every row of one seeded unit per head, against all keys.
Operands are drawn on the device from a CUDA generator seeded with the stable hash of the row id (the same data in every run on
the same software); weights are scaled 1/sqrt(K) like production. u16 = 2^-8, u32 = 2^-24.
"""
import math
import time
import zlib

import pytest
import torch
import torch.nn.functional as F

import test_gpu_kernel_contract as KC
from test_gpu_kernel_contract import U16, U32, assert_within, bf16_out_bound

pytestmark = pytest.mark.gpu

SMS = 132                    # SMs of an H100 SXM: the planners' argument in the CPU guards
EPI = dict(BF16=0, GELU=1, F32=2, GATE_RES=3, GELU_ERF=4, RES_BF16=5)     # include/yume_b200.h

# ------------------------------------------------------------------------------------------------------------
# the production-shape table
# ------------------------------------------------------------------------------------------------------------
# DiT configurations: (name, C, heads, F, layers, Lq, Lk of self-attention, gate flags of the gated GATE_RES launches)
DIT_CFGS = {
    "5b": dict(C=3072, heads=24, F=14336, layers=30, L=18480, Lk=18480, gated=("gate", "tok_idx"), img=False),
    "14b_chunk": dict(C=5120, heads=40, F=13824, layers=40, L=21930, Lk=21930, gated=("gate",), img=True),
    # the 81-frame regular grid (latent [16, 21, 68, 120]): seq_len = L_grid = 21 x 34 x 60, every row a key
    "14b_grid": dict(C=5120, heads=40, F=13824, layers=40, L=42840, Lk=42840, gated=("gate",), img=True),
}
TEXT_LEN, N_IMG = 512, 257


def _dit_rows():
    rows = []
    for cfg, d in DIT_CFGS.items():
        C, L, H = d["C"], d["L"], d["heads"]
        g = frozenset(d["gated"])

        def gemm(name, M, N, K, epi, flags=frozenset(), layers=1, raster=False):
            rows.append(dict(id=f"{cfg}.{name}", entry="gemm", cfg=cfg, M=M, N=N, K=K, epi=EPI[epi], flags=frozenset(flags),
                             layers=layers, raster=raster))
        gemm("qkv", L, 3 * C, C, "BF16")
        gemm("o", L, C, C, "GATE_RES", g)
        gemm("cross_q", L, C, C, "BF16", {"out_window"})          # q2 = qkv[:, :C]: ldo = 3C
        gemm("cross_o", L, C, C, "GATE_RES")
        gemm("ffn0", L, d["F"], C, "GELU")
        gemm("ffn2", L, C, d["F"], "GATE_RES", g)
        # one GEMM per forward for every block's K|V (N = layers * 2C); recorded per layer from a one-layer engine
        gemm("cross_kv_all", TEXT_LEN, d["layers"] * 2 * C, C, "BF16", layers=d["layers"], raster=True)
        if d["img"]:
            gemm("img_kv_all", N_IMG, d["layers"] * 2 * C, C, "BF16", layers=d["layers"], raster=True)

        def att(name, Lq, Lk, acc=False, self_attn=False):
            rows.append(dict(id=f"{cfg}.{name}", entry="attention", cfg=cfg, Lq=Lq, Lk=Lk, heads=H, accumulate=acc,
                             self_attn=self_attn))
        att("self_attention", L, d["Lk"], self_attn=True)
        att("text_attention", L, TEXT_LEN)
        if d["img"]:
            att("img_attention", L, N_IMG, acc=True)
    # a caller passing seq_len > L_grid (the k_lens form: the padded rows are queries but not keys). Not the default shape
    # (the engine's callers pass seq_len = L_grid); kept for its partial last KV tile under full query units
    rows.append(dict(id="14b_grid_seq_len_43008.self_attention", entry="attention", cfg="14b_grid_seq_len_43008", Lq=43008,
                     Lk=42840, heads=40, accumulate=False, self_attn=True))
    return rows


# Ulysses per-rank launches, all P ranks emulated on one GPU (5B: 24 heads; Lp = 18480 / P)
SP_ROWS = [
    dict(id="5b.sp8.attention_sp", entry="attention_sp", cfg="5b", P=8, Lp=2310, heads=3, self_attn=True),
    dict(id="5b.sp4.attention_sp", entry="attention_sp", cfg="5b", P=4, Lp=4620, heads=6, self_attn=True),
    dict(id="5b.sp8.gemm_sp_qkv", entry="gemm_sp_qkv", cfg="5b", P=8, Lp=2310, C=3072, K=3072),
]

# VAE conv launches: (T, H, W) input extents, Cp input channels (padded), Cout, taps, oob_zero_pad (Wan) or replicate-padded
# input (hyvideo), out_t_mul (time_conv's frame interleave), stride_t / stride_hw (the encoders' Resample convs), epilogue.
# Decodes at production spatial size with a short frame count (frames only scale M; full spatial size is where the box
# decomposition changes).
def _conv(cfg, name, T, H, W, Cp, Cout, taps=(3, 3, 3), epi="BF16", wan=True, t_mul=1, t_add=0, st_t=1, st_hw=1):
    return dict(id=f"{cfg}.{name}", entry="conv", cfg=cfg, T=T, H=H, W=W, Cp=Cp, Cout=Cout, taps=tuple(taps), epi=EPI[epi],
                oob_zero_pad=wan, out_t_mul=t_mul, out_t_add=t_add, stride_t=st_t, stride_hw=st_hw)


VAE_CONV_ROWS = []            # filled below
VAE_GEMM_ROWS = []


def _gemm_row(cfg, name, M, N, K, epi="BF16", flags=()):
    return dict(id=f"{cfg}.{name}", entry="gemm", cfg=cfg, M=M, N=N, K=K, epi=EPI[epi], flags=frozenset(flags), layers=1,
                raster=False)


# the VAE decoders' launches at production spatial size with 2 latent frames (test_table_covers_the_engines_launches records
# them): Wan2.2 latent 44x80 -> 352x640 (before unpatchify), Wan2.1 68x120 -> 544x960, one hyvideo 32x32 latent tile.
# conv: (T, H, W, Cp, Cout, taps, epilogue, oob_zero_pad, out_t_mul) — time_conv (out_t_mul 2) runs once per channel group,
# out_t_add 1 and 2; gemm: (M, N, K, epilogue[, operand windows]) — b_window: the mid-attention P.vT reads
# B = vT[:, f*Lf:(f+1)*Lf] (ldb > K); out_window: the latent 1x1 conv writes x0[:, :32] of a 64-wide buffer
_VAE_LAUNCHES = {
    "wan22_dec": [
        (7040, 64, 64, 0), (2, 44, 80, 64, 1024, (3, 3, 3), 0, True, 1), (2, 44, 80, 1024, 1024, (3, 3, 3), 0, True, 1),
        (2, 44, 80, 1024, 1024, (3, 3, 3), 5, True, 1), (7040, 1024, 1024, 0), (1024, 7072, 1024, 0), (3520, 3520, 1024, 2),
        (3520, 1024, 3520, 0, ("b_window",)), (7040, 1024, 1024, 5), (1, 44, 80, 1024, 1024, (3, 1, 1), 0, True, 2),
        (3, 88, 160, 1024, 1024, (1, 3, 3), 0, True, 1), (3, 88, 160, 1024, 1024, (3, 3, 3), 0, True, 1),
        (3, 88, 160, 1024, 1024, (3, 3, 3), 5, True, 1), (2, 88, 160, 1024, 1024, (3, 1, 1), 0, True, 2),
        (5, 176, 320, 1024, 1024, (1, 3, 3), 0, True, 1), (5, 176, 320, 1024, 512, (3, 3, 3), 0, True, 1),
        (281600, 512, 1024, 0), (5, 176, 320, 512, 512, (3, 3, 3), 5, True, 1), (5, 176, 320, 512, 512, (3, 3, 3), 0, True, 1),
        (5, 352, 640, 512, 512, (1, 3, 3), 0, True, 1), (5, 352, 640, 512, 256, (3, 3, 3), 0, True, 1), (1126400, 256, 512, 0),
        (5, 352, 640, 256, 256, (3, 3, 3), 5, True, 1), (5, 352, 640, 256, 256, (3, 3, 3), 0, True, 1),
        (5, 352, 640, 256, 32, (3, 3, 3), 2, True, 1)],
    "wan21_dec": [
        (16320, 32, 64, 0, ("out_window",)), (2, 68, 120, 64, 384, (3, 3, 3), 0, True, 1), (2, 68, 120, 384, 384, (3, 3, 3), 0, True, 1),
        (2, 68, 120, 384, 384, (3, 3, 3), 5, True, 1), (16320, 384, 384, 0), (384, 16352, 384, 0), (8160, 8160, 384, 2),
        (8160, 384, 8160, 0, ("b_window",)), (16320, 384, 384, 5), (1, 68, 120, 384, 384, (3, 1, 1), 0, True, 2),
        (3, 136, 240, 384, 192, (1, 3, 3), 0, True, 1), (3, 136, 240, 192, 384, (3, 3, 3), 0, True, 1), (97920, 384, 192, 0),
        (3, 136, 240, 384, 384, (3, 3, 3), 5, True, 1), (3, 136, 240, 384, 384, (3, 3, 3), 0, True, 1),
        (2, 136, 240, 384, 384, (3, 1, 1), 0, True, 2), (5, 272, 480, 384, 192, (1, 3, 3), 0, True, 1),
        (5, 272, 480, 192, 192, (3, 3, 3), 0, True, 1), (5, 272, 480, 192, 192, (3, 3, 3), 5, True, 1),
        (5, 544, 960, 192, 96, (1, 3, 3), 0, True, 1), (5, 544, 960, 128, 96, (3, 3, 3), 0, True, 1),
        (5, 544, 960, 128, 96, (3, 3, 3), 5, True, 1), (5, 544, 960, 128, 32, (3, 3, 3), 2, True, 1)],
    "hy_tile": [
        (2048, 32, 64, 0, ("out_window",)), (2, 32, 32, 64, 512, (3, 3, 3), 0, False, 1), (2, 32, 32, 512, 512, (3, 3, 3), 0, False, 1),
        (2, 32, 32, 512, 512, (3, 3, 3), 5, False, 1), (2048, 512, 512, 0), (512, 2048, 512, 0), (2048, 2048, 512, 2),
        (2048, 512, 2048, 0), (2048, 512, 512, 5), (2, 64, 64, 512, 512, (3, 3, 3), 0, False, 1),
        (2, 64, 64, 512, 512, (3, 3, 3), 5, False, 1), (3, 128, 128, 512, 512, (3, 3, 3), 0, False, 1),
        (3, 128, 128, 512, 256, (3, 3, 3), 0, False, 1), (49152, 256, 512, 0), (3, 128, 128, 256, 256, (3, 3, 3), 5, False, 1),
        (3, 128, 128, 256, 256, (3, 3, 3), 0, False, 1), (5, 256, 256, 256, 256, (3, 3, 3), 0, False, 1),
        (5, 256, 256, 256, 128, (3, 3, 3), 0, False, 1), (327680, 128, 256, 0), (5, 256, 256, 128, 128, (3, 3, 3), 5, False, 1),
        (5, 256, 256, 128, 128, (3, 3, 3), 0, False, 1), (5, 256, 256, 128, 32, (3, 3, 3), 2, False, 1)],
}
for _cfg, _launches in _VAE_LAUNCHES.items():
    for _i, _l in enumerate(_launches):
        if len(_l) <= 5:
            VAE_GEMM_ROWS.append(_gemm_row(_cfg, f"gemm{_i}_M{_l[0]}_N{_l[1]}_K{_l[2]}", *_l[:3],
                                           epi={0: "BF16", 2: "F32", 5: "RES_BF16"}[_l[3]], flags=_l[4] if len(_l) == 5 else ()))
        else:
            T, H, W, Cp, Co, taps, e, wan, mul = _l
            for _add in ((1, 2) if mul > 1 else (0,)):
                VAE_CONV_ROWS.append(_conv(_cfg, f"conv{_i}_{T}x{H}x{W}_{Cp}to{Co}_k{''.join(map(str, taps))}" +
                                           (f"_add{_add}" if mul > 1 else ""), T, H, W, Cp, Co, taps,
                                           epi={0: "BF16", 2: "F32", 5: "RES_BF16"}[e], wan=wan, t_mul=mul, t_add=_add))
# the encoders' strided Resample forms at full size (Wan2.1 encoder: ZeroPad2d + Conv2d stride 2 on the 544x960 frames;
# time_conv stride 2 of downsample3d)
VAE_CONV_ROWS += [_conv("wan21_enc", "down2d_stride2_544x960", 5, 544, 960, 128, 96, (1, 3, 3), st_hw=2),
                  _conv("wan21_enc", "down3d_time_stride2_136x240", 5, 136, 240, 384, 384, (3, 1, 1), st_t=2)]

PROD_TABLE = _dit_rows() + SP_ROWS + VAE_CONV_ROWS + VAE_GEMM_ROWS

# rows allowed below 3 tiles per CTA at 132 SMs, and why: the decode launches them at this size. tests/test_kernel_contract_cpu.py
# requires every other GEMM / conv row to reach 3, and every row listed here to be below 3 (no stale entries).
_LAT22 = "Wan2.2 latent level: 2 frames of 44x80 voxels"
_LAT21 = "Wan2.1 latent level: 2 frames of 68x120 voxels (time_conv: 1 frame)"
_HY = "hyvideo 32x32 latent tile (256x256 pixels): the levels below the last one are this small"
WAVE_EXEMPT = {
    "wan22_dec.conv1_2x44x80_64to1024_k333": _LAT22, "wan22_dec.conv2_2x44x80_1024to1024_k333": _LAT22,
    "wan22_dec.conv3_2x44x80_1024to1024_k333": _LAT22, "wan22_dec.conv9_1x44x80_1024to1024_k311_add1": _LAT22,
    "wan22_dec.conv9_1x44x80_1024to1024_k311_add2": _LAT22,
    "wan22_dec.gemm0_M7040_N64_K64": _LAT22 + ", the 48 -> 48 channel conv2 as a GEMM",
    "wan22_dec.gemm4_M7040_N1024_K1024": _LAT22 + ", mid-attention q", "wan22_dec.gemm8_M7040_N1024_K1024": _LAT22 + ", proj",
    "wan22_dec.gemm5_M1024_N7072_K1024": _LAT22 + ", mid-attention v^T", "wan22_dec.gemm6_M3520_N3520_K1024": _LAT22 +
    ", one frame's S = q.k^T", "wan22_dec.gemm7_M3520_N1024_K3520": _LAT22 + ", one frame's P.v^T",
    "wan21_dec.conv9_1x68x120_384to384_k311_add1": _LAT21, "wan21_dec.conv9_1x68x120_384to384_k311_add2": _LAT21,
    "wan21_dec.gemm0_M16320_N32_K64": _LAT21 + ", the 16 -> 16 channel conv2 as a GEMM",
    "wan21_dec.gemm4_M16320_N384_K384": _LAT21 + ", mid-attention q", "wan21_dec.gemm8_M16320_N384_K384": _LAT21 + ", proj",
    "wan21_dec.gemm5_M384_N16352_K384": _LAT21 + ", mid-attention v^T", "wan21_dec.gemm7_M8160_N384_K8160": _LAT21 +
    ", one frame's P.v^T",
    **{f"hy_tile.{n}": _HY for n in (
        "conv1_2x32x32_64to512_k333", "conv2_2x32x32_512to512_k333", "conv3_2x32x32_512to512_k333",
        "conv9_2x64x64_512to512_k333", "conv10_2x64x64_512to512_k333", "conv12_3x128x128_512to256_k333",
        "conv14_3x128x128_256to256_k333", "conv15_3x128x128_256to256_k333", "gemm0_M2048_N32_K64", "gemm4_M2048_N512_K512",
        "gemm5_M512_N2048_K512", "gemm6_M2048_N2048_K512", "gemm7_M2048_N512_K2048", "gemm8_M2048_N512_K512",
        "gemm13_M49152_N256_K512")},
}


# ------------------------------------------------------------------------------------------------------------
# plans (host-only planners of the library: no GPU needed)
# ------------------------------------------------------------------------------------------------------------
def _lib():
    from yume_b200 import _lib as L
    return L.load()


def _c_out(n, fn, *args):
    import ctypes as C
    out = (C.c_int * n)()
    assert fn(*args, out) == 0, (fn, args)
    return tuple(out)


def conv_out_dims(row):
    kt, kh, kw = row["taps"]
    T, H, W, st, sh = row["T"], row["H"], row["W"], row["stride_t"], row["stride_hw"]
    To = (T - kt) // st + 1 if st > 1 else T
    Ho, Wo = ((H + 1 - kh) // sh + 1, (W + 1 - kw) // sh + 1) if sh > 1 else (H, W)
    return To, Ho, Wo


def row_plan(row, sms=SMS):
    """The launch decomposition of a row as the library plans it: tiles (or work units), the CTAs that run them, per-CTA
    tiles, and what the sampler needs (tile sizes / boxes / units)."""
    lib = _lib()
    e = row["entry"]
    if e == "gemm":
        pair, bn, mt, nt = _c_out(4, lib.yb_gemm_plan, row["M"], row["N"], sms)
        return dict(block_m=128, block_n=bn, tiles=mt * nt, ctas=sms, per_cta=mt * nt / sms, m_tiles=mt, n_tiles=nt)
    if e == "gemm_sp_qkv":             # SM-pair kernel: 256-row tiles, block_n 256, one CTA pair per cluster slot
        M, N = row["Lp"], 3 * row["C"]
        mt, nt = -(-M // 256), -(-N // 256)
        return dict(block_m=256, block_n=256, tiles=mt * nt, ctas=sms // 2, per_cta=mt * nt / (sms // 2), m_tiles=mt,
                    n_tiles=nt)
    if e == "conv":
        kt, kh, kw = row["taps"]
        oT, oH, oW = conv_out_dims(row)
        strided = row["stride_t"] > 1 or row["stride_hw"] > 1
        TW, TH, TT, fused = _c_out(4, lib.yb_conv3d_plan, oT, oH, oW, row["Cout"], kw, 1 if strided else 0)
        boxes = -(-oT // TT) * -(-oH // TH) * -(-oW // TW)
        bn = 256 if row["Cout"] % 256 == 0 else 128
        nt = -(-row["Cout"] // bn)
        return dict(box=(TT, TH, TW), fused=fused, block_n=bn, boxes=boxes, tiles=boxes * nt, ctas=sms,
                    per_cta=boxes * nt / sms, dims=(oT, oH, oW))
    Lq, Lk, heads = (row["Lp"] * row["P"], row["Lp"] * row["P"], row["heads"]) if e == "attention_sp" else \
        (row["Lq"], row["Lk"], row["heads"])
    flags = 2 if row.get("accumulate") else 0          # YB_ATT_ACCUMULATE
    full, tail, ns, per = _c_out(4, lib.yb_attention_plan, Lq, Lk, heads, sms, flags)
    nq = -(-Lq // 256)
    return dict(units=nq * heads, nq=nq, full_units=full, tail=tail, ns=ns, kv_per_segment=per, nkv=-(-Lk // 128),
                ctas=full + tail * ns, per_cta=nq * heads / sms, Lq=Lq, Lk=Lk, heads=heads)


# ------------------------------------------------------------------------------------------------------------
# sample sets (pure functions: tests/test_kernel_contract_cpu.py checks them against every row's plan)
# ------------------------------------------------------------------------------------------------------------
def _cpu_gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def band_sample(n, band, key):
    """Two indices of every `band`-wide band of range(n): a seeded one and the band's last valid index (sorted, unique)."""
    starts = torch.arange(0, n, band)
    ends = torch.clamp(starts + band, max=n)
    seeded = starts + (torch.rand(len(starts), generator=_cpu_gen("band", n, band, key)) * (ends - starts)).long()
    return torch.unique(torch.cat([seeded, ends - 1]))


def gemm_sample(M, N, key):
    """Full rows (2 per 128-row band) and full columns (2 per 64-column band) whose fp64 reference is computed."""
    return band_sample(M, 128, ("rows", key)), band_sample(N, 64, ("cols", key))


def gemm_sp_qkv_sample(row):
    """Rows of the [P*Lp, 3C] reassembled receive buffers (2 per 128-row band of every rank's Lp tokens) and columns (2 per
    64-column band) of the fused QKV + all-to-all GEMM."""
    Lp, P, C = row["Lp"], row["P"], row["C"]
    rows = torch.cat([r * Lp + band_sample(Lp, 128, ("rows", row["id"], r)) for r in range(P)])
    return rows, band_sample(3 * C, 64, ("cols", row["id"]))


def gemm_tiles_missed(rows, cols, M, N, block_m, block_n):
    """Output tiles (i, j) of a block_m x block_n plan that hold no sampled element (a sampled row or column inside it)."""
    mt, nt = -(-M // block_m), -(-N // block_n)
    row_hit = torch.zeros(mt, dtype=torch.bool)
    row_hit[rows // block_m] = True
    col_hit = torch.zeros(nt, dtype=torch.bool)
    col_hit[cols // block_n] = True
    miss = ~(row_hit[:, None] | col_hit[None, :])
    return [tuple(int(v) for v in ij) for ij in miss.nonzero()]


def conv_sample(dims, box, key):
    """Linear output-voxel indices (t*oH*oW + h*oW + w): two of every (TT, TH, TW) box, a seeded one and the box's last
    valid voxel."""
    (oT, oH, oW), (TT, TH, TW) = dims, box
    bt, bh, bw = torch.meshgrid(torch.arange(0, oT, TT), torch.arange(0, oH, TH), torch.arange(0, oW, TW), indexing="ij")
    bt, bh, bw = bt.flatten(), bh.flatten(), bw.flatten()
    et, eh, ew = torch.clamp(bt + TT, max=oT), torch.clamp(bh + TH, max=oH), torch.clamp(bw + TW, max=oW)
    g = _cpu_gen("conv", dims, box, key)
    r = torch.rand(3, len(bt), generator=g)
    st = bt + (r[0] * (et - bt)).long()
    sh = bh + (r[1] * (eh - bh)).long()
    sw = bw + (r[2] * (ew - bw)).long()
    lin = lambda t, h, w: (t * oH + h) * oW + w                             # noqa: E731
    return torch.unique(torch.cat([lin(st, sh, sw), lin(et - 1, eh - 1, ew - 1)]))


def conv_boxes_missed(vox, dims, box):
    (oT, oH, oW), (TT, TH, TW) = dims, box
    t, rem = vox // (oH * oW), vox % (oH * oW)
    h, w = rem // oW, rem % oW
    nbh, nbw = -(-oH // TH), -(-oW // TW)
    nb = -(-oT // TT) * nbh * nbw
    hit = torch.zeros(nb, dtype=torch.bool)
    hit[((t // TT) * nbh + h // TH) * nbw + w // TW] = True
    return [int(i) for i in (~hit).nonzero().flatten()]


def attention_sample(Lq, heads, key, per_tile=4):
    """Query rows per head: `per_tile` rows of every 128-row query tile of every 256-row unit (seeded rows and the tile's last
    valid row), plus every row of one seeded unit. Four per tile, not one: a defect confined to one unit (one KV tile dropped
    in its loop) moves few rows past the bound, and 2 rows per unit saw a dropped tile of 145 in only 3 of 8 seeds where 8
    rows saw it in all 8 (tests/test_kernel_contract_cpu.py keeps such a case)."""
    out = []
    nq = -(-Lq // 256)
    ntile = -(-Lq // 128)
    for h in range(heads):
        g = _cpu_gen("att", Lq, h, key)
        starts = torch.arange(ntile) * 128
        ends = torch.clamp(starts + 128, max=Lq)
        seeded = starts[:, None] + (torch.rand(ntile, per_tile - 1, generator=g) * (ends - starts)[:, None]).long()
        u = int(torch.randint(nq, (1,), generator=g))
        whole = torch.arange(u * 256, min(Lq, u * 256 + 256))
        out.append(torch.unique(torch.cat([seeded.flatten(), ends - 1, whole])))
    return out


def attention_units_missed(rows_per_head, Lq, heads):
    """(head, unit, query tile) triples with valid rows but no sampled row: every 128-row query tile of every unit counts."""
    missed = []
    ntile = -(-Lq // 128)
    for h in range(heads):
        hit = torch.zeros(ntile, dtype=torch.bool)
        hit[rows_per_head[h] // 128] = True
        missed += [(h, int(i) // 2, int(i) % 2) for i in (~hit).nonzero().flatten()]
    return missed


# ------------------------------------------------------------------------------------------------------------
# bounds
# ------------------------------------------------------------------------------------------------------------
def attention_bound_prod(q, k, v, scale, nkv, ns=1):
    """attention_bound of part one (output rounding, P in bf16, logit error) plus the fp32 terms that grow with the number of
    KV tiles nkv, which at 8 tiles are negligible and at 335 are not (each relative to sum_j p_ij |v_j|, the scale of o / l):
      (8*nkv + 4)*u32   the normaliser l: each thread adds 8 pair-sums per KV tile into its running l0 / l1, sequentially over
                        all tiles (a pair-sum of 4 terms rounds twice more), then a 2-level shuffle: a recursive fp32 sum of
                        8*nkv + 4 roundings, each <= u32 * (the sum so far) <= u32 * l
      nkv*u32           l *= alpha once per tile (alpha multiplies o and l alike, so its own error cancels in o / l)
      nkv*u32           o *= alpha once per tile
      2*(8*nkv + 16)*u32  o += P.V: 8 wgmma k-steps of 16 keys per tile chain 8*nkv fp32 additions into o, each k-step's 16
                        products summed inside the tensor core (truncation allowed: factor 2, as gemm_bounds)
      3*ns*u32          the combine of ns KV segments (weights 2^(m_s - M), the weighted sums of O and l): only when split
    total (26*nkv + 36 + 3*ns)*u32. Returns (ref, bound) in fp64 for q [R, 128] sampled rows, k / v [Lk, 128] of one head."""
    s = (q @ k.t()) * scale
    p = torch.softmax(s, dim=-1)
    ref = p @ v
    pv = p @ v.abs()
    e = (2 * 128 * U32 * scale * (q.abs() @ k.abs().t()) + 4 * U32 * s.abs()).amax(dim=-1, keepdim=True)
    extra = (26 * nkv + 36 + (3 * ns if ns > 1 else 0)) * U32
    return ref, U16 * ref.abs() + (2 * U16 + 2 * e + extra) * pv


def gemm_epilogue_ref(epi, acc, Fb, bias=None, res=None, x0=None, gate=None):
    """(ref, bound) of one epilogue from the fp64 accumulator acc = A.B^T and F = gemm_bounds at the same elements (the
    bounds of test_gpu_kernel_contract.test_gemm_every_epilogue_per_element)."""
    b = bias if bias is not None else torch.zeros_like(acc)
    accb = acc + b
    f32 = Fb + 4 * U32 * (acc.abs() + b.abs())
    if epi == EPI["BF16"]:
        return accb, bf16_out_bound(accb, f32)
    if epi == EPI["GELU"]:
        ref = F.gelu(accb, approximate="tanh")
        return ref, bf16_out_bound(ref, 1.13 * f32 + 2.0 ** -12 * accb.abs() + 4 * U32 * accb.abs())
    if epi == EPI["GELU_ERF"]:
        ref = F.gelu(accb)
        return ref, bf16_out_bound(ref, 1.13 * f32 + 2.0 ** -20 * accb.abs() + 4 * U32 * accb.abs())
    if epi == EPI["F32"]:
        return accb, f32
    if epi == EPI["RES_BF16"]:
        ref = accb + res
        return ref, bf16_out_bound(ref, f32 + 4 * U32 * res.abs())
    g = gate if gate is not None else torch.ones_like(acc)
    return x0 + accb * g, g.abs() * f32 + 4 * U32 * (x0.abs() + (g * accb).abs())


def gemm_ref_rows_cols(A, B, rows, cols, chunk=1 << 14):
    """fp64 acc and F = 2*K*u32*(|A||B|^T) at the sampled full rows ([len(rows), N]) and full columns ([M, len(cols)]),
    chunked so that no fp64 copy of a large operand exists at once."""
    K = A.shape[1]
    Ar = A[rows].double()
    accR = torch.empty(len(rows), B.shape[0], dtype=torch.float64, device=A.device)
    FR = torch.empty_like(accR)
    for n0 in range(0, B.shape[0], chunk):
        Bd = B[n0:n0 + chunk].double()
        accR[:, n0:n0 + chunk] = Ar @ Bd.t()
        FR[:, n0:n0 + chunk] = 2.0 * K * U32 * (Ar.abs() @ Bd.abs().t())
    Bc = B[cols].double()
    accC = torch.empty(A.shape[0], len(cols), dtype=torch.float64, device=A.device)
    FC = torch.empty_like(accC)
    for m0 in range(0, A.shape[0], chunk):
        Ad = A[m0:m0 + chunk].double()
        accC[m0:m0 + chunk] = Ad @ Bc.t()
        FC[m0:m0 + chunk] = 2.0 * K * U32 * (Ad.abs() @ Bc.abs().t())
    return (accR, FR), (accC, FC)


# ------------------------------------------------------------------------------------------------------------
# device helpers
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()
    return "cuda"


STATS = {}                   # family -> [wall seconds, peak bytes]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if KC.WORST:
        import json
        import os
        print("[contract] worst |err|/bound per family: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(KC.WORST.items())))
        for k, (sec, peak) in sorted(STATS.items()):
            print(f"[contract] {k}: {sec:.1f} s, peak max_memory_allocated {peak / 2 ** 30:.2f} GiB")
        path = os.environ.get("YB_CONTRACT_REPORT")
        if path:
            data = {"worst_ratio": {}}
            if os.path.exists(path):
                with open(path) as f:
                    data = json.load(f)
            worst = data.setdefault("worst_ratio", {})
            for k, v in KC.WORST.items():
                worst[k] = max(worst.get(k, 0.0), v)
            data.setdefault("prod_stats", {}).update({k: dict(seconds=s, peak_bytes=p) for k, (s, p) in STATS.items()})
            if torch.cuda.is_available():
                data["device"] = torch.cuda.get_device_name(0)
            with open(path, "w") as f:
                json.dump(data, f, indent=1, sort_keys=True)


@pytest.fixture()
def measure(request):
    """Frees the previous case's memory, then records wall time and peak max_memory_allocated per family."""
    import gc
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    box = {}
    yield box
    torch.cuda.synchronize()
    fam = box.get("family")
    if fam:
        s = STATS.setdefault(fam, [0.0, 0])
        s[0] += time.time() - t0
        s[1] = max(s[1], torch.cuda.max_memory_allocated())


def _cuda_gen(key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(key).encode()))


def _rand(g, rows, cols, scale=1.0, dtype=torch.bfloat16, chunk=1 << 14):
    """[rows, cols] standard normal * scale drawn on the device in row chunks (no fp32 copy of a large bf16 tensor)."""
    out = torch.empty(rows, cols, dtype=dtype, device="cuda")
    for r0 in range(0, rows, chunk):
        n = min(chunk, rows - r0)
        out[r0:r0 + n] = torch.randn(n, cols, generator=g, device="cuda").mul_(scale)
    return out


class Lean:
    """A NaN-poisoned (or seeded) [rows, cols] view with `pr` guard rows above and below and `pc` guard columns on both sides
    (the column window production writes into); the guard is checked against its bit pattern directly and the NaN check runs
    in row chunks, so no full-size mask or copy exists."""

    def __init__(self, rows, cols, dtype, pr=128, pc=0, fill=None):
        self.itype, self.pattern = KC._GUARD_BITS[dtype]
        self.pr, self.pc = pr, pc
        self.backing = torch.full((rows + 2 * pr, cols + 2 * pc), self.pattern, dtype=self.itype, device="cuda").view(dtype)
        self.view = self.backing[pr:pr + rows, pc:pc + cols]
        if fill is None:
            self.view.fill_(float("nan"))
        else:
            self.view.copy_(fill)

    def check(self, what, written_rows=None):
        bits = self.backing.view(self.itype)
        pr, pc = self.pr, self.pc
        parts = [bits[:pr], bits[bits.shape[0] - pr:]]
        if pc:
            parts += [bits[pr:bits.shape[0] - pr, :pc], bits[pr:bits.shape[0] - pr, bits.shape[1] - pc:]]
        for p in parts:
            if p.numel() and not bool((p == self.pattern).all()):
                raise AssertionError(f"{what}: {int((p != self.pattern).sum())} guard element(s) changed")
        rows = self.view if written_rows is None else self.view[written_rows]
        for r0 in range(0, rows.shape[0], 1 << 14):
            bad = torch.isnan(rows[r0:r0 + (1 << 14)])
            if bool(bad.any()):
                i = tuple(int(v) for v in bad.nonzero()[0])
                raise AssertionError(f"{what}: {int(bad.sum())} output element(s) never written (still NaN), first at "
                                     f"({i[0] + r0}, {i[1]})")


def _ids(rows):
    return [r["id"] for r in rows]


def _rows(entry):
    return [r for r in PROD_TABLE if r["entry"] == entry]


# ------------------------------------------------------------------------------------------------------------
# GEMM rows
# ------------------------------------------------------------------------------------------------------------
def _check_gemm_sampled(got, A, B, rows, cols, epi, tag, family, bias=None, res=None, x0=None, gate_rows=None):
    """Sampled fp64 check of a GEMM output `got` [M, N]: the full rows `rows` and full columns `cols`. gate_rows: the
    per-token gate table [M -> gate row] as a callable idx -> [len(idx), N] (or None)."""
    (accR, FR), (accC, FC) = gemm_ref_rows_cols(A, B, rows.to(A.device), cols.to(A.device))
    r, c = rows.to(A.device), cols.to(A.device)
    bd = None if bias is None else bias.double()
    kw = lambda ri, ci: dict(                                                        # noqa: E731
        bias=None if bd is None else bd[ci][None].expand(len(ri) if ri is not None else A.shape[0], -1),
        res=None if res is None else (res[ri] if ri is not None else res[:, ci]).double(),
        x0=None if x0 is None else (x0[ri] if ri is not None else x0[:, ci]).double(),
        gate=None if gate_rows is None else (gate_rows(ri) if ri is not None else gate_rows(None)[:, ci]))
    allc = torch.arange(B.shape[0], device=A.device)
    ref, bound = gemm_epilogue_ref(epi, accR, FR, **kw(r, allc))
    assert_within(got[r], ref, bound, tag + " sampled rows", family)
    ref, bound = gemm_epilogue_ref(epi, accC, FC, **kw(None, c))
    assert_within(got[:, c], ref, bound, tag + " sampled columns", family)


@pytest.mark.parametrize("rid", _ids(_rows("gemm")))
def test_prod_gemm(dev, measure, rid):
    """One GEMM launch of the table at its production shape, as the engine makes it (1-CTA kernel, automatic tile plan): poison
    / guard checks on the whole output, the fp64 reference on the sampled rows and columns (gemm_sample), bounds of
    gemm_epilogue_ref with the actual K. GATE_RES runs in place on seeded xs (gate rows from a 2-row [U, 6, N] table through
    tok_idx where the row is gated that way), then once more under F32 into a NaN buffer: every element written."""
    from yume_b200 import ops
    row = next(r for r in PROD_TABLE if r["id"] == rid)
    measure["family"] = "prod_gemm"
    M, N, K, epi = row["M"], row["N"], row["K"], row["epi"]
    g = _cuda_gen(rid)
    A = _rand(g, M, K)
    if "b_window" in row["flags"]:                             # B a column window of a wider buffer (ldb > K), as vT[:, f*Lf:]
        B = _rand(g, N, K + 64, 1 / math.sqrt(K))[:, 32:32 + K]
    else:
        B = _rand(g, N, K, 1 / math.sqrt(K))
    bias = None if epi == EPI["F32"] else torch.randn(N, generator=g, device=dev)
    rows, cols = gemm_sample(M, N, rid)
    pc = 64 if "out_window" in row["flags"] else 0             # out a column window (ldo > N), as q2 = qkv[:, :C]
    tag = f"prod gemm {rid} M{M} N{N} K{K}"
    if epi == EPI["GATE_RES"]:
        x0 = _rand(g, M, N, dtype=torch.float32)
        extra, gate_rows = {}, None
        if "gate" in row["flags"]:
            U = 2 if "tok_idx" in row["flags"] else 1
            gate6 = torch.randn(U, 6, N, generator=g, device=dev)
            tok = (torch.arange(M, device=dev) >= M // 3).to(torch.int32) if U == 2 else None   # history | new tokens
            extra = dict(gate=gate6[:, 2], tok_idx=tok)
            gate_rows = (lambda ri: gate6[(tok.long() if tok is not None else torch.zeros(M, dtype=torch.long, device=dev))
                                          [ri if ri is not None else slice(None)], 2].double())
        out = Lean(M, N, torch.float32, fill=x0)
        ops.gemm(A, B, bias, out.view, epi, **extra)
        torch.cuda.synchronize()
        out.check(tag + " GATE_RES")
        _check_gemm_sampled(out.view, A, B, rows, cols, epi, tag + " GATE_RES", "prod_gemm", bias=bias, x0=x0,
                            gate_rows=gate_rows)
        del out, x0
        o32 = Lean(M, N, torch.float32)
        ops.gemm(A, B, None, o32.view, EPI["F32"])
        torch.cuda.synchronize()
        o32.check(tag + " F32 coverage run")
        _check_gemm_sampled(o32.view, A, B, rows, cols, EPI["F32"], tag + " F32 coverage run", "prod_gemm")
        return
    res = _rand(g, M, N) if epi == EPI["RES_BF16"] else None
    out = Lean(M, N, torch.float32 if epi == EPI["F32"] else torch.bfloat16, pc=pc)
    ops.gemm(A, B, bias, out.view, epi, res=res)
    torch.cuda.synchronize()
    out.check(tag)
    _check_gemm_sampled(out.view, A, B, rows, cols, epi, tag, "prod_gemm", bias=bias, res=res)


# ------------------------------------------------------------------------------------------------------------
# attention rows
# ------------------------------------------------------------------------------------------------------------
def _check_attention_sampled(got, q, k, v, heads, scale, plan, key, tag, family, fill=None):
    """got [Lq, heads*128]; reference per head on the sampled query rows (attention_sample) against all keys."""
    samples = attention_sample(q.shape[0], heads, key)
    for h in range(heads):
        sl = slice(h * 128, (h + 1) * 128)
        kd, vd = k[:, sl].double(), v[:, sl].double()
        refs, bounds = [], []
        r = samples[h].to(q.device)
        for c0 in range(0, len(r), 1024):                       # row chunks: [1024, Lk] fp64 intermediates at most
            rc = r[c0:c0 + 1024]
            ref, bound = attention_bound_prod(q[rc, sl].double(), kd, vd, scale, plan["nkv"], plan["ns"])
            if fill is not None:           # out += result: one more bf16 rounding of the result before the add
                f = fill[rc, sl].double()
                bound = bound + U16 * ref.abs() + U16 * (ref + f).abs()
                ref = ref + f
            refs.append(ref)
            bounds.append(bound)
        assert_within(got[r, sl], torch.cat(refs), torch.cat(bounds), f"{tag} head{h}", family)


@pytest.mark.parametrize("rid", _ids(_rows("attention")))
def test_prod_attention(dev, measure, rid):
    """One attention launch of the table at its production shape with the automatic split policy (q, k, v as column slices of
    one fused [L, 3*heads*128] buffer, keys cut to Lk as the k_lens contract does). The output is poisoned and guarded; for
    the accumulating image branch it is seeded, and the same operands run once more without accumulate into a NaN buffer.
    Bound: attention_bound_prod with the launch's nkv and segment count."""
    from yume_b200 import ops
    row = next(r for r in PROD_TABLE if r["id"] == rid)
    measure["family"] = "prod_attention"
    plan = row_plan(row)
    Lq, Lk, H = row["Lq"], row["Lk"], row["heads"]
    g = _cuda_gen(rid)
    W = H * 128
    buf = _rand(g, max(Lq, Lk), 3 * W)
    q, k, v = buf[:Lq, :W], buf[:Lk, W:2 * W], buf[:Lk, 2 * W:]
    q.mul_(2.0)                                                   # logits spread ~N(0, 4): the softmax is not flat
    scale = 1 / math.sqrt(128.0)
    tag = f"prod attention {rid} Lq{Lq} Lk{Lk} h{H} tail{plan['tail']} ns{plan['ns']}"
    fill = _rand(g, Lq, W) if row["accumulate"] else None
    out = Lean(Lq, W, torch.bfloat16, fill=fill)
    ops.attention(q, k, v, out.view, H, scale=scale, accumulate=row["accumulate"])
    torch.cuda.synchronize()
    out.check(tag)
    _check_attention_sampled(out.view, q, k, v, H, scale, plan, rid, tag, "prod_attention", fill=fill)
    if row["accumulate"]:
        del out
        o2 = Lean(Lq, W, torch.bfloat16)
        ops.attention(q, k, v, o2.view, H, scale=scale)
        torch.cuda.synchronize()
        o2.check(tag + " coverage run")
        _check_attention_sampled(o2.view, q, k, v, H, scale, row_plan(dict(row, accumulate=False)), rid, tag + " coverage run",
                                 "prod_attention")


@pytest.mark.parametrize("rid", _ids(_rows("attention_sp")))
def test_prod_attention_sp(dev, measure, rid):
    """yb_attention_sp at a Ulysses per-rank shape, every rank's launch emulated on one GPU: rank r attends over all P*Lp
    gathered query rows for its heads/P heads and stores row t into receiver t // Lp's [P(src), Lp, Hl*128] buffer (guarded,
    NaN-poisoned). The receive buffers, reassembled into global [L, heads*128] order, are checked on the sampled rows."""
    from yume_b200 import ops
    row = next(r for r in PROD_TABLE if r["id"] == rid)
    measure["family"] = "prod_sp"
    P, Lp, Hl = row["P"], row["Lp"], row["heads"]
    plan = row_plan(row)
    L, Wh = P * Lp, Hl * 128
    g = _cuda_gen(rid)
    scale = 1 / math.sqrt(128.0)
    bufs = [Lean(P * Lp, Wh, torch.bfloat16) for _ in range(P)]
    ptrs = [b.view.data_ptr() for b in bufs]
    qkvs = []
    for r in range(P):
        full = _rand(g, L, 3 * Wh)                                # rank r's gathered q|k|v [L, 3*Wh]
        full[:, :Wh].mul_(2.0)
        ops.attention_sp(full[:, :Wh], full[:, Wh:2 * Wh], full[:, 2 * Wh:], ptrs, Wh, Hl, r, Lp, scale=scale)
        qkvs.append(full)
    torch.cuda.synchronize()
    tag = f"prod attention_sp {rid} P{P} Lp{Lp} h{Hl} tail{plan['tail']} ns{plan['ns']}"
    for p in range(P):
        bufs[p].check(f"{tag} receiver{p}")
    recv = torch.stack([b.view.view(P, Lp, Wh) for b in bufs])     # [receiver, src, Lp, Wh]
    for r in range(P):
        got = recv[:, r].reshape(L, Wh)                              # rank r's output rows in global order
        full = qkvs[r]
        _check_attention_sampled(got, full[:, :Wh], full[:, Wh:2 * Wh], full[:, 2 * Wh:], Hl, scale, plan, (rid, r),
                                 f"{tag} rank{r}", "prod_sp")


@pytest.mark.parametrize("rid", _ids(_rows("gemm_sp_qkv")))
def test_prod_gemm_sp_qkv(dev, measure, rid):
    """yb_gemm_sp_qkv at a Ulysses per-rank shape (SM-pair kernel, 256-row tiles), every rank emulated on one GPU: rank r
    projects its Lp tokens and stores head block p of q|k|v into receiver p's guarded [P(src), Lp, 3*Wh] buffer. The
    buffers reassembled into [L, 3C] are checked on the sampled rows (2 per 128-row band of every rank) and columns; the
    per-token sums of squares that yb_sp_bcast_sums delivers must match the received rows (sumsq_bound)."""
    from yume_b200 import ops
    import test_gpu_kernel_contract_ext as KX
    row = next(r for r in PROD_TABLE if r["id"] == rid)
    measure["family"] = "prod_sp"
    P, Lp, C, K = row["P"], row["Lp"], row["C"], row["K"]
    L, Wh = P * Lp, C // P
    g = _cuda_gen(rid)
    h = _rand(g, L, K)
    w = _rand(g, 3 * C, K, 1 / math.sqrt(K))
    bias = torch.randn(3 * C, generator=g, device=dev)
    bufs = [Lean(P * Lp, 3 * Wh, torch.bfloat16, pr=8) for _ in range(P)]
    tables = [Lean(P * Lp, 2, torch.float32, pr=4) for _ in range(P)]
    local = torch.zeros(Lp, 2, device=dev)
    for r in range(P):
        ops.gemm_sp_qkv(h[r * Lp:(r + 1) * Lp], w, bias, [b.view.data_ptr() for b in bufs], r, Lp, local)
        ops.sp_bcast_sums(local, [t.view.data_ptr() for t in tables], r, Lp)
    torch.cuda.synchronize()
    tag = f"prod gemm_sp_qkv {rid} P{P} Lp{Lp} C{C}"
    for p in range(P):
        bufs[p].check(f"{tag} receiver{p}")
        tables[p].check(f"{tag} table{p}")
        assert torch.equal(tables[p].view, tables[0].view), f"{tag}: table {p} differs from table 0"
    # receiver p, source r, row i, part, column j  ->  global row r*Lp + i, column part*C + p*Wh + j
    got = torch.stack([b.view.view(P, Lp, 3, Wh) for b in bufs]).permute(1, 2, 3, 0, 4).reshape(L, 3 * C)
    rows, cols = gemm_sp_qkv_sample(row)
    _check_gemm_sampled(got, h, w, rows, cols, EPI["BF16"], tag, "prod_sp", bias=bias)
    S = tables[0].view.double()
    for part, name in ((0, "q"), (1, "k")):
        xsq = got[:, part * C:(part + 1) * C].double().pow(2).sum(1)
        assert_within(S[:, part], xsq, KX.sumsq_bound(xsq, C), f"{tag} sum {name}^2", "prod_sp")


# ------------------------------------------------------------------------------------------------------------
# conv rows
# ------------------------------------------------------------------------------------------------------------
def conv_ref_at(x, wt, row, vox, chunk=2048):
    """fp64 acc [len(vox), Cout] and F = 2*K*u32*(|patch|.|w|) at the sampled output voxels, from the im2col rows of those
    voxels (zero outside the input for the Wan forms, the replicate-padded buffer as it is for hyvideo)."""
    kt, kh, kw = row["taps"]
    oT, oH, oW = conv_out_dims(row)
    Cp = x.shape[-1]
    K = kt * kh * kw * Cp
    wd = wt.double()
    dt, dh, dw = torch.meshgrid(torch.arange(kt), torch.arange(kh), torch.arange(kw), indexing="ij")
    dt, dh, dw = (d.flatten().to(x.device) for d in (dt, dh, dw))
    accs, Fs = [], []
    for v0 in range(0, len(vox), chunk):
        v = vox[v0:v0 + chunk].to(x.device)
        t, rem = v // (oH * oW), v % (oH * oW)
        hh, ww = rem // oW, rem % oW
        if not row["oob_zero_pad"]:
            ti, hi, wi = t[:, None] + dt, hh[:, None] + dh, ww[:, None] + dw
        elif row["stride_hw"] > 1:
            ti, hi, wi = t[:, None] + dt, 2 * hh[:, None] + dh, 2 * ww[:, None] + dw
        elif row["stride_t"] > 1:
            ti, hi, wi = 2 * t[:, None] + dt, hh[:, None] + dh, ww[:, None] + dw
        else:
            ti, hi, wi = t[:, None] + dt - (kt - 1), hh[:, None] + dh - kh // 2, ww[:, None] + dw - kw // 2
        Tn, Hn, Wn = x.shape[:3]
        ok = (ti >= 0) & (ti < Tn) & (hi >= 0) & (hi < Hn) & (wi >= 0) & (wi < Wn)
        patch = x[ti.clamp(0, Tn - 1), hi.clamp(0, Hn - 1), wi.clamp(0, Wn - 1)].double() * ok[..., None]
        patch = patch.reshape(len(v), K)
        accs.append(patch @ wd.t())
        Fs.append(2.0 * K * U32 * (patch.abs() @ wd.abs().t()))
    return torch.cat(accs), torch.cat(Fs)


@pytest.mark.parametrize("rid", _ids(_rows("conv")))
def test_prod_conv(dev, measure, rid):
    """One VAE conv launch of the table at its production size (automatic plan: box shape, kw fusion): NaN-poisoned, guarded
    output (time_conv: out_t_mul = 2 into a buffer with the other group's frames, which must stay NaN), fp64 reference on 2
    voxels of every box (conv_sample) at all Cout, bound: the GEMM's with K = taps*Cp plus one fp32 add per epilogue operand,
    then bf16 rounding for bf16 outputs."""
    from yume_b200 import ops
    row = next(r for r in PROD_TABLE if r["id"] == rid)
    measure["family"] = "prod_conv"
    plan = row_plan(row)
    T, H, W, Cp, Co, taps = row["T"], row["H"], row["W"], row["Cp"], row["Cout"], row["taps"]
    kt, kh, kw = taps
    K = kt * kh * kw * Cp
    oT, oH, oW = plan["dims"]
    g = _cuda_gen(rid)
    shape = (T, H, W) if row["oob_zero_pad"] else (T + kt - 1, H + kh - 1, W + kw - 1)
    x = _rand(g, shape[0] * shape[1] * shape[2], Cp).view(*shape, Cp)
    wt = _rand(g, Co, K, 1 / math.sqrt(K))
    epi = row["epi"]
    b = torch.randn(Co, generator=g, device=dev)
    M = oT * oH * oW
    res = _rand(g, M, Co) if epi == EPI["RES_BF16"] else None
    mul = row["out_t_mul"]
    add = row["out_t_add"]
    rows_out = ((oT - 1) * mul + add + 1) * oH * oW
    out = Lean(rows_out, Co, torch.float32 if epi == EPI["F32"] else torch.bfloat16, pr=64, pc=16)
    ops.conv3d_causal(x, wt, b, out.view, T, H, W, epi, res, taps=taps, oob_zero_pad=row["oob_zero_pad"], out_t_mul=mul,
                      out_t_add=add, stride_t=row["stride_t"], stride_hw=row["stride_hw"])
    torch.cuda.synchronize()
    tag = f"prod conv {rid} box{plan['box']} fused{plan['fused']} boxes{plan['boxes']}"
    frame_of = torch.arange(rows_out, device=dev) // (oH * oW)
    written = ((frame_of - add) % mul == 0) & (frame_of >= add)
    out.check(tag, written_rows=written if mul > 1 else None)
    if mul > 1:
        assert bool(torch.isnan(out.view[~written]).all()), tag + ": the other group's frames were written"
    vox = conv_sample(plan["dims"], plan["box"], rid)
    acc, Fb = conv_ref_at(x, wt, row, vox)
    v = vox.to(dev)
    orow = ((v // (oH * oW)) * mul + add) * oH * oW + v % (oH * oW)
    ref, bound = gemm_epilogue_ref(epi if epi != EPI["F32"] else EPI["BF16"], acc, Fb, bias=b.double()[None].expand_as(acc),
                                   res=None if res is None else res[v].double())
    if epi == EPI["F32"]:
        bound = Fb + 4 * U32 * (acc.abs() + b.double().abs())
    assert_within(out.view[orow], ref, bound, tag, "prod_conv")


# ------------------------------------------------------------------------------------------------------------
# the table against the engines' launches
# ------------------------------------------------------------------------------------------------------------
def _record(monkeypatch):
    """Recording wrappers around ops.gemm / attention / conv3d_causal (they record, then call through)."""
    from yume_b200 import ops
    calls = []
    real = dict(gemm=ops.gemm, attention=ops.attention, conv3d_causal=ops.conv3d_causal)

    def gemm(a, w, bias, out, epilogue, **kw):
        K = w.shape[1]
        flags = {f for f in ("gate", "tok_idx") if kw.get(f) is not None}
        flags |= {n for n, t in (("a_window", a.stride(0) != K and kw.get("shape") is None), ("b_window", w.stride(0) != K),
                                 ("out_window", out.stride(0) != w.shape[0] and kw.get("shape") is None)) if t}
        flags = frozenset(flags)
        calls.append(dict(entry="gemm", M=(kw.get("shape") or a.shape)[0], N=w.shape[0], K=w.shape[1], epi=epilogue,
                          flags=flags))
        return real["gemm"](a, w, bias, out, epilogue, **kw)

    def attention(q, k, v, out, heads, **kw):
        calls.append(dict(entry="attention", Lq=q.shape[0], Lk=k.shape[0], heads=heads, accumulate=bool(kw.get("accumulate"))))
        return real["attention"](q, k, v, out, heads, **kw)

    def conv3d_causal(x, w, bias, out, T, H, W, epilogue=0, res=None, taps=(3, 3, 3), oob_zero_pad=False, out_t_mul=1,
                      out_t_add=0, fuse_w=0, cta_pair=None, stride_t=1, stride_hw=1):
        calls.append(dict(entry="conv", T=T, H=H, W=W, Cp=x.shape[-1], Cout=w.shape[0], taps=tuple(taps), epi=epilogue,
                          oob_zero_pad=bool(oob_zero_pad), out_t_mul=out_t_mul, out_t_add=out_t_add, stride_t=stride_t,
                          stride_hw=stride_hw))
        return real["conv3d_causal"](x, w, bias, out, T, H, W, epilogue, res, taps, oob_zero_pad, out_t_mul, out_t_add, fuse_w,
                                     cta_pair, stride_t, stride_hw)
    monkeypatch.setattr(ops, "gemm", gemm)
    monkeypatch.setattr(ops, "attention", attention)
    monkeypatch.setattr(ops, "conv3d_causal", conv3d_causal)
    return calls


def unmatched_launches(calls, cfg):
    """Recorded launches of configuration `cfg` without a table row. GEMMs match on (N per layer, K, epilogue, flags) and
    then M (the all-layer K|V rows are recorded from a one-layer engine: N = row N / layers); attention on (Lq, Lk, heads,
    accumulate); convs on every argument that shapes the launch (the plan follows from them)."""
    rows = [r for r in PROD_TABLE if r["cfg"] == cfg]
    bad = []
    for c in calls:
        if c["entry"] == "gemm":
            ok = any(r["entry"] == "gemm" and r["N"] // r["layers"] == c["N"] and r["K"] == c["K"] and r["epi"] == c["epi"]
                     and r["flags"] == c["flags"] and r["M"] == c["M"] for r in rows)
        elif c["entry"] == "attention":
            ok = any(r["entry"] == "attention" and all(r[k] == c[k] for k in ("Lq", "Lk", "heads", "accumulate")) for r in rows)
        else:
            keys = ("T", "H", "W", "Cp", "Cout", "taps", "epi", "oob_zero_pad", "out_t_mul", "out_t_add", "stride_t",
                    "stride_hw")
            ok = any(r["entry"] == "conv" and all(r[k] == c[k] for k in keys) for r in rows)
        if not ok and c not in bad:
            bad.append(c)
    return bad


# the latents the DiT configurations run on (bench.py's workloads); production_L derives the sequence length from them by the
# engine's rules, independently of the table
DIT_LATENTS = {"5b": ("grid", 21, 44, 80), "14b_chunk": ("framepack", 13, 68, 120, 8), "14b_grid": ("grid", 21, 68, 120)}


def production_L(cfg_name):
    """Tokens of one forward: F * H/2 * W/2 on the regular grid (the callers pass seq_len = L_grid, so every row is a key);
    on the 14B FramePack path the history segments of framepack_plan plus latent_frame_zero new frames, counted as
    WanDiT._forward_eager counts them."""
    kind, F_, H, W, *rest = DIT_LATENTS[cfg_name]
    if kind == "grid":
        return F_ * (H // 2) * (W // 2)
    from yume_b200.dit import framepack_plan
    lfz = rest[0]
    n = 0
    for seg in framepack_plan(F_ - lfz, F_ - 9):                 # 14B: branch history = Ftot - 9
        f = seg.frames.stop - seg.frames.start
        hh, ww = (-(-H // 4), -(-W // 4)) if seg.pre_2x_f else (H, W)
        n += f * ((hh // 2) * (ww // 2) if seg.name == "patch_embedding" else -(-hh // seg.patch) * -(-ww // seg.patch))
    return n + lfz * (H // 2) * (W // 2)


def _dit_launches(cfg_name, monkeypatch):
    from oracle import synth
    from yume_b200.dit import WanDiT
    d = DIT_CFGS[cfg_name]
    cfg = synth.CFG_5B if cfg_name == "5b" else synth.CFG_14B
    sd = synth.make_state_dict(cfg, 1234, num_layers=1)
    kw = synth.oracle_kwargs(cfg)
    variant = kw.pop("variant")
    kw["num_layers"] = 1
    eng = WanDiT(sd, variant, device="cuda", **kw)
    del sd
    L, C = production_L(cfg_name), d["C"]                      # not the table's L: the launches must match it on their own
    g = _cuda_gen(("coverage", cfg_name))
    xs = torch.randn(L, C, generator=g, device="cuda")
    ctx = _rand(g, (N_IMG if d["img"] else 0) + TEXT_LEN, C)
    t_unique = torch.tensor([0.0, 900.0] if cfg_name == "5b" else [500.0], device="cuda")
    _, mod, _ = eng._time_tables(t_unique)
    tok_idx = (torch.arange(L, device="cuda") >= L // 3).to(torch.int32) if cfg_name == "5b" else None
    rope = eng._rope_table([(1, 1, L, 0)])
    calls = _record(monkeypatch)
    kv = eng._cross_kv(ctx)
    eng._block(0, xs, mod, tok_idx, rope, L, kv, L)
    torch.cuda.synchronize()
    monkeypatch.undo()
    return calls


def _vae_launches(cfg_name, monkeypatch):
    from oracle import hyvae, wan21vae, wan22vae
    from yume_b200 import vae, vae21, vae22
    mod, Eng, cfg, z = {
        "wan22_dec": (wan22vae, vae22.Wan22VaeDecoder, dict(dec_dim=256, z_dim=48), (48, 2, 44, 80)),
        "wan21_dec": (wan21vae, vae21.Wan21VaeDecoder, dict(dim=96, z_dim=16), (16, 2, 68, 120)),
        "hy_tile": (hyvae, vae.HyVaeDecoder, dict(), (1, 16, 2, 32, 32))}[cfg_name]
    eng = Eng(mod.make_state_dict(0, **cfg), device="cuda", **cfg)
    calls = _record(monkeypatch)
    eng.decode(torch.randn(*z, generator=torch.Generator().manual_seed(1)).cuda())
    torch.cuda.synchronize()
    monkeypatch.undo()
    return calls


@pytest.mark.parametrize("cfg_name", list(DIT_CFGS) + list(_VAE_LAUNCHES))
def test_table_covers_the_engines_launches(dev, measure, monkeypatch, cfg_name):
    """Runs one real-width, one-layer DiT block (the engine's own _block, after its all-layer cross K|V GEMM) at the table's
    L, or a VAE decoder at production spatial size with 2 latent frames, with recording wrappers around ops.gemm /
    attention / conv3d_causal: every launch must have a row in PROD_TABLE (M checked against the row's configuration)."""
    measure["family"] = "prod_coverage"
    calls = _dit_launches(cfg_name, monkeypatch) if cfg_name in DIT_CFGS else _vae_launches(cfg_name, monkeypatch)
    assert calls, "nothing was recorded"
    bad = unmatched_launches(calls, cfg_name)
    assert not bad, f"{cfg_name}: {len(bad)} launch(es) without a table row: {bad}"


COVERS = {
    "yb_gemm_bf16": ["test_prod_gemm", "test_table_covers_the_engines_launches"],
    "yb_attention_ex": ["test_prod_attention"],
    "yb_attention_sp": ["test_prod_attention_sp"],
    "yb_gemm_sp_qkv": ["test_prod_gemm_sp_qkv"],
    "yb_sp_bcast_sums": ["test_prod_gemm_sp_qkv"],
    "yb_conv3d_causal": ["test_prod_conv"],
}
