"""CPU side of Wan22VaeDecoder(precision="fp8") (include/yume_b200_fp8_vae.h):
  * the activation twin and its layout (tests/helpers/torch_ops_fp8_vae.py);
  * the engine's fp8 host logic over torch stand-ins for the two new ops, against the fp8-qdq oracle (oracle/wan22vae_fp8.py) on
    the wan22vae_tiny cases, one-pass and streamed;
  * the per-conv rule at tiny and at real width, the precision switches and their rejections;
  * the C-ABI guards (header symbols bound, struct layout, a contract test per entry point);
  * the GPU contract's conv bound against a tile-by-tile model of the kernel and five modelled defects."""
import math
import re
import types
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

import test_gpu_kernel_contract_fp8_vae as KV
from helpers import torch_ops_fp8_vae
from oracle import wan21vae, wan22vae
from oracle.fp8 import quantize_act, quantize_weight
from oracle.wan22vae_fp8 import Wan22VaeOracleFp8, converted
from test_fp8_cpu import _truncate
from test_kernel_contract_cpu import _entry_problems
from yume_b200 import vae21, vae22, vae_enc
from yume_b200._lib import YumeB200Error

HEADER = Path(__file__).resolve().parents[1] / "include" / "yume_b200_fp8_vae.h"
E4M3 = torch.float8_e4m3fn


def psnr(a, b):
    mse = float((a.double() - b.double()).pow(2).mean())
    return math.inf if mse == 0 else 10 * math.log10(4.0 / mse)


# ------------------------------------------------------------------------------------------------------------
# the activation twin
# ------------------------------------------------------------------------------------------------------------
def test_rms_act_fp8_twin_layout_and_zero_groups():
    """Frame-major scales [T, Cp/128, H, W]; channels past C and all-zero groups are zero with scale 0; the values are
    quantize_act of what vae_rms_act writes."""
    T, Hs, Ws, C, Cp = 2, 3, 4, 200, 256
    g = torch.Generator().manual_seed(0)
    x = torch.randn(T * Hs * Ws, C, generator=g).to(torch.bfloat16)
    x[5].zero_()
    q = torch.empty(T, 2 * Hs, 2 * Ws, Cp, dtype=E4M3)
    s = torch.empty(T, Cp // 128, 2 * Hs, 2 * Ws)
    torch_ops_fp8_vae.vae_rms_act_fp8(x, (T, Hs, Ws), q, s, None, 2, True)
    bf = torch.empty(T, 2 * Hs, 2 * Ws, Cp, dtype=torch.bfloat16)
    torch_ops_fp8_vae.torch_ops.vae_rms_act(x, (T, Hs, Ws), bf, None, 2, True)
    for t in range(T):                                    # each frame of both is its own block
        tq, ts = quantize_act(bf[t].float().reshape(-1, Cp))
        assert torch.equal(q[t].view(torch.uint8).reshape(-1, Cp), tq.view(torch.uint8))
        assert torch.equal(s[t].reshape(Cp // 128, -1), ts)
    assert (q[..., C:].view(torch.uint8) == 0).all()
    v5 = (0, 1, 2)                                        # voxel 5 of frame 0 (row 1, column 1) upsampled to rows 2-3, columns 2-3
    assert float(s[v5[0], :, 2:4, 2:4].abs().max()) == 0.0
    back = torch_ops_fp8_vae.dequantize_frames(q, s)
    assert float((back - bf.float()).abs().max()) <= float(bf.float().abs().max()) * 2 ** -4


# ------------------------------------------------------------------------------------------------------------
# the engine's fp8 host logic
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def cpu_ops(monkeypatch):
    monkeypatch.setattr(vae22, "ops", torch_ops_fp8_vae)
    torch_ops_fp8_vae.calls.clear()


def _tiny(golden_dir):
    g = torch.load(golden_dir / "wan22vae_tiny.pt", weights_only=False)
    return g, wan22vae.make_state_dict(g["seed_w"], **g["cfg"])


# Measured over the four cases (engine over the stand-ins vs the fp8-qdq oracle): rel-Frobenius 4.8e-2 .. 5.3e-2, PSNR 39.0 ..
# 43.5 dB, short of the bf16 engine's bars (3e-2, 40 dB). The engine quantises the bf16 values of its own bf16 layer chain, the
# oracle those of its fp32 chain: a last-bit bf16 difference moves a value across an e4m3 rounding boundary (3 mantissa bits,
# a 6 % step), and 18 converted convs in a row compound these whole-step flips. The fp8-qdq oracle is itself 6e-2 from the
# fp32 oracle at this width. The kernels' own numerics are pinned per element by the GPU contract; this test checks the wiring.
QDQ_BAR = 8e-2
PSNR_BAR = 36.0


@pytest.mark.parametrize("case", ["t1", "t2", "t5", "t3_wide"])
def test_fp8_host_logic_matches_the_oracle(cpu_ops, golden_dir, case):
    g, sd = _tiny(golden_dir)
    c = g["cases"][case]
    eng = vae22.Wan22VaeDecoder(sd, mean=g["mean"], std=g["std"], device="cpu", precision="fp8", **g["cfg"])
    z = torch.randn(g["cfg"]["z_dim"], c["T"], c["H"], c["W"], generator=torch.Generator().manual_seed(c["seed"]))
    got = eng.decode(z)
    want = Wan22VaeOracleFp8(sd, mean=g["mean"], std=g["std"], **g["cfg"]).decode(z)
    rel, p = float((got - want).norm() / want.norm()), psnr(got, want)
    print(f"{case}: fp8 host logic vs fp8 oracle rel {rel:.2e}, PSNR {p:.1f} dB")
    assert "conv3d_fp8" in torch_ops_fp8_vae.calls and "vae_rms_act_fp8" in torch_ops_fp8_vae.calls
    assert rel < QDQ_BAR and p >= PSNR_BAR
    if case == "t5":                                      # one streamed partition: carried e4m3 frames and scales
        torch_ops_fp8_vae.calls.clear()
        out = eng._decode_chunks(z, [2, 3])
        assert "conv3d_causal_hist" in torch_ops_fp8_vae.calls
        assert float((out - got).norm() / got.norm()) < 2e-2      # the bar of the bf16 streaming host test


def test_streamed_fp8_stream_carries_value_and_scale_frames(cpu_ops, golden_dir, monkeypatch):
    """After the first chunk every converted conv reads its carried frames: a (values, scales) pair of HIST frames each."""
    g, sd = _tiny(golden_dir)
    eng = vae22.Wan22VaeDecoder(sd, mean=g["mean"], std=g["std"], device="cpu", precision="fp8", **g["cfg"])
    seen = []
    real = torch_ops_fp8_vae.conv3d_fp8

    def spy(x, x_scale, *a, **k):
        seen.append((x.shape[0] - a[4], x_scale.shape[0] == x.shape[0]))     # a[4] = T
        return real(x, x_scale, *a, **k)
    monkeypatch.setattr(torch_ops_fp8_vae, "conv3d_fp8", spy)
    z = torch.randn(g["cfg"]["z_dim"], 3, 4, 8, generator=torch.Generator().manual_seed(1))
    eng._decode_chunks(z, [1, 2])
    hist = {h for h, _ in seen}
    assert hist == {0, 2} and all(ok for _, ok in seen)


def _rule(dec_dim):
    shapes = vae22.decoder_param_shapes(dec_dim=dec_dim, z_dim=48)
    out = set()
    for k, shp in shapes.items():
        if k.endswith(".weight") and len(shp) in (4, 5) and tuple(shp[2:]) != (1, 1, 1) and "to_qkv" not in k and ".proj." not in k:
            name, co, ci = k[:-7], shp[0], shp[1]
            if name.endswith(".time_conv"):
                co //= 2
            if vae22.fp8_conv(name, -(-ci // 64) * 64, -(-co // 32) * 32):
                out.add(name)
            assert converted(name, ci, co) == (name in out), name          # the oracle restates the same rule
    return out, shapes


def test_per_conv_rule_at_real_and_tiny_width():
    conv8, shapes = _rule(256)
    want = {k[:-7] for k in shapes if k.endswith((".residual.2.weight", ".residual.6.weight", ".resample.1.weight"))}
    assert conv8 == want and len(want) == 2 * 14 + 3                 # every res conv and every Resample Conv2d at real width
    tiny, _ = _rule(32)                                               # dims 128, 128, 128, 64, 32: levels 0-1 convert, 2-3 do not
    assert "decoder.middle.0.residual.2" in tiny and "decoder.upsamples.1.upsamples.3.resample.1" in tiny
    assert "decoder.upsamples.2.upsamples.0.residual.2" not in tiny and "decoder.upsamples.3.upsamples.1.residual.6" not in tiny
    assert not any(n.endswith((".time_conv", ".shortcut")) or n in ("decoder.conv1", "decoder.head.2") for n in conv8 | tiny)


def test_engine_applies_the_rule_once_and_keeps_no_bf16_copy(cpu_ops, golden_dir):
    g, sd = _tiny(golden_dir)
    eng = vae22.Wan22VaeDecoder(sd, mean=g["mean"], std=g["std"], device="cpu", precision="fp8", **g["cfg"])
    tiny, _ = _rule(32)
    assert set(eng.conv8) == tiny and not set(eng.conv) & tiny
    for wq, sw, b, taps in eng.conv8.values():
        assert wq.dtype == E4M3 and sw.dtype == torch.float32 and wq.shape[1] % 128 == 0
    name = "decoder.middle.0.residual.2"
    w = sd[name + ".weight"]
    tq, ts = quantize_weight(w.to(torch.bfloat16).float().permute(0, 2, 3, 4, 1).reshape(w.shape[0], -1))
    assert torch.equal(eng.conv8[name][1], ts)
    bf = vae22.Wan22VaeDecoder(sd, mean=g["mean"], std=g["std"], device="cpu", **g["cfg"])
    assert bf.precision == "bf16" and not bf.conv8


def _stub_vae(which):
    cfg = dict(dim=32, z_dim=16) if which == "wan21" else dict(dec_dim=32, z_dim=16)
    return cfg


def test_precision_rejections():
    sd21 = wan21vae.make_state_dict(0, dim=32, z_dim=16)
    with pytest.raises(YumeB200Error, match="fp8 path is Wan22VaeDecoder"):
        vae21.Wan21VaeDecoder(sd21, dim=32, z_dim=16, device="cpu", precision="fp8")
    m = types.SimpleNamespace(state_dict=lambda: sd21, dim=32, z_dim=16, dim_mult=[1, 2, 4, 4], num_res_blocks=2,
                              temperal_upsample=[True, True, False], temperal_downsample=[False, True, True])
    vae = types.SimpleNamespace(model=m, mean=torch.zeros(16), std=torch.ones(16))
    with pytest.raises(YumeB200Error, match="precision"):
        vae21.install_wan21_vae(vae, device="cpu", precision="fp8")
    with pytest.raises(YumeB200Error, match="precision"):
        vae_enc.install_wan21_vae_encoder(vae, device="cpu", precision="fp8")
    for Enc, kw in ((vae_enc.Wan22VaeEncoder, dict(dim=32, z_dim=16)), (vae_enc.Wan21VaeEncoder, dict(dim=32, z_dim=16))):
        with pytest.raises(YumeB200Error, match="fp8 path is Wan22VaeDecoder"):
            Enc({}, device="cpu", precision="fp8", **kw)
    with pytest.raises(YumeB200Error, match="'bf16' or 'fp8'"):
        vae22.Wan22VaeDecoder({}, dec_dim=32, z_dim=16, device="cpu", precision="int8")


# ------------------------------------------------------------------------------------------------------------
# C-ABI guards over include/yume_b200_fp8_vae.h
# ------------------------------------------------------------------------------------------------------------
def test_fp8_vae_header_symbols_are_bound():
    from yume_b200 import _lib
    declared = set(re.findall(r"^\s*(?:int|long long)\s+(yb_\w+)\s*\(", HEADER.read_text(), flags=re.M))
    assert declared == set(_lib.FP8_VAE_SIGNATURES) == {"yb_conv3d_fp8", "yb_vae_rms_act_fp8"}
    others = (set(_lib.SIGNATURES) | set(_lib.CLIP_SIGNATURES) | set(_lib.T5_SIGNATURES) | set(_lib.STREAM_SIGNATURES)
              | set(_lib.FP8_SIGNATURES) | set(_lib.FP8_ATTN_SIGNATURES))
    assert not declared & others


def test_conv_fp8_args_mirror_the_header_struct():
    """Field names in header order, one ctypes field per declarator, struct_bytes first (the library refuses another size)."""
    from yume_b200 import _lib
    body = re.search(r"typedef struct yb_conv3d_fp8_args \{(.*?)\} yb_conv3d_fp8_args;", HEADER.read_text(), re.S).group(1)
    names = []
    for line in body.split("\n"):
        decl = re.sub(r"/\*.*?(\*/|$)", "", line).strip()
        m = re.match(r"^(?:const\s+)?(?:unsigned|int|long long|void\*)\s+(.*);$", decl)
        if m:
            names += [re.sub(r"[*\s]", "", n) for n in m.group(1).split(",")]
    assert names == [f[0] for f in _lib.Conv3dFp8Args._fields_] and names[0] == "struct_bytes"


def test_every_fp8_vae_entry_point_has_a_contract_test():
    assert _entry_problems(HEADER, modules=(KV,)) == []


def test_fp8_vae_entry_point_guard_notices_a_missing_test(monkeypatch):
    covers = dict(KV.COVERS)
    del covers["yb_conv3d_fp8"]
    monkeypatch.setattr(KV, "COVERS", covers)
    assert _entry_problems(HEADER, modules=(KV,)) == ["entry point without a contract test: yb_conv3d_fp8"]


def test_table_rows_are_the_converted_convs_of_a_real_width_decode():
    conv8, _ = _rule(256)
    keys = {KV.table_key(r["H"], r["W"], r["Cp"], r["Cout"], r["taps"], r["epi"], r["t_hist"]) for r in KV.FP8_VAE_TABLE}
    assert (44, 80, 1024, 1024, (3, 3, 3), 5, 2) in keys and (352, 640, 512, 512, (1, 3, 3), 0, 0) in keys
    assert len(conv8) == 31


# ------------------------------------------------------------------------------------------------------------
# the GPU contract's conv bound against a tile-by-tile model of the kernel
# ------------------------------------------------------------------------------------------------------------
T_, H_, W_, CP, CO, TH_ = 3, 4, 5, 256, 8, 2           # a later chunk: two carried frames in front


def _operands(positive):
    g = torch.Generator().manual_seed(3)
    x = torch.randn((TH_ + T_) * H_ * W_, CP, generator=g) * (0.3 + 2 * torch.rand((TH_ + T_) * H_ * W_, 1, generator=g))
    w = torch.randn(CO, 27 * CP, generator=g) / math.sqrt(27 * CP)
    if positive:                                        # all products positive: where an unpromoted accumulator's truncations add up
        x, w = x.abs() + 0.5, w.abs() + 0.5 / math.sqrt(27 * CP)
    q, s = torch_ops_fp8_vae.quantize_frames(x.to(torch.bfloat16).view(TH_ + T_, H_, W_, CP))
    wq, sw = quantize_weight(w)
    return q, s, wq, sw, 0.1 * torch.randn(CO, generator=g)


def _kernel_model(q, s, wq, sw, bias, defect=None):
    """The kernel per output voxel in fp64: for every (tap, g) the inner sum over 128 channels in four k32 steps, each truncated
    to ACC_BITS; promotion acc += s_a[tap-shifted voxel, g] * inner; out = bf16(acc * s_w + bias). Padded voxels read zeros."""
    bits = KV.ACC_BITS
    inT = TH_ + T_
    qd, sd = q.double(), s.double()
    wd = wq.double().view(CO, 27, CP)
    out = torch.zeros(T_ * H_ * W_, CO, dtype=torch.float64)
    for t in range(T_):
        for h in range(H_):
            for w in range(W_):
                acc = torch.zeros(CO, dtype=torch.float64)
                for tap in range(27):
                    dt, dh, dw = tap // 9, (tap // 3) % 3, tap % 3
                    ti, hi, wi = t + dt, h - 1 + dh, w - 1 + dw          # t_hist = kt - 1: input frame t + dt
                    inside = 0 <= ti < inT and 0 <= hi < H_ and 0 <= wi < W_
                    for g in range(CP // 128):
                        if inside:
                            a = qd[ti, hi, wi, g * 128:(g + 1) * 128]
                            sa = float(sd[ti, g, hi, wi])
                        else:
                            a = torch.zeros(128, dtype=torch.float64)
                            sa = float("nan") if defect == "nonzero_padded_scale" else 0.0
                        if defect == "unshifted_scale":
                            sa = float(sd[t + 2, g, h, w])
                        if defect == "no_act_scale":
                            sa = 1.0
                        if defect == "no_promotion":             # one tensor-core accumulator across every group
                            for c in range(0, 128, 32):
                                acc = _truncate(acc + sa * (wd[:, tap, g * 128 + c:g * 128 + c + 32] @ a[c:c + 32]), bits)
                            continue
                        inner = torch.zeros(CO, dtype=torch.float64)
                        for c in range(0, 128, 32):
                            inner = _truncate(inner + wd[:, tap, g * 128 + c:g * 128 + c + 32] @ a[c:c + 32], bits)
                        acc = acc + sa * inner
                f = 1.0 if defect == "no_weight_scale" else sw.double()
                out[(t * H_ + h) * W_ + w] = acc * f + bias.double()
    return out.float().to(torch.bfloat16).double()


@pytest.mark.parametrize("defect", [None, "no_act_scale", "unshifted_scale", "no_weight_scale", "no_promotion",
                                    "nonzero_padded_scale"])
def test_conv_bound_accepts_the_kernel_model_and_rejects_defects(defect):
    q, s, wq, sw, bias = _operands(positive=defect == "no_promotion")
    wd = (wq.double() * sw.double()[:, None]).view(CO, 27, CP)
    t, h, w = torch.meshgrid(torch.arange(T_), torch.arange(H_), torch.arange(W_), indexing="ij")
    t, h, w = t.flatten(), h.flatten(), w.flatten()
    ref, sabs = KV.conv_fp8_reference(q, s, wd, bias, None, t, h, w, T_, TH_, (3, 3, 3))
    bound = KV.conv_fp8_bound(sabs, 27 * CP // 128, 2.0 ** -8, ref)
    got = _kernel_model(q, s, wq, sw, bias, defect)
    ratio = float(((got - ref).abs() / bound).max()) if torch.isfinite(got).all() else math.inf
    print(f"{defect}: worst |err|/bound {ratio:.3f}")
    if defect is None:
        assert ratio <= 1.0
    else:
        assert ratio > 1.0
