"""Per-element contract of the fp8 VAE entry points (include/yume_b200_fp8_vae.h) on the H100.

- FP8_VAE_TABLE lists every e4m3 conv launch of a real-width Wan2.2 decode (dec_dim 256) at the production 704 x 1280 output
  (latent 44 x 80, 13 latent frames): the res convs of the four levels (1024, 1024 -> 512, 512 -> 256 and their square forms),
  the three Resample Conv2d shapes, both epilogues, one-pass (t_hist 0) and after-the-first-chunk (t_hist 2) forms, plus ragged
  small shapes. test_fp8_vae_table_covers_the_engines_launches runs a real-width engine with a recording wrapper and fails on a
  launch without a row.
- yb_conv3d_fp8, every row: outputs land in a NaN-poisoned buffer whose guard rows / columns must stay NaN and whose every output
  element must be written; sampled voxels (one in every 128-voxel box of the launch's tile plan, plus the corners) are checked
  against an fp64 conv of the DEQUANTISED operands within `conv_fp8_bound`.
- yb_vae_rms_act_fp8: bit-identical to `quantize_act` (oracle/fp8.py) of what yb_vae_rms_act writes for the same arguments.

`conv_fp8_bound` is plain torch and is also exercised on the CPU (tests/test_fp8_vae_cpu.py) against a tile-by-tile model of the
kernel and its modelled defects."""
import ctypes as C

import pytest
import torch

from oracle.fp8 import quantize_act, quantize_weight
from test_gpu_kernel_contract_fp8 import ACC_BITS, ROUNDS_PER_GROUP


def conv_fp8_bound(s: torch.Tensor, groups: int, out_ulp: float, ref: torch.Tensor) -> torch.Tensor:
    """Per-element error bound of one fp8 conv launch, `gemm_bound` with taps * Cp / 128 groups: s = sum of |products| of the
    dequantised operands of the element, ref its fp64 value (bias and residual included). Each group's tensor-core sum loses at
    most ROUNDS_PER_GROUP * 2^-ACC_BITS of its sum of |products|; promotion and the epilogue add fp32 roundings; the bf16 store
    adds out_ulp * |ref|."""
    return (ROUNDS_PER_GROUP * 2.0 ** -ACC_BITS + (groups + 4) * 2.0 ** -23) * s + out_ulp * ref.abs() + 1e-30


# ------------------------------------------------------------------------------------------------------------
# the launch table
# ------------------------------------------------------------------------------------------------------------
EPI = dict(BF16=0, RES_BF16=5)
# (level, frames, H, W of the res convs, level input width, level output width, Resample of the level: (frames, H, W) of its
# Conv2d output or None) of a 13-latent-frame decode at 704 x 1280
LEVELS = [(0, 13, 44, 80, 1024, 1024, (25, 88, 160)), (1, 25, 88, 160, 1024, 1024, (49, 176, 320)),
          (2, 49, 176, 320, 1024, 512, (49, 352, 640)), (3, 49, 352, 640, 512, 256, None)]
CHUNK_T = {0: 3, 1: 6, 2: 12, 3: 12}           # frames of a later chunk at each level (t_hist = 2 rows)


def _rows():
    rows = []

    def add(rid, T, H, W, Cp, Cout, epi, t_hist, taps=(3, 3, 3)):
        rows.append(dict(id=rid, T=T, H=H, W=W, Cp=Cp, Cout=Cout, taps=taps, epi=EPI[epi], t_hist=t_hist))
    for lv, T, H, W, ci, co, rs in LEVELS:
        for th in (0, 2):
            Tr = T if th == 0 else CHUNK_T[lv]
            if ci != co:
                add(f"L{lv}.res{ci}to{co}.t{th}", Tr, H, W, ci, co, "BF16", th)
            add(f"L{lv}.res{co}.t{th}", Tr, H, W, co, co, "BF16", th)
            add(f"L{lv}.res{co}_res.t{th}", Tr, H, W, co, co, "RES_BF16", th)
        if rs is not None:
            add(f"L{lv}.resample{co}", *rs, co, co, "BF16", 0, taps=(1, 3, 3))
    add("ragged.t2", 3, 5, 7, 256, 128, "RES_BF16", 2)
    add("ragged.t0", 2, 3, 9, 128, 256, "BF16", 0)
    add("ragged.2d", 3, 6, 5, 384, 128, "RES_BF16", 0, taps=(1, 3, 3))
    return rows


FP8_VAE_TABLE = _rows()


def _row(rid):
    return next(r for r in FP8_VAE_TABLE if r["id"] == rid)


def table_key(H, W, Cp, Cout, taps, epi, t_hist):
    """What a row stands for: the frame count of a launch varies with the chunk, everything else is the launch's shape."""
    return (H, W, Cp, Cout, tuple(taps), epi, t_hist)


# ------------------------------------------------------------------------------------------------------------
# everything below needs the GPU
# ------------------------------------------------------------------------------------------------------------
gpu = pytest.mark.gpu
E4M3 = torch.float8_e4m3fn
BF = torch.bfloat16

COVERS = {
    "yb_conv3d_fp8": ["test_conv3d_fp8_per_element_at_production_shapes", "test_conv3d_fp8_rejects_bad_arguments",
                      "test_fp8_vae_table_covers_the_engines_launches"],
    "yb_vae_rms_act_fp8": ["test_vae_rms_act_fp8_bit_identical_to_twin", "test_vae_rms_act_fp8_rejects_bad_arguments"],
}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()
    return "cuda"


def quantize_volume(x_rows: torch.Tensor, T: int, H: int, W: int):
    """f32 rows [T*H*W, Cp] -> (e4m3 [T, H, W, Cp], f32 scales [T, Cp/128, H, W]) of their bf16 rounding, frame by frame."""
    Cp = x_rows.shape[1]
    q = torch.empty(T, H, W, Cp, dtype=E4M3, device=x_rows.device)
    s = torch.empty(T, Cp // 128, H, W, device=x_rows.device)
    n = H * W
    for t in range(T):
        qt, st = quantize_act(x_rows[t * n:(t + 1) * n].to(BF).float())
        q[t].copy_(qt.view(H, W, Cp))
        s[t].copy_(st.view(Cp // 128, H, W))
    return q, s


def _plan(T, H, W, Cout):
    from yume_b200 import _lib as L
    out = (C.c_int * 4)()
    assert L.load().yb_conv3d_plan(T, H, W, Cout, 3, 1, out) == 0
    return out[0], out[1], out[2]


def sample_voxels(T, H, W, Cout, gen):
    """One voxel in every TT x TH x TW box of the launch's tile plan (inside the output), plus the eight corners."""
    TW, TH, TT = _plan(T, H, W, Cout)
    nt, nh, nw = -(-T // TT), -(-H // TH), -(-W // TW)
    bt, bh, bw = torch.meshgrid(torch.arange(nt), torch.arange(nh), torch.arange(nw), indexing="ij")
    n = bt.numel()
    t = (bt.flatten() * TT + torch.randint(0, TT, (n,), generator=gen)).clamp(max=T - 1)
    h = (bh.flatten() * TH + torch.randint(0, TH, (n,), generator=gen)).clamp(max=H - 1)
    w = (bw.flatten() * TW + torch.randint(0, TW, (n,), generator=gen)).clamp(max=W - 1)
    ct, ch, cw = torch.meshgrid(torch.tensor([0, T - 1]), torch.tensor([0, H - 1]), torch.tensor([0, W - 1]), indexing="ij")
    return torch.cat([t, ct.flatten()]), torch.cat([h, ch.flatten()]), torch.cat([w, cw.flatten()])


def conv_fp8_reference(q, s, wd, bias, res, t, h, w, T, t_hist, taps):
    """fp64 (ref, sum of |products|) at output voxels (t, h, w) of the conv of the dequantised input (q, s) with wd
    [Cout, taps, Cp] (fp64): tap (dt, dh, dw) reads input frame t + t_hist - (kt - 1) + dt, row h - 1 + dh, column w - 1 + dw,
    zero outside the input."""
    kt = taps[0]
    inT, H, W, Cp = q.shape
    G = Cp // 128
    dt, dh, dw = torch.meshgrid(torch.arange(kt), torch.arange(3), torch.arange(3), indexing="ij")
    dev = q.device
    ti = (t[:, None] + t_hist - (kt - 1) + dt.flatten()[None]).to(dev)
    hi = (h[:, None] - 1 + dh.flatten()[None]).to(dev)
    wi = (w[:, None] - 1 + dw.flatten()[None]).to(dev)
    ok = (ti >= 0) & (ti < inT) & (hi >= 0) & (hi < H) & (wi >= 0) & (wi < W)
    idx = torch.where(ok, (ti * H + hi) * W + wi, torch.zeros_like(ti))
    xv = q.view(-1, Cp)[idx].double()                                          # [S, taps, Cp]
    sc = s.permute(0, 2, 3, 1).reshape(-1, G)[idx].double() * ok[..., None]    # [S, taps, G]
    xd = (xv.view(*xv.shape[:2], G, 128) * sc[..., None]).view(xv.shape[0], -1)
    wf = wd.reshape(wd.shape[0], -1)
    ref = xd @ wf.t() + bias.double()
    vox = ((t * H + h) * W + w).to(dev)
    if res is not None:
        ref = ref + res[vox].double()
    return ref, xd.abs() @ wf.abs().t()


@gpu
@pytest.mark.parametrize("rid", [r["id"] for r in FP8_VAE_TABLE])
def test_conv3d_fp8_per_element_at_production_shapes(dev, rid):
    from yume_b200 import ops
    r = _row(rid)
    T, H, W, Cp, Cout, taps, epi, th = r["T"], r["H"], r["W"], r["Cp"], r["Cout"], r["taps"], r["epi"], r["t_hist"]
    inT, n = T + th, T * H * W
    K = taps[0] * 9 * Cp
    g = torch.Generator(device=dev).manual_seed(T * 131 + H + W + Cp + Cout + epi + th)
    q = torch.empty(inT, H, W, Cp, dtype=E4M3, device=dev)
    s = torch.empty(inT, Cp // 128, H, W, device=dev)
    for t in range(inT):                                       # SiLU-like activations with a per-voxel magnitude
        x = torch.randn(H * W, Cp, device=dev, generator=g) * (0.2 + 2 * torch.rand(H * W, 1, device=dev, generator=g))
        qt, st = quantize_volume(torch.nn.functional.silu(x), 1, H, W)
        q[t], s[t] = qt[0], st[0]
    if rid == "ragged.t2":
        s[0, 0, 0, 0] = 0.0                                    # a zero group among the carried frames
        q[0, 0, 0, :128] = 0.0
    w = torch.randn(Cout, K, device=dev, generator=g) * K ** -0.5
    wq, sw = quantize_weight(w)
    del w
    bias = torch.randn(Cout, device=dev, generator=g) * 0.1
    res = torch.randn(n, Cout, device=dev, generator=g).to(BF) if epi == EPI["RES_BF16"] else None
    ldo = Cout + 32
    buf = torch.full((n + 8, ldo), float("nan"), dtype=BF, device=dev)
    out = buf[:n, :Cout]
    ops.conv3d_fp8(q, s, wq, sw, bias, out, T, H, W, th, epi, res, taps=taps)
    torch.cuda.synchronize()
    assert torch.isnan(buf[n:]).all() and torch.isnan(buf[:, Cout:]).all(), "write outside [T*H*W, Cout]"
    assert torch.isfinite(out).all(), "an output element was not written"
    wd = (wq.double() * sw.double()[:, None]).view(Cout, -1, Cp)
    t, h, w_ = sample_voxels(T, H, W, Cout, torch.Generator().manual_seed(7))
    worst = 0.0
    for i in range(0, t.numel(), 2048):
        sl = slice(i, i + 2048)
        ref, sabs = conv_fp8_reference(q, s, wd, bias, res, t[sl], h[sl], w_[sl], T, th, taps)
        got = out[((t[sl] * H + h[sl]) * W + w_[sl]).to(dev)].double()
        bound = conv_fp8_bound(sabs, K // 128, 2.0 ** -8, ref)
        worst = max(worst, float(((got - ref).abs() / bound).max()))
    print(f"{rid} T={T} H={H} W={W} Cp={Cp} Cout={Cout} taps={taps} t_hist={th}: {t.numel()} voxels, worst |err|/bound {worst:.3f}")
    assert worst <= 1.0


@gpu
def test_conv3d_fp8_rejects_bad_arguments(dev):
    from yume_b200 import _lib as L
    from yume_b200 import ops
    T, H, W, Cp, Cout = 2, 4, 6, 256, 128
    q = torch.zeros(T + 2, H, W, Cp, dtype=E4M3, device=dev)
    s = torch.zeros(T + 2, Cp // 128, H, W, device=dev)
    wq = torch.zeros(Cout, 27 * Cp, dtype=E4M3, device=dev)
    sw = torch.zeros(Cout, device=dev)
    out = torch.zeros(T * H * W, Cout, dtype=BF, device=dev)
    lib = L.load()

    def call(**kw):
        base = dict(struct_bytes=C.sizeof(L.Conv3dFp8Args), x=q.data_ptr(), x_scale=s.data_ptr(), w=wq.data_ptr(),
                    w_scale=sw.data_ptr(), bias=None, out=out.data_ptr(), res=None, ldo=Cout, res_ld=0, T=T, H=H, W=W, Cp=Cp,
                    Cout=Cout, kt=3, kh=3, kw=3, t_hist=2, epilogue=0)
        base.update(kw)
        return lib.yb_conv3d_fp8(C.byref(L.Conv3dFp8Args(**base)), ops._stream())

    assert call() == 0
    assert call(t_hist=0) == 0
    assert call(struct_bytes=8) == -1
    assert call(x=None) == -1
    assert call(t_hist=1) == -1                       # history is kt - 1 frames or none
    assert call(epilogue=2) == -1                     # F32 is not an fp8 conv epilogue
    assert call(epilogue=5) == -1                     # RES_BF16 without res
    assert call(Cp=192) == -2                         # whole 128-channel groups only
    assert call(Cout=96) == -2
    assert call(kt=3, kh=1, kw=1) == -2               # time_conv taps stay bf16
    assert call(kt=1, t_hist=2) == -1                 # a (1,3,3) conv has no history
    assert call(ldo=Cout + 4) == -3
    torch.cuda.synchronize()


@gpu
@pytest.mark.parametrize("C_,up,silu,gamma,hist", [
    (1024, 1, True, True, 0), (1024, 1, True, True, 2), (1024, 2, False, False, 0), (512, 1, True, True, 2),
    (512, 2, False, False, 0), (256, 1, True, True, 0), (256, 2, True, False, 2), (128, 1, True, True, 2),
    (128, 2, False, True, 0), (96, 1, True, True, 0), (320, 1, False, True, 2)])
def test_vae_rms_act_fp8_bit_identical_to_twin(dev, C_, up, silu, gamma, hist):
    from yume_b200 import ops
    T, Hs, Ws = 3, 22, 40
    Cp = -(-C_ // 128) * 128
    g = torch.Generator(device=dev).manual_seed(C_ + up)
    ldx = C_ + 64
    xb = (torch.randn(T * Hs * Ws, ldx, device=dev, generator=g) * torch.exp(torch.randn(T * Hs * Ws, 1, device=dev, generator=g)))
    xb = xb.to(BF)
    x = xb[:, :C_]
    x[0].zero_()                                                          # an all-zero voxel: scale 0
    gm = (1 + 0.1 * torch.randn(C_, device=dev, generator=g)) if gamma else None
    H, W = Hs * up, Ws * up
    want = torch.empty(T, H, W, Cp, dtype=BF, device=dev)
    ops.vae_rms_act(x, (T, Hs, Ws), want, gm, up, silu)
    q = torch.full((hist + T, H, W, Cp), 0x7F, dtype=torch.uint8, device=dev).view(E4M3)   # 0x7F: e4m3 NaN
    s = torch.full((hist + T, Cp // 128, H, W), float("nan"), device=dev)
    ops.vae_rms_act_fp8(x, (T, Hs, Ws), q[hist:], s[hist:], gm, up, silu)
    torch.cuda.synchronize()
    assert (q[:hist].view(torch.uint8) == 0x7F).all() and torch.isnan(s[:hist]).all(), "write before the output frames"
    tq, ts = quantize_act(want.float().view(-1, Cp))
    assert torch.equal(q[hist:].view(torch.uint8).view(-1, Cp), tq.view(torch.uint8)), "e4m3 values differ from the twin"
    got_s = s[hist:].transpose(0, 1).reshape(Cp // 128, -1)
    assert torch.equal(got_s, ts), "scales differ from the twin"
    assert float(got_s[:, 0].abs().max()) == 0.0


@gpu
def test_vae_rms_act_fp8_rejects_bad_arguments(dev):
    from yume_b200 import _lib as L
    from yume_b200 import ops
    lib = L.load()
    x = torch.zeros(2 * 4 * 4, 256, dtype=BF, device=dev)
    q = torch.zeros(2, 4, 4, 256, dtype=E4M3, device=dev)
    s = torch.zeros(2, 2, 4, 4, device=dev)

    def call(C_=256, Cp=256, up=1, out_scale=True):
        return lib.yb_vae_rms_act_fp8(x.data_ptr(), 256, q.data_ptr(), s.data_ptr() if out_scale else None, None, 2, 4, 4, C_, Cp,
                                      up, 1, ops._stream())
    assert call() == 0
    assert call(Cp=192) == -2                          # not whole 128-channel groups
    assert call(C_=96, Cp=256) == -2                   # Cp must be rup(C, 128)
    assert call(up=3) == -2
    assert call(out_scale=False) == -1
    torch.cuda.synchronize()


@gpu
def test_fp8_vae_table_covers_the_engines_launches(dev, monkeypatch):
    """A real-width engine (dec_dim 256) decodes a 3-frame latent at the production 44 x 80 in chunks [1, 2] (one-pass forms
    in the first chunk, history forms in the second) with a recording wrapper around ops.conv3d_fp8: every launch must have a
    table row."""
    from oracle import wan22vae
    from yume_b200 import ops, vae22
    eng = vae22.Wan22VaeDecoder(wan22vae.make_state_dict(0, dec_dim=256, z_dim=48), dec_dim=256, z_dim=48, device=dev,
                                precision="fp8")
    calls = []
    real = ops.conv3d_fp8

    def rec(x, x_scale, w, w_scale, bias, out, T, H, W, t_hist=0, epilogue=0, res=None, taps=(3, 3, 3)):
        calls.append(table_key(H, W, x.shape[-1], w.shape[0], taps, epilogue, t_hist))
        return real(x, x_scale, w, w_scale, bias, out, T, H, W, t_hist, epilogue, res, taps)
    monkeypatch.setattr(ops, "conv3d_fp8", rec)
    z = torch.randn(48, 3, 44, 80, generator=torch.Generator().manual_seed(1)).to(dev)
    out = eng._decode_chunks(z, [1, 2])
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    rows = {table_key(r["H"], r["W"], r["Cp"], r["Cout"], r["taps"], r["epi"], r["t_hist"]) for r in FP8_VAE_TABLE}
    assert calls
    missing = sorted(set(calls) - rows)
    print(f"{len(calls)} fp8 conv launches, {len(set(calls))} distinct")
    assert not missing, f"launches without a table row: {missing}"
