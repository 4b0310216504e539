"""Per-element contract of include/yume_b200_vae_rows.h on one H100 (`-m gpu`), at the band shapes a row-parallel decode
launches on P = 2, 4 and 8 ranks (Wan2.2 at 704x1280: latent 44x80 and every level up to 352x640; Wan2.1 at 544x960):
  * the row-halo conv, one-pass (one and two frames) and history forms, into NaN-poisoned outputs with guard bands: the band's first, middle and last
    rows against an fp64 convolution of the same bf16 operands, and every element `torch.equal` to the same rows of the
    full-height launch (yb_conv3d_causal / yb_conv3d_causal_hist) on the input the band was cut from;
  * a recording decode on every band size fails on a launch without a row in the table;
  * the band norm pass, the halo pack / unpack and the two band tails exactly against their full-height twins, rows they must
    not write left NaN."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()
    return "cuda"


def _bands(H, P):
    return [(r * H // P, (r + 1) * H // P) for r in range(P)]


# (latent H, W, [(level, taps, Cp, Cout, epilogue)]): every conv with kh = 3 of the two decoders; level k runs at 2^k x the
# latent size. 0 = BF16, 2 = F32 (the heads), 5 = RES_BF16 (the second conv of a residual block)
DECODERS = {
    "wan22": (44, 80, [(0, (3, 3, 3), 64, 1024, 0), (0, (3, 3, 3), 1024, 1024, 0), (0, (3, 3, 3), 1024, 1024, 5),
                       (1, (1, 3, 3), 1024, 1024, 0), (1, (3, 3, 3), 1024, 1024, 0), (1, (3, 3, 3), 1024, 1024, 5),
                       (2, (1, 3, 3), 1024, 1024, 0), (2, (3, 3, 3), 1024, 512, 0), (2, (3, 3, 3), 512, 512, 0),
                       (2, (3, 3, 3), 512, 512, 5), (3, (1, 3, 3), 512, 512, 0), (3, (3, 3, 3), 512, 256, 0),
                       (3, (3, 3, 3), 256, 256, 0), (3, (3, 3, 3), 256, 256, 5), (3, (3, 3, 3), 256, 32, 2)]),
    "wan21": (68, 120, [(0, (3, 3, 3), 64, 384, 0), (0, (3, 3, 3), 384, 384, 0), (0, (3, 3, 3), 384, 384, 5),
                        (1, (1, 3, 3), 384, 192, 0), (1, (3, 3, 3), 192, 384, 0), (1, (3, 3, 3), 384, 384, 0),
                        (1, (3, 3, 3), 384, 384, 5), (2, (1, 3, 3), 384, 192, 0), (2, (3, 3, 3), 192, 192, 0),
                        (2, (3, 3, 3), 192, 192, 5), (3, (1, 3, 3), 192, 96, 0), (3, (3, 3, 3), 128, 96, 0),
                        (3, (3, 3, 3), 128, 96, 5), (3, (3, 3, 3), 128, 32, 2)]),
}

# (taps, H, band rows, W, Cp, Cout, epilogue, first row, P): one row per band size of every conv, P = 2, 4, 8, the band of an
# interior rank where there is one (both halos are then a neighbour's rows)
BAND_ROWS = []
for _H0, _W0, _convs in DECODERS.values():
    for _lvl, _taps, _cp, _co, _epi in _convs:
        _seen = set()
        for _P in (2, 4, 8):
            for _r, (_a, _b) in sorted(enumerate(_bands(_H0, _P)), key=lambda rb: (rb[0] in (0, _P - 1), rb[0])):
                if (_b - _a) not in _seen:
                    _seen.add(_b - _a)
                    s = 2 ** _lvl
                    BAND_ROWS.append((_taps, _H0 * s, (_b - _a) * s, _W0 * s, _cp, _co, _epi, _a * s, _P))


def _row_id(r):
    return "x".join(map(str, r[0])) + f"_{r[1]}-{r[2]}x{r[3]}_c{r[4]}-{r[5]}_e{r[6]}_p{r[8]}at{r[7]}"


@pytest.mark.parametrize("hist,T", [(0, 2), (0, 1), (1, 2)], ids=["one_pass", "one_frame", "hist"])
@pytest.mark.parametrize("row", BAND_ROWS, ids=_row_id)
def test_conv_rows_contract(dev, row, hist, T):
    import torch.nn.functional as F
    from yume_b200 import ops
    taps, H, hs, W, Cp, Cout, epi, r0_lvl, P = row
    kt, kh, kw = taps
    t_hist = (kt - 1) if hist else 0
    if hist and kt == 1:
        pytest.skip("a (1,3,3) conv carries no frames")
    r0 = r0_lvl
    g = torch.Generator(device="cuda").manual_seed(7)
    seq = torch.randn(t_hist + T, H, W, Cp, device="cuda", generator=g).to(BF)
    w = (torch.randn(Cout, kt * kh * kw * Cp, device="cuda", generator=g) / (kt * kh * kw * Cp) ** 0.5).to(BF)
    b = torch.randn(Cout, device="cuda", generator=g)
    full_res = torch.randn(T * H * W, Cout, device="cuda", generator=g).to(BF) if epi == ops.YB_EPI_RES_BF16 else None
    odt = torch.float32 if epi == ops.YB_EPI_F32 else BF
    # the band buffer cut from the full input: own rows, the neighbours' rows as halos, zeros at the image's edge
    buf = torch.zeros(t_hist + T, hs + 2, W, Cp, device="cuda", dtype=BF)
    lo, hi = max(r0 - 1, 0), min(r0 + hs + 1, H)
    buf[:, lo - (r0 - 1):hi - (r0 - 1)] = seq[:, lo:hi]
    res = None if full_res is None else full_res.view(T, H, W, Cout)[:, r0:r0 + hs].reshape(-1, Cout).contiguous()
    rows = T * hs * W
    guard = 2 * W
    out = torch.full((guard + rows + guard, Cout), float("nan"), device="cuda", dtype=odt)
    ops.conv3d_rows(buf, w, b, out[guard:guard + rows], T, hs, W, t_hist, epi, res, taps=taps, full_h=H)
    assert torch.isnan(out[:guard]).all() and torch.isnan(out[-guard:]).all(), "write outside the output"
    got = out[guard:guard + rows].view(T, hs, W, Cout)
    # bit identity with the full-height launch
    full = torch.empty(T * H * W, Cout, device="cuda", dtype=odt)
    if t_hist:
        ops.conv3d_causal_hist(seq, w, b, full, T, H, W, t_hist, epi, full_res, taps=taps)
    else:
        ops.conv3d_causal(seq, w, b, full, T, H, W, epi, full_res, taps=taps, oob_zero_pad=True)
    assert torch.equal(got, full.view(T, H, W, Cout)[:, r0:r0 + hs])
    # fp64 bound on the band's first, middle and last rows
    wt = w.double().view(Cout, kt, kh, kw, Cp).permute(0, 4, 1, 2, 3)
    for h in sorted({0, hs // 2, hs - 1}):
        xn = F.pad(buf[:, h:h + 3].double().permute(3, 0, 1, 2)[None], (kw // 2, kw // 2, 0, 0, kt - 1 - t_hist, 0))
        ref = F.conv3d(xn, wt, b.double())[0].permute(1, 2, 3, 0)[:, 0]
        mag = F.conv3d(xn.abs(), wt.abs(), b.double().abs())[0].permute(1, 2, 3, 0)[:, 0]
        if res is not None:
            ref = ref + res.view(T, hs, W, Cout)[:, h].double()
            mag = mag + res.view(T, hs, W, Cout)[:, h].double().abs()
        ulp = 2.0 ** -24 if odt == torch.float32 else 2.0 ** -8
        bound = ulp * ref.abs() + kt * kh * kw * Cp * 2.0 ** -23 * mag + 1e-30
        ratio = float(((got[:, h].double() - ref).abs() / bound).max())
        assert ratio <= 1.0, (h, ratio)


class _Ranks:
    """A RowGroup stand-in for one rank of P in one process: halo rows and gathered bands are zeros (the launches' shapes are
    those of the real decode)."""

    def __init__(self, P, rank):
        self.world, self.rank = P, rank

    def band(self, H, r=None):
        return _bands(H, self.world)[self.rank if r is None else r]

    def sizes(self, H):
        return [b - a for a, b in _bands(H, self.world)]

    def exchange(self, send):
        return (None if self.rank == 0 else torch.zeros_like(send[0]),
                None if self.rank == self.world - 1 else torch.zeros_like(send[1]))

    def gather(self, x, dim, sizes):
        out = []
        for r, s in enumerate(sizes):
            shape = list(x.shape)
            shape[dim] = s
            out.append(x if r == self.rank else torch.zeros(shape, dtype=x.dtype, device=x.device))
        return out

    def min_int(self, v):
        return v


@pytest.mark.parametrize("which", ["wan22", "wan21"])
def test_table_covers_the_band_launches(dev, monkeypatch, which):
    """Decodes of every band size (one pass and 3 chunks) with a recording wrapper around ops.conv3d_rows: every launch must
    have a row in BAND_ROWS."""
    from yume_b200 import ops, vae21, vae22
    table = {(t, hs, W, cp, co, e) for t, H, hs, W, cp, co, e, _, _ in BAND_ROWS}
    seen = []
    real = ops.conv3d_rows

    def record(xbuf, w, bias, out, T, H, W, t_hist=0, epilogue=ops.YB_EPI_BF16, res=None, taps=(3, 3, 3), full_h=None):
        seen.append((tuple(taps), H, W, xbuf.shape[-1], w.shape[0], epilogue))
        return real(xbuf, w, bias, out, T, H, W, t_hist, epilogue, res, taps, full_h)
    monkeypatch.setattr(ops, "conv3d_rows", record)
    zero = lambda shapes: {k: torch.zeros(v) for k, v in shapes.items()}             # noqa: E731
    if which == "wan22":
        eng, zd, (H, W) = vae22.Wan22VaeDecoder(zero(vae22.decoder_param_shapes()), device=dev), 48, DECODERS["wan22"][:2]
    else:
        eng, zd, (H, W) = vae21.Wan21VaeDecoder(zero(vae21.decoder_param_shapes()), device=dev), 16, DECODERS["wan21"][:2]
    z = torch.zeros(zd, 3, H, W, device=dev)
    for P in (2, 4, 8):
        done = set()
        for r, (a, b) in enumerate(_bands(H, P)):
            if (b - a, r in (0, P - 1)) in done:
                continue
            done.add((b - a, r in (0, P - 1)))
            eng._rows = _Ranks(P, r)
            eng._band = (a, b - a, H)
            for parts in ([3], [1, 1, 1]):
                eng._decode_chunks(z, parts)
    torch.cuda.synchronize()
    assert seen, "no row-halo launch"
    missing = sorted(set(seen) - table)
    assert not missing, missing


@pytest.mark.parametrize("T,Hs,Ws,C,up", [(2, 5, 80, 1024, 1), (2, 6, 80, 1024, 2), (2, 11, 160, 1024, 2), (2, 22, 320, 512, 2),
                                          (2, 44, 640, 256, 1), (3, 1, 120, 384, 1), (2, 9, 120, 384, 2), (2, 17, 480, 96, 1)])
def test_rms_act_rows_exact(dev, T, Hs, Ws, C, up):
    """The band norm pass writes rows 1 .. Hs*up exactly as yb_vae_rms_act writes the dense frames, leaves the halo rows alone,
    and its send rows are the first and last written rows."""
    from yume_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    Cp = (C + 63) // 64 * 64
    x = torch.randn(T * Hs * Ws, C, device="cuda", generator=g).to(BF)
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    dense = torch.empty(T, Hs * up, Ws * up, Cp, device="cuda", dtype=BF)
    ops.vae_rms_act(x, (T, Hs, Ws), dense, gamma, up, True)
    buf = torch.full((T, Hs * up + 2, Ws * up, Cp), float("nan"), device="cuda", dtype=BF)
    send = torch.full((2, T, Ws * up, Cp), float("nan"), device="cuda", dtype=BF)
    ops.vae_rms_act_rows(x, (T, Hs, Ws), buf, gamma, up, True, send=send)
    assert torch.equal(buf[:, 1:-1], dense)
    assert torch.isnan(buf[:, 0]).all() and torch.isnan(buf[:, -1]).all()
    assert torch.equal(send[0], dense[:, 0]) and torch.equal(send[1], dense[:, -1])
    # pack reads the same rows back; unpack fills the halos (zeros for an edge)
    packed = torch.full_like(send, float("nan"))
    ops.vae_rows_pack(buf, packed)
    assert torch.equal(packed, send)
    top = torch.randn(T, Ws * up, Cp, device="cuda", generator=g).to(BF)
    ops.vae_rows_unpack(top, None, buf)
    assert torch.equal(buf[:, 0], top) and not buf[:, -1].any() and torch.equal(buf[:, 1:-1], dense)


@pytest.mark.parametrize("T,H,W,r0,hs", [(3, 44, 80, 11, 11), (2, 44, 80, 38, 6), (2, 8, 12, 0, 3)])
def test_unpatchify2_clamp_rows_exact(dev, T, H, W, r0, hs):
    from yume_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(4)
    y = torch.randn(T * H * W, 32, device="cuda", generator=g) * 2
    want = torch.empty(3, T, 2 * H, 2 * W, device="cuda")
    ops.vae_unpatchify2_clamp(y, want, T, H, W)
    video = torch.full((3, T + 2, 2 * H, 2 * W), float("nan"), device="cuda")
    band = y.view(T, H, W, 32)[:, r0:r0 + hs].reshape(-1, 32).contiguous()
    ops.vae_unpatchify2_clamp_rows(band, video[:, 1:T + 1, 2 * r0:2 * (r0 + hs)], T, hs, W)
    assert torch.equal(video[:, 1:T + 1, 2 * r0:2 * (r0 + hs)], want[:, :, 2 * r0:2 * (r0 + hs)])
    video[:, 1:T + 1, 2 * r0:2 * (r0 + hs)] = 0
    assert torch.isnan(video[:, 1:T + 1]).sum() == 3 * T * 2 * (H - hs) * 2 * W and torch.isnan(video[:, 0]).all()


@pytest.mark.parametrize("T,H,W,r0,hs", [(3, 544, 960, 136, 136), (2, 544, 960, 472, 72), (2, 8, 12, 5, 3)])
def test_nhwc_to_nchw_f32_clamp_rows_exact(dev, T, H, W, r0, hs):
    from yume_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(T * H * W, 32, device="cuda", generator=g) * 2
    want = torch.empty(3, T, H, W, device="cuda")
    ops.nhwc_to_nchw_f32_win(x, want, (-1.0, 1.0))
    video = torch.full((3, T + 2, H, W), float("nan"), device="cuda")
    band = x.view(T, H, W, 32)[:, r0:r0 + hs].reshape(-1, 32).contiguous()
    ops.nhwc_to_nchw_f32_rows(band, video[:, 1:T + 1, r0:r0 + hs], (-1.0, 1.0))
    assert torch.equal(video[:, 1:T + 1, r0:r0 + hs], want[:, :, r0:r0 + hs])
    video[:, 1:T + 1, r0:r0 + hs] = 0
    assert torch.isnan(video[:, 1:T + 1]).sum() == 3 * T * (H - hs) * W and torch.isnan(video[:, 0]).all()
