"""Per-element contract of include/yume_b200_vae_rows_enc.h, and of yb_conv3d_rows at the encoders' shapes, on one H100
(`-m gpu`), at the band shapes a row-parallel encode launches on P = 2, 4 and 8 ranks (Wan2.2 at 704x1280: latent 44x80 and
every level up to the patchified 352x640; Wan2.1 at 544x960: latent 68x120 up to 544x960):
  * the strided band conv at every Resample level, into NaN-poisoned outputs with guard bands, from a band buffer whose unused
    row 0 is NaN: the first, middle and last output rows against an fp64 convolution of the same bf16 operands, and every element
    `torch.equal` to the same rows of the full-height yb_conv3d_causal(stride_hw = 2);
  * the row-halo conv at the encoders' shapes (conv1 at 64 -> 160 / 96 channels, the residual convs, the head), every element
    `torch.equal` to the full-height launch;
  * the two video readers `torch.equal` to the _win readers' rows, zero halo rows at the image's edges, nothing written outside
    the band buffer;
  * a recording encode on every band size fails on a band launch without a row in the tables."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()
    yield "cuda"
    torch.cuda.empty_cache()          # the full-height operands are large: leave no cached blocks to the modules after this one


def _bands(H, P):
    return [(r * H // P, (r + 1) * H // P) for r in range(P)]


# (latent H, W, unit-stride convs [(scale, Cp, Cout, epilogue)], Resample convs [(scale of the input, Cp, Cout)]): level `scale`
# runs at scale x the latent size. Every conv with kh = 3 has taps (3,3,3) in the encoders. 0 = BF16, 5 = RES_BF16
ENCODERS = {
    "wan22": (44, 80, [(8, 64, 160, 0), (8, 192, 160, 0), (8, 192, 160, 5), (4, 192, 320, 0), (4, 320, 320, 0),
                       (4, 320, 320, 5), (2, 320, 640, 0), (2, 640, 640, 0), (2, 640, 640, 5), (1, 640, 640, 0),
                       (1, 640, 640, 5), (1, 640, 96, 0)],
              [(8, 192, 160), (4, 320, 320), (2, 640, 640)]),
    "wan21": (68, 120, [(8, 64, 96, 0), (8, 128, 96, 0), (8, 128, 96, 5), (4, 128, 192, 0), (4, 192, 192, 0),
                        (4, 192, 192, 5), (2, 192, 384, 0), (2, 384, 384, 0), (2, 384, 384, 5), (1, 384, 384, 0),
                        (1, 384, 384, 5), (1, 384, 32, 0)],
              [(8, 128, 96), (4, 192, 192), (2, 384, 384)]),
}


def _band_rows(table_of):
    """One row per band size of every conv at P = 2, 4, 8, the band of an interior rank where there is one, and the last band
    (its halo below is the image's edge): (H, band rows, W, Cp, Cout, extra, first row, P) at the conv's level."""
    rows = []
    for H0, W0, convs, downs in ENCODERS.values():
        for s, cp, co, extra in table_of(convs, downs):
            seen = set()
            for P in (2, 4, 8):
                bands = list(enumerate(_bands(H0, P)))
                for r, (a, b) in sorted(bands, key=lambda rb: (rb[0] in (0, P - 1), rb[0])) + [bands[-1]]:
                    key = (b - a, r == P - 1)
                    if key not in seen:
                        seen.add(key)
                        rows.append((H0 * s, (b - a) * s, W0 * s, cp, co, extra, a * s, P))
    return rows


CONV_ROWS = _band_rows(lambda convs, downs: convs)
DOWN_ROWS = _band_rows(lambda convs, downs: [(s, cp, co, None) for s, cp, co in downs])


def _row_id(r):
    return f"{r[1]}of{r[0]}x{r[2]}_c{r[3]}-{r[4]}_e{r[5]}_p{r[7]}at{r[6]}"


def _cut(seq, r0, hs, row0=0.0):
    """The band buffer of rows [r0, r0 + hs) cut from seq [T, H, W, C]: the neighbours' rows as halos, zeros beyond the image;
    row 0 set to row0 (NaN: a row the launch must not read)."""
    T, H, W, C = seq.shape
    buf = torch.zeros(T, hs + 2, W, C, device=seq.device, dtype=seq.dtype)
    lo, hi = max(r0 - 1, 0), min(r0 + hs + 1, H)
    buf[:, lo - (r0 - 1):hi - (r0 - 1)] = seq[:, lo:hi]
    if row0 != 0.0:
        buf[:, 0] = row0
    return buf


@pytest.mark.parametrize("row", DOWN_ROWS, ids=_row_id)
def test_conv_rows_down_contract(dev, row):
    from yume_b200 import ops
    H, hs, W, Cp, Cout, _, r0, P = row
    T = 2
    g = torch.Generator(device="cuda").manual_seed(11)
    seq = torch.randn(T, H, W, Cp, device="cuda", generator=g).to(BF)
    w = (torch.randn(Cout, 9 * Cp, device="cuda", generator=g) / (9 * Cp) ** 0.5).to(BF)
    b = torch.randn(Cout, device="cuda", generator=g)
    buf = _cut(seq, r0, hs, float("nan"))
    ho, wo = hs // 2, W // 2
    rows = T * ho * wo
    guard = 2 * wo
    out = torch.full((guard + rows + guard, Cout), float("nan"), device="cuda", dtype=BF)
    ops.conv3d_rows_down(buf, w, b, out[guard:guard + rows], T, hs, W)
    assert torch.isnan(out[:guard]).all() and torch.isnan(out[-guard:]).all(), "write outside the output"
    got = out[guard:guard + rows].view(T, ho, wo, Cout)
    full = torch.empty(T * (H // 2) * wo, Cout, device="cuda", dtype=BF)
    ops.conv3d_causal(seq, w, b, full, T, H, W, taps=(1, 3, 3), oob_zero_pad=True, stride_hw=2)
    assert torch.equal(got, full.view(T, H // 2, wo, Cout)[:, r0 // 2:r0 // 2 + ho])
    # fp64 bound on the band's first, middle and last output rows: ZeroPad2d((0,1,0,1)) + 3x3 stride 2
    wt = w.double().view(Cout, 1, 3, 3, Cp).permute(0, 4, 1, 2, 3)
    xn = F.pad(seq.double().permute(3, 0, 1, 2)[None], (0, 1, 0, 1))
    for h in sorted({0, ho // 2, ho - 1}):
        oh = r0 // 2 + h
        win = xn[:, :, :, 2 * oh:2 * oh + 3]
        ref = F.conv3d(win, wt, b.double(), stride=(1, 1, 2))[0].permute(1, 2, 3, 0)[:, 0]
        mag = F.conv3d(win.abs(), wt.abs(), b.double().abs(), stride=(1, 1, 2))[0].permute(1, 2, 3, 0)[:, 0]
        bound = 2.0 ** -8 * ref.abs() + 9 * Cp * 2.0 ** -23 * mag + 1e-30
        ratio = float(((got[:, h].double() - ref).abs() / bound).max())
        assert ratio <= 1.0, (h, ratio)


@pytest.mark.parametrize("row", CONV_ROWS, ids=_row_id)
def test_conv_rows_at_encoder_shapes(dev, row):
    from yume_b200 import ops
    H, hs, W, Cp, Cout, epi, r0, P = row
    T, taps = 2, (3, 3, 3)
    g = torch.Generator(device="cuda").manual_seed(12)
    seq = torch.randn(T, H, W, Cp, device="cuda", generator=g).to(BF)
    w = (torch.randn(Cout, 27 * Cp, device="cuda", generator=g) / (27 * Cp) ** 0.5).to(BF)
    b = torch.randn(Cout, device="cuda", generator=g)
    full_res = torch.randn(T * H * W, Cout, device="cuda", generator=g).to(BF) if epi == ops.YB_EPI_RES_BF16 else None
    res = None if full_res is None else full_res.view(T, H, W, Cout)[:, r0:r0 + hs].reshape(-1, Cout).contiguous()
    rows, guard = T * hs * W, 2 * W
    out = torch.full((guard + rows + guard, Cout), float("nan"), device="cuda", dtype=BF)
    ops.conv3d_rows(_cut(seq, r0, hs), w, b, out[guard:guard + rows], T, hs, W, 0, epi, res, taps=taps, full_h=H)
    assert torch.isnan(out[:guard]).all() and torch.isnan(out[-guard:]).all(), "write outside the output"
    full = torch.empty(T * H * W, Cout, device="cuda", dtype=BF)
    ops.conv3d_causal(seq, w, b, full, T, H, W, epi, full_res, taps=taps, oob_zero_pad=True)
    assert torch.equal(out[guard:guard + rows].view(T, hs, W, Cout), full.view(T, H, W, Cout)[:, r0:r0 + hs])


# (video H, W, latent rows, reader level scale): the reader writes rows of the level encoder.conv1 reads
READERS = {"wan22": (704, 1280, 44, 8), "wan21": (544, 960, 68, 8)}


@pytest.mark.parametrize("which", ["wan22", "wan21"])
@pytest.mark.parametrize("P", [2, 4, 8])
def test_band_readers_exact(dev, which, P):
    from yume_b200 import ops
    H, W, Hl, s = READERS[which]
    T, t0 = 2, 1
    g = torch.Generator(device="cuda").manual_seed(13)
    whole = torch.randn(3, T + 2, H, W, device="cuda", generator=g)
    win = whole[:, t0:t0 + T]
    if which == "wan22":
        rows, cols = H // 2, W // 2
        dense = torch.empty(T * rows * cols, 64, device="cuda", dtype=BF)
        ops.vae_patchify2_bf16_win(win, dense)
        read = ops.vae_patchify2_bf16_rows
    else:
        rows, cols = H, W
        dense = torch.empty(T * rows * cols, 64, device="cuda", dtype=BF)
        ops.nchw_to_nhwc_bf16_win(win, dense)
        read = ops.nchw_to_nhwc_bf16_rows
    dense = dense.view(T, rows, cols, 64)
    for r, (a, b) in enumerate(_bands(Hl, P)):
        r0, hs = a * s, (b - a) * s
        n = T * (hs + 2) * cols * 64
        guard = cols * 64
        flat = torch.full((guard + n + guard,), float("nan"), device="cuda", dtype=BF)
        buf = flat[guard:guard + n].view(T, hs + 2, cols, 64)
        read(win, buf, r0)
        assert torch.isnan(flat[:guard]).all() and torch.isnan(flat[-guard:]).all(), "write outside the band buffer"
        assert torch.equal(buf, _cut(dense, r0, hs)), (r, P)
        if r == 0:
            assert not buf[:, 0].any()
        if r == P - 1:
            assert not buf[:, -1].any()


class _Ranks:
    """A RowGroup stand-in for one rank of P in one process: halo rows and gathered bands are zeros (the launches' shapes are
    those of the real encode)."""

    def __init__(self, P, rank):
        self.world, self.rank = P, rank

    def band(self, H, r=None):
        return _bands(H, self.world)[self.rank if r is None else r]

    def sizes(self, H):
        return [b - a for a, b in _bands(H, self.world)]

    def exchange(self, send):
        return (None if self.rank == 0 else torch.zeros_like(send[0]),
                None if self.rank == self.world - 1 else torch.zeros_like(send[1]))

    def from_below(self, send):
        return None if self.rank == self.world - 1 else torch.zeros_like(send[0])

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
    """Encodes of every band size (one pass and 3 chunks) with recording wrappers around ops.conv3d_rows and
    ops.conv3d_rows_down: every launch must have a row in CONV_ROWS / DOWN_ROWS."""
    from yume_b200 import ops, vae_enc
    conv_table = {(hs, W, cp, co, e) for _, hs, W, cp, co, e, _, _ in CONV_ROWS}
    down_table = {(hs, W, cp, co) for _, hs, W, cp, co, _, _, _ in DOWN_ROWS}
    seen, seen_down = [], []
    real, real_down = ops.conv3d_rows, ops.conv3d_rows_down

    def record(xbuf, w, bias, out, T, H, W, t_hist=0, epilogue=ops.YB_EPI_BF16, res=None, taps=(3, 3, 3), full_h=None):
        seen.append((H, W, xbuf.shape[-1], w.shape[0], epilogue) if taps == (3, 3, 3) else ("taps", taps))
        return real(xbuf, w, bias, out, T, H, W, t_hist, epilogue, res, taps, full_h)

    def record_down(xbuf, w, bias, out, T, H, W, epilogue=ops.YB_EPI_BF16):
        seen_down.append((H, W, xbuf.shape[-1], w.shape[0]))
        return real_down(xbuf, w, bias, out, T, H, W, epilogue)
    monkeypatch.setattr(ops, "conv3d_rows", record)
    monkeypatch.setattr(ops, "conv3d_rows_down", record_down)
    zero = lambda shapes: {k: torch.zeros(v) for k, v in shapes.items()}             # noqa: E731
    if which == "wan22":
        eng = vae_enc.Wan22VaeEncoder(zero(vae_enc.encoder_param_shapes_22()), device=dev)
    else:
        eng = vae_enc.Wan21VaeEncoder(zero(vae_enc.encoder_param_shapes_21()), device=dev)
    H, W, Hl, _ = READERS[which]
    v = torch.zeros(3, 9, H, W, device=dev)
    for P in (2, 4, 8):
        done = set()
        for r, (a, b) in enumerate(_bands(Hl, P)):
            if (b - a, r in (0, P - 1)) in done:
                continue
            done.add((b - a, r in (0, P - 1)))
            eng._rows = _Ranks(P, r)
            for parts in ([3], [1, 1, 1]):
                eng._encode_chunks(v, parts)
    torch.cuda.synchronize()
    assert seen and seen_down, "no band launch"
    missing = sorted(set(seen) - conv_table, key=str) + sorted(set(seen_down) - down_table, key=str)
    assert not missing, missing
