"""Chunk-streamed decode and encode of the Wan VAEs on the GPU (`-m gpu`):
  * bit identity: at real channel widths every partition of the latent gives the one-pass video `torch.equal` — each conv output
    voxel sums the same taps x channel chunks in the same order whatever the chunk (the tile plan depends only on the output
    extents, and the history frames replace the zero fill in the same K slots), the norms are per voxel, the mid attention is per
    frame and the GEMMs have no split-K;
  * causal prefix at production spatial size: decode(z)[:, :4k-3] == decode(z[:, :k]) bit for bit;
  * the encoders the same way: every legal partition (1 + 4a frames first, then 4b) bit-identical to the one pass,
    encode(v)[:, :1+k] == encode(v[:, :1+4k]) at production size;
  * long sequences in bounded memory: 145-frame Wan2.1 decode and 177-frame Wan2.1 encode (each with 28 GB held on the device,
    standing in for the 14B DiT weights), 81-frame 704x1280 Wan2.2 decode and encode (the encode fits one pass on an empty
    80 GB card, so 40 GB are held to make the planner split it), peak allocation within the planner's bound, two chunk lengths
    bit-identical;
  * the per-element contract of every entry point of include/yume_b200_stream.h at the shapes the streams launch, on NaN-poisoned
    outputs with guard bands: the history-form conv at every launch shape of the four streams against an fp64 convolution
    (every element) and bit for bit against the one-pass launch, with a recording run that fails on a launch without a row;
    the index kernels against torch exactly."""
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


def _engine(which, dev):
    from oracle import wan21vae, wan22vae
    from yume_b200 import vae21, vae22
    mod, Eng, cfg = ((wan22vae, vae22.Wan22VaeDecoder, dict(dec_dim=256, z_dim=48)) if which == "wan22" else
                     (wan21vae, vae21.Wan21VaeDecoder, dict(dim=96, z_dim=16)))
    gen = torch.Generator().manual_seed(3)
    zd = cfg["z_dim"]
    return Eng(mod.make_state_dict(0, **cfg), mean=0.2 * torch.randn(zd, generator=gen),
               std=0.5 + torch.rand(zd, generator=gen), device=dev, **cfg)


@pytest.fixture(scope="module")
def engines(dev):
    return {w: _engine(w, dev) for w in ("wan22", "wan21")}


def _z(engine, T, H, W, seed=1):
    return torch.randn(engine.z_dim, T, H, W, generator=torch.Generator().manual_seed(seed)).cuda()


@pytest.mark.parametrize("which", ["wan22", "wan21"])
def test_every_partition_is_bit_identical_to_one_pass(engines, which):
    eng = engines[which]
    z = _z(eng, 9, 4, 6)
    ref = eng._decode_chunks(z, [9])
    assert torch.isfinite(ref).all()
    for parts in ([1] * 9, [2, 7], [4, 5], [1, 3, 5], [8, 1], [3, 3, 3]):
        got = eng._decode_chunks(z, parts)
        assert torch.equal(got, ref), (parts, float((got - ref).abs().max()))


@pytest.mark.parametrize("which,H,W", [("wan22", 44, 80), ("wan21", 68, 120)])
def test_causal_prefix_at_production_size(engines, which, H, W):
    eng = engines[which]
    z = _z(eng, 4, H, W, seed=2)
    full = eng._decode_chunks(z, [1, 3])
    for k in (1, 2):
        assert torch.equal(full[:, :4 * k - 3], eng.decode(z[:, :k].contiguous())), k


@pytest.mark.parametrize("which,T,H,W,hold_gb", [("wan21", 37, 68, 120, 28), ("wan22", 21, 44, 80, 0)])
def test_long_sequence_in_bounded_memory(engines, which, T, H, W, hold_gb):
    eng = engines[which]
    z = _z(eng, T, H, W, seed=4)
    held = torch.empty(hold_gb << 30, dtype=torch.uint8, device="cuda") if hold_gb else None
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    plan = eng.plan_chunks(T, H, W)
    assert len(plan) > 1, plan
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = eng.decode(z)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    bound = eng.chunk_bytes(plan[0], T, H, W)
    print(f"{which} T={T}: chunks {plan}, peak {peak / 2**30:.2f} GiB, planner bound {bound / 2**30:.2f} GiB")
    assert peak <= bound
    assert tuple(out.shape) == eng._out_shape(T, H, W) and torch.isfinite(out).all()
    n = max(1, plan[0] // 2)
    other = [n] * (T // n) + ([T % n] if T % n else [])
    assert torch.equal(eng._decode_chunks(z, other), out), other
    del held


# ------------------------------------------------------------------------------------------------------------
# encoders
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def encoders(dev):
    from oracle import wan21vae_enc, wan22vae_enc
    from yume_b200 import vae_enc
    out = {}
    for which, mod, Eng, cfg in (("wan22", wan22vae_enc, vae_enc.Wan22VaeEncoder, dict(dim=160, z_dim=48)),
                                 ("wan21", wan21vae_enc, vae_enc.Wan21VaeEncoder, dict(dim=96, z_dim=16))):
        gen = torch.Generator().manual_seed(8)
        zd = cfg["z_dim"]
        out[which] = Eng(mod.make_state_dict(0, **cfg), mean=0.2 * torch.randn(zd, generator=gen),
                         std=0.5 + torch.rand(zd, generator=gen), device=dev, **cfg)
    return out


def _video(T, H, W, seed):
    return torch.randn(3, T, H, W, generator=torch.Generator().manual_seed(seed)).clamp_(-1, 1).cuda()


@pytest.mark.parametrize("which,H,W", [("wan22", 32, 48), ("wan21", 16, 24)])
def test_every_encode_partition_is_bit_identical_to_one_pass(encoders, which, H, W):
    eng = encoders[which]
    v = _video(27, H, W, 11)                                     # 27 frames: the reference encodes the first 25 (7 latent frames)
    ref = eng._encode_chunks(v, [7])
    assert torch.isfinite(ref).all() and ref.shape[1] == 7
    for parts in ([1] * 7, [2, 5], [4, 3], [1, 3, 3], [6, 1]):
        got = eng._encode_chunks(v, parts)
        assert torch.equal(got, ref), (parts, float((got - ref).abs().max()))


@pytest.mark.parametrize("which,H,W", [("wan22", 704, 1280), ("wan21", 544, 960)])
def test_encode_causal_prefix_at_production_size(encoders, which, H, W):
    eng = encoders[which]
    v = _video(9, H, W, 12)
    full = eng._encode_chunks(v, [1, 2])
    for k in (0, 1):
        assert torch.equal(full[:, :1 + k], eng.encode(v[:, :1 + 4 * k].contiguous())), k


@pytest.mark.parametrize("which,T,H,W,hold_gb", [("wan21", 177, 544, 960, 28), ("wan22", 81, 704, 1280, 40)])
def test_long_encode_in_bounded_memory(encoders, which, T, H, W, hold_gb):
    eng = encoders[which]
    v = _video(T, H, W, 13)
    held = torch.empty(hold_gb << 30, dtype=torch.uint8, device="cuda") if hold_gb else None
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    plan = eng.plan_chunks(T, H, W)
    assert len(plan) > 1, plan
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = eng.encode(v)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    bound = eng.chunk_bytes(plan[0], T, H, W)
    print(f"{which} encode T={T}: chunks {plan}, peak {peak / 2**30:.2f} GiB, planner bound {bound / 2**30:.2f} GiB")
    assert peak <= bound
    assert out.shape[1] == 1 + (T - 1) // 4 and torch.isfinite(out).all()
    n = max(1, plan[0] // 2)
    Tl = out.shape[1]
    other = [n] * (Tl // n) + ([Tl % n] if Tl % n else [])
    assert torch.equal(eng._encode_chunks(v, other), out), other
    del held


# ------------------------------------------------------------------------------------------------------------
# per-element contract of include/yume_b200_stream.h
# ------------------------------------------------------------------------------------------------------------
# (taps, H, W, Cp, Cout, stride_t, out_t_mul, epilogue): every history-form launch of the four streams at production spatial size
# (test_table_covers_the_streams_launches checks that no launch is missing); 0 = BF16, 2 = F32 (the decoder heads), 5 = RES_BF16
CONV_ROWS = sorted({
    # Wan2.2 decoder, latent 44x80
    ((3, 1, 1), 44, 80, 1024, 1024, 1, 2, 0), ((3, 1, 1), 88, 160, 1024, 1024, 1, 2, 0), ((3, 3, 3), 44, 80, 64, 1024, 1, 1, 0),
    ((3, 3, 3), 44, 80, 1024, 1024, 1, 1, 0), ((3, 3, 3), 44, 80, 1024, 1024, 1, 1, 5), ((3, 3, 3), 88, 160, 1024, 1024, 1, 1, 0),
    ((3, 3, 3), 88, 160, 1024, 1024, 1, 1, 5), ((3, 3, 3), 176, 320, 512, 512, 1, 1, 0), ((3, 3, 3), 176, 320, 512, 512, 1, 1, 5),
    ((3, 3, 3), 176, 320, 1024, 512, 1, 1, 0), ((3, 3, 3), 352, 640, 256, 32, 1, 1, 2), ((3, 3, 3), 352, 640, 256, 256, 1, 1, 0),
    ((3, 3, 3), 352, 640, 256, 256, 1, 1, 5), ((3, 3, 3), 352, 640, 512, 256, 1, 1, 0),
    # Wan2.1 decoder, latent 68x120
    ((3, 1, 1), 68, 120, 384, 384, 1, 2, 0), ((3, 1, 1), 136, 240, 384, 384, 1, 2, 0), ((3, 3, 3), 68, 120, 64, 384, 1, 1, 0),
    ((3, 3, 3), 68, 120, 384, 384, 1, 1, 0), ((3, 3, 3), 68, 120, 384, 384, 1, 1, 5), ((3, 3, 3), 136, 240, 192, 384, 1, 1, 0),
    ((3, 3, 3), 136, 240, 384, 384, 1, 1, 0), ((3, 3, 3), 136, 240, 384, 384, 1, 1, 5), ((3, 3, 3), 272, 480, 192, 192, 1, 1, 0),
    ((3, 3, 3), 272, 480, 192, 192, 1, 1, 5), ((3, 3, 3), 544, 960, 128, 32, 1, 1, 2), ((3, 3, 3), 544, 960, 128, 96, 1, 1, 0),
    ((3, 3, 3), 544, 960, 128, 96, 1, 1, 5),
    # Wan2.2 encoder, 704x1280
    ((3, 1, 1), 44, 80, 640, 640, 2, 1, 0), ((3, 1, 1), 88, 160, 320, 320, 2, 1, 0), ((3, 3, 3), 44, 80, 640, 96, 1, 1, 0),
    ((3, 3, 3), 44, 80, 640, 640, 1, 1, 0), ((3, 3, 3), 44, 80, 640, 640, 1, 1, 5), ((3, 3, 3), 88, 160, 320, 640, 1, 1, 0),
    ((3, 3, 3), 88, 160, 640, 640, 1, 1, 0), ((3, 3, 3), 88, 160, 640, 640, 1, 1, 5), ((3, 3, 3), 176, 320, 192, 320, 1, 1, 0),
    ((3, 3, 3), 176, 320, 320, 320, 1, 1, 0), ((3, 3, 3), 176, 320, 320, 320, 1, 1, 5), ((3, 3, 3), 352, 640, 64, 160, 1, 1, 0),
    ((3, 3, 3), 352, 640, 192, 160, 1, 1, 0), ((3, 3, 3), 352, 640, 192, 160, 1, 1, 5),
    # Wan2.1 encoder, 544x960
    ((3, 1, 1), 68, 120, 384, 384, 2, 1, 0), ((3, 1, 1), 136, 240, 192, 192, 2, 1, 0), ((3, 3, 3), 68, 120, 384, 32, 1, 1, 0),
    ((3, 3, 3), 136, 240, 192, 384, 1, 1, 0), ((3, 3, 3), 272, 480, 128, 192, 1, 1, 0), ((3, 3, 3), 272, 480, 192, 192, 1, 1, 0),
    ((3, 3, 3), 272, 480, 192, 192, 1, 1, 5), ((3, 3, 3), 544, 960, 64, 96, 1, 1, 0),
})


def _row_id(r):
    return "x".join(map(str, r[0])) + f"_{r[1]}x{r[2]}_c{r[3]}-{r[4]}_s{r[5]}_m{r[6]}_e{r[7]}"


@pytest.mark.parametrize("row", CONV_ROWS, ids=_row_id)
def test_conv_hist_contract(dev, row):
    """Every output element of the history form against an fp64 convolution of the same bf16 operands (|err| <= half a bf16 ulp
    of the result plus fp32 accumulation over the K products), bit for bit against the one-pass launch over the whole sequence,
    into a NaN-poisoned output with a guard band on both sides (interleaved time_conv frames of the other group stay NaN)."""
    import torch.nn.functional as F
    from yume_b200 import ops
    taps, H, W, Cp, Cout, st, mul, epi = row
    kt, kh, kw = taps
    hist = 1 if st == 2 else kt - 1
    T = 4 if st == 2 else 2                                      # new frames: 2 output frames either way
    To = T // st
    g = torch.Generator(device="cuda").manual_seed(5)
    P = 2 if st == 2 else 3                                      # frames before this chunk's history (even: stride-2 windows align)
    seq = torch.randn(P + hist + T, H, W, Cp, device="cuda", generator=g).to(BF)
    w = (torch.randn(Cout, kt * kh * kw * Cp, device="cuda", generator=g) / (kt * kh * kw * Cp) ** 0.5).to(BF)
    b = torch.randn(Cout, device="cuda", generator=g)
    res = torch.randn(T * H * W, Cout, device="cuda", generator=g).to(BF) if epi == ops.YB_EPI_RES_BF16 else None
    odt = torch.float32 if epi == ops.YB_EPI_F32 else BF
    Tall = seq.shape[0]
    buf = seq[Tall - hist - T:].contiguous()
    rows = To * mul * H * W
    guard = 2 * H * W
    out = torch.full((guard + rows + guard, Cout), float("nan"), device="cuda", dtype=odt)
    ops.conv3d_causal_hist(buf, w, b, out[guard:guard + rows], T, H, W, hist, epi, res, taps=taps, out_t_mul=mul, stride_t=st)
    assert torch.isnan(out[:guard]).all() and torch.isnan(out[-guard:]).all(), "write outside the output"
    got = out[guard:guard + rows].view(To * mul, H * W, Cout)
    frames = list(range(0, To * mul, mul))
    for t in set(range(To * mul)) - set(frames):
        assert torch.isnan(got[t]).all(), f"interleaved frame {t} written"
    got = got[frames].float()
    # fp64 reference: the buffer frames stand in front (no time padding), H / W zero padded
    wt = w.double().view(Cout, kt, kh, kw, Cp).permute(0, 4, 1, 2, 3)
    xn = F.pad(buf.double().permute(3, 0, 1, 2)[None], (kw // 2, kw // 2, kh // 2, kh // 2, 0, 0))
    ref = F.conv3d(xn, wt, b.double(), stride=(st, 1, 1))[0].permute(1, 2, 3, 0).reshape(To, H * W, Cout)
    mag = F.conv3d(xn.abs(), wt.abs(), b.double().abs(), stride=(st, 1, 1))[0].permute(1, 2, 3, 0).reshape(To, H * W, Cout)
    if res is not None:
        ref = ref + res.double().view(To, H * W, Cout)
        mag = mag + res.double().abs().view(To, H * W, Cout)
    K = kt * kh * kw * Cp
    ulp = 2.0 ** -24 if odt == torch.float32 else 2.0 ** -8
    bound = ulp * ref.abs() + K * 2.0 ** -23 * mag + 1e-30
    ratio = float(((got.double() - ref).abs() / bound).max())
    assert ratio <= 1.0, ratio
    # bit identity with the one-pass launch over the whole sequence (the stream's premise)
    if st == 1:
        full_res = None if res is None else torch.cat([torch.zeros((Tall - T) * H * W, Cout, device="cuda", dtype=BF), res])
        full = torch.empty(Tall * mul * H * W, Cout, device="cuda", dtype=odt)
        ops.conv3d_causal(seq, w, b, full, Tall, H, W, epi, full_res, taps=taps, oob_zero_pad=True, out_t_mul=mul)
        want = full.view(Tall * mul, H * W, Cout)[(Tall - T) * mul:][frames]
    else:
        full = torch.empty(((Tall - 3) // 2 + 1) * H * W, Cout, device="cuda", dtype=odt)
        ops.conv3d_causal(seq, w, b, full, Tall, H, W, epi, None, taps=taps, oob_zero_pad=True, stride_t=2)
        want = full.view(-1, H * W, Cout)[-To:]
    assert torch.equal(got, want.float())


def _stream_engines(dev):
    from yume_b200 import vae21, vae22, vae_enc
    zero = lambda shapes: {k: torch.zeros(v) for k, v in shapes.items()}             # noqa: E731
    return {
        "wan22_dec": (vae22.Wan22VaeDecoder(zero(vae22.decoder_param_shapes()), device=dev),
                      lambda e: e._decode_chunks(torch.zeros(48, 3, 44, 80, device=dev), [1, 1, 1])),
        "wan21_dec": (vae21.Wan21VaeDecoder(zero(vae21.decoder_param_shapes()), device=dev),
                      lambda e: e._decode_chunks(torch.zeros(16, 3, 68, 120, device=dev), [1, 1, 1])),
        "wan22_enc": (vae_enc.Wan22VaeEncoder(zero(vae_enc.encoder_param_shapes_22()), device=dev),
                      lambda e: e._encode_chunks(torch.zeros(3, 9, 704, 1280, device=dev), [1, 1, 1])),
        "wan21_enc": (vae_enc.Wan21VaeEncoder(zero(vae_enc.encoder_param_shapes_21()), device=dev),
                      lambda e: e._encode_chunks(torch.zeros(3, 9, 544, 960, device=dev), [1, 1, 1])),
    }


@pytest.mark.parametrize("name", ["wan22_dec", "wan21_dec", "wan22_enc", "wan21_enc"])
def test_table_covers_the_streams_launches(dev, monkeypatch, name):
    """A 3-chunk stream at production spatial size with a recording wrapper around ops.conv3d_causal_hist: every launch must
    have a row in CONV_ROWS."""
    from yume_b200 import ops
    seen = []
    real = ops.conv3d_causal_hist

    def record(xbuf, w, bias, out, T, H, W, t_hist, epilogue=ops.YB_EPI_BF16, res=None, taps=(3, 3, 3), out_t_mul=1,
               out_t_add=0, stride_t=1, stride_hw=1):
        seen.append((tuple(taps), H, W, xbuf.shape[-1], w.shape[0], stride_t, out_t_mul, epilogue))
        return real(xbuf, w, bias, out, T, H, W, t_hist, epilogue, res, taps, out_t_mul, out_t_add, stride_t, stride_hw)
    monkeypatch.setattr(ops, "conv3d_causal_hist", record)
    eng, run = _stream_engines(dev)[name]
    run(eng)
    torch.cuda.synchronize()
    assert seen, "no history-form launch"
    missing = sorted(set(seen) - set(CONV_ROWS))
    assert not missing, missing


@pytest.mark.parametrize("Ts,Hs,Ws,in_c,out_c,ft", [(2, 44, 80, 1024, 1024, 2), (2, 88, 160, 1024, 512, 2),
                                                   (2, 176, 320, 512, 256, 1)])
def test_dupup_add_cont_exact(dev, Ts, Hs, Ws, in_c, out_c, ft):
    from yume_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(Ts, Hs, Ws, in_c, device="cuda", generator=g).to(BF)
    main = torch.randn(ft * Ts, 2 * Hs, 2 * Ws, out_c, device="cuda", generator=g).to(BF)
    rep = out_c * ft * 4 // in_c
    y = x.float().permute(3, 0, 1, 2).repeat_interleave(rep, dim=0).view(out_c, ft, 2, 2, Ts, Hs, Ws)
    up = y.permute(4, 1, 5, 2, 6, 3, 0).reshape(ft * Ts, 2 * Hs, 2 * Ws, out_c)
    want = (main.float() + up).to(BF)
    ops.vae_dupup_add_cont(main, x, (Ts, Hs, Ws), in_c, out_c, ft, 2)
    assert torch.equal(main, want)


def _video_window(C, Tall, h, w, t0, T):
    video = torch.full((C, Tall, h, w), float("nan"), device="cuda")
    return video, video[:, t0:t0 + T]


def test_unpatchify2_clamp_win_exact(dev):
    from yume_b200 import ops
    T, H, W = 4, 352, 640
    y = 1.5 * torch.randn(T * H * W, 32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))
    video, win = _video_window(3, 9, 2 * H, 2 * W, 5, T)
    ops.vae_unpatchify2_clamp_win(y, win, T, H, W)
    v = y[:, :12].view(T, H, W, 12).permute(3, 0, 1, 2)[None]
    want = v.reshape(1, 3, 2, 2, T, H, W).permute(0, 1, 4, 5, 3, 6, 2).reshape(3, T, 2 * H, 2 * W).clamp(-1, 1)
    assert torch.equal(win, want)
    assert torch.isnan(video[:, :5]).all()


@pytest.mark.parametrize("C,h,w,clamp", [(3, 544, 960, (-1.0, 1.0)), (16, 68, 120, None), (48, 44, 80, None)])
def test_nhwc_to_nchw_f32_win_exact(dev, C, h, w, clamp):
    """The Wan2.1 decoder tail (clamped) and both encoders' mu writes (no clamp) into a frame window of a NaN-filled result."""
    from yume_b200 import ops
    T = 4
    x = 1.5 * torch.randn(T * h * w, 64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(8))
    video, win = _video_window(C, 10, h, w, 3, T)
    ops.nhwc_to_nchw_f32_win(x, win, clamp)
    want = x[:, :C].t().reshape(C, T, h, w)
    assert torch.equal(win, want if clamp is None else want.clamp(*clamp))
    assert torch.isnan(video[:, :3]).all() and torch.isnan(video[:, 7:]).all()


@pytest.mark.parametrize("T,H,W", [(4, 704, 1280), (5, 32, 48)])
def test_patchify2_bf16_win_exact(dev, T, H, W):
    """The Wan2.2 encoder input read from frames 3.. of a longer video, into a NaN-poisoned buffer with guard rows."""
    from yume_b200 import ops
    video = torch.randn(3, 11, H, W, device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    n, g = T * (H // 2) * (W // 2), 64
    out = torch.full((g + n + g, 64), float("nan"), device="cuda", dtype=BF)
    ops.vae_patchify2_bf16_win(video[:, 3:3 + T], out[g:g + n])
    x = video[:, 3:3 + T].reshape(3, T, H // 2, 2, W // 2, 2).permute(0, 5, 3, 1, 2, 4).reshape(12, T, H // 2, W // 2)
    want = torch.zeros(n, 64, device="cuda", dtype=BF)
    want[:, :12] = x.permute(1, 2, 3, 0).reshape(-1, 12).to(BF)
    assert torch.equal(out[g:g + n], want)
    assert torch.isnan(out[:g].float()).all() and torch.isnan(out[g + n:].float()).all()


@pytest.mark.parametrize("T,H,W", [(4, 544, 960), (5, 16, 24)])
def test_nchw_to_nhwc_bf16_win_exact(dev, T, H, W):
    """The Wan2.1 encoder input read from frames 3.. of a longer video, into a NaN-poisoned buffer with guard rows."""
    from yume_b200 import ops
    video = torch.randn(3, 11, H, W, device="cuda", generator=torch.Generator(device="cuda").manual_seed(10))
    n, g = T * H * W, 64
    out = torch.full((g + n + g, 64), float("nan"), device="cuda", dtype=BF)
    ops.nchw_to_nhwc_bf16_win(video[:, 3:3 + T], out[g:g + n])
    want = torch.zeros(n, 64, device="cuda", dtype=BF)
    want[:, :3] = video[:, 3:3 + T].reshape(3, -1).t().to(BF)
    assert torch.equal(out[g:g + n], want)
    assert torch.isnan(out[:g].float()).all() and torch.isnan(out[g + n:].float()).all()


# entry point -> tests that exercise it (tests/test_host_logic_vae_stream.py: every entry point of include/yume_b200_stream.h)
COVERS = {
    "yb_conv3d_causal_hist": ["test_conv_hist_contract", "test_table_covers_the_streams_launches",
                              "test_every_partition_is_bit_identical_to_one_pass"],
    "yb_vae_dupup_add_cont": ["test_dupup_add_cont_exact", "test_every_partition_is_bit_identical_to_one_pass"],
    "yb_vae_unpatchify2_clamp_win": ["test_unpatchify2_clamp_win_exact"],
    "yb_nhwc_to_nchw_f32_clamp_win": ["test_nhwc_to_nchw_f32_win_exact"],
    "yb_vae_patchify2_bf16_win": ["test_patchify2_bf16_win_exact", "test_every_encode_partition_is_bit_identical_to_one_pass"],
    "yb_nchw_to_nhwc_bf16_win": ["test_nchw_to_nhwc_bf16_win_exact", "test_every_encode_partition_is_bit_identical_to_one_pass"],
}
