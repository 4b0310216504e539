"""Resuming Wan VAE sessions on the GPU (`-m gpu`):
  * Wan2.1 at real width, 544x960: a decode session of 49 -> 81 -> 113 -> 145 frames and an encode session of the 14B sampler's
    [history, zeros(32)] inputs of the same lengths, each call `torch.equal` to a fresh engine's full call;
  * Wan2.2 at 704x1280: decode sessions in bf16 and precision="fp8", the same check;
  * yb_vae_frame_match against the bitwise reference (tests/helpers/torch_ops_resume.frame_match): a difference in the first, the
    last or no frame, kept inputs shorter and longer than the new one, -0.0, NaN payloads, all-zero and subnormal frames, every
    element size and load width, frames whose bytes are not a multiple of the widest load, inside NaN guard bands;
  * memory: retained_bytes() is the bytes of the kept tensors, and reset() returns memory_allocated to its level before the
    session; resume=False issues the launches of the plain call."""
import pytest
import torch

from helpers.torch_ops_resume import frame_match

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()
    return "cuda"


def _sd(which):
    from oracle import wan21vae, wan21vae_enc, wan22vae
    if which == "wan21":
        return {**wan21vae.make_state_dict(0, dim=96, z_dim=16), **wan21vae_enc.make_state_dict(1, dim=96, z_dim=16)}
    return wan22vae.make_state_dict(0, dec_dim=256, z_dim=48)


def _stats(zd):
    g = torch.Generator().manual_seed(3)
    return dict(mean=0.2 * torch.randn(zd, generator=g), std=0.5 + torch.rand(zd, generator=g))


@pytest.fixture(scope="module")
def wan21(dev):
    from yume_b200 import vae21, vae_enc
    sd, st = _sd("wan21"), _stats(16)
    return {r: (vae21.Wan21VaeDecoder(sd, dim=96, z_dim=16, device=dev, resume=r, **st),
                vae_enc.Wan21VaeEncoder(sd, dim=96, z_dim=16, device=dev, resume=r, **st)) for r in (False, True)}


def _z(zd, T, H, W, seed):
    return torch.randn(zd, T, H, W, generator=torch.Generator().manual_seed(seed)).cuda()


def test_wan21_decode_session_at_real_width(wan21):
    (full, _), (eng, _) = wan21[False], wan21[True]
    z = _z(16, 37, 68, 120, seed=1)
    for T in (13, 21, 29, 37):                                    # 49, 81, 113, 145 frames
        zt = z[:, :T].contiguous()
        got = eng.decode(zt)
        want = full.decode(zt)
        assert got.shape == (3, 4 * T - 3, 544, 960) and torch.equal(got, want), T
        del want
    assert eng._kept.snaps.keys() == {37}
    eng.reset()


def test_wan21_encode_session_at_real_width(wan21):
    """[history, zeros(32)] with history 17, 49, 81, 113 frames: every call after the first resumes where the zeros began."""
    (_, full), (_, eng) = wan21[False], wan21[True]
    video = (torch.randn(3, 113, 544, 960, generator=torch.Generator().manual_seed(2)).clamp_(-1, 1)).cuda()
    zeros = torch.zeros(3, 32, 544, 960, device="cuda")
    for n in (17, 49, 81, 113):
        v = torch.cat([video[:, :n], zeros], 1)
        got = eng.encode(v)
        assert set(eng._kept.snaps) == {n, n + 32}
        want = full.encode(v)
        assert got.shape == (16, (n + 31) // 4 + 1, 68, 120) and torch.equal(got, want), n
        del v, want
    eng.reset()


@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_wan22_decode_session_at_704x1280(dev, precision):
    from yume_b200 import vae22
    sd, st = _sd("wan22"), _stats(48)
    full = vae22.Wan22VaeDecoder(sd, dec_dim=256, z_dim=48, device=dev, precision=precision, **st)
    eng = vae22.Wan22VaeDecoder(sd, dec_dim=256, z_dim=48, device=dev, precision=precision, resume=True, **st)
    del sd
    z = _z(48, 7, 44, 80, seed=4)
    for T in (3, 5, 7):
        zt = z[:, :T].contiguous()
        got = eng.decode(zt)
        want = full.decode(zt)
        assert got.shape == (3, 4 * T - 3, 704, 1280) and torch.equal(got, want), (precision, T)
        del want
    if precision == "fp8":                                        # the (values, scales) carry pairs are kept
        assert any(isinstance(c, tuple) for c in eng._kept.snaps[7][1].values())
    eng.reset()


# ------------------------------------------------------------------------------------------------------------
# yb_vae_frame_match
# ------------------------------------------------------------------------------------------------------------
def _match(kept, x):
    from yume_b200 import ops
    res = torch.tensor([-7, -7], dtype=torch.int32, device="cuda")             # overwritten, not accumulated into
    ops.vae_frame_match(kept, x, res)
    return tuple(res.tolist())


def _check(kept, x):
    want = frame_match(None if kept is None else kept.cpu(), x.cpu())
    assert _match(kept, x) == want, want
    return want


def test_frame_match_edge_cases(dev):
    g = torch.Generator().manual_seed(5)
    x = torch.randn(3, 9, 24, 40, generator=g).cuda()
    x[:, 6:] = 0
    assert _check(None, x) == (0, 6)
    assert _check(x.clone(), x) == (9, 6)                        # no difference
    assert _check(x[:, :4].contiguous(), x) == (4, 6)            # kept shorter
    assert _check(torch.cat([x, x[:, :2]], 1), x) == (9, 6)      # kept longer
    for f in (0, 5, 8):                                          # first, an interior, the last frame
        y = x.clone()
        y.view(torch.int32)[2, f, 23, 39] ^= 1 << 30
        assert _check(x, y) == (f, 9 if f == 8 else 6)
    y = x.clone()
    y[1, 7, 0, 0] = -0.0                                         # -0.0 is neither equal bitwise nor a zero frame
    assert _check(x, y) == (7, 8)
    y = x.clone()
    y[0, 3, 5, 5] = float("nan")
    k = y.clone()
    k.view(torch.int32)[0, 3, 5, 5] ^= 1                         # another NaN payload
    assert _check(k, y) == (3, 6)
    assert _check(y, y.clone()) == (9, 6)                        # the same NaN bits compare equal
    y = x.clone()
    y[2, 6, 10, 10] = torch.finfo(torch.float32).smallest_normal / 4      # a subnormal frame is not zero
    assert _check(x, y) == (6, 7)
    assert _check(None, torch.zeros(3, 5, 24, 40, device="cuda")) == (0, 0)
    z = torch.zeros(3, 5, 24, 40, device="cuda")
    assert _check(z[:, :2].contiguous(), z) == (2, 0)


@pytest.mark.parametrize("dtype,elems,pad", [(torch.float32, 16 * 9, 64), (torch.float32, 146, 64), (torch.float32, 37 * 5, 64),
                                             (torch.float32, 37 * 5, 37), (torch.bfloat16, 12 * 7, 64), (torch.bfloat16, 37 * 5, 37),
                                             (torch.uint8, 37 * 5, 37), (torch.float64, 37 * 5, 37)])
def test_frame_match_in_nan_guard_bands(dev, dtype, elems, pad):
    """Frames of `elems` elements `pad` elements into a buffer of NaN (0xff bytes): 16-, 8-, 4-, 2- and 1-byte loads, frames whose
    bytes are not a multiple of 16. A read past either end would see a set bit in x's zero tail or a difference from kept."""
    g = torch.Generator().manual_seed(elems)
    C, T, Tk = 3, 7, 5
    back = torch.full(((C * T * elems + 2 * pad) * dtype.itemsize,), 0xff, dtype=torch.uint8, device="cuda")
    kback = torch.full(((C * Tk * elems + 2 * pad) * dtype.itemsize,), 0xfe, dtype=torch.uint8, device="cuda")
    x = back.view(dtype)[pad:pad + C * T * elems].view(C, T, elems)
    kept = kback.view(dtype)[pad:pad + C * Tk * elems].view(C, Tk, elems)
    data = (torch.rand(C, T, elems, generator=g) * 100 + 1).to(dtype).cuda()
    data[:, 4:] = 0
    x.copy_(data)
    kept.copy_(data[:, :Tk])
    assert _check(kept, x) == (5, 4)
    x[0, 2, elems - 1] = 0                                       # the last element of an interior frame
    assert _check(kept, x) == (2, 4)
    x[0, 2, elems - 1] = data[0, 2, elems - 1]
    x[C - 1, T - 1, elems - 1] = 1                               # the very last element
    assert _check(kept, x) == (5, 7)
    assert (back[:pad * dtype.itemsize] == 0xff).all() and (back[-pad * dtype.itemsize:] == 0xff).all()


def test_frame_match_large_input(dev):
    """A 250 MB input: many blocks per frame, one launch grid of persistent blocks."""
    x = torch.randn(3, 40, 544, 960, generator=torch.Generator().manual_seed(6)).cuda()
    x[:, 33:] = 0
    k = x[:, :33].clone()
    k[1, 20, 543, 959] += 1
    assert _match(k, x) == (20, 33)


# ------------------------------------------------------------------------------------------------------------
# memory, default launches
# ------------------------------------------------------------------------------------------------------------
def test_retained_bytes_and_reset_return_memory(dev):
    from yume_b200 import vae_enc
    sd, st = _sd("wan21"), _stats(16)
    eng = vae_enc.Wan21VaeEncoder(sd, dim=96, z_dim=16, device=dev, resume=True, **st)
    video = torch.randn(3, 25, 272, 480, generator=torch.Generator().manual_seed(7)).clamp_(-1, 1)
    eng.encode(video[:, :5])                                      # anything the first launches allocate for good
    eng.reset()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    for n in (9, 17):
        out = eng.encode(torch.cat([video[:, :n], torch.zeros(3, 8, 272, 480)], 1))
        k = eng._kept
        tensors = {t.data_ptr(): t for t in [k.src, k.out] + [c for _, cs in k.snaps.values() for c in cs.values()]}
        assert eng.retained_bytes() == sum(t.numel() * t.element_size() for t in tensors.values()) > 0
        del out, k, tensors
    eng.reset()
    torch.cuda.synchronize()
    assert eng.retained_bytes() == 0 and torch.cuda.memory_allocated() == base


def test_resume_off_issues_the_plain_launches(wan21):
    from yume_b200 import ops
    dec = wan21[False][0]
    z = _z(16, 5, 34, 60, seed=8)
    ops.reset_launch_count()
    want = dec._decode_chunks(z, dec.plan_chunks(*z.shape[1:]))
    n = ops.launch_count()
    ops.reset_launch_count()
    got = dec.decode(z)
    assert ops.launch_count() == n and torch.equal(got, want) and dec.retained_bytes() == 0
