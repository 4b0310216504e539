"""The four Wan VAE engines launch by launch on the H100 (tests/helpers/vae_dataflow.py): the engines run unchanged with a
checking wrapper in front of the ops of vae22 / vae21 / vae_enc. Every launch of every chunk must be the spec's next stage,
take exactly the operands the spec names (buffers, frame windows, carried history frames and their count, e4m3 scale frames),
and produce an output within its kernel's contract bound; layout kernels and quantisers bit for bit, windowed writers leaving
the rest of the result untouched.

  * real channel widths, small latents (5 latent frames at 6 x 10): every engine one-pass and in chunks [1, 2, 2], the fp8
    decode included, and one resumed session per side (Wan2.1 decode, Wan2.2 encode with its zero-tail fork);
  * production spatial size, few frames, chunks [1, 1]: Wan2.2 decode at a 44 x 80 latent (bf16 and fp8), Wan2.1 decode at
    68 x 120, Wan2.2 encode at 704 x 1280 and Wan2.1 encode at 544 x 960 (5 frames each).
Each cell prints its worst |err| / bound per entry and its wall time."""
import time

import pytest
import torch

from helpers import vae_dataflow as VF
from oracle import wan21vae, wan21vae_enc, wan22vae, wan22vae_enc
from yume_b200 import vae21, vae22, vae_enc

pytestmark = pytest.mark.gpu

MODULES = (vae22, vae21, vae_enc)
CFGS = {"wan22_dec": (wan22vae, dict(dec_dim=256, z_dim=48)), "wan21_dec": (wan21vae, dict(dim=96, z_dim=16)),
        "wan22_enc": (wan22vae_enc, dict(dim=160, z_dim=48)), "wan21_enc": (wan21vae_enc, dict(dim=96, z_dim=16))}
ENGINES = {"wan22_dec": lambda: vae22.Wan22VaeDecoder, "wan21_dec": lambda: vae21.Wan21VaeDecoder,
           "wan22_enc": lambda: vae_enc.Wan22VaeEncoder, "wan21_enc": lambda: vae_enc.Wan21VaeEncoder}
SCALE = {"wan22_enc": 16, "wan21_enc": 8}
SMALL = [(k, "bf16", p) for k in CFGS for p in ([5], [1, 2, 2])] + [("wan22_dec", "fp8", p) for p in ([5], [1, 2, 2])]
# (engine, precision, latent H x W): 2 latent frames in chunks [1, 1] (5 video frames for the encoders)
PROD = [("wan22_dec", "bf16", 44, 80), ("wan22_dec", "fp8", 44, 80), ("wan21_dec", "bf16", 68, 120),
        ("wan22_enc", "bf16", 44, 80), ("wan21_enc", "bf16", 68, 120)]

_ENG = {}


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()
    yield
    _ENG.clear()
    torch.cuda.empty_cache()


def _stats(zd):
    g = torch.Generator().manual_seed(3)
    return 0.2 * torch.randn(zd, generator=g), 0.5 + torch.rand(zd, generator=g)


def _setup(kind, precision, resume=False):
    key = (kind, precision, resume)
    if key not in _ENG:
        _ENG.clear()
        torch.cuda.empty_cache()
        mod, cfg = CFGS[kind]
        sd = mod.make_state_dict(0, **cfg)
        mean, std = _stats(cfg["z_dim"])
        eng = ENGINES[kind]()(sd, mean=mean, std=std, device="cuda", precision=precision, resume=resume, **cfg)
        _ENG[key] = (eng, VF.Spec(kind, sd, cfg, mean, std, "cuda", precision))
    return _ENG[key]


def _input(kind, units, H, W, seed=1):
    g = torch.Generator().manual_seed(seed)
    if kind.endswith("dec"):
        return torch.randn(CFGS[kind][1]["z_dim"], units, H, W, generator=g).cuda()
    s = SCALE[kind]
    return torch.randn(3, 1 + 4 * (units - 1), H * s, W * s, generator=g).clamp_(-1, 1).cuda()


def _run(eng, x, parts):
    if isinstance(eng, vae_enc.WanVaeEncoder):
        return eng._encode_chunks(x, parts)
    return eng._decode_chunks(x, parts)


def _cell(monkeypatch, kind, precision, parts, H, W):
    eng, spec = _setup(kind, precision)
    x = _input(kind, sum(parts), H, W)
    tag = f"{kind}/{precision} latent {sum(parts)}x{H}x{W} chunks {parts}"
    t0 = time.time()
    ck = VF.install(monkeypatch, MODULES, eng, spec, tag)
    ck.expect(parts)
    out = _run(eng, x, parts)
    torch.cuda.synchronize()
    VF.finish(ck)
    assert torch.isfinite(out).all()
    print(f"\n[vae dataflow] {tag}: {ck.chunks_run} chunks, wall {time.time() - t0:.1f} s; worst |err|/bound per entry: "
          f"{ck.report()}")
    del out, x, ck
    torch.cuda.empty_cache()


@pytest.mark.parametrize("kind,precision,parts", SMALL, ids=[f"{k}-{p}-{'_'.join(map(str, c))}" for k, p, c in SMALL])
def test_real_width_small_latent(monkeypatch, kind, precision, parts):
    _cell(monkeypatch, kind, precision, parts, 6, 10)


@pytest.mark.parametrize("kind,precision,H,W", PROD, ids=[f"{k}-{p}-{h}x{w}" for k, p, h, w in PROD])
def test_production_spatial_size(monkeypatch, kind, precision, H, W):
    _cell(monkeypatch, kind, precision, [1, 1], H, W)


@pytest.mark.parametrize("kind", ["wan21_dec", "wan22_enc"])
def test_resumed_session(monkeypatch, kind):
    """Three resume=True calls at real width: a growing latent (decoder); [video_k, 4 zero frames] with video_{k+1} extending
    video_k (encoder: each call forks at the start of its zero tail, the next one resumes there)."""
    eng, spec = _setup(kind, "bf16", resume=True)
    t0 = time.time()
    ck = VF.install(monkeypatch, MODULES, eng, spec, f"{kind} session", keep_snaps=True)
    H, W = 6, 10
    if kind.endswith("dec"):
        z = _input(kind, 5, H, W, seed=2)
        for T, parts, u0 in ((2, [2], 0), (3, [1], 2), (5, [2], 3)):
            ck.expect(parts, u0, resume=True)
            eng.decode(z[:, :T].clone())
    else:
        v = _input(kind, 4, H, W, seed=2)
        zeros = torch.zeros(3, 4, *v.shape[2:], device="cuda")
        for T, parts, u0 in ((5, [2, 1], 0), (9, [1, 1], 2), (13, [1, 1], 3)):
            ck.expect(parts, u0, resume=True)
            eng.encode(torch.cat([v[:, :T], zeros], 1))
    torch.cuda.synchronize()
    VF.finish(ck)
    print(f"\n[vae dataflow] {kind} session: {ck.chunks_run} chunks, wall {time.time() - t0:.1f} s; worst |err|/bound per "
          f"entry: {ck.report()}")
