"""Wan22VaeDecoder(precision="fp8") end to end on the H100:
  * against the fp8-qdq oracle (oracle/wan22vae_fp8.py) on the tiny fixtures (mixed fp8 / bf16 layers) and at real width, within
    the bars below (the measured values are printed);
  * against the fp32 oracle and the bf16 engine at real width: PSNR >= 30 dB;
  * every chunk partition is `torch.equal` to the one-pass fp8 decode, and the causal prefix property holds at production size;
  * a streamed decode stays within the planner's `chunk_bytes`;
  * precision="bf16" is `torch.equal` to an engine built without the argument."""
import math

import pytest
import torch

from oracle import wan22vae
from oracle.wan22vae_fp8 import Wan22VaeOracleFp8

pytestmark = pytest.mark.gpu

REAL = dict(dec_dim=256, z_dim=48)
# fp8 engine against the fp8-qdq oracle, measured on an H100: tiny fixtures rel-Frobenius 4.8e-2 .. 5.6e-2, PSNR 39.0 .. 43.0 dB;
# real width (3 x 6 x 10 latent) 7.1e-2, 36.9 dB. This misses the bf16 engine's bars (3e-2, 40 dB): the engine quantises the
# bf16 values of its own layer chain and the oracle those of its fp32 chain, so a last-bit bf16 difference moves a value across
# an e4m3 rounding boundary (a 6 % step) and the converted convs in a row compound these flips. The fp8-qdq oracle is itself
# 6e-2 (tiny) from the fp32 oracle. The kernels are pinned per element by tests/test_gpu_kernel_contract_fp8_vae.py.
TINY_BAR, TINY_PSNR = 8e-2, 36.0
REAL_BAR, REAL_PSNR = 1e-1, 34.0


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()
    return "cuda"


def _stats(seed, zd):
    gen = torch.Generator().manual_seed(seed)
    return 0.2 * torch.randn(zd, generator=gen), 0.5 + torch.rand(zd, generator=gen)


@pytest.fixture(scope="module")
def real(dev):
    from yume_b200.vae22 import Wan22VaeDecoder
    sd = wan22vae.make_state_dict(0, **REAL)
    mean, std = _stats(3, REAL["z_dim"])
    kw = dict(mean=mean, std=std, device=dev, **REAL)
    return dict(sd=sd, mean=mean, std=std, fp8=Wan22VaeDecoder(sd, precision="fp8", **kw),
                bf16=Wan22VaeDecoder(sd, precision="bf16", **kw), default=Wan22VaeDecoder(sd, **kw))


def _z(zd, T, H, W, seed=1):
    return torch.randn(zd, T, H, W, generator=torch.Generator().manual_seed(seed)).cuda()


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def psnr(a, b):
    """PSNR of two videos in [-1, 1] (peak-to-peak 2)."""
    mse = float((a.double() - b.double()).pow(2).mean())
    return math.inf if mse == 0 else 10 * math.log10(4.0 / mse)


@pytest.mark.parametrize("case", ["t1", "t2", "t5", "t3_wide"])
def test_tiny_fixture_against_the_fp8_oracle(dev, golden_dir, case):
    from yume_b200.vae22 import Wan22VaeDecoder
    g = torch.load(golden_dir / "wan22vae_tiny.pt", weights_only=False)
    sd = wan22vae.make_state_dict(g["seed_w"], **g["cfg"])
    c = g["cases"][case]
    eng = Wan22VaeDecoder(sd, mean=g["mean"], std=g["std"], device=dev, precision="fp8", **g["cfg"])
    assert eng.conv8 and any(n.endswith((".residual.2", ".residual.6")) for n in eng.conv), "tiny width mixes fp8 and bf16"
    z = torch.randn(g["cfg"]["z_dim"], c["T"], c["H"], c["W"], generator=torch.Generator().manual_seed(c["seed"]))
    got = eng.decode(z.to(dev)).cpu()
    want = Wan22VaeOracleFp8(sd, mean=g["mean"], std=g["std"], **g["cfg"]).decode(z)
    rel, p = _rel(got, want), psnr(got, want)
    print(f"{case}: fp8 engine vs fp8 oracle rel {rel:.2e}, PSNR {p:.1f} dB")
    assert rel < TINY_BAR and p >= TINY_PSNR


def test_real_width_against_the_oracles_and_the_bf16_engine(real):
    z = _z(48, 3, 6, 10, seed=5)
    got = real["fp8"].decode(z)
    bf = real["bf16"].decode(z)
    sd = {k: v.cuda() for k, v in real["sd"].items()}
    kw = dict(mean=real["mean"].cuda(), std=real["std"].cuda(), **REAL)
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        want8 = Wan22VaeOracleFp8(sd, **kw).decode(z)
        want32 = wan22vae.Wan22VaeOracle(sd, **kw).decode(z)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    r8, p8 = _rel(got, want8), psnr(got, want8)
    p32, pbf = psnr(got, want32), psnr(got, bf)
    print(f"real width: fp8 engine vs fp8 oracle rel {r8:.2e} PSNR {p8:.1f} dB; vs fp32 oracle PSNR {p32:.1f} dB; "
          f"vs bf16 engine PSNR {pbf:.1f} dB (bf16 engine vs fp32 oracle {psnr(bf, want32):.1f} dB)")
    assert r8 < REAL_BAR and p8 >= REAL_PSNR
    assert p32 >= 30.0 and pbf >= 30.0


def test_every_partition_is_bit_identical_to_one_pass(real):
    eng = real["fp8"]
    z = _z(48, 9, 4, 6)
    ref = eng._decode_chunks(z, [9])
    assert torch.isfinite(ref).all()
    for parts in ([1] * 9, [2, 7], [4, 5], [1, 3, 5], [8, 1], [3, 3, 3]):
        got = eng._decode_chunks(z, parts)
        assert torch.equal(got, ref), (parts, float((got - ref).abs().max()))


def test_causal_prefix_at_production_size(real):
    eng = real["fp8"]
    z = _z(48, 4, 44, 80, seed=2)
    full = eng._decode_chunks(z, [1, 3])
    for k in (1, 2):
        assert torch.equal(full[:, :4 * k - 3], eng.decode(z[:, :k].contiguous())), k


def test_streamed_decode_within_the_planner_bound(real):
    eng = real["fp8"]
    T, H, W = 21, 44, 80
    z = _z(48, T, H, W, seed=4)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    plan = eng.plan_chunks(T, H, W)
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = eng._decode_chunks(z, [6, 6, 6, 3])
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    bound = eng.chunk_bytes(6, T, H, W)
    print(f"fp8 T={T} chunks of 6 (planner: {plan}): peak {peak / 2**30:.2f} GiB, planner bound {bound / 2**30:.2f} GiB")
    assert peak <= bound
    assert torch.isfinite(out).all()


def test_bf16_precision_is_the_default(real):
    z = _z(48, 3, 6, 10, seed=6)
    assert torch.equal(real["bf16"].decode(z), real["default"].decode(z))
    assert not real["bf16"].conv8 and not real["default"].conv8
