"""umT5 text encoder on the GPU (`-m gpu`): yume_b200/t5.py on the sm_90a kernels against
  * the reference fixtures (tests/golden/t5_tiny.pt, the reference's own T5Encoder.forward in fp32);
  * oracle/t5.py in fp32 on the device at the real umT5-XXL width (24 layers, dim 4096, 64 heads of 64, ffn 10240; bf16
    weights generated on the device, vocabulary cut to 32 768 rows: only the gather depends on it), L = 512 with a 120-token
    prompt, the reference's own regime (the oracle in bf16) measured against the same fp32 oracle and printed;
and checks the bucket table the engine builds on the device against the reference's CPU table, and install_t5 on a stand-in
T5EncoderModel at that width (bf16 [1, 512, 4096] out, `.to()` still accepted).
Bars are twice the measured error. Peak memory of the real-width tests: the bf16 weights and the engine's re-packed copy at
once (9.5 GB each at the cut vocabulary), plus one fp32 layer of the oracle: 15.0 GiB measured on an H100 80GB HBM3."""
import gc

import pytest
import torch

from helpers import t5_standin
from oracle import t5 as ot5

pytestmark = pytest.mark.gpu

CASES = ["L512_m1", "L512_m37", "L512_m512", "B2_L77", "L64_none", "L96_holed", "L600", "shared_B2_L77", "shared_L600_holed"]
XXL = dict(ot5.UMT5_XXL, vocab=32768)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import yume_b200
    yume_b200.load()
    return "cuda"


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(golden_dir / "t5_tiny.pt", weights_only=False)


@pytest.fixture(scope="module")
def tiny(gold, dev):
    from yume_b200.t5 import T5TextEncoder
    return {name: T5TextEncoder(ot5.make_state_dict(gold["seed_w"][name], **cfg), **cfg, device=dev)
            for name, cfg in gold["cfg"].items()}


# Measured on the stand-in ops (same roundings, tests/test_t5_cpu.py): 4.8e-3; bar 9.6e-3 as there.
FIXTURE_BAR = 9.6e-3


@pytest.mark.parametrize("case", CASES)
def test_engine_matches_reference_fixture(tiny, gold, dev, case):
    c = gold["cases"][case]
    ids = c["ids"].long().to(dev)
    mask = None if c["mask"] is None else c["mask"].long().to(dev)
    out = tiny[c["model"]](ids, mask)
    assert out.device == ids.device and out.dtype == torch.float32 and tuple(out.shape) == tuple(c["out_shape"])
    out = out.cpu()
    got = torch.stack([out[b, c["out_rows"][b].long()] for b in range(out.shape[0])])
    err = _rel(got, c["out"])
    print(f"[t5] engine vs reference fixture {case}: rel-Frobenius {err:.3g}")
    assert err <= FIXTURE_BAR


def test_device_bucket_table_matches_the_reference_cpu_table(tiny, gold, dev):
    """The engine computes the buckets with the reference's torch expression on its own device, as the reference does on the
    device its embedding lives on. The CPU table has |j - i| = 16, 32 and 64 exactly on a truncation boundary; a
    disagreement of the device's evaluation would show here (the engine follows the device)."""
    import test_gpu_kernel_contract_t5 as KT
    enc = tiny["tiny"]
    bk = enc.buckets(600)
    assert bk.device.type == "cuda"
    got = bk.cpu()[KT.rel_index(600)]
    want = gold["buckets_L600"].long()
    diff = got != want
    print(f"[t5] device bucket table vs reference CPU table at L = 600: {int(diff.sum())} entries differ")
    assert not diff.any(), f"bucket offsets differ at j - i = {sorted({int(j - i) for i, j in diff.nonzero().tolist()})}"
    assert torch.equal(ot5.bucket_table(600, 32, device=dev).cpu(), want)


@pytest.fixture(scope="module")
def xxl(dev):
    """Seeded umT5-XXL-width bf16 weights on the device, and the 512-token inputs with a 120-token prompt."""
    sd = ot5.make_state_dict(4321, **XXL, device=dev, dtype=torch.bfloat16)
    g = torch.Generator().manual_seed(8)
    ids = torch.randint(0, XXL["vocab"], (1, 512), generator=g)
    ids[0, 120:] = 0                                              # the tokenizer's padding id
    mask = torch.zeros(1, 512, dtype=torch.long)
    mask[0, :120] = 1
    yield sd, ids.to(dev), mask.to(dev)
    del sd
    gc.collect()
    torch.cuda.empty_cache()


# The 24-layer fp32 oracle against the engine at the real width, L = 512, 120-token prompt. Measured on an H100 80GB HBM3:
# rel-Frobenius 1.08e-2; the reference's own regime (the oracle in bf16) measures 2.4e-2 against the same oracle. Bar 2.2e-2
# (2x). Peak max_memory_allocated of this test: 15.0 GiB.
XXL_BAR = 2.2e-2


def test_engine_at_umt5_xxl_width_matches_fp32_oracle(dev, xxl):
    from yume_b200.t5 import T5TextEncoder
    sd, ids, mask = xxl
    torch.cuda.reset_peak_memory_stats()
    enc = T5TextEncoder(sd, **XXL, device=dev)
    out = enc(ids, mask)
    del enc
    gc.collect()
    torch.cuda.empty_cache()
    with torch.no_grad():
        ref = ot5.encode(sd, ids, mask, **XXL, dtype=torch.float32)
        reg = ot5.encode(sd, ids, mask, **XXL, dtype=torch.bfloat16)
    assert out.shape == ref.shape == (1, 512, 4096) and out.dtype == torch.bfloat16
    err, err_reg = _rel(out, ref), _rel(reg, ref)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"[t5] umT5-XXL width, L 512, 120-token prompt: engine vs fp32 oracle rel-Frobenius {err:.3g}; reference regime "
          f"(bf16) {err_reg:.3g}; peak max_memory_allocated {peak:.2f} GiB")
    assert err <= XXL_BAR


def test_install_t5_on_standin_at_umt5_xxl_width(dev, xxl):
    from yume_b200.t5 import install_t5
    sd, ids, mask = xxl
    te = t5_standin.make_text_encoder(sd, XXL, dtype=torch.bfloat16, device=dev)
    install_t5(te, device=dev)
    out = te.model(ids, mask)
    assert out.dtype == torch.bfloat16 and tuple(out.shape) == (1, 512, 4096) and torch.isfinite(out).all()
    assert out.device == ids.device
    te.model.to(dev)                                              # moves only the reference's copy: still accepted
    assert torch.equal(te.model(ids, mask), out)
    del te
    gc.collect()
    torch.cuda.empty_cache()
