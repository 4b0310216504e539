"""umT5 text encoder (yume_b200/t5.py, oracle/t5.py, include/yume_b200_t5.h) without a GPU:
  * oracle/t5.py reproduces tests/golden/t5_tiny.pt, which tools/make_golden_t5.py wrote by running the reference's own
    T5Encoder.forward (fp32 on CPU), and the reference's bucket table bit for bit;
  * the engine's host logic (weight re-packing, the bias tables, the fp32 stream, the launch sequence) reproduces the same
    fixtures over the torch stand-in of its ops (tests/helpers/torch_ops_t5.py);
  * the umT5-XXL state-dict layout the engine reads is the reference's, and every key is read;
  * install_t5 re-binds T5Encoder.forward on a stand-in, and each configuration and input it rejects is rejected before
    anything runs;
  * the C-ABI guards of include/yume_b200.h applied to include/yume_b200_t5.h, and the bounds of
    tests/test_gpu_kernel_contract_t5.py accept the kernels' arithmetic and reject one realistic defect each.
"""
import re
import types
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

import test_gpu_kernel_contract_t5 as KT
from helpers import t5_standin, torch_ops_t5
from oracle import t5 as ot5
from test_gpu_kernel_contract import assert_within
from test_kernel_contract_cpu import _entry_problems

ROOT = Path(__file__).resolve().parents[1]
T5_HEADER = ROOT / "include" / "yume_b200_t5.h"
CASES = ["L512_m1", "L512_m37", "L512_m512", "B2_L77", "L64_none", "L96_holed", "L600", "shared_B2_L77", "shared_L600_holed"]


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(golden_dir / "t5_tiny.pt", weights_only=False)


def _sd(gold, name):
    cfg = gold["cfg"][name]
    sd = ot5.make_state_dict(gold["seed_w"][name], **cfg)
    got = float(sum(v.abs().sum() for v in sd.values()))
    assert abs(got - gold["weight_abs_sum"][name]) <= 1e-5 * gold["weight_abs_sum"][name], "weight RNG drifted"
    return sd


def _inputs(c):
    return c["ids"].long(), None if c["mask"] is None else c["mask"].long()


def _check_rows(out, c):
    """out [B, L, dim] against the fixture's stored rows: full shape, then rel-Frobenius over the stored rows."""
    assert tuple(out.shape) == tuple(c["out_shape"])
    got = torch.stack([out[b, c["out_rows"][b].long()] for b in range(out.shape[0])])
    return _rel(got, c["out"])


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference_fixture(gold, case):
    c = gold["cases"][case]
    cfg = gold["cfg"][c["model"]]
    ids, mask = _inputs(c)
    out = ot5.encode(_sd(gold, c["model"]), ids, mask, **cfg)
    assert out.dtype == torch.float32
    assert _check_rows(out, c) <= 2e-5


def test_bucket_table_is_the_reference_table(gold):
    """The oracle's and the engine's bucket computations reproduce the reference's [600, 600] table on the CPU bit for bit
    (the engine's 1-D form [2L-1] indexed by j - i + L - 1)."""
    want = gold["buckets_L600"].long()
    assert torch.equal(ot5.bucket_table(600, 32), want)
    from yume_b200.t5 import relative_position_bucket
    rel = torch.arange(2 * 600 - 1) - 599
    assert torch.equal(relative_position_bucket(rel, 32, 128)[KT.rel_index(600)], want)
    # the boundaries that sit on a truncation: |j - i| = 16, 32, 64 open buckets 10, 12 and 14 (+16 for j > i)
    assert [int(want[0, d]) for d in (15, 16, 31, 32, 63, 64)] == [25, 26, 27, 28, 29, 30]


def _engine(gold, name, monkeypatch, sd=None, device="cpu"):
    from yume_b200 import t5 as eng
    monkeypatch.setattr(eng, "ops", torch_ops_t5)
    return eng.T5TextEncoder(sd if sd is not None else _sd(gold, name), **gold["cfg"][name], device=device)


# The engine over the stand-in differs from the fp32 fixture by its bf16 GEMM operands, bf16 q / k / v, P and FFN activations.
# Measured worst rel-Frobenius over the cases: 4.8e-3 (L64_none); bar 9.6e-3 (2x).
ENGINE_BAR = 9.6e-3


@pytest.mark.parametrize("case", CASES)
def test_engine_host_logic_matches_reference_fixture(gold, monkeypatch, case):
    c = gold["cases"][case]
    enc = _engine(gold, c["model"], monkeypatch)
    ids, mask = _inputs(c)
    out = enc(ids, mask)
    assert out.dtype == torch.float32                         # the fp32 model's dtype
    err = _check_rows(out, c)
    print(f"[t5] engine (stand-in ops) vs reference fixture {case}: rel-Frobenius {err:.3g}")
    assert err <= ENGINE_BAR


def test_umt5_xxl_layout_is_the_reference_layout(gold):
    """The recorded umt5_xxl encoder state dict (keys and shapes), oracle.t5.param_shapes and the stand-in's keys agree."""
    assert gold["umt5_xxl_cfg"] == ot5.UMT5_XXL
    want = {k: tuple(v) for k, v in gold["umt5_xxl_shapes"].items()}
    assert ot5.param_shapes(**ot5.UMT5_XXL) == want
    with torch.device("meta"):
        standin = t5_standin.T5EncoderStandin(**ot5.UMT5_XXL)
    assert {k: tuple(v.shape) for k, v in standin.state_dict().items()} == want


class _Recording(dict):
    def __init__(self, *a):
        super().__init__(*a)
        self.read = set()

    def __getitem__(self, k):
        self.read.add(k)
        return super().__getitem__(k)


@pytest.mark.parametrize("name", ["tiny", "tiny_shared"])
def test_engine_reads_every_key(gold, monkeypatch, name):
    sd = _Recording(_sd(gold, name))
    _engine(gold, name, monkeypatch, sd)
    assert sd.read == set(sd)


def test_key_mapping_consumes_every_umt5_xxl_key(gold, monkeypatch):
    """The engine's key reads at the umT5-XXL layout (meta tensors: shapes only) are exactly the recorded keys."""
    from yume_b200 import t5 as eng
    monkeypatch.setattr(eng, "ops", torch_ops_t5)
    sd = _Recording({k: torch.empty(v, device="meta", dtype=torch.bfloat16) for k, v in gold["umt5_xxl_shapes"].items()})
    enc = eng.T5TextEncoder(sd, **ot5.UMT5_XXL, device="meta")
    assert sd.read == set(gold["umt5_xxl_shapes"])
    b = enc.blocks[0]
    assert tuple(b.w_qkv.shape) == (3 * 4096, 4096) and tuple(b.w_ug.shape) == (2 * 10240, 4096)
    assert tuple(b.w_fc2.shape) == (4096, 10240) and tuple(b.emb.shape) == (32, 64) and len(enc.blocks) == 24


def test_engine_repacks_in_the_reference_order(gold, monkeypatch):
    sd = _sd(gold, "tiny")
    enc = _engine(gold, "tiny", monkeypatch, sd)
    b = enc.blocks[1]
    bf = lambda k: sd["blocks.1." + k].bfloat16()                   # noqa: E731
    assert torch.equal(b.w_qkv, torch.cat([bf("attn.q.weight"), bf("attn.k.weight"), bf("attn.v.weight")]))
    assert torch.equal(b.w_ug, torch.cat([bf("ffn.fc1.weight"), bf("ffn.gate.0.weight")]))
    assert torch.equal(b.emb, sd["blocks.1.pos_embedding.embedding.weight"])
    tabs = enc.bias_tables(77)
    want = ot5.position_bias(sd["blocks.1.pos_embedding.embedding.weight"], 77)[0]          # [heads, L, L]
    assert torch.equal(tabs[1][:, KT.rel_index(77)], want)


def test_install_t5_rebinds_forward(gold, monkeypatch):
    from yume_b200 import t5 as eng
    monkeypatch.setattr(eng, "ops", torch_ops_t5)
    sd, cfg = _sd(gold, "tiny"), gold["cfg"]["tiny"]
    te = t5_standin.make_text_encoder(sd, cfg, dtype=torch.float32)
    enc = eng.install_t5(te, device="cpu")
    assert te.yume_b200_t5 is enc and enc.layers == cfg["num_layers"]
    c = gold["cases"]["B2_L77"]
    ids, mask = _inputs(c)
    out = te.model(ids, mask)                                     # nn.Module.__call__ -> the re-bound forward
    assert out.dtype == torch.float32 and _check_rows(out, c) <= ENGINE_BAR
    # the shipped regime: bf16 weights -> bf16 result; .to() / .cpu() still work and move only the reference's copy
    te16 = t5_standin.make_text_encoder(sd, cfg, dtype=torch.bfloat16)
    eng.install_t5(te16, device="cpu")
    te16.model.to("cpu")
    te16.model.cpu()
    out16 = te16.model(ids, mask)
    assert out16.dtype == torch.bfloat16 and tuple(out16.shape) == (2, 77, 256)
    assert _check_rows(out16.float(), c) <= 2 * ENGINE_BAR


def _raise_on_launch():
    def boom(*a, **k):
        raise AssertionError("a kernel was launched")
    return types.SimpleNamespace(**{n: boom for n in ("gemm", "t5_attention", "t5_rmsnorm", "t5_geglu")},
                                 YB_EPI_BF16=0, YB_EPI_GATE_RES=3)


@pytest.mark.parametrize("variant", ["head_dim_128", "fp16", "training"])
def test_install_t5_rejects_unimplemented_configs(gold, monkeypatch, variant):
    from yume_b200 import t5 as eng
    cfg = dict(gold["cfg"]["tiny"])
    dtype = torch.float32
    if variant == "head_dim_128":
        cfg["num_heads"] = 2
    elif variant == "fp16":
        dtype = torch.float16
    sd = ot5.make_state_dict(1, **cfg)
    te = t5_standin.make_text_encoder(sd, cfg, dtype=dtype)
    if variant == "training":
        monkeypatch.setattr(eng, "ops", _raise_on_launch())
        eng.install_t5(te, device="cpu")
        te.model.train()
        with pytest.raises(NotImplementedError, match="training"):
            te.model(torch.zeros(1, 8, dtype=torch.long))
        return
    with pytest.raises(NotImplementedError, match="head_dim" if variant == "head_dim_128" else "fp16"):
        eng.install_t5(te, device="cpu")


@pytest.mark.parametrize("bad,exc,match", [
    ("mask_3d", NotImplementedError, "3-D"), ("id_negative", IndexError, "out of range"),
    ("id_vocab", IndexError, "out of range"), ("mask_empty_row", ValueError, "no nonzero")])
def test_rejected_inputs_never_launch(gold, monkeypatch, bad, exc, match):
    from yume_b200 import t5 as eng
    sd, cfg = _sd(gold, "tiny"), gold["cfg"]["tiny"]
    monkeypatch.setattr(eng, "ops", _raise_on_launch())
    te = t5_standin.make_text_encoder(sd, cfg, dtype=torch.float32)
    eng.install_t5(te, device="cpu")
    ids = torch.randint(0, cfg["vocab"], (2, 16), generator=torch.Generator().manual_seed(0))
    mask = torch.ones(2, 16, dtype=torch.long)
    if bad == "mask_3d":
        mask = torch.ones(2, 16, 16, dtype=torch.long)
    elif bad == "id_negative":
        ids[1, 3] = -1
    elif bad == "id_vocab":
        ids[0, 5] = cfg["vocab"]
    else:
        mask[1] = 0
    with pytest.raises(exc, match=match):
        te.model(ids, mask)
    if bad.startswith("id_"):                     # nn.Embedding on the CPU raises IndexError for the same ids
        with pytest.raises(IndexError):
            F.embedding(ids, sd["token_embedding.weight"])


def test_mask_of_any_dtype_nonzero_means_attend(gold, monkeypatch):
    """A bool, int8 or float mask gives the result of the long mask (the reference tests mask == 0)."""
    c = gold["cases"]["L96_holed"]
    enc = _engine(gold, "tiny", monkeypatch)
    ids, mask = _inputs(c)
    want = enc(ids, mask)
    for m in (mask.bool(), mask.to(torch.int8), mask.float() * 3.5):
        assert torch.equal(enc(ids, m), want)


# ------------------------------------------------------------------------------------------------------------
# C-ABI guards over include/yume_b200_t5.h
# ------------------------------------------------------------------------------------------------------------
def test_library_exports_every_t5_header_symbol():
    import yume_b200
    from yume_b200 import _lib
    declared = set(re.findall(r"^\s*(?:int|long long)\s+(yb_\w+)\s*\(", T5_HEADER.read_text(), flags=re.M))
    assert declared == {"yb_t5_attention", "yb_t5_rmsnorm", "yb_t5_geglu"}
    lib = yume_b200.load()
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/yume_b200_t5.h but not exported"
    assert declared == set(_lib.T5_SIGNATURES)
    assert not declared & (set(_lib.SIGNATURES) | set(_lib.CLIP_SIGNATURES))


def test_every_t5_entry_point_has_a_contract_test():
    assert _entry_problems(T5_HEADER, modules=(KT,)) == []


def test_t5_entry_point_guard_notices_a_missing_test(monkeypatch):
    covers = dict(KT.COVERS)
    del covers["yb_t5_geglu"]
    monkeypatch.setattr(KT, "COVERS", covers)
    assert _entry_problems(T5_HEADER, modules=(KT,)) == ["entry point without a contract test: yb_t5_geglu"]


def test_rmsnorm_widths_match_the_kernel_instances():
    from yume_b200.t5 import RMSNORM_WIDTHS
    src = (ROOT / "yume_b200" / "csrc" / "t5.cu").read_text()
    cases = {int(c): int(nv) for c, nv in re.findall(r"case (\d+): return launch_rmsnorm<(\d+)>", src)}
    assert all(c == 128 * nv for c, nv in cases.items())
    assert tuple(sorted(cases)) == RMSNORM_WIDTHS == KT.RMS_WIDTHS


# ------------------------------------------------------------------------------------------------------------
# the bounds: accept the kernels' arithmetic, reject the defects
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def att_case():
    g = KT._gen("t5att cpu")
    B, L, heads = 2, 150, 3
    q, k, v, bias, keep = KT.attention_inputs(g, B, L, heads, "holed")
    ref, bound = KT.t5_attention_ref(q, k, v, bias, keep, B, heads)
    return q, k, v, bias, keep, B, heads, ref, bound


def _emulated_attention(q, k, v, bias, keep, B, heads):
    out = torch.empty(q.shape[0], heads * 64, dtype=torch.bfloat16)
    return torch_ops_t5.t5_attention(q, k, v, out, B, heads, bias, None if keep is None else keep.to(torch.uint8))


def test_attention_bound_accepts_the_kernel_arithmetic(att_case):
    q, k, v, bias, keep, B, heads, ref, bound = att_case
    assert assert_within(_emulated_attention(q, k, v, bias, keep, B, heads), ref, bound, "t5_attention emulated") <= 1.0


def test_attention_bound_rejects_a_flipped_bias_sign(att_case):
    q, k, v, bias, keep, B, heads, ref, bound = att_case
    bad, _ = KT.t5_attention_ref(q, k, v, bias, keep, B, heads, flip=True)
    with pytest.raises(AssertionError, match="out of bound"):
        assert_within(bad.to(torch.bfloat16), ref, bound, "t5_attention bias(i - j)")


def test_attention_bound_rejects_one_masked_key_included(att_case):
    q, k, v, bias, keep, B, heads, ref, bound = att_case
    leaky = keep.clone()
    j = int((~keep[1]).nonzero()[0])
    leaky[1, j] = True                                             # one masked key of sample 1 attends
    with pytest.raises(AssertionError, match="out of bound"):
        assert_within(_emulated_attention(q, k, v, bias, leaky, B, heads), ref, bound, "t5_attention leaky key")


def test_attention_bound_rejects_a_scaled_score(att_case):
    q, k, v, bias, keep, B, heads, ref, bound = att_case
    bad, _ = KT.t5_attention_ref(q, k, v, bias, keep, B, heads, scale=0.125)
    with pytest.raises(AssertionError, match="out of bound"):
        assert_within(bad.to(torch.bfloat16), ref, bound, "t5_attention 1/8 scale")


@pytest.fixture(scope="module")
def geglu_case():
    g = KT._gen("t5geglu cpu")
    L, F_ = 256, 1024
    ug = (torch.randn(L, 2 * F_, generator=g) * 2).to(torch.bfloat16)
    ref, bound = KT.geglu_ref(ug, F_)
    return ug, F_, ref, bound


def test_geglu_bound_accepts_the_kernel_arithmetic(geglu_case):
    ug, F_, ref, bound = geglu_case
    got = torch_ops_t5.t5_geglu(ug, torch.empty(ug.shape[0], F_, dtype=torch.bfloat16))
    assert assert_within(got, ref, bound, "t5_geglu fp32") <= 1.0


@pytest.mark.parametrize("defect", ["erf", "swap"])
def test_geglu_bound_rejects_the_defects(geglu_case, defect):
    ug, F_, ref, bound = geglu_case
    u, g = ug[:, :F_].float(), ug[:, F_:].float()
    bad = (u * F.gelu(g)) if defect == "erf" else (g * F.gelu(u, approximate="tanh"))
    with pytest.raises(AssertionError, match="out of bound"):
        assert_within(bad.to(torch.bfloat16), ref, bound, f"t5_geglu {defect}")


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
def test_rmsnorm_bound_accepts_fp32_and_rejects_a_subtracted_mean(out_dtype):
    from test_gpu_kernel_contract import U32, bf16_out_bound
    g = KT._gen("t5rms cpu")
    x = (torch.randn(64, 4096, generator=g) + 0.5) * torch.exp(torch.randn(64, 1, generator=g))
    w = 1.0 + 0.3 * torch.randn(4096, generator=g)
    ref, f32 = KT.rmsnorm_ref(x, w)
    bound = bf16_out_bound(ref, f32) if out_dtype == torch.bfloat16 else f32 + U32 * ref.abs()
    got = torch_ops_t5.t5_rmsnorm(x, torch.empty(64, 4096, dtype=out_dtype), w)
    assert assert_within(got, ref, bound, "t5_rmsnorm fp32") <= 1.0
    bad = x - x.mean(dim=1, keepdim=True)
    bad = torch_ops_t5.t5_rmsnorm(bad, torch.empty(64, 4096, dtype=out_dtype), w)
    with pytest.raises(AssertionError, match="out of bound"):
        assert_within(bad, ref, bound, "t5_rmsnorm mean subtracted")
