"""Chunk-streamed decode of the Wan VAE decoders (yume_b200/vae22.py, vae21.py) without a GPU, over the torch stand-in of the ops
extended with the streaming entry points (tests/helpers/torch_ops_stream.py):
  * every chunk partition reproduces the reference's own chunked, feature-cached decode of 9 latent frames and encode of 25 and
    27 frames (tests/golden/wan_vae_stream_tiny.pt, tools/make_golden_vae_stream.py) within the VAE bar, and the one-pass
    result within bf16 noise;
  * a one-chunk decode or encode issues the one-pass launches only: no history-form conv, no continuation or window form, no
    carry;
  * the chunk planner: one chunk when the sequence fits and always off CUDA, monotone in the budget, a partition of T;
  * the C-ABI guards applied to include/yume_b200_stream.h.
The encoders stream in chunks of 1 + 4a, then 4b video frames and are checked the same way against the reference's 25- and 27-frame
encodes (27 exercises its trim to 1 + 4k). The stand-in rounds every activation to bf16 and its CPU convolutions round differently for different buffer lengths, so two
partitions agree here to bf16 noise (rel ~1e-2, against > 0.1 when the carried frames are dropped or taken one frame
early); the GPU twin
(tests/test_gpu_vae_stream.py) checks that they agree bit for bit."""
import re
from pathlib import Path

import pytest
import torch

import test_gpu_vae_stream as KS
from helpers import torch_ops_stream
from oracle import wan21vae, wan21vae_enc, wan22vae, wan22vae_enc
from test_kernel_contract_cpu import _entry_problems
from yume_b200 import vae21, vae22, vae_enc, wan_vae

STREAM_HEADER = Path(__file__).resolve().parents[1] / "include" / "yume_b200_stream.h"
DEC_PARTS = [[1] * 9, [2, 7], [4, 5], [1, 3, 5], [8, 1], [3, 3, 3]]
ENC_PARTS = [[1] * 7, [2, 5], [4, 3], [1, 3, 3], [6, 1]]          # latent frames: 1 + 4(n-1) video frames first, then 4n


@pytest.fixture()
def cpu_ops(monkeypatch):
    for mod in (vae22, vae21, vae_enc):
        monkeypatch.setattr(mod, "ops", torch_ops_stream)
    torch_ops_stream.calls.clear()


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(golden_dir / "wan_vae_stream_tiny.pt", weights_only=False)


def _decoder(gold, which):
    g = gold[which]
    mod, Engine = (wan22vae, vae22.Wan22VaeDecoder) if which == "wan22" else (wan21vae, vae21.Wan21VaeDecoder)
    eng = Engine(mod.make_state_dict(g["dec_seed"], **g["dec_cfg"]), mean=g["mean"], std=g["std"], device="cpu", **g["dec_cfg"])
    c = g["decode"]
    return eng, torch.randn(16, c["T"], c["H"], c["W"], generator=torch.Generator().manual_seed(c["seed"])), c


def _encoder(gold, which, T):
    g = gold[which]
    mod, Engine = (wan22vae_enc, vae_enc.Wan22VaeEncoder) if which == "wan22" else (wan21vae_enc, vae_enc.Wan21VaeEncoder)
    eng = Engine(mod.make_state_dict(g["enc_seed"], **g["enc_cfg"]), mean=g["mean"], std=g["std"], device="cpu", **g["enc_cfg"])
    c = g["encode"][T]
    x = torch.randn(3, T, c["H"], c["W"], generator=torch.Generator().manual_seed(c["seed"])).clamp_(-1, 1)
    return eng, x, c


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _check_decode(out, c):
    assert tuple(out.shape) == c["shape"]
    for key, got in (("sample", out[..., ::3, ::3]), ("rowsum", out.sum(-1)), ("colsum", out.sum(-2))):
        assert _rel(got, c[key]) < 3e-2, key                  # the bar of tests/test_host_logic_vae_dec.py


@pytest.mark.parametrize("which", ["wan22", "wan21"])
def test_streamed_decode_reproduces_reference_fixture(cpu_ops, gold, which):
    eng, z, c = _decoder(gold, which)
    one = eng.decode(z)
    _check_decode(one, c)
    for parts in DEC_PARTS:
        torch_ops_stream.calls.clear()
        out = eng._decode_chunks(z, parts)
        _check_decode(out, c)
        assert _rel(out, one) < 2e-2, parts
        assert "conv3d_causal_hist" in torch_ops_stream.calls
        assert ("vae_dupup_add_cont" in torch_ops_stream.calls) == (which == "wan22")


@pytest.mark.parametrize("which", ["wan22", "wan21"])
@pytest.mark.parametrize("T", [25, 27])
def test_streamed_encode_reproduces_reference_fixture(cpu_ops, gold, which, T):
    eng, x, c = _encoder(gold, which, T)
    one = eng.encode(x)
    assert tuple(one.shape) == c["shape"] and _rel(one, c["mu"]) < 3e-2     # the bar of tests/test_host_logic_vae_enc.py
    for parts in ENC_PARTS:
        torch_ops_stream.calls.clear()
        out = eng._encode_chunks(x, parts)
        assert tuple(out.shape) == c["shape"] and _rel(out, c["mu"]) < 3e-2, parts
        assert _rel(out, one) < 2e-2, parts
        assert "conv3d_causal_hist" in torch_ops_stream.calls
        assert ("vae_patchify2_bf16_win" if which == "wan22" else "nchw_to_nhwc_bf16_win") in torch_ops_stream.calls


def test_dropped_or_shifted_carries_are_detected(cpu_ops, gold, monkeypatch):
    """The bars above reject a stream that forgets its history, or carries the frames one position off."""
    eng, z, c = _decoder(gold, "wan22")
    one = eng.decode(z)
    keep = vae22.Wan22VaeDecoder._keep
    for defect in ("zero", "shift"):
        def bad_keep(self, key, frames, n=0, defect=defect):
            keep(self, key, frames, n)
            if self._more:
                cur = self._carry[key]
                if defect == "zero":
                    cur.zero_()
                elif frames.shape[0] > cur.shape[0]:               # the frames before the last ones
                    cur.copy_(frames[frames.shape[0] - cur.shape[0] - 1:frames.shape[0] - 1])
        monkeypatch.setattr(vae22.Wan22VaeDecoder, "_keep", bad_keep)
        assert _rel(eng._decode_chunks(z, [1, 3, 5]), one) > 0.1, defect


@pytest.mark.parametrize("which", ["wan22", "wan21"])
def test_one_chunk_decode_and_encode_issue_the_one_pass_launches(cpu_ops, gold, monkeypatch, which):
    kept = []
    keep = wan_vae.WanVaeEngine._keep                            # every engine's carries go through the base's _keep
    monkeypatch.setattr(wan_vae.WanVaeEngine, "_keep", lambda self, key, f, n=0: (kept.append(key) if self._more else None,
                                                                                 keep(self, key, f, n)))
    streaming = {"conv3d_causal_hist", "vae_dupup_add_cont", "vae_unpatchify2_clamp_win", "nhwc_to_nchw_f32_win",
                 "vae_patchify2_bf16_win", "nchw_to_nhwc_bf16_win"}
    eng, z, c = _decoder(gold, which)
    eng.decode(z)
    assert not streaming & set(torch_ops_stream.calls)
    assert torch_ops_stream.calls.count("vae_unpatchify2_clamp" if which == "wan22" else "nhwc_to_nchw_f32") == 1
    torch_ops_stream.calls.clear()
    enc, x, _ = _encoder(gold, which, 25)
    enc.encode(x)
    assert not streaming & set(torch_ops_stream.calls)
    assert kept == [] and eng._carry is None and enc._carry is None


def test_bad_partitions_are_rejected(cpu_ops, gold):
    eng, z, _ = _decoder(gold, "wan21")
    for parts in ([2, 2], [9, 0], [10]):
        with pytest.raises(vae22.YumeB200Error, match="partition"):
            eng._decode_chunks(z, parts)
    enc, x, _ = _encoder(gold, "wan21", 27)
    for parts in ([3, 3], [8]):
        with pytest.raises(vae22.YumeB200Error, match="partition"):
            enc._encode_chunks(x, parts)


# ------------------------------------------------------------------------------------------------------------
# chunk planner
# ------------------------------------------------------------------------------------------------------------
def _real_width(which):
    mod, Eng, cfg = ((vae22, vae22.Wan22VaeDecoder, dict(dec_dim=256, z_dim=48)) if which == "wan22" else
                     (vae21, vae21.Wan21VaeDecoder, dict(dim=96, z_dim=16)))
    return Eng({k: torch.zeros(v) for k, v in mod.decoder_param_shapes(**cfg).items()}, device="cpu", **cfg)


@pytest.mark.parametrize("which,T,H,W", [("wan22", 21, 44, 80), ("wan21", 37, 68, 120)])
def test_planner_bytes_grow_with_the_chunk_and_cover_the_video(which, T, H, W):
    eng = _real_width(which)
    b = [eng.chunk_bytes(n, T, H, W) for n in range(1, T + 1)]
    assert all(x < y for x, y in zip(b, b[1:]))
    assert b[0] > 4 * 3 * eng._out_shape(T, H, W)[1] * eng._out_shape(T, H, W)[2] * eng._out_shape(T, H, W)[3]


def test_chunk_lengths_rules():
    cost = lambda n: 10 * n + 5                                  # noqa: E731
    assert vae22.chunk_lengths(9, cost, 95) == [9]               # fits: one chunk
    assert vae22.chunk_lengths(9, cost, 94) == [8, 1]
    assert vae22.chunk_lengths(9, cost, 40) == [3, 3, 3]
    assert vae22.chunk_lengths(9, cost, 0) == [1] * 9            # never shorter than one frame
    prev = None
    for budget in range(0, 120, 3):                              # monotone in the budget
        n = vae22.chunk_lengths(9, cost, budget)
        assert sum(n) == 9 and min(n) >= 1
        assert prev is None or n[0] >= prev
        prev = n[0]


def _real_width_encoder(which):
    Eng, shapes, cfg = ((vae_enc.Wan22VaeEncoder, vae_enc.encoder_param_shapes_22, dict(dim=160, z_dim=48)) if which == "wan22" else
                        (vae_enc.Wan21VaeEncoder, vae_enc.encoder_param_shapes_21, dict(dim=96, z_dim=16)))
    return Eng({k: torch.zeros(v) for k, v in shapes(**cfg).items()}, device="cpu", **cfg)


@pytest.mark.parametrize("which,T,H,W", [("wan22", 81, 704, 1280), ("wan21", 177, 544, 960)])
def test_encoder_planner_bytes_grow_with_the_chunk(which, T, H, W):
    eng = _real_width_encoder(which)
    Tl = 1 + (T - 1) // 4
    b = [eng.chunk_bytes(n, T, H, W) for n in range(1, Tl + 1)]
    assert all(x < y for x, y in zip(b, b[1:]))
    assert b[0] > 4 * 3 * T * H * W


def test_planner_is_one_chunk_off_cuda():
    assert _real_width("wan22").plan_chunks(21, 44, 80) == [21]
    assert _real_width_encoder("wan21").plan_chunks(177, 544, 960) == [45]


# ------------------------------------------------------------------------------------------------------------
# C-ABI guards over include/yume_b200_stream.h
# ------------------------------------------------------------------------------------------------------------
def test_library_exports_every_stream_header_symbol():
    import yume_b200
    from yume_b200 import _lib
    declared = set(re.findall(r"^\s*(?:int|long long)\s+(yb_\w+)\s*\(", STREAM_HEADER.read_text(), flags=re.M))
    assert declared == {"yb_conv3d_causal_hist", "yb_vae_dupup_add_cont", "yb_vae_unpatchify2_clamp_win",
                        "yb_nhwc_to_nchw_f32_clamp_win", "yb_vae_patchify2_bf16_win", "yb_nchw_to_nhwc_bf16_win"}
    lib = yume_b200.load()
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/yume_b200_stream.h but not exported"
    assert declared == set(_lib.STREAM_SIGNATURES)
    assert not declared & (set(_lib.SIGNATURES) | set(_lib.CLIP_SIGNATURES) | set(_lib.T5_SIGNATURES))


def test_every_stream_entry_point_has_a_contract_test():
    assert _entry_problems(STREAM_HEADER, modules=(KS,)) == []


def test_stream_entry_point_guard_notices_a_missing_test(monkeypatch):
    covers = dict(KS.COVERS)
    del covers["yb_vae_dupup_add_cont"]
    monkeypatch.setattr(KS, "COVERS", covers)
    assert _entry_problems(STREAM_HEADER, modules=(KS,)) == ["entry point without a contract test: yb_vae_dupup_add_cont"]
