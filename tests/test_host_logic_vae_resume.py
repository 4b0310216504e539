"""Resuming Wan VAE sessions (`resume=True`, WanVaeEngine._resumed) without a GPU, over the torch stand-in of the ops extended with
the frame comparison's twin and an input-voxel count (tests/helpers/torch_ops_resume.py), on the Wan2.1 and Wan2.2 tiny fixtures
of tests/golden/wan_vae_stream_tiny.pt:
  * the 14B sampler's call pattern over 4 calls — a growing latent for the decoders, [video_k, zeros] with
    video_{k+1} = [video_k, new] for the encoders (which resume from the start of the zero tail) — reads only the new frames;
  * the fallbacks (one flipped bit, a -0.0 in the prefix, another H or W, an in-place edit of the returned result, a zero tail
    that does not start on a latent-frame boundary, a shorter input) read the whole input;
  * resume=False keeps nothing and issues the launches of the plain call; the installers pass `resume=` through.
The stand-in's CPU convolutions round differently for different buffer lengths (tests/test_host_logic_vae_stream.py), so each
call is checked `torch.equal` against a fresh engine run over the chunk partition the session amounts to, and within bf16 noise
of the fresh one-pass call; on the GPU every partition is the one pass bit for bit, and tests/test_gpu_vae_resume.py checks each
resumed call `torch.equal` against a fresh full call."""
import types

import pytest
import torch

from helpers import torch_ops_resume as R
from helpers import torch_ops_stream
from oracle import wan21vae, wan21vae_enc, wan22vae, wan22vae_enc
from yume_b200 import vae21, vae22, vae_enc


@pytest.fixture()
def cpu_ops(monkeypatch):
    for mod in (vae22, vae21, vae_enc):
        monkeypatch.setattr(mod, "ops", R)
    torch_ops_stream.calls.clear()
    R.read_voxels.clear()


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(golden_dir / "wan_vae_stream_tiny.pt", weights_only=False)


def _decoder(gold, which, resume=True):
    g = gold[which]
    mod, Engine = (wan22vae, vae22.Wan22VaeDecoder) if which == "wan22" else (wan21vae, vae21.Wan21VaeDecoder)
    return Engine(mod.make_state_dict(g["dec_seed"], **g["dec_cfg"]), mean=g["mean"], std=g["std"], device="cpu", resume=resume,
                  **g["dec_cfg"])


def _encoder(gold, which, resume=True):
    g = gold[which]
    mod, Engine = (wan22vae_enc, vae_enc.Wan22VaeEncoder) if which == "wan22" else (wan21vae_enc, vae_enc.Wan21VaeEncoder)
    eng = Engine(mod.make_state_dict(g["enc_seed"], **g["enc_cfg"]), mean=g["mean"], std=g["std"], device="cpu", resume=resume,
                 **g["enc_cfg"])
    return eng, g["encode"][25]["H"], g["encode"][25]["W"]


def _z(T, H=4, W=6, seed=5):
    return torch.randn(16, T, H, W, generator=torch.Generator().manual_seed(seed))


def _video(T, H, W, seed):
    return torch.randn(3, T, H, W, generator=torch.Generator().manual_seed(seed)).clamp_(-1, 1)


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _reads():
    n = sum(R.read_voxels)
    R.read_voxels.clear()
    return n


def _check_decode(eng, fresh, z, parts, new_frames):
    """One resumed decode: it read `new_frames` latent frames, equals the fresh engine over `parts`, and the one pass to bf16 noise."""
    got = eng.decode(z)
    assert _reads() == new_frames * z.shape[2] * z.shape[3], parts
    want = fresh._decode_chunks(z, parts)
    R.read_voxels.clear()
    assert torch.equal(got, want), parts
    assert _rel(got, fresh.decode(z)) < 2e-2
    R.read_voxels.clear()
    return got


def _check_encode(eng, fresh, v, parts, new_frames):
    got = eng.encode(v)
    assert _reads() == new_frames * v.shape[2] * v.shape[3], parts
    want = fresh._encode_chunks(v, parts)
    R.read_voxels.clear()
    assert torch.equal(got, want), parts
    assert _rel(got, fresh.encode(v)) < 2e-2
    R.read_voxels.clear()
    return got


# ------------------------------------------------------------------------------------------------------------
# the frame comparison's twin
# ------------------------------------------------------------------------------------------------------------
def test_frame_match_twin_is_bitwise():
    x = torch.randn(3, 6, 4, 5)
    x[:, 4:] = 0
    assert R.frame_match(None, x) == (0, 4)
    assert R.frame_match(x.clone(), x) == (6, 4)
    assert R.frame_match(x[:, :3].clone(), x) == (3, 4)
    y = x.clone()
    y[2, 1, 3, 4] = -y[2, 1, 3, 4]
    assert R.frame_match(x, y) == (1, 4)
    y = x.clone()
    y[0, 4, 0, 0] = -0.0                                         # -0.0 == 0.0 numerically, but not bitwise: not a zero frame
    assert R.frame_match(x, y) == (4, 5)
    assert R.frame_match(torch.zeros(3, 2, 4, 5), torch.zeros(3, 3, 4, 5)) == (2, 0)
    n = torch.full((1, 2, 3), float("nan"))
    m = n.clone().view(torch.int32)
    m[0, 1, 2] ^= 1                                              # another NaN payload
    assert R.frame_match(n, m.view(torch.float32)) == (1, 2)


# ------------------------------------------------------------------------------------------------------------
# the 14B sampler's call patterns
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["wan22", "wan21"])
def test_decode_session_runs_only_new_latent_frames(cpu_ops, gold, which):
    eng, fresh = _decoder(gold, which), _decoder(gold, which, resume=False)
    z = _z(9)
    done = 0
    for T in (2, 4, 6, 9):
        parts = [2, 2, 2, 3][:len([t for t in (2, 4, 6, 9) if t <= T])]
        _check_decode(eng, fresh, z[:, :T].contiguous(), parts, T - done)
        done = T
    assert eng.retained_bytes() > 0


@pytest.mark.parametrize("which", ["wan22", "wan21"])
def test_encode_session_resumes_at_the_zero_tail(cpu_ops, gold, which):
    """[video_k, zeros(8)], video_{k+1} = [video_k, 4 new frames]: each call after the first reads the 4 new frames and the zeros."""
    eng, H, W = _encoder(gold, which)
    fresh = _encoder(gold, which, resume=False)[0]
    video = _video(17, H, W, seed=6)
    for k in range(1, 5):
        v = torch.cat([video[:, :1 + 4 * k], torch.zeros(3, 8, H, W)], 1)
        parts = [2] + [1] * (k - 1) + [2]                        # frames 0-4, then 4 per new latent frame, then the zero tail
        _check_encode(eng, fresh, v, parts, v.shape[1] if k == 1 else 12)
        assert set(eng._kept.snaps) == {1 + 4 * k, v.shape[1]}


def test_repeated_call_runs_nothing(cpu_ops, gold):
    eng = _decoder(gold, "wan21")
    z = _z(4)
    first = eng.decode(z)
    _reads()
    again = eng.decode(z.clone())
    assert _reads() == 0 and torch.equal(again, first) and again is not first


# ------------------------------------------------------------------------------------------------------------
# fallbacks: each reads the whole input and equals a fresh full call
# ------------------------------------------------------------------------------------------------------------
def _flip_bit(z, frame):
    z = z.clone()
    z.view(torch.int32)[1, frame, 1, 2] ^= 1
    return z


@pytest.mark.parametrize("which", ["wan22", "wan21"])
@pytest.mark.parametrize("edit", ["bit", "negative_zero"])
def test_decode_falls_back_on_a_changed_prefix(cpu_ops, gold, which, edit):
    eng, fresh = _decoder(gold, which), _decoder(gold, which, resume=False)
    z = _z(6)
    if edit == "negative_zero":                                  # the kept latent holds +0.0 there, the new one -0.0
        z[5, 1, 2, 3] = 0.0
    eng.decode(z[:, :4].contiguous())
    _reads()
    z2 = _flip_bit(z, 2) if edit == "bit" else z.clone()
    if edit == "negative_zero":
        z2[5, 1, 2, 3] = -0.0
    _check_decode(eng, fresh, z2, [6], 6)


def test_decode_falls_back_on_another_size_or_a_shorter_latent(cpu_ops, gold):
    eng, fresh = _decoder(gold, "wan22"), _decoder(gold, "wan22", resume=False)
    z = _z(6)
    eng.decode(z[:, :4].contiguous())
    _reads()
    _check_decode(eng, fresh, _z(6, H=4, W=4), [6], 6)          # another W
    _check_decode(eng, fresh, _z(6, H=2, W=4), [6], 6)          # another H
    _check_decode(eng, fresh, z, [6], 6)
    _check_decode(eng, fresh, z[:, :3].contiguous(), [3], 3)    # shorter than the kept latent


def test_decode_falls_back_after_an_in_place_edit_of_the_result(cpu_ops, gold):
    eng, fresh = _decoder(gold, "wan21"), _decoder(gold, "wan21", resume=False)
    z = _z(6)
    out = eng.decode(z[:, :4].contiguous())
    _reads()
    out[:, 0].mul_(0.5)                                          # the caller edits the video it was handed
    _check_decode(eng, fresh, z, [6], 6)
    eng.decode(z[:, :4].contiguous())
    _reads()
    _check_decode(eng, fresh, z, [4, 2], 2)                      # an untouched result resumes


@pytest.mark.parametrize("which", ["wan22", "wan21"])
def test_encode_with_an_unaligned_zero_tail_falls_back(cpu_ops, gold, which):
    """History of 6 frames (not 1 + 4k) and 7 zero frames: no snapshot at the zero tail, so the next call runs in full."""
    eng, H, W = _encoder(gold, which)
    fresh = _encoder(gold, which, resume=False)[0]
    video = _video(10, H, W, seed=8)
    v1 = torch.cat([video[:, :6], torch.zeros(3, 7, H, W)], 1)
    _check_encode(eng, fresh, v1, [4], 13)
    assert set(eng._kept.snaps) == {13}
    v2 = torch.cat([video[:, :10], torch.zeros(3, 7, H, W)], 1)[:, :17]
    _check_encode(eng, fresh, v2, [5], 17)


def test_encode_flipped_bit_before_the_fork_falls_back(cpu_ops, gold):
    eng, H, W = _encoder(gold, "wan21")
    fresh = _encoder(gold, "wan21", resume=False)[0]
    video = _video(9, H, W, seed=9)
    eng.encode(torch.cat([video[:, :5], torch.zeros(3, 8, H, W)], 1))
    _reads()
    v = _flip_bit(torch.cat([video, torch.zeros(3, 8, H, W)], 1), 3)
    _check_encode(eng, fresh, v, [3, 2], 17)                    # a full run, split where its own zero tail starts


# ------------------------------------------------------------------------------------------------------------
# default unchanged, state accounting
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["wan22", "wan21"])
def test_resume_off_keeps_nothing_and_issues_the_plain_launches(cpu_ops, gold, which):
    eng = _decoder(gold, which, resume=False)
    z = _z(5)
    torch_ops_stream.calls.clear()
    eng._decode_chunks(z, [5])
    plain = list(torch_ops_stream.calls)
    for _ in range(2):
        torch_ops_stream.calls.clear()
        eng.decode(z)
        assert torch_ops_stream.calls == plain and "vae_frame_match" not in plain
    assert eng.retained_bytes() == 0 and eng._kept is None
    enc, H, W = _encoder(gold, which, resume=False)
    v = _video(9, H, W, seed=3)
    torch_ops_stream.calls.clear()
    enc._encode_chunks(v, [3])
    plain = list(torch_ops_stream.calls)
    torch_ops_stream.calls.clear()
    enc.encode(v)
    assert torch_ops_stream.calls == plain and enc.retained_bytes() == 0


def test_retained_bytes_counts_the_kept_tensors_and_reset_drops_them(cpu_ops, gold):
    eng, H, W = _encoder(gold, "wan22")
    v = torch.cat([_video(5, H, W, seed=2), torch.zeros(3, 8, H, W)], 1)
    out = eng.encode(v)
    k = eng._kept
    tensors = {t.data_ptr(): t for t in [k.src, k.out] + [x for _, c in k.snaps.values() for x in c.values()]}
    assert k.out is out and len(k.snaps) == 2
    assert eng.retained_bytes() == sum(t.numel() * t.element_size() for t in tensors.values())
    eng.reset()
    assert eng.retained_bytes() == 0 and eng._kept is None
    _reads()
    eng.encode(v)
    assert _reads() == 13 * H * W                                # after reset() the next call runs in full


# ------------------------------------------------------------------------------------------------------------
# installers, on the recorded reference interfaces
# ------------------------------------------------------------------------------------------------------------
def test_installers_pass_resume_through(cpu_ops, golden_dir):
    """A 3-call session through each installed hook (a prefix, the whole input, the whole input again) against the reference
    objects' recorded outputs, at the bars of tests/test_host_logic_vae_install.py (the prefix against the output's prefix: the
    VAEs are causal)."""
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tools"))
    import make_golden_install as recipe
    golden = torch.load(golden_dir / "install_hooks.pt")

    def model(g, sd):
        return types.SimpleNamespace(state_dict=lambda: dict(sd), **g["attrs"])

    for tree in ("wan22", "wan21"):
        g = golden[tree]
        mean, std, video, z = recipe.wan_vae_inputs(tree)
        sd = recipe.wan22_state_dict() if tree == "wan22" else recipe.wan21_state_dict()
        wrapper = types.SimpleNamespace(model=model(g, sd), mean=mean, std=std, scale=[mean, 1.0 / std], dtype=torch.float)
        if tree == "wan22":
            vae_enc.install_wan22_vae_encoder(wrapper, device="cpu", resume=True)
            vae22.install_wan22_vae(wrapper, device="cpu", resume=True)
        else:
            vae_enc.install_wan21_vae_encoder(wrapper, device="cpu", resume=True)
            vae21.install_wan21_vae(wrapper, device="cpu", resume=True)
        assert wrapper._yb_encoder.resume and wrapper._yb_decoder.resume
        _reads()
        for n_lat, n_vid in ((1, 1), (2, 5), (2, 5)):
            x = wrapper.decode([z[:, :n_lat].contiguous()])[0]
            mu = wrapper.encode([video[:, :n_vid].contiguous()])[0]
            assert x.shape == g["x"][:, :1 + 4 * (n_lat - 1)].shape and _rel(x, g["x"][:, :1 + 4 * (n_lat - 1)]) < 3e-2
            assert mu.shape == g["mu"][:, :n_lat].shape and _rel(mu, g["mu"][:, :n_lat]) < 3e-2
        # latent frames 0, 1, then none; video frames 0, 1-4, then none
        assert _reads() == z.shape[2] * z.shape[3] * 2 + video.shape[2] * video.shape[3] * 5


# ------------------------------------------------------------------------------------------------------------
# C-ABI guards over include/yume_b200_vae_resume.h
# ------------------------------------------------------------------------------------------------------------
def test_library_exports_the_resume_header_symbol():
    import re
    from pathlib import Path

    import yume_b200
    from yume_b200 import _lib
    header = Path(__file__).resolve().parents[1] / "include" / "yume_b200_vae_resume.h"
    declared = set(re.findall(r"^\s*(?:int|long long)\s+(yb_\w+)\s*\(", header.read_text(), flags=re.M))
    assert declared == set(_lib.RESUME_SIGNATURES) == {"yb_vae_frame_match"}
    assert hasattr(yume_b200.load(), "yb_vae_frame_match")
    others = (set(_lib.SIGNATURES) | set(_lib.CLIP_SIGNATURES) | set(_lib.T5_SIGNATURES) | set(_lib.STREAM_SIGNATURES)
              | set(_lib.FP8_SIGNATURES) | set(_lib.FP8_ATTN_SIGNATURES) | set(_lib.FP8_VAE_SIGNATURES))
    assert not declared & others


def test_frame_match_is_a_gpu_op():
    from yume_b200 import YumeB200Error, ops
    with pytest.raises(YumeB200Error, match="CUDA"):
        ops.vae_frame_match(None, torch.zeros(3, 2, 4), torch.zeros(2, dtype=torch.int32))
