"""The launch-by-launch dataflow check of the four Wan VAE engines (tests/helpers/vae_dataflow.py) over the torch stand-ins at
tiny width.

The clean engines must pass one-pass and chunked runs, the fp8 decode, and resumed sessions: every launch of every chunk is the
spec's stage, with the spec's operands (carried history frames included), and its output is within the kernel contract's
bound. Each wiring defect below, patched into an engine, must fail with a message that names the stage and the operand (for a
wrong entry, the operand 'entry'); the model-level metric the end-to-end tests use (relative Frobenius error against the
matching oracle) is printed beside the bar it would face, which shows the defects those tests miss."""
import types

import pytest
import torch

from helpers import torch_ops_fp8_vae, torch_ops_resume
from helpers import vae_dataflow as VF
from oracle import wan21vae, wan21vae_enc, wan22vae, wan22vae_enc
from oracle.wan22vae_fp8 import Wan22VaeOracleFp8
from yume_b200 import vae21, vae22, vae_enc

MODULES = (vae22, vae21, vae_enc)
# the stand-ins of every entry the engines launch (bf16, streaming, fp8 and the resume frame comparison)
OPS = types.ModuleType("vae_standin_ops")
OPS.__dict__.update({k: v for k, v in vars(torch_ops_fp8_vae).items() if not k.startswith("__")})
OPS.vae_frame_match = torch_ops_resume.vae_frame_match

DEC_CFG = {"wan22_dec": dict(dec_dim=32, z_dim=16), "wan21_dec": dict(dim=32, z_dim=16)}
ENC_CFG = {"wan22_enc": dict(dim=32, z_dim=16), "wan21_enc": dict(dim=32, z_dim=16)}
# latent H x W of a decode (4 x 6: H*W a multiple of 8, dense attention rows; 3 x 5: per-frame slots), video H x W of an encode
DEC_HW = {"wan22_dec": (4, 6), "wan21_dec": (3, 5)}
ENC_HW = {"wan22_enc": (32, 48), "wan21_enc": (32, 48)}      # latents 2 x 3 (slots) and 4 x 6 (dense)
PARTS = {"dec": ([3], [1, 2], [2, 1], [1, 1, 1]), "enc": ([3], [1, 2], [2, 1])}
# the end-to-end bars of tests/test_gpu_parity.py (bf16) and tests/test_gpu_vae_fp8.py (fp8, tiny fixtures)
BARS = {"bf16": 3e-2, "fp8": 8e-2}


@pytest.fixture()
def cpu(monkeypatch):
    for m in MODULES:
        monkeypatch.setattr(m, "ops", OPS)
    return monkeypatch


def _stats(zd):
    g = torch.Generator().manual_seed(3)
    return 0.2 * torch.randn(zd, generator=g), 0.5 + torch.rand(zd, generator=g)


def _setup(kind, precision="bf16", resume=False):
    """(engine, spec, oracle, input) of one tiny engine."""
    if kind.endswith("dec"):
        cfg = DEC_CFG[kind]
        mod, Eng = (wan22vae, vae22.Wan22VaeDecoder) if kind == "wan22_dec" else (wan21vae, vae21.Wan21VaeDecoder)
        H, W = DEC_HW[kind]
        x = torch.randn(cfg["z_dim"], 3, H, W, generator=torch.Generator().manual_seed(1))
    else:
        cfg = ENC_CFG[kind]
        mod, Eng = (wan22vae_enc, vae_enc.Wan22VaeEncoder) if kind == "wan22_enc" else (wan21vae_enc, vae_enc.Wan21VaeEncoder)
        H, W = ENC_HW[kind]
        x = torch.randn(3, 9, H, W, generator=torch.Generator().manual_seed(1)).clamp_(-1, 1)
    sd = mod.make_state_dict(0, **cfg)
    mean, std = _stats(cfg["z_dim"])
    eng = Eng(sd, mean=mean, std=std, device="cpu", precision=precision, resume=resume, **cfg)
    spec = VF.Spec(kind, sd, cfg, mean, std, "cpu", precision)
    if kind == "wan22_dec" and precision == "fp8":
        orc = Wan22VaeOracleFp8(sd, mean=mean, std=std, **cfg)
    else:
        orc = spec.orc
    return eng, spec, orc, x


def _run(eng, x, parts):
    if isinstance(eng, vae_enc.WanVaeEncoder):
        return eng._encode_chunks(x, parts)
    return eng._decode_chunks(x, parts)


def _want(orc, x):
    return orc.encode(x) if hasattr(orc, "encode") else orc.decode(x)


CLEAN = [(k, "bf16", p) for k in ("wan22_dec", "wan21_dec") for p in PARTS["dec"]] + \
        [(k, "bf16", p) for k in ("wan22_enc", "wan21_enc") for p in PARTS["enc"]] + \
        [("wan22_dec", "fp8", p) for p in PARTS["dec"]]


@pytest.mark.parametrize("kind,precision,parts", CLEAN, ids=[f"{k}-{p}-{'_'.join(map(str, c))}" for k, p, c in CLEAN])
def test_clean_engine_meets_the_spec(cpu, kind, precision, parts):
    eng, spec, _, x = _setup(kind, precision)
    tag = f"{kind}/{precision} chunks {parts}"
    ck = VF.install(cpu, MODULES, eng, spec, tag)
    ck.expect(parts)
    _run(eng, x, parts)
    VF.finish(ck)
    assert ck.chunks_run == len(parts)
    print(f"{tag}: worst |err|/bound per entry: {ck.report()}")


@pytest.mark.parametrize("kind", ["wan21_dec", "wan22_enc"])
def test_resumed_session_meets_the_spec(cpu, kind):
    """Three resume=True calls: a growing latent (decoder), or the 14B sampler's [video_k, zero frames] with video_{k+1}
    extending video_k (encoder: each call forks at the start of its zero tail and the next resumes there)."""
    eng, spec, _, x = _setup(kind, resume=True)
    ck = VF.install(cpu, MODULES, eng, spec, f"{kind} session", keep_snaps=True)
    if kind.endswith("dec"):
        z = torch.randn(x.shape[0], 5, *x.shape[2:], generator=torch.Generator().manual_seed(2))
        calls = [(z[:, :2], [2], 0), (z[:, :3], [1], 2), (z[:, :5], [2], 3)]
        for inp, parts, u0 in calls:
            ck.expect(parts, u0, resume=True)
            eng.decode(inp.clone())
    else:
        H, W = x.shape[2:]
        v = torch.randn(3, 13, H, W, generator=torch.Generator().manual_seed(2)).clamp_(-1, 1)
        zeros = torch.zeros(3, 4, H, W)
        calls = [(torch.cat([v[:, :5], zeros], 1), [2, 1], 0), (torch.cat([v[:, :9], zeros], 1), [1, 1], 2),
                 (torch.cat([v[:, :13], zeros], 1), [1, 1], 3)]
        for inp, parts, u0 in calls:
            ck.expect(parts, u0, resume=True)
            eng.encode(inp)
    VF.finish(ck)
    print(f"{kind} session: {ck.chunks_run} chunks, worst |err|/bound per entry: {ck.report()}")


# ------------------------------------------------------------------------------------------------------------
# defects
# ------------------------------------------------------------------------------------------------------------
BLOCK = "decoder.upsamples.1.upsamples.1"
SHORTCUT = "decoder.upsamples.2.upsamples.0.shortcut"
RES6 = "decoder.upsamples.0.upsamples.0.residual.6"


def _swap_gammas(mp, eng):
    """residual.0 / residual.3 gammas swapped in one block."""
    g = dict(eng.gamma)
    g[BLOCK + ".residual.0"], g[BLOCK + ".residual.3"] = g[BLOCK + ".residual.3"], g[BLOCK + ".residual.0"]
    mp.setattr(eng, "gamma", g)


def _shortcut_bias(mp, eng):
    """One shortcut's bias dropped in the re-pack."""
    lin = dict(eng.lin)
    w, b = lin[SHORTCUT]
    lin[SHORTCUT] = (w, torch.zeros_like(b))
    mp.setattr(eng, "lin", lin)


def _res6_bias(mp, eng):
    """One residual.6 conv's bias dropped in the re-pack (its e4m3 form on the fp8 path)."""
    if RES6 in eng.conv8:
        c8 = dict(eng.conv8)
        wq, sw, b, taps = c8[RES6]
        c8[RES6] = (wq, sw, torch.zeros_like(b), taps)
        mp.setattr(eng, "conv8", c8)
    else:
        cv = dict(eng.conv)
        w, b, taps = cv[RES6]
        cv[RES6] = (w, torch.zeros_like(b), taps)
        mp.setattr(eng, "conv", cv)


def _mid_norm_ones(mp, eng):
    """The mid-attention norm's gamma replaced by ones."""
    g = dict(eng.gamma)
    g["decoder.middle.1.norm"] = torch.ones_like(g["decoder.middle.1.norm"])
    mp.setattr(eng, "gamma", g)


def _time_conv_carry(mp, eng):
    """The stride-2 time_conv carries (and reads back) 2 frames, as a 3-tap conv does, instead of 1."""
    real_keep, real_buf = eng._keep, eng._hist_buf
    mp.setattr(eng, "_keep", lambda key, frames, n=0: real_keep(key, frames, 0 if key.endswith("time_conv") else n))
    mp.setattr(eng, "_hist_buf", lambda key, T, H, W, Cp, zero=False, n=0, fp8=False:
               real_buf(key, T, H, W, Cp, zero, 0 if (key or "").endswith("time_conv") else n, fp8))


def _dupup_cont_first(mp, eng):
    """DupUp3D's continuation form (no frame dropped) in the first chunk too."""
    ops = vae22.ops

    class Shim:
        def __getattr__(self, name):
            return getattr(ops, name)

        def vae_dupup_add(self, *a, **k):
            return ops.vae_dupup_add_cont(*a, **k)
    mp.setattr(vae22, "ops", Shim())


def _scales_wrong_stream(mp, eng):
    """After the first chunk each residual.6 e4m3 input buffer takes its carried scale frames from the block's residual.2
    stream."""
    real = eng._hist_buf

    def hist_buf(key, T, H, W, Cp, zero=False, n=0, fp8=False):
        buf = real(key, T, H, W, Cp, zero, n, fp8)
        if fp8 and key and key.endswith(".residual.6") and eng._chunk > 0:
            other = eng._carry[key[:-len(".residual.6")] + ".residual.2"][1]
            buf[1][:other.shape[0]].copy_(other)
        return buf
    mp.setattr(eng, "_hist_buf", hist_buf)


def _key_slice_off(mp, eng):
    """Each frame after the first of the mid attention scores its queries against the previous frame's keys."""
    ops = vae22.ops

    class Shim:
        def __getattr__(self, name):
            return getattr(ops, name)

        def gemm(self, a, w, bias, out, epilogue, *r, **k):
            if bias is None and epilogue == ops.YB_EPI_F32 and w.storage_offset() > 0:
                rows = a.shape[0]
                w = w.as_strided(w.shape, w.stride(), w.storage_offset() - rows * w.stride(0))
            return ops.gemm(a, w, bias, out, epilogue, *r, **k)
    mp.setattr(vae22, "ops", Shim())


# name: (defect, engine, precisions, chunks, installed after the checker, (stage, operand))
DEFECTS = {
    "res_gammas_swapped": (_swap_gammas, "wan22_dec", ("bf16", "fp8"), [1, 2], False, (BLOCK + ".residual.0", "gamma")),
    "shortcut_bias_dropped": (_shortcut_bias, "wan22_dec", ("bf16", "fp8"), [1, 2], False, (SHORTCUT, "bias")),
    "residual6_bias_dropped": (_res6_bias, "wan22_dec", ("bf16", "fp8"), [1, 2], False, (RES6, "bias")),
    "mid_norm_gamma_ones": (_mid_norm_ones, "wan22_dec", ("bf16", "fp8"), [1, 2], False, ("decoder.middle.1.norm", "gamma")),
    "time_conv_carry_two_frames": (_time_conv_carry, "wan22_enc", ("bf16",), [1, 2], False,
                                   ("encoder.downsamples.1.downsamples.2.resample.1", "out")),
    "dupup_cont_in_first_chunk": (_dupup_cont_first, "wan22_dec", ("bf16",), [1, 2], True,
                                  ("decoder.upsamples.0.shortcut", "entry")),
    "fp8_scales_from_wrong_stream": (_scales_wrong_stream, "wan22_dec", ("fp8",), [1, 2], False,
                                     ("decoder.middle.0.residual.6", "x_scale")),
    "attention_keys_one_frame_off": (_key_slice_off, "wan22_dec", ("bf16",), [3], True, ("decoder.middle.1.frame1.S", "w")),
}
DEFECT_CASES = [(d, p) for d, spec in DEFECTS.items() for p in spec[2]]


def _model_metric(kind, precision, parts, defect):
    """Relative Frobenius error of the defective engine against the matching oracle (what the end-to-end tests see)."""
    with pytest.MonkeyPatch.context() as mp:
        for m in MODULES:
            mp.setattr(m, "ops", OPS)
        eng, _, orc, x = _setup(kind, precision)
        defect(mp, eng)
        try:
            got = _run(eng, x, parts)
        except Exception as e:             # noqa: BLE001  (a defect may break the stand-in's shape logic)
            return f"the run raises {type(e).__name__}"
    want = _want(orc, x)
    return float((got - want).norm() / want.norm())


@pytest.mark.parametrize("name,precision", DEFECT_CASES)
def test_defect_is_caught_at_its_stage_and_operand(cpu, name, precision):
    defect, kind, _, parts, after, (stage, operand) = DEFECTS[name]
    eng, spec, _, x = _setup(kind, precision)
    if not after:
        defect(cpu, eng)
    ck = VF.install(cpu, MODULES, eng, spec, f"{kind}/{precision} chunks {parts}")
    if after:
        defect(cpu, eng)
    ck.expect(parts)
    with pytest.raises(AssertionError) as err:
        _run(eng, x, parts)
    msg = str(err.value)
    cpu.undo()
    rel = _model_metric(kind, precision, parts, defect)
    bar = BARS[precision]
    verdict = rel if isinstance(rel, str) else f"{rel:.3e} against the {precision} oracle, bar {bar:.0e}: " \
        f"{'missed' if rel < bar else 'caught'} by the end-to-end test"
    print(f"{name} [{kind}/{precision}]: caught: {msg}\n    model level: {verdict}")
    assert f"stage '{stage}'" in msg and f"operand '{operand}'" in msg, msg
