"""Row-parallel Wan VAE encode across processes (`-m gpu`): `torchrun --nproc-per-node P` runs tests/helpers/vae_rows_enc_mp.py,
and every rank's mu of a seeded real-width 49-frame video (Wan2.2 at 704x1280, Wan2.1 at 544x960) must be `torch.equal` to the
one-process encode — in one call, forced into several chunks, and in the 14B loop's resumed [history, zeros] pair.
  * P = 2, 3 and 8 processes on one H100 over gloo (device tensors through host memory; uneven bands at P = 3 and 8);
  * P = 2 and 8 over NCCL, one GPU per rank, skipped when the machine has fewer GPUs.
Each run is a subprocess with a timeout, so no rank outlives the test."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
WORKER = ROOT / "tests" / "helpers" / "vae_rows_enc_mp.py"


@pytest.fixture(scope="module")
def want(tmp_path_factory):
    """The one-process mus, written where the ranks read them."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    sys.path.insert(0, str(ROOT / "tests" / "helpers"))
    import vae_rows_enc_mp
    out = {}
    d = tmp_path_factory.mktemp("rows_enc")
    for which in ("wan22", "wan21"):
        eng = vae_rows_enc_mp.engine(which, "cuda")
        v = vae_rows_enc_mp.video(which).cuda()
        first, second = vae_rows_enc_mp.resumed_pair(v)
        mus = {"mu": eng.encode(v).cpu(), "first": eng.encode(first).cpu(), "second": eng.encode(second).cpu()}
        out[which] = d / f"{which}.pt"
        torch.save(mus, out[which])
        del eng, v, first, second
    torch.cuda.empty_cache()
    return out


def _run(P, which, backend, want_file, same_device):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc-per-node={P}", str(WORKER),
           "--which", which, "--backend", backend, "--want", str(want_file)] + (["--same-device"] if same_device else [])
    env = dict(os.environ, OMP_NUM_THREADS="2", PYTHONPATH=str(ROOT))
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    log = r.stdout + r.stderr[-4000:]
    assert r.returncode == 0, log
    assert log.count("equal") - log.count("DIFFERS") == 4 * P, log


@pytest.mark.parametrize("which", ["wan22", "wan21"])
@pytest.mark.parametrize("P", [2, 3, 8])
def test_processes_on_one_gpu_over_gloo(want, P, which):
    _run(P, which, "gloo", want[which], True)


@pytest.mark.parametrize("which", ["wan22", "wan21"])
@pytest.mark.parametrize("P", [2, 8])
def test_gpus_over_nccl(want, P, which):
    if torch.cuda.device_count() < P:
        pytest.skip(f"needs {P} GPUs")
    _run(P, which, "nccl", want[which], False)
