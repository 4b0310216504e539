"""precision="fp8" and "fp8_attn" under Ulysses sequence parallelism on 2, 4 and 8 GPUs: tools/sp_parity.py under torchrun with
YB_SP_PRECISION, every golden forward case of the tiny and 8-head models, transports p2p (NVLink peer-memory kernels: the q|k|v
scatter in the norm/RoPE pass, the output scatter in the fp8 attention's epilogue) and nccl (the pack into the send buffer, two
all-to-alls), with the KV tail split forced through the peer-scatter combine or not. The tool holds each output to the one-GPU CPU
bars (3e-2 of the fp8 oracle, 5e-2 of the reference's forward) and prints the distance to the same engine on one GPU.
Skipped on boxes with fewer GPUs than the world size."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("split", ["0", "2"])
@pytest.mark.parametrize("precision", ["fp8", "fp8_attn"])
@pytest.mark.parametrize("transport", ["p2p", "nccl"])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_fp8_ulysses_matches_golden(world, transport, precision, split):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    root = Path(__file__).resolve().parents[1]
    env = dict(os.environ, YB_SP_TRANSPORT=transport, YB_SP_PRECISION=precision)
    if split != "0":
        env["YB_ATT_FORCE_SPLIT"] = split
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29633 + world), str(root / "tools" / "sp_parity.py")],
                       capture_output=True, text=True, timeout=1800, env=env)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
