"""TEST INFRASTRUCTURE: the torch-CPU stand-in of tests/helpers/torch_ops_stream.py extended with the frame comparison of
include/yume_b200_vae_resume.h (`frame_match`, the twin the GPU test checks the kernel against) and a count of the input voxels
each engine reads, so a test can see which frames a resumed call ran. Tests monkeypatch it in; the package never imports it."""
import torch

from helpers import torch_ops_stream
from helpers.torch_ops_stream import *  # noqa: F401,F403  (every stand-in the engines call)

read_voxels = []    # input voxels (frames x H x W of the latent or video) each input gather read since the last clear()

_BITS = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def frame_match(kept, x):
    """(first frame < min(Tk, T) at which kept [C, Tk, ...] and x [C, T, ...] differ in any bit, else min(Tk, T); start of x's
    trailing run of all-zero frames) — the contract of yb_vae_frame_match, on the raw bits."""
    C, T = x.shape[:2]
    xb = x.contiguous().view(_BITS[x.element_size()]).reshape(C, T, -1)
    n = 0 if kept is None else min(kept.shape[1], T)
    first = n
    if n:
        kb = kept.contiguous().view(_BITS[kept.element_size()]).reshape(C, kept.shape[1], -1)
        diff = (kb[:, :n] != xb[:, :n]).any(-1).any(0).nonzero()
        first = int(diff[0]) if len(diff) else n
    nz = (xb != 0).any(-1).any(0).nonzero()
    return first, (int(nz[-1]) + 1 if len(nz) else 0)


def vae_frame_match(kept, x, result):
    torch_ops_stream.calls.append("vae_frame_match")
    result.copy_(torch.tensor(frame_match(kept, x), dtype=torch.int32))
    return result


def _reads(fn, voxels):
    def wrapper(*a, **k):
        read_voxels.append(voxels(*a))
        return fn(*a, **k)
    return wrapper


nchw_to_nhwc_bf16 = _reads(torch_ops_stream.nchw_to_nhwc_bf16, lambda x, out: out.shape[0])
nchw_to_nhwc_bf16_win = _reads(torch_ops_stream.nchw_to_nhwc_bf16_win, lambda x, out: out.shape[0])
vae_patchify2_bf16 = _reads(torch_ops_stream.vae_patchify2_bf16, lambda v, out: v.shape[1] * v.shape[2] * v.shape[3])
vae_patchify2_bf16_win = _reads(torch_ops_stream.vae_patchify2_bf16_win, lambda v, out: v.shape[1] * v.shape[2] * v.shape[3])
