"""Build libyume_b200.so (sm_90a only) in-tree with nvcc.

The library is plain C ABI (include/yume_b200.h); there is no torch / pybind dependency in it, so it is built
with a direct nvcc invocation rather than torch.utils.cpp_extension. nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
LIB = CSRC / "libyume_b200.so"
SOURCES = ["gemm.cu", "attention.cu", "elementwise.cu", "vae_elementwise.cu", "probe.cu", "clip.cu", "t5.cu", "gemm_fp8.cu",
           "attention_fp8.cu"]
HEADERS = ["yb_ptx.cuh", "yb_host.h", "../../include/yume_b200.h", "../../include/yume_b200_clip.h",
           "../../include/yume_b200_t5.h", "../../include/yume_b200_stream.h",
           "../../include/yume_b200_fp8.h", "../../include/yume_b200_fp8_attn.h",
           "../../include/yume_b200_fp8_vae.h", "../../include/yume_b200_vae_resume.h",
           "../../include/yume_b200_fp8_sp.h", "../../include/yume_b200_vae_rows.h",
           "../../include/yume_b200_vae_rows_enc.h"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: libyume_b200.so cannot be built")


def _digest() -> str:
    h = hashlib.sha256()
    for name in SOURCES + HEADERS:
        h.update((CSRC / name).read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every .cu under csrc/ into one shared library. Returns the library path."""
    stamp = CSRC / ".build_stamp"
    digest = _digest()
    if not force and LIB.exists() and stamp.exists() and stamp.read_text().strip() == digest:
        return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in SOURCES:
        obj = CSRC / (src[:-3] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(CSRC / src), "-o", str(obj)]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, obj, pr in procs:
        out, _ = pr.communicate()
        log.append(f"== {src}\n{out}")
        if pr.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed on {src}")
        objs.append(str(obj))
    tmp = LIB.with_suffix(".so.tmp")          # link beside the target, then rename: a reader never sees a half-written library
    cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(tmp), *objs]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("nvcc link failed")
    os.replace(tmp, LIB)
    (CSRC / "build.log").write_text("\n".join(log))
    stamp.write_text(digest)
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose=True)
    print(f"built {p}")
