"""Build libemoport.so (all sm_90a kernels + the C-ABI) in-tree with nvcc.

    python -m emoportraits_b200.csrc.build [--force]

The library is built next to the sources so that it travels with the gpurun snapshot.
"""
from __future__ import annotations

import hashlib
import os
import pathlib
import shutil
import subprocess
import sys

HERE = pathlib.Path(__file__).resolve().parent
LIB = HERE / "libemoport.so"
SOURCES = ["conv_igemm.cu", "grid_sample.cu", "norm.cu", "misc.cu", "masks.cu", "video.cu"]
HEADERS = ["common.cuh", "pose_math.cuh", "wgmma.cuh", "../../include/emoportraits_b200.h"]
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc() -> str:
    for cand in [os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"]:
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _digest() -> str:
    h = hashlib.sha256()
    for f in SOURCES + HEADERS + ["build.py"]:
        h.update((HERE / f).read_bytes())
    h.update(os.environ.get("EMO_NVCC_EXTRA", "").encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False, debug: bool = False) -> pathlib.Path:
    """debug=True: the instrumented build (-DEMO_CONV_DEBUG: parts of the conv kernel can be switched off at run time,
    tools/conv_bound_probe.py) as libemoport_dbg.so next to the product library; loaded only through EMO_LIB=<path>."""
    LIB = HERE / ("libemoport_dbg.so" if debug else "libemoport.so")
    stamp = HERE / (".build_stamp_dbg" if debug else ".build_stamp")
    dig = _digest()
    if LIB.exists() and not force and stamp.exists() and stamp.read_text() == dig:
        return LIB
    flags = [*ARCH_FLAGS, "-O3", "-std=c++17", "-lineinfo"]  # no --use_fast_math: expf/tanhf/division stay IEEE-accurate
    flags += ["-Xcompiler", "-fPIC", "-cudart", "shared"]
    flags += os.environ.get("EMO_NVCC_EXTRA", "").split()
    if debug:
        flags += ["-DEMO_CONV_DEBUG"]
    if verbose:
        flags += ["-Xptxas", "-v"]
    # one nvcc per source, side by side (conv_igemm.cu alone is most of the wall time), then one link
    objdir = HERE / ("_obj_dbg" if debug else "_obj")
    objdir.mkdir(exist_ok=True)
    procs = []
    for src in SOURCES:
        obj = objdir / (pathlib.Path(src).stem + ".o")
        procs.append((src, obj, subprocess.Popen([_nvcc(), *flags, "-c", str(HERE / src), "-o", str(obj)], stdout=subprocess.PIPE,
                                                 stderr=subprocess.STDOUT, text=True)))
    log, failed = "", False
    for src, obj, pr in procs:
        out, _ = pr.communicate()
        log += out
        failed |= pr.returncode != 0
    if failed:
        sys.stderr.write(log)
        raise RuntimeError("nvcc failed building libemoport.so")
    tmp = LIB.with_name(LIB.name + ".tmp")  # link into a temporary name, then rename: a reader (or a gpurun snapshot)
    r = subprocess.run([_nvcc(), *ARCH_FLAGS, "-shared", "-cudart", "shared", "-o", str(tmp)] + [str(o) for _, o, _ in procs],
                       capture_output=True, text=True)  # never sees a half-written library
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        tmp.unlink(missing_ok=True)
        raise RuntimeError("nvcc failed linking libemoport.so")
    r.stdout = log + r.stdout
    os.replace(tmp, LIB)
    if verbose:
        sys.stderr.write(r.stdout + r.stderr)
    stamp.write_text(dig)
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv, debug="--debug" in sys.argv)
    print(p)
