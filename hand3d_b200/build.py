"""Builds libhand3d_b200.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc.

The shared library links the CUDA runtime statically and resolves the driver's
cuTensorMapEncodeTiled at run time, so it loads (and exports every symbol of include/hand3d_b200.h)
on a machine without a GPU; every compute entry point then fails with H3D_ENODEVICE.

`python -m hand3d_b200.build --skew` builds the schedule-skew variant libhand3d_b200_skew.so instead: the same sources with
-DH3D_SKEW_BUILD, which turns the H3D_SKEW hooks of csrc/skew.cuh into configurable delays (tests/test_gpu_schedule_skew.py).  It has its
own objects, log (build/skew/nvcc.log) and stamp, and nothing loads it by default.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libhand3d_b200.so")
STAMP = os.path.join(HERE, ".libhand3d_b200.stamp")
LIB_SKEW = os.path.join(HERE, "libhand3d_b200_skew.so")
STAMP_SKEW = os.path.join(HERE, ".libhand3d_b200_skew.stamp")
SKEW_FLAGS = ["-DH3D_SKEW_BUILD"]
SOURCES = ["api.cu", "elementwise.cu", "reader.cu", "reader_aug.cu", "conv_direct.cu", "conv_wgmma.cu", "conv_wgrad.cu", "train.cu", "train_lift.cu",
           "frames.cu", "eval.cu", "track.cu", "draw.cu", "dropout.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--cudart=static", "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]
# per-source additions: frames.cu builds Pillow's resampling coefficients on the host in double, which must not be fused into FMAs;
# draw.cu's coverage rule is restated in numpy float32, so its device arithmetic must not be contracted either
SOURCE_FLAGS = {"frames.cu": ["-Xcompiler", "-ffp-contract=off"], "draw.cu": ["-fmad=false"]}


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _digest(skew=False):
    h = hashlib.sha256()
    names = sorted(os.listdir(CSRC)) + [os.path.join("..", "..", "include", h) for h in ("hand3d_b200.h", "hand3d_b200_rig.h")]
    for n in names:
        p = os.path.join(CSRC, n)
        if os.path.isfile(p):
            h.update(n.encode())
            h.update(open(p, "rb").read())
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(repr(sorted(SOURCE_FLAGS.items())).encode())
    if skew:
        h.update(" ".join(SKEW_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False, skew: bool = False) -> str:
    """Builds the product library, or with skew=True the schedule-skew variant (its own objects, log and stamp)."""
    lib, stamp = (LIB_SKEW, STAMP_SKEW) if skew else (LIB, STAMP)
    objdir = os.path.join(HERE, "build", "skew") if skew else os.path.join(HERE, "build")
    dig = _digest(skew)
    if not force and os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return lib
    objs = []
    procs = []
    os.makedirs(objdir, exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [_nvcc(), *NVCC_FLAGS, *(SKEW_FLAGS if skew else []), *SOURCE_FLAGS.get(src, []), "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append("== %s ==\n%s" % (src, out))
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError("nvcc failed on %s" % src)
    tmp = lib + ".tmp"       # link next to the target and rename: a reader (or a repo snapshot) never sees a half-written library
    cmd = [_nvcc(), "-shared", "--cudart=static", "-gencode", "arch=compute_90a,code=sm_90a", "-o", tmp, *objs]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    os.replace(tmp, lib)
    with open(os.path.join(objdir, "nvcc.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    open(stamp, "w").write(dig)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, skew="--skew" in sys.argv))
