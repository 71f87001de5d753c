"""Builds libhand3d_b200.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc.

The shared library links the CUDA runtime statically and resolves the driver's
cuTensorMapEncodeTiled at run time, so it loads (and exports every symbol of include/hand3d_b200.h)
on a machine without a GPU; every compute entry point then fails with H3D_ENODEVICE.
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
SOURCES = ["api.cu", "elementwise.cu", "reader.cu", "conv_direct.cu", "conv_wgmma.cu", "conv_wgrad.cu", "train.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--cudart=static", "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _digest():
    h = hashlib.sha256()
    names = sorted(os.listdir(CSRC)) + [os.path.join("..", "..", "include", "hand3d_b200.h")]
    for n in names:
        p = os.path.join(CSRC, n)
        if os.path.isfile(p):
            h.update(n.encode())
            h.update(open(p, "rb").read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == dig:
        return LIB
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [_nvcc(), *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append("== %s ==\n%s" % (src, out))
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError("nvcc failed on %s" % src)
    tmp = LIB + ".tmp"       # link next to the target and rename: a reader (or a repo snapshot) never sees a half-written library
    cmd = [_nvcc(), "-shared", "--cudart=static", "-gencode", "arch=compute_90a,code=sm_90a", "-o", tmp, *objs]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    os.replace(tmp, LIB)
    with open(os.path.join(HERE, "build", "nvcc.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    open(STAMP, "w").write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
