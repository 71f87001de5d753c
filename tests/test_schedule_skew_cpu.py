"""The schedule-skew hooks (csrc/skew.cuh) on the host: they compile away in the product library, exist in every hooked kernel of the
skew variant, leave the register allocation the warp-specialised kernels rely on, and the product library refuses their tuning keys.
No GPU needed: SASS comes from cuobjdump, registers from the -Xptxas -v logs of the two builds."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hand3d_b200")
LIB, LIB_SKEW = os.path.join(PKG, "libhand3d_b200.so"), os.path.join(PKG, "libhand3d_b200_skew.so")
LOG, LOG_SKEW = os.path.join(PKG, "build", "nvcc.log"), os.path.join(PKG, "build", "skew", "nvcc.log")

# mangled-name pattern -> number of instances; every one carries at least one hook
HOOKED = {
    r"conv_tc_kernelILi": 9, r"conv_c3_tc_kernelI": 4, r"fc_chain_kernelI": 2, r"conv_wgrad_tc_kernelILi": 4,
    r"mask_grow_cluster_kernel": 1, r"seg_prob_kernelI": 2, r"heatmap_argmax_kernel": 1, r"resize_argmax_kernelI": 1,
    r"resize_argmax_pow2_kernelI": 1, r"adam_step_kernel": 1,
}
SETMAXNREG = (r"conv_tc_kernelILi", r"conv_wgrad_tc_kernelILi")   # launched at 168 registers, redistributed by setmaxnreg
# registers per thread at which the launch bounds still give the product's occupancy: (384, 1) -> 168, (256, 2) -> 128, (1024, 1) -> 64
REG_BOUND = {r"fc_chain_kernelI": 168, r"conv_c3_tc_kernelI": 128, r"mask_grow_cluster_kernel": 64}


def _cuobjdump():
    for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if c and os.path.exists(c):
            return c
    pytest.skip("cuobjdump not found")


def _sleeps(lib):
    """{mangled kernel name: number of plain NANOSLEEP instructions}.  NANOSLEEP.SYNCS is mbarrier.try_wait's suspend hint, not a hook."""
    sass = subprocess.run([_cuobjdump(), "-sass", lib], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    out, fn = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            out[fn] = 0
        elif fn and re.search(r"\bNANOSLEEP\s", line):
            out[fn] += 1
    return out


def _hooked(names):
    got = {pat: [n for n in names if re.search(pat, n)] for pat in HOOKED}
    for pat, n in HOOKED.items():
        assert len(got[pat]) == n, (pat, got[pat])
    return got


def _log(path):
    out = {}
    for sec in open(path).read().split("Compiling entry function")[1:]:
        out[sec.split("'")[1]] = (int(re.search(r"Used (\d+) registers", sec).group(1)),
                                  int(re.search(r"(\d+) bytes spill stores", sec).group(1)))
    return out


def test_product_library_has_no_hook():
    if not os.path.exists(LIB):
        pytest.skip("no library: run python -m hand3d_b200.build first")
    sleeps = _sleeps(LIB)
    for pat, names in _hooked(sleeps).items():
        for n in names:
            assert sleeps[n] == 0, "%s: %d NANOSLEEP in the product build" % (n, sleeps[n])


def test_skew_library_has_a_hook_in_every_hooked_kernel():
    if not os.path.exists(LIB_SKEW):
        pytest.skip("no skew variant: run python -m hand3d_b200.build --skew first")
    sleeps = _sleeps(LIB_SKEW)
    for pat, names in _hooked(sleeps).items():
        for n in names:
            assert sleeps[n] > 0, "%s has no hook in the skew build" % n


def test_skew_build_keeps_the_register_allocation():
    """setmaxnreg only redistributes what the launch allocated: the skew build of the warp-specialised kernels must be allocated
    exactly as the product build (168) and spill nothing, or a skewed run would not run the product's register budget."""
    if not (os.path.exists(LOG) and os.path.exists(LOG_SKEW)):
        pytest.skip("build logs missing: run python -m hand3d_b200.build and python -m hand3d_b200.build --skew first")
    prod, skew = _log(LOG), _log(LOG_SKEW)
    assert set(prod) == set(skew)
    for pat, names in _hooked(skew).items():
        for n in names:
            regs, spill = skew[n]
            assert spill == 0 and prod[n][1] == 0, "%s spills %d bytes in the skew build" % (n, spill)
            if pat in SETMAXNREG:
                assert regs == prod[n][0] == 168, "%s allocated at %d registers (product %d)" % (n, regs, prod[n][0])
            elif pat in REG_BOUND:
                assert regs <= REG_BOUND[pat], "%s uses %d registers, past its launch bound's %d" % (n, regs, REG_BOUND[pat])


@pytest.mark.parametrize("key", ["skew_reset", "skew_producer_ns", "skew_consumer_role", "skew_cluster_period", "skew_ticket_seed"])
def test_product_library_rejects_skew_keys(key):
    from hand3d_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("no library: run python -m hand3d_b200.build first")
    lib = _lib.load()
    assert lib.h3d_set_tuning(None, key.encode(), 1) == _lib.EINVAL
    assert "unknown key" in _lib.last_error()
