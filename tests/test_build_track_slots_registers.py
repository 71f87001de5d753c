"""Register allocation of the slot-selection kernels and of every kernel that takes a device-counted batch (HandSegNet's counted
plan), read from the -Xptxas -v log the build writes (no GPU needed): sm_90a, no spills, and conv_tc_kernel still allocated at 168
registers per thread."""
import os
import re

import pytest

LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hand3d_b200", "build", "nvcc.log")
KERNELS = ["track_select_kernel", "track_merge_kernel", "conv_tc_kernel", "conv_c3_tc_kernel", "conv3x3_c3_kernel", "conv_direct_kernel",
           "maxpool_split_kernel", "maxpool_f32_kernel", "resize_bilinear_tf1_kernel", "seg_prob_kernel", "mask_grow_kernel",
           "mask_grow_cluster_kernel"]


def _sections():
    if not os.path.exists(LOG):
        pytest.skip("no build log: run python -m hand3d_b200.build first")
    for sec in open(LOG).read().split("Compiling entry function")[1:]:
        yield sec.split("'")[1], sec


def _kernel_of(name):
    for k in sorted(KERNELS, key=len, reverse=True):   # mask_grow_cluster_kernel before mask_grow_kernel
        if re.search(r"\d+%s" % k, name):
            return k
    return None


def test_counted_kernels_compile_for_sm90a_without_spills():
    found = {}
    for name, sec in _sections():
        k = _kernel_of(name)
        if k is None:
            continue
        assert "for 'sm_90a'" in sec, name
        spill = int(re.search(r"(\d+) bytes spill stores", sec).group(1))
        assert spill == 0, "%s spills %d bytes" % (name, spill)
        found.setdefault(k, 0)
        found[k] += 1
        if k == "conv_tc_kernel":
            regs = int(re.search(r"Used (\d+) registers", sec).group(1))
            assert regs == 168, "%s: %d registers per thread at launch" % (name, regs)
    assert sorted(found) == sorted(KERNELS), sorted(set(KERNELS) - set(found))
