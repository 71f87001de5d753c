"""Register allocation of the wgmma weight-gradient kernel, read from the -Xptxas -v log the build writes (no GPU needed)."""
import os
import re

import pytest

LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hand3d_b200", "build", "nvcc.log")


def test_conv_wgrad_tc_kernel_no_spills():
    if not os.path.exists(LOG):
        pytest.skip("no build log: run python -m hand3d_b200.build first")
    entries = {}
    for sec in open(LOG).read().split("Compiling entry function")[1:]:
        name = sec.split("'")[1]
        m = re.search(r"conv_wgrad_tc_kernelILi(\d+)ELi(\d)E", name)
        if m:
            entries[m.groups()] = (int(re.search(r"(\d+) bytes spill stores", sec).group(1)), int(re.search(r"Used (\d+) registers", sec).group(1)))
    assert sorted(entries) == [("128", "1"), ("128", "3"), ("64", "1"), ("64", "3")], sorted(entries)   # BN 64 / 128 x passes 1 / 3
    for inst, (spill, regs) in entries.items():
        assert spill == 0, "conv_wgrad_tc_kernel<BN=%s, PASSES=%s> spills %d bytes" % (*inst, spill)
        # setmaxnreg moves registers between warpgroups of the 384 x 168 allocated at launch (producer 40, consumers 232)
        assert regs == 168, "conv_wgrad_tc_kernel<BN=%s, PASSES=%s> allocated at %d registers" % (*inst, regs)
