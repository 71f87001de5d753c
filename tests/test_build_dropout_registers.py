"""Register allocation of the dropout kernels (csrc/dropout.cu), read from the -Xptxas -v log the build writes (no GPU needed)."""
import os
import re

import pytest

LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hand3d_b200", "build", "nvcc.log")
KERNELS = ["dropout_kernelILi0E", "dropout_kernelILi1E", "dropout_kernelILi2E", "dropout_backward_kernel", "dropout_advance_kernel"]


def test_dropout_kernels_compile_for_sm90a_without_spills():
    if not os.path.exists(LOG):
        pytest.skip("no build log: run python -m hand3d_b200.build first")
    found = {}
    for sec in open(LOG).read().split("Compiling entry function")[1:]:
        name = sec.split("'")[1]
        for k in KERNELS:
            if k in name and "dropout_cu" in name:
                assert "for 'sm_90a'" in sec, name
                found[k] = int(re.search(r"(\d+) bytes spill stores", sec).group(1))
    assert sorted(found) == sorted(KERNELS), sorted(set(KERNELS) - set(found))
    for k, spill in found.items():
        assert spill == 0, "%s spills %d bytes" % (k, spill)
