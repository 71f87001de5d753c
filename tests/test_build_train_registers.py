"""Register allocation of the training kernels (csrc/train.cu), read from the -Xptxas -v log the build writes (no GPU needed)."""
import os
import re

import pytest

LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hand3d_b200", "build", "nvcc.log")
KERNELS = ["resize_grad_cols_kernelILi0E", "resize_grad_cols_kernelILi2E", "resize_grad_cols_kernelILi21E", "resize_grad_rows_kernel",
           "scoremap_sq_partial_kernel", "scoremap_loss_finalize_kernel", "scoremap_loss_grad_kernel", "xent_partial_kernel",
           "xent_finalize_kernel", "xent_grad_kernel", "adam_step_kernel", "adam_state_set_kernel"]


def test_train_kernels_no_spills():
    if not os.path.exists(LOG):
        pytest.skip("no build log: run python -m hand3d_b200.build first")
    found = {}
    for sec in open(LOG).read().split("Compiling entry function")[1:]:
        name = sec.split("'")[1]
        for k in KERNELS:
            if k in name and "train_cu" in name:
                found[k] = int(re.search(r"(\d+) bytes spill stores", sec).group(1))
    assert sorted(found) == sorted(KERNELS), sorted(set(KERNELS) - set(found))
    for k, spill in found.items():
        assert spill == 0, "%s spills %d bytes" % (k, spill)
