"""Register allocation of the tensor-core convolution, read from the -Xptxas -v log the build writes (no GPU needed).

conv_tc_kernel moves registers from its producer warpgroup to the two wgmma warpgroups (setmaxnreg); without that, the BN = 128
instances spill their fp32 accumulator fragment to local memory inside the K loop."""
import os
import re

import pytest

LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hand3d_b200", "build", "nvcc.log")


def _conv_tc_entries():
    if not os.path.exists(LOG):
        pytest.skip("no build log: run python -m hand3d_b200.build first")
    out = {}
    for sec in open(LOG).read().split("Compiling entry function")[1:]:
        name = sec.split("'")[1]
        m = re.search(r"conv_tc_kernelILi(\d+)ELi(\d)ELb(\d)E", name)
        if m:
            out[m.groups()] = (int(re.search(r"(\d+) bytes spill stores", sec).group(1)), int(re.search(r"Used (\d+) registers", sec).group(1)))
    return out


def test_conv_tc_kernel_no_spills():
    entries = _conv_tc_entries()
    assert len(entries) == 9, sorted(entries)    # BN 64 / 128 x passes 1 / 3 x bf16 / fp16, + BN 64 fp16_f8c
    for inst, (spill, regs) in entries.items():
        assert spill == 0, "conv_tc_kernel<BN=%s, PASSES=%s, FP16=%s> spills %d bytes" % (*inst, spill)
        # setmaxnreg redistributes the registers allocated at launch: 384 threads x 168 = the producer's 40 + the consumers' 232
        assert regs == 168, "conv_tc_kernel<BN=%s, PASSES=%s, FP16=%s> allocated at %d registers" % (*inst, regs)
