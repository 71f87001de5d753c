"""Register allocation of every pixel-format instance of the frame kernels (csrc/frames.cu: resize_frames_kernel<F> and
convert_frames_kernel<F>, F = H3D_PIXEL_RGB .. H3D_PIXEL_YUYV), read from the -Xptxas -v log the build writes (no GPU needed): sm_90a,
no spills, and at most 64 registers, so that two 512-thread resize CTAs fit on an SM."""
import os
import re

import pytest

LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hand3d_b200", "build", "nvcc.log")
KERNELS = ["%s_frames_kernelILi%dE" % (k, f) for k in ("resize", "convert") for f in range(5)]


def test_frame_format_kernels_compile_for_sm90a_within_64_registers_without_spills():
    if not os.path.exists(LOG):
        pytest.skip("no build log: run python -m hand3d_b200.build first")
    found = {}
    for sec in open(LOG).read().split("Compiling entry function")[1:]:
        name = sec.split("'")[1]
        for k in KERNELS:
            if k in name and "frames_cu" in name:
                assert "for 'sm_90a'" in sec, name
                found[k] = (int(re.search(r"(\d+) bytes spill stores", sec).group(1)), int(re.search(r"Used (\d+) registers", sec).group(1)))
    assert sorted(found) == sorted(KERNELS), sorted(set(KERNELS) - set(found))
    for k, (spill, regs) in found.items():
        assert spill == 0, "%s spills %d bytes" % (k, spill)
        assert regs <= 64, "%s uses %d registers" % (k, regs)
