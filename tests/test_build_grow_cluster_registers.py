"""The cluster mask grower (csrc/elementwise.cu, images above 512 px a side): compiled for sm_90a without register spills, and one CTA's
shared memory fits the 227 KB of an H100 SM at the 2048x2048 limit.  Read from the -Xptxas -v log the build writes (no GPU needed)."""
import os
import re

import pytest

LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hand3d_b200", "build", "nvcc.log")


def _section():
    if not os.path.exists(LOG):
        pytest.skip("no build log: run python -m hand3d_b200.build first")
    for sec in open(LOG).read().split("Compiling entry function")[1:]:
        if "mask_grow_cluster_kernel" in sec.split("'")[1]:
            return sec
    raise AssertionError("mask_grow_cluster_kernel not in the build log")


def test_grow_cluster_kernel_compiles_for_sm90a_without_spills():
    sec = _section()
    assert "for 'sm_90a'" in sec
    assert int(re.search(r"(\d+) bytes spill stores", sec).group(1)) == 0
    assert int(re.search(r"(\d+) bytes spill loads", sec).group(1)) == 0
    assert int(re.search(r"Used (\d+) registers", sec).group(1)) <= 64   # 1024 threads per CTA


def test_grow_cluster_shared_memory_fits_at_2048():
    """Per CTA: det and obj [bp][Ww] and hor [10 + bp + 17][Ww] words (grow_smem_bytes), bp = the largest band rounded up to 8 rows.
    At 2048x2048 on 8 CTAs a band is 256 rows of 64 words: (3 * 256 + 27) * 64 * 4 = 203 520 bytes, plus the static words."""
    static = int(re.search(r"(\d+) bytes smem", _section()).group(1))
    H = W = 2048
    cs = max(1, min(8, H // 16))
    bp = (-(-H // cs) + 7) // 8 * 8
    ww = (W + 31) // 32
    dynamic = (3 * bp + 27) * ww * 4
    assert dynamic == 203520
    assert dynamic + static <= 227 * 1024
