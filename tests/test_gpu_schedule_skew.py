"""The tensor-core rings, cluster handshakes, dependent launches and tickets under injected delays (csrc/skew.cuh).

These kernels are deterministic by design (no float atomics, fixed reduction orders), so no schedule may change a bit of their
output.  A child process builds and loads the schedule-skew library (schedule_skew_cases.main) and runs every case of
schedule_skew_cases.CASES under every delay pattern of PATTERNS: producer slow, either consumer warpgroup slow, the window between wgmma
commit and wait widened, one warpgroup's epilogue slow, cluster rank 0 or the last rank slow, the primary's tail slow after it let its
PDL dependents launch, and three seeded random mixes.  This process runs the same cases on the product library.  Checks:
  * every pattern's output equals the product library's, bit for bit (pattern "none": the hooks compiled in but idle change nothing);
  * the product output holds against the suite's existing reference at the existing bound, so every skewed output does too."""
import os
import subprocess
import sys

import numpy as np
import pytest

import schedule_skew_cases as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def product():
    from hand3d_b200 import runtime
    ctx = runtime.Context()
    out = S.run_cases(ctx)
    return {c: d for (_, c), d in out.items()}


@pytest.fixture(scope="module")
def skewed(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("skew") / "skew.npz")
    r = subprocess.run([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)), "schedule_skew_cases.py"), path],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, "skew child failed:\n" + r.stdout[-6000:]
    print(r.stdout.strip().splitlines()[-1])
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


def _first_diff(a, b):
    bad = a.view(np.uint8).reshape(-1) != b.view(np.uint8).reshape(-1)
    return int(bad.sum()), np.unravel_index(int(np.argmax(bad)) // a.itemsize, a.shape)


@pytest.mark.parametrize("pattern", list(S.PATTERNS))
@pytest.mark.parametrize("case", list(S.CASES))
def test_skewed_output_equals_product(product, skewed, case, pattern):
    want = product[case]
    for name, a in want.items():
        key = "%s/%s/%s" % (pattern, case, name)
        assert key in skewed, key
        a, b = np.atleast_1d(a), np.atleast_1d(skewed[key])
        assert a.shape == b.shape and a.dtype == b.dtype, (name, a.shape, b.shape, a.dtype, b.dtype)
        if not np.array_equal(a.view(np.uint8), b.view(np.uint8)):
            n, at = _first_diff(a, b)
            raise AssertionError("%s under %s: %d bytes differ from the product library, first at %s: %r vs %r"
                                 % (name, pattern, n, at, a[at], b[at]))


@pytest.mark.parametrize("case", [c for c, (_, check) in S.CASES.items() if check is not None])
def test_product_output_vs_reference(product, case):
    S.CASES[case][1](product[case])
