"""Golden learning rates produced by the UNMODIFIED reference LearningRateScheduler (utils/general.py:480-519 of a checkout of
lmb-freiburg/hand3d named by $H3D_REFERENCE, read-only) run over the eager `tensorflow` stand-in oracle/tf1_eager.py, at the boundary
steps of 1-, 2- and 3-value schedules (the two training scripts' schedules among them).  tests/test_training_oracle.py pins
hand3d_b200.utils.general.LearningRateScheduler against golden_reference_lr.npz.

    python tests/golden/make_golden_reference_lr.py        # H3D_REFERENCE=<checkout of lmb-freiburg/hand3d>
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "golden_reference_lr.npz")

# (steps, values): a constant, a single switch, the two training scripts' schedules and an uneven 4-value one
SCHEDULES = [
    ([], [1e-3]),
    ([100], [1e-4, 1e-5]),
    ([10000, 20000], [1e-4, 1e-5, 1e-6]),       # training_posenet.py:29-30
    ([20000, 30000], [1e-5, 1e-6, 1e-7]),       # training_handsegnet.py:29-30
    ([5, 7, 40], [0.5, 0.25, 3e-3, 1e-9]),
]


def query_steps(steps):
    q = {0, 1, 50000}
    for s in steps:
        q.update({s - 1, s, s + 1})
    return sorted(v for v in q if v >= 0)


def main():
    sys.path.insert(0, os.path.dirname(HERE))
    from golden.make_golden_reference_graph import setup_imports
    tfe, _, _, ref_general, _ = setup_imports()
    out = {}
    for i, (steps, values) in enumerate(SCHEDULES):
        sched = ref_general.LearningRateScheduler(steps=steps, values=values)
        q = query_steps(steps)
        out["s%d_steps" % i] = np.array(steps, np.int64)
        out["s%d_values" % i] = np.array(values, np.float64)
        out["s%d_query" % i] = np.array(q, np.int64)
        out["s%d_lr" % i] = np.array([np.asarray(sched.get_lr(np.int64(t))) for t in q], np.float32)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", len(SCHEDULES), "schedules")


if __name__ == "__main__":
    main()
