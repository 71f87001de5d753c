"""Which kernels of csrc/train.cu and csrc/train_lift.cu the tables of tests/test_gpu_train_paths.py reach, and what their rows hold,
checked without a GPU.  Every __global__ of the two files must be the marked kernel of some table row or be excluded here with the
reason and the test that covers it; every row must take the path it is marked with under the launchers' policies (restated in
tests/train_order_oracle.py and checked on the device by that module's test_dispatch); the tables must reach every instance, pass,
chunking, block count, alignment and batch edge the module promises."""
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_gpu_train_paths as Tp  # noqa: E402
import train_order_oracle as R  # noqa: E402

SOURCES = [os.path.join(os.path.dirname(HERE), "hand3d_b200", "csrc", f) for f in ("train.cu", "train_lift.cu")]

# kernel: (why no row of the tables reaches it, the test that covers it)
EXCLUDED = {
    "bone_rel_trafo_kernel": ("the 'local' target, a forward analysis without a gradient, pinned to the reference's own graph",
                              "test_gpu_lifting_training.py::test_bone_rel_trafo_vs_oracle_and_reference_graph"),
    "adam_state_set_kernel": ("writes the Adam state words; every Adam row calls it through adam_state_set and adam_set_lr",
                              "test_gpu_training.py::test_adam_bit_identical_to_tf_restatement_100_steps"),
}


def global_kernels():
    names = set()
    for path in SOURCES:
        src = open(path).read()
        found = re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", src)
        assert len(found) == src.count("__global__"), "a __global__ of %s the parser does not read" % path
        names |= set(found)
    return names


def _base(name):
    return name.split("<")[0]


def test_every_kernel_is_reached_or_excluded():
    kernels = global_kernels()
    reached = {_base(k) for k in Tp.expected_kernels() if k != "copy"}
    assert reached <= kernels, "table rows marked with kernels the sources do not have: %s" % sorted(reached - kernels)
    assert not reached & set(EXCLUDED), "reached and excluded: %s" % sorted(reached & set(EXCLUDED))
    missing = kernels - reached - set(EXCLUDED)
    assert not missing, "kernels neither reached by a table row nor excluded: %s" % sorted(missing)
    assert set(EXCLUDED) <= kernels, "exclusions of kernels that no longer exist: %s" % sorted(set(EXCLUDED) - kernels)


def test_exclusions_name_existing_tests():
    for kernel, (reason, test) in EXCLUDED.items():
        path, name = test.split("::")
        src = open(os.path.join(HERE, path)).read()
        assert re.search(r"^def %s\(" % name, src, re.M), "%s: %s has no %s" % (kernel, path, name)
        assert reason


def test_rows_take_their_marked_path():
    for B, H, W, C, oh, ow, path in Tp.RESIZE_GRAD:
        assert Tp.resize_grad_path(H, W, C, oh, ow) == path, (B, H, W, C, oh, ow)
    for B, H, W, path in Tp.SCOREMAP:
        assert Tp.scoremap_path(B, H, W) == path, (B, H, W)
    for n, path in Tp.XENT + Tp.MSE:
        assert Tp.reduction_path(n) == path, n


def test_resize_rows_reach_every_case():
    rows = [r for r in Tp.RESIZE_GRAD if r[-1] != "copy"]
    assert {r[3] for r in Tp.RESIZE_GRAD} >= {21, 2, 1, 3, 64}
    for inst in ("cols<21>", "cols<2>", "cols<0>"):
        paths = {r[-1] for r in rows if inst in r[-1]}
        assert {inst, inst + "+rows"} <= paths, "%s: W alone and both dimensions" % inst
    assert any(r[-1] == "rows" for r in rows), "H alone"
    assert {r[3] for r in Tp.RESIZE_GRAD if r[-1] == "copy"} >= {21, 2, 1, 64}, "the copy"
    up = [r for r in rows if r[4] >= r[1] and r[5] >= r[2]]
    down = [r for r in rows if r[4] <= r[1] and r[5] <= r[2]]
    assert up and down
    assert any((r[4] % r[1] and r[1] % r[4]) or (r[5] % r[2] and r[2] % r[5]) for r in rows), "a non-integer ratio"
    assert any(r[1] == r[2] == 1 for r in rows) and any(r[4] == r[5] == 1 for r in rows), "1-pixel inputs and outputs"
    assert any(max(r[1], r[2]) >= 1000 and r[4] * r[5] <= 9 for r in rows), "a 1000 -> 3 downscale"
    loops = set()
    for B, H, W, C, oh, ow, _ in rows:
        loops |= Tp.resize_grad_loops(B, H, W, C, oh, ow)
    assert loops == {"cols", "rows"}, "the grid-stride loop of both passes: %s" % loops


def test_scoremap_rows_reach_every_case():
    tags = {t for r in Tp.SCOREMAP for t in r[-1].split(", ")}
    assert {"1 chunk (HW <= 256)", "1 chunk (B >= 264)", "33 chunks", "short last", "idle groups", "laps"} <= tags
    assert {r[0] for r in Tp.SCOREMAP} >= {1, 8, 13, 265, 65536, 70001}
    assert {r[1] * r[2] for r in Tp.SCOREMAP} >= {1, 6, 100, 256, 257, 65536}
    assert any(r[0] > 65535 for r in Tp.SCOREMAP), "more images than a grid has rows"
    assert set(Tp.SCOREMAP_KINDS) == {"binary", "fractional", "canary"}


def test_reduction_rows_reach_every_case():
    xr = [n for n, _ in Tp.XENT]
    assert xr == [1, 255, 2048, 2049, 524288, 2097152, 2097153, 3000001]
    assert [R.reduction_blocks(n) for n in xr[-3:]] == [(1024, 2048), (1024, 2049), (1024, 2930)]
    assert [n for n, _ in Tp.MSE] == [1, 255, 504, 2048, 2049, 2 ** 21, 2 ** 21 + 1, 3000007]
    for table in (Tp.XENT, Tp.MSE):
        paths = [p for _, p in table]
        assert any(p.startswith("1 x ") for p in paths) and any(p.startswith("2 x ") for p in paths)
        assert any("laps" in p for p in paths) and any(R.reduction_blocks(n)[1] > 2048 for n, _ in table)
    assert set(Tp.XENT_LABELS) == {"one_hot", "soft", "unnormalised"}


def test_adam_tables_reach_every_case():
    tables = dict(Tp.ADAM)
    per = R.adam_chunks_per_block([n for n, _ in tables["several chunks per block"]])
    assert per.max() >= 2 and R.adam_chunk_prefix([n for n, _ in tables["several chunks per block"]])[-1] > R.ADAM_BLOCKS
    sizes = {n for _, rows in Tp.ADAM for n, _ in rows}
    assert {0, 1, 3, 4, 8191, 8192, 8193, 16387} <= sizes
    assert len(tables["1024 tensors"]) == R.ADAM_MAX_TENSORS
    mis = [off for n, off in tables["one misaligned array"]]
    assert {(a, o) for off in mis for a, o in enumerate(off) if o} == {(a, o) for a in range(4) for o in (1, 2, 3)}
    assert all(sum(1 for o in off if o) <= 1 for off in mis) and (0, 0, 0, 0) in mis, "one array misaligned at a time, aligned beside"
    assert tables["one element"] == [(1, (0, 0, 0, 0))]
    assert R.adam_chunks_per_block([1]).sum() == 1, "527 blocks idle"
    assert {off for _, off in Tp.ADAM_OPTIM} == {0, 1, 2, 3}


def test_adjoint_batches_cross_the_blocks():
    blocks = {R.cdiv(B * 6, 128) for B in Tp.BONE_B}
    assert {1, 2, 3} <= blocks and any(B * 6 % 128 for B in Tp.BONE_B if R.cdiv(B * 6, 128) == 1)
    assert 21 * 6 < 128 < 22 * 6
    assert max(Tp.ROTATE_B) > 65535
    ties = [hs for hs in Tp.TIES if hs[0] == hs[1]]
    assert len(ties) >= 3 and {float(hs[0]) for hs in ties} >= {0.0, 1.0}


def test_tables_hold_no_duplicates():
    for name in ("RESIZE_GRAD", "SCOREMAP", "XENT", "MSE", "ADAM_OPTIM", "BONE_B", "ROTATE_B"):
        rows = getattr(Tp, name)
        assert len(set(rows)) == len(rows), name
    keys = [(name, tuple(rows)) for name, rows in Tp.ADAM]
    assert len({k for k, _ in keys}) == len(keys) and len({r for _, r in keys}) == len(keys)
