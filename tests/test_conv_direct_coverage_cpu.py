"""Which paths the shape tables of tests/test_gpu_conv_direct_paths.py reach, asked from the launchers' own choosers
(h3d_conv2d_f32_geometry, h3d_fully_connected_f32_geometry: host only, no device needed).  If a predicate of launch_conv_direct or
launch_fc changes and a path drops out of a table, or an entry stops taking the path it is marked with, this fails without a GPU."""
import os
import re
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_conv_direct_paths as Tp  # noqa: E402
from hand3d_b200 import _lib, runtime  # noqa: E402

KC, TM, TN = 16, 64, 64          # conv_direct.cu: reduction chunk, output pixels and channels per CTA
FCB, FCN = 32, 64                # batch rows and outputs per FC CTA
PATHS = {"vec", "scalar", "vec+splitk", "scalar+splitk", "c3_ffma", "c3_tc"}


def _cd(a, b):
    return -(-a // b)


def _entry_facts(shape):
    B, H, W, Cin, Cout, k, s = shape[:7]
    M = B * _cd(H, s) * _cd(W, s)
    return M, _cd(M, TM) * _cd(Cout, TN), k * k * Cin


def test_queries_refuse_bad_arguments():
    lib = _lib.load()
    out = (_lib.C.c_int * 6)()
    S = _lib.CONV_SPLITK_SCRATCH_FLOATS
    ok = [1, 8, 8, 16, 16, 0, 8, 8, 0, 1, 0, 0, 0, 3, 1, 1, S]
    assert lib.h3d_conv2d_f32_geometry(*ok, out) == _lib.OK
    for i, bad in ((0, 0), (3, 0), (4, 15), (5, 1), (6, 0), (7, 7), (8, 1), (10, 6), (13, 0), (14, 0), (16, -1)):
        args = list(ok)
        args[i] = bad
        assert lib.h3d_conv2d_f32_geometry(*args, out) == _lib.EINVAL, (i, bad)
    args = list(ok)
    args[9] = 0                                   # neither fp32 output nor planes
    assert lib.h3d_conv2d_f32_geometry(*args, out) == _lib.EINVAL
    assert "no output" in _lib.last_error()
    args[10], args[11], args[12] = _lib.PRECISIONS["bf16"], 8, 1      # planes past Cs_total
    assert lib.h3d_conv2d_f32_geometry(*args, out) == _lib.EINVAL
    assert lib.h3d_conv2d_f32_geometry(*ok, None) == _lib.EINVAL
    assert lib.h3d_fully_connected_f32_geometry(0, 8, 8, out) == _lib.EINVAL
    assert lib.h3d_fully_connected_f32_geometry(1, 0, 8, out) == _lib.EINVAL
    assert lib.h3d_fully_connected_f32_geometry(1, 8, 8, None) == _lib.EINVAL


def test_header_constants_match_the_binding():
    txt = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "hand3d_b200.h")).read()
    m = re.search(r"#define H3D_CONV_SPLITK_SCRATCH_FLOATS \((\d+)LL \* (\d+) \* (\d+)\)", txt)
    assert m and int(m.group(1)) * int(m.group(2)) * int(m.group(3)) == _lib.CONV_SPLITK_SCRATCH_FLOATS
    kernels = dict((int(v), k) for k, v in re.findall(r"#define H3D_DIRECT_(\w+) (\d+)", txt))
    assert {i: k.lower() for i, k in kernels.items()} == _lib.DIRECT_KERNELS


def test_queries_on_known_layers():
    """The first layers, the c3_ffma switch, the lifting pyramid's stride-2 layers and the FC stacks of the lifting stage."""
    assert runtime.conv2d_f32_geometry(8, 240, 320, 3, 64, 3, yf=False, planes="bf16x3") == ("c3_tc", (0, 0, 0), 1, 27)
    assert runtime.conv2d_f32_geometry(8, 240, 320, 3, 64, 3) == ("c3_ffma", (600, 1, 1), 1, 27)
    assert runtime.conv2d_f32_geometry(8, 240, 320, 3, 64, 3, yf=False, planes="fp16_f8c")[0] == "c3_ffma"
    lib = _lib.load()
    try:
        assert lib.h3d_set_tuning(None, b"c3_ffma", 1) == _lib.OK
        assert runtime.conv2d_f32_geometry(8, 240, 320, 3, 64, 3, yf=False, planes="bf16x3")[0] == "c3_ffma"
    finally:
        assert lib.h3d_set_tuning(None, b"c3_ffma", 0) == _lib.OK
    # PosePrior conv_pose_0_1 (32 x 32 x 21 -> 32, stride 1) and conv_pose_1_1 (stride 2), B = 8
    assert runtime.conv2d_f32_geometry(8, 32, 32, 21, 32, 3) == ("scalar", (128, 1, 1), 1, 192)
    assert runtime.conv2d_f32_geometry(8, 32, 32, 32, 64, 3, 2) == ("vec", (32, 1, 3), 3, 96)
    assert runtime.conv2d_f32_geometry(8, 32, 32, 32, 64, 3, 2, splitk_scratch_floats=0) == ("vec", (32, 1, 1), 1, 288)
    assert runtime.conv2d_f32_geometry(8, 32, 32, 32, 64, 3, 2, yf=False, planes="bf16")[2] == 1   # planes never split K
    assert runtime.fully_connected_f32_geometry(8, 2050, 512) == (33, 64, (8, 33, 1))
    assert runtime.fully_connected_f32_geometry(8, 128, 3) == (2, 64, (1, 2, 1))


def test_every_entry_takes_its_marked_path():
    for s in Tp.ENTRY_SHAPES:
        assert Tp.path_of(Tp.entry_geometry(s)) == s[8], "%s runs %s" % (s, Tp.entry_geometry(s))
    for layer in Tp.LAYERS:
        assert Tp.path_of(Tp.layer_geometry(layer)) == layer[-1], "%s runs %s" % (layer, Tp.layer_geometry(layer))


def test_tables_reach_every_path():
    entry = {s[8] for s in Tp.ENTRY_SHAPES}
    layer = {layer[-1] for layer in Tp.LAYERS}
    assert entry | layer == PATHS
    assert entry >= PATHS - {"c3_tc"}, "the operator entry writes fp32 only, so it runs every path but c3_tc"
    assert layer >= {"c3_tc", "c3_ffma", "vec", "scalar"}


def test_grids_and_splits_are_consistent():
    for s in Tp.ENTRY_SHAPES:
        kernel, grid, ksplit, kps = Tp.entry_geometry(s)
        M, ctas, K = _entry_facts(s)
        if kernel.startswith("c3"):
            B, H, W = s[:3]
            assert grid == (_cd(_cd(W, 32) * _cd(H, 8) * B, 4), 1, 1) and (ksplit, kps) == (1, 27)
            continue
        assert grid[:2] == (_cd(M, TM), _cd(s[4], TN)) and grid[2] == ksplit
        assert kps % KC == 0 and (ksplit - 1) * kps < K <= ksplit * kps, "the slices tile K: %s" % (s,)


def test_split_k_boundaries():
    """Each side of ctas < 296 (with one and several channel tiles), of Ktot >= 256, of the entry's B Ho Wo <= 64 x 295, a split count
    lowered by the rounding of k_per_split, and the fallback when the partial sums do not fit the scratch."""
    facts = {s[:8]: (_entry_facts(s), Tp.entry_geometry(s)) for s in Tp.ENTRY_SHAPES}
    sides = set()
    for (M, ctas, K), (kernel, grid, ksplit, kps) in facts.values():
        if K >= 256 and ctas in (295, 296):
            sides.add(("ctas", ctas, grid[1] > 1, ksplit > 1))
        if ctas < 296 and K in (255, 256):
            sides.add(("K", K, ksplit > 1))
        if M in (64 * 295, 64 * 295 + 1):
            sides.add(("M", M, ksplit > 1))
    assert {("ctas", 295, False, True), ("ctas", 296, False, False), ("ctas", 295, True, True), ("ctas", 296, True, False)} <= sides
    assert {("K", 255, False), ("K", 256, True), ("M", 18880, True), ("M", 18881, False)} <= sides
    recomputed = [s for s, ((M, ctas, K), g) in facts.items() if g[2] > 1 and g[2] < min(_cd(K, 128), max(1, 592 // ctas))]
    assert recomputed, "no shape whose split count is lowered by the rounding of k_per_split"
    # fallback: the library's scratch holds every split its policy asks for (ksplit M Cout <= (592 / ctas) 64 ctas 64), so only a
    # smaller scratch reaches it; the GPU cannot, and the query shows the policy falling back to one pass
    assert 592 * TM * TN <= _lib.CONV_SPLITK_SCRATCH_FLOATS
    for s in [s for s in Tp.ENTRY_SHAPES if s[8].endswith("+splitk")]:
        B, H, W, Cin, Cout, k, st, al = s[:8]
        (M, ctas, K), (_, _, ksplit, _) = _entry_facts(s), Tp.entry_geometry(s)
        need = min(_cd(K, 128), max(1, 592 // ctas)) * M * Cout          # the split the policy asks for, before the rounding
        small = runtime.conv2d_f32_geometry(B, H, W, Cin, Cout, k, st, x_aligned=al, splitk_scratch_floats=need - 1)
        assert small[2] == 1 and small[1][2] == 1 and small[3] == _cd(k * k * Cin, KC) * KC, (s, small)
        assert runtime.conv2d_f32_geometry(B, H, W, Cin, Cout, k, st, x_aligned=al, splitk_scratch_floats=need)[2] == ksplit


def test_vec_scalar_boundary():
    """Cin % 16, Cin_total % 4, an unaligned x: each alone moves an otherwise float4 layer to the scalar gather."""
    entries = {(s[3], s[7]): s[8].split("+")[0] for s in Tp.ENTRY_SHAPES}
    assert entries[(16, True)] == "vec" and entries[(16, False)] == "scalar" and entries[(21, True)] == "scalar"
    assert any(layer[3] == layer[4] + 1 and layer[4] % 16 == 0 and layer[-1] == "scalar" for layer in Tp.LAYERS)
    assert any(layer[3] > layer[4] and layer[-1] == "vec" for layer in Tp.LAYERS)
    for shape in [s for s in Tp.ENTRY_SHAPES if s[3] % 16 == 0 and s[7]]:
        vec, scalar = Tp.entry_geometry(shape), Tp.entry_geometry(shape[:7] + (False,))
        assert vec[0] == "vec" and scalar[0] == "scalar" and vec[1:] == scalar[1:]


def test_tables_cover_kernel_sizes_strides_and_channels():
    rows = Tp.ENTRY_SHAPES
    assert {(s[5], s[6]) for s in rows} >= {(1, 1), (1, 2), (3, 1), (3, 2), (3, 3), (5, 1), (5, 2), (5, 3), (7, 1), (7, 2), (7, 3)}
    assert any(s[1] % 2 == 0 for s in rows) and any(s[1] % 2 for s in rows) and any(s[2] % 2 == 0 for s in rows) and any(s[2] % 2 for s in rows)
    couts = {s[4] for s in rows} | {layer[5] for layer in Tp.LAYERS}
    assert couts >= {1, 2, 3, 5, 21, 63, 64, 65, 129, 256}
    assert {c & 3 for c in couts} == {0, 1, 2, 3}, "every Cout & 3 tail of the weight loads and the epilogue"
    assert {s[3] for s in rows} >= {3, 16, 21, 32, 149}
    assert any(layer[3] > layer[4] for layer in Tp.LAYERS)
    # TF SAME puts the odd padding pixel at the bottom / right: some shape pads its top and left differently
    pads = set()
    for B, H, W, Cin, Cout, k, s in [r[:7] for r in rows]:
        pt = max((_cd(H, s) - 1) * s + k - H, 0) // 2
        pl = max((_cd(W, s) - 1) * s + k - W, 0) // 2
        pads.add(pt != pl)
    assert True in pads


def test_first_layer_tiles():
    """conv3x3_c3_kernel: H % 8 and W % 32 ragged, a last CTA of fewer than 4 tiles, a CTA whose tiles lie in two images (B up to
    9), the fp32 output at an aligned offset of a wider tensor, and shapes one step outside is_c3_case that run the generic kernel."""
    c3 = [s for s in Tp.ENTRY_SHAPES if s[8] == "c3_ffma"] + [(layer[0], layer[1], layer[2]) for layer in Tp.LAYERS
                                                               if layer[-1].startswith("c3")]
    assert any(H % 8 and W % 32 for B, H, W in [s[:3] for s in c3])
    per_img = [(B, _cd(W, 32) * _cd(H, 8)) for B, H, W in [s[:3] for s in c3]]
    assert any((B * t) % 4 for B, t in per_img), "no last CTA with fewer than 4 tiles"
    assert any(B > 1 and t % 4 for B, t in per_img) and max(B for B, _ in per_img) == 9, "no CTA straddling two images"
    assert any(layer[-1] == "c3_ffma" and layer[10] and layer[10] > 64 and layer[11] % 4 == 0 and layer[11] for layer in Tp.LAYERS)
    outside = [s for s in Tp.ENTRY_SHAPES if s[3] == 3 and s[5] == 3 and not s[8].startswith("c3")]
    assert {s[6] for s in outside} >= {2} and {s[4] for s in outside} >= {63, 65}
    layers_out = [layer for layer in Tp.LAYERS if layer[4] == 3 and layer[5] == 64 and not layer[-1].startswith("c3")]
    assert any(layer[3] == 4 for layer in layers_out)
    assert any(layer[10] and layer[11] % 4 for layer in layers_out)
    assert any(layer[7] and layer[9] % 8 for layer in layers_out)


def test_plane_epilogues():
    """conv_direct_kernel's plane epilogue in every format at a plane offset != 0, with and without the fp32 output."""
    generic = [layer for layer in Tp.LAYERS if layer[-1] in ("vec", "scalar") and layer[7]]
    assert {layer[7] for layer in generic if layer[9]} == {"bf16x3", "fp16x3", "bf16", "fp16", "fp16_f8c"}
    assert any(layer[10] for layer in generic) and any(not layer[10] for layer in generic)
    assert {layer[7] for layer in Tp.LAYERS if layer[-1] == "c3_ffma"} >= {"fp16x3", "fp16_f8c", "bf16"}
    for layer in [layer for layer in Tp.LAYERS if layer[7] and not layer[10] and layer[-1] != "c3_tc"]:
        assert Tp.layer_geometry(layer, Tp._identity_yf(layer))[0] == layer[-1], "the added fp32 output keeps %s on its kernel" % (layer,)


def test_fc_table_reaches_every_split_regime():
    B_ = {s[0] for s in Tp.FC_SHAPES}
    assert B_ >= {1, 31, 32, 33, 64, 65, 160, 300}
    assert {s[1] for s in Tp.FC_SHAPES} >= {1, 30, 33, 512, 2050, 4098}
    assert {s[2] for s in Tp.FC_SHAPES} >= {1, 3, 63, 64, 65, 512}
    regimes = set()
    for B, n_in, n_out in Tp.FC_SHAPES:
        ksplit, kps, grid = runtime.fully_connected_f32_geometry(B, n_in, n_out)
        assert grid == (_cd(n_out, FCN), ksplit, _cd(B, FCB)) and kps % 32 == 0 and (ksplit - 1) * kps < n_in + ksplit * kps
        ctas = grid[0] * grid[2]
        if ksplit == 1:
            regimes.add("one")
        elif ksplit == _cd(n_in, 64) and ksplit <= 296 // ctas:
            regimes.add("by in_features")
        else:
            assert ksplit == 296 // ctas
            regimes.add("by tiles")
        if ksplit > 1 and (ksplit - 1) * kps >= n_in:
            regimes.add("empty last slices")
        if grid[2] > 1:
            regimes.add("several batch tiles")
        if B % FCB:
            regimes.add("ragged batch tile")
    assert regimes == {"one", "by in_features", "by tiles", "empty last slices", "several batch tiles", "ragged batch tile"}


@pytest.mark.parametrize("table", ["ENTRY_SHAPES", "LAYERS", "FC_SHAPES"])
def test_tables_hold_no_duplicates_and_stay_small(table):
    rows = getattr(Tp, table)
    assert len(set(rows)) == len(rows)
    for r in rows:
        if table == "FC_SHAPES":
            macs = r[0] * r[1] * r[2]
        elif table == "ENTRY_SHAPES":
            M, _, K = _entry_facts(r)
            macs = M * K * r[4]
        else:
            macs = r[0] * r[1] * r[2] * r[6] * r[6] * r[4] * r[5]
        assert macs < 1e9, "keep the fp64 reference of %s quick" % (r,)
