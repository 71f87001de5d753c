"""Which tiles the shape tables of tests/test_gpu_conv_tiles.py reach, asked from the library's own choosers (h3d_conv2d_tc_geometry,
h3d_conv2d_wgrad_geometry: host only, no device needed).  If a chooser changes and a candidate drops out of a table, or a shape stops
being ragged where it claims to be, this fails without a GPU.  The same holds for the training geometries of
tests/test_gpu_conv_backward.py (TRAIN_CASES)."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_conv_backward as Tb  # noqa: E402
import test_gpu_conv_tiles as Tt  # noqa: E402
from test_gpu_conv_layer_planes import POOL_LEGAL, TILE_SHAPES  # noqa: E402
from hand3d_b200 import _lib, arch, runtime  # noqa: E402

# the candidate lists of choose_tile (conv_wgmma.cu) and wgrad_geometry (conv_wgrad.cu), TW x TH x TB
FWD_TILES = [(16, 8, 1), (8, 16, 1), (32, 4, 1), (4, 32, 1), (64, 2, 1), (128, 1, 1), (8, 8, 2), (16, 4, 2), (4, 16, 2), (8, 4, 4),
             (4, 8, 4), (4, 4, 8), (8, 2, 8), (2, 2, 32), (1, 1, 128)]
WGRAD_TILES = [(8, 8, 1), (16, 4, 1), (4, 16, 1), (32, 2, 1), (2, 32, 1), (64, 1, 1), (1, 64, 1), (8, 4, 2), (4, 8, 2), (4, 4, 4),
               (4, 2, 8), (2, 4, 8), (2, 2, 16), (1, 1, 64)]


def _cd(a, b):
    return -(-a // b)


def fwd_geometry(shape, prec="bf16x3"):
    B, H, W, Cin, Cout, k, s = shape[:7]
    g = runtime.conv2d_tc_geometry(B, H, W, Cout, 2 if s == 2 else 0, prec)
    return g[:3], g[3]


def wgrad_geometry(shape):
    B, H, W, Cin, Cout, k, s = shape[:7]
    g = runtime.conv2d_wgrad_geometry(B, H, W, k, Cin, Cout)
    return g[:3], g[3], g[4], g[5]


def _ragged(shape, tile):
    B, H, W = shape[:3]
    return [W % tile[0] != 0, H % tile[1] != 0, B % tile[2] != 0]


def _check_raggedness(shapes, geometry):
    plus_one = set()
    for s in shapes:
        tile = geometry(s)[0]
        assert tile[0] * tile[1] * tile[2] in (64, 128)
        if s[7]:
            assert not any(_ragged(s, tile)), "%s is marked as an exact fit of %s" % (s, tile)
        else:
            assert any(_ragged(s, tile)), "%s fits %s exactly and is not marked so" % (s, tile)
        if tile[2] > 1 and s[0] == tile[2] + 1:
            plus_one.add(tile)
    return plus_one


def test_queries_refuse_bad_arguments():
    lib = _lib.load()
    out = (_lib.C.c_int * 6)()
    assert lib.h3d_conv2d_tc_geometry(0, 8, 8, 64, 0, _lib.PRECISIONS["bf16x3"], out) == _lib.EINVAL
    assert lib.h3d_conv2d_tc_geometry(1, 8, 8, 64, 3, _lib.PRECISIONS["bf16x3"], out) == _lib.EINVAL
    assert lib.h3d_conv2d_tc_geometry(1, 8, 8, 64, 0, _lib.PRECISIONS["fp32_ffma"], out) == _lib.EINVAL
    assert lib.h3d_conv2d_tc_geometry(1, 8, 8, 64, 0, _lib.PRECISIONS["bf16x3"], None) == _lib.EINVAL
    assert lib.h3d_conv2d_wgrad_geometry(1, 8, 8, 4, 64, 64, out) == _lib.EINVAL
    assert lib.h3d_conv2d_wgrad_geometry(1, 8, 8, 3, 0, 64, out) == _lib.EINVAL
    assert "ksize" in _lib.last_error() or "bad argument" in _lib.last_error()


def test_queries_on_known_layers():
    """Shapes whose geometry DESIGN states: 30x40 HandSegNet maps at B = 8, the lifting pyramids' 4x4 maps, FC-as-1x1 rows."""
    assert runtime.conv2d_tc_geometry(8, 30, 40, 128) == (8, 2, 8, 128)
    assert runtime.conv2d_tc_geometry(8, 4, 4, 256) == (4, 4, 8, 64)            # H W <= 256: N = 64
    assert runtime.conv2d_tc_geometry(128, 1, 1, 512) == (1, 1, 128, 64)
    assert runtime.conv2d_tc_geometry(1, 64, 64, 512, 0, "fp16_f8c")[3] == 64   # the fp8-corrected instance has N = 64 only
    assert runtime.conv2d_tc_geometry(1, 64, 64, 72)[3] == 128                  # align_up(Cout, 64) is what counts
    assert runtime.conv2d_tc_geometry(1, 64, 64, 136)[3] == 64
    assert runtime.conv2d_tc_geometry(1, 2, 256, 64, 1)[:3] == (16, 8, 1)       # fused pool: no 64x2 tile
    assert runtime.conv2d_wgrad_geometry(8, 128, 128, 3, 64, 64) == (8, 8, 1, 64, 9, 44)
    assert runtime.conv2d_wgrad_geometry(1, 16, 8, 7, 128, 64)[3:5] == (128, 49)


def test_forward_table_reaches_every_tile_with_both_n_tiles():
    """All 15 x 2 (tile, N tile) pairs are reachable from the geometry alone (N = 128 needs a map of more than 256 pixels, which the
    multi-image tiles get from a batch of thin maps), so none needs the tc_bn switch."""
    reached = {}
    for s in Tt.FWD_SHAPES:
        reached.setdefault(fwd_geometry(s), []).append(s)
    missing = [(t, bn) for t in FWD_TILES for bn in (64, 128) if (t, bn) not in reached]
    assert not missing, "no forward shape runs on %s" % missing
    assert {t for t, _ in reached} == set(FWD_TILES)
    for prec in ("fp16x3", "bf16", "fp16"):
        assert all(fwd_geometry(s, prec) in reached for s in Tt.FWD_SHAPES)


def test_forward_table_raggedness_and_batch_boxes():
    plus_one = _check_raggedness(Tt.FWD_SHAPES, fwd_geometry)
    assert plus_one == {t for t in FWD_TILES if t[2] > 1}, "every multi-image tile needs a shape with B = TB + 1"


def test_forward_table_kernel_sizes_and_strides():
    for stride, sizes in ((1, (1, 3, 5, 7)), (2, (3, 5, 7))):
        rows = [s for s in Tt.FWD_SHAPES if s[6] == stride]
        assert {_cd(s[3], 64) for s in rows} >= {1, 2, 3}
        for k in sizes:
            with_k = [s for s in rows if s[5] == k]
            assert len({fwd_geometry(s)[0] for s in with_k}) >= 2, "ksize %d at stride %d runs on fewer than two tiles" % (k, stride)
            assert all(s[1] % stride == 0 and s[2] % stride == 0 for s in with_k)


def test_single_pass_shapes_cover_the_kernel_instances():
    inst = {(fwd_geometry(s, p)[1], p) for s, p in Tt.SINGLE_PASS}
    assert inst == {(64, "bf16"), (128, "bf16"), (64, "fp16"), (128, "fp16"), (64, "fp16_f8c")}
    assert any(Cout % 128 == 0 and H * W > 256 for (_, H, W, _, Cout, _, _), p in Tt.SINGLE_PASS if p == "fp16_f8c")


def test_fold_tables_sit_on_the_fold_boundaries():
    assert {c[3] // 64 for c in Tt.FOLD_3PASS} == {8, 9, 10, 18, 19}
    assert {c[3] // 64 for c in Tt.FOLD_1PASS} == {26, 27, 28}
    for table in (Tt.FOLD_3PASS, Tt.FOLD_1PASS):
        assert {runtime.conv2d_tc_geometry(B, H, W, Cout)[3] for B, H, W, _, Cout in table} == {64, 128}


def test_forced_n_tile_is_what_the_query_reports():
    lib = _lib.load()
    default = [fwd_geometry(s)[1] for s in Tt.BN_SHAPES]
    assert sorted(default) == [64, 128]
    try:
        for bn in (64, 128):
            assert lib.h3d_set_tuning(None, b"tc_bn", bn) == _lib.OK
            assert [fwd_geometry(s)[1] for s in Tt.BN_SHAPES] == [bn, bn]
            assert [fwd_geometry(s)[0] for s in Tt.BN_SHAPES] == [fwd_geometry(s)[0] for s in Tt.BN_SHAPES]
            assert runtime.conv2d_tc_geometry(1, 25, 21, 64)[3] == 64            # Cout_pad = 64 cannot take N = 128
            assert runtime.conv2d_tc_geometry(1, 25, 21, 128, 0, "fp16_f8c")[3] == 64
    finally:
        assert lib.h3d_set_tuning(None, b"tc_bn", 0) == _lib.OK
    assert [fwd_geometry(s)[1] for s in Tt.BN_SHAPES] == default


def test_pooled_table_reaches_every_pool_legal_tile():
    assert len(POOL_LEGAL) == 11 and set(POOL_LEGAL) < set(FWD_TILES)
    for tile, (B, H, W) in TILE_SHAPES.items():
        assert runtime.conv2d_tc_geometry(B, H, W, 64, 1)[:3] == tile, (tile, (B, H, W))
    assert set(TILE_SHAPES) == set(POOL_LEGAL)


def test_backward_table_reaches_every_wgrad_tile_and_split():
    reached, bns, splits = set(), set(), set()
    for s in Tt.BWD_SHAPES:
        tile, bn, num_tiles, sp = wgrad_geometry(s)
        B, H, W, Cin, Cout, k = s[:6]
        blocks = _cd(W, tile[0]) * _cd(H, tile[1]) * _cd(B, tile[2])
        assert bn == (128 if _cd(Cin, 64) % 2 == 0 else 64)
        assert num_tiles == k * k * _cd(Cout, 64) * (_cd(Cin, 64) * 64 // bn)
        assert 1 <= sp <= blocks
        reached.add(tile); bns.add(bn)
        if blocks > 2:
            splits.add("one" if sp == 1 else "every block" if sp == blocks else "between")
    assert reached == set(WGRAD_TILES), "no backward shape runs on %s" % sorted(set(WGRAD_TILES) - reached)
    assert bns == {64, 128}
    assert splits == {"one", "every block", "between"}
    assert {wgrad_geometry(s)[1] for s in Tt.BWD_BF16} == {64, 128}


def test_backward_table_raggedness_kernel_sizes_and_strides():
    plus_one = _check_raggedness(Tt.BWD_SHAPES, lambda s: wgrad_geometry(s))
    assert plus_one == {t for t in WGRAD_TILES if t[2] > 1}
    assert {(s[5], s[6]) for s in Tt.BWD_SHAPES} >= {(1, 1), (3, 1), (5, 1), (7, 1), (3, 2), (5, 2), (7, 2)}
    # the data gradient runs the forward kernel on (B, H, W) with Cin output channels
    dx_tiles = {runtime.conv2d_tc_geometry(s[0], s[1], s[2], s[3])[:3] for s in Tt.BWD_SHAPES}
    assert len(dx_tiles) >= 8


@pytest.mark.parametrize("table", ["FWD_SHAPES", "BWD_SHAPES"])
def test_tables_hold_no_duplicates_and_stay_small(table):
    shapes = getattr(Tt, table)
    assert len(set(shapes)) == len(shapes)
    for B, H, W, Cin, Cout, k, s, _ in shapes:
        assert 2.0 * B * H * W * k * k * Cin * Cout < 2.5e9, "keep the fp64 reference of %s quick" % ((B, H, W, Cin, Cout, k),)


def _training_layers(B=8, S=256):
    """{scope/layer: (B, H, W, Cin, Cout, k, stride, leaky)} of every convolution of the HandSegNet and PoseNet2D training graphs at
    B x S x S, from the variables' weight shapes and the number of pools before each layer."""
    shapes = arch.variable_shapes()
    out = {}
    for scope, pool_after in (("HandSegNet", arch.HANDSEGNET_POOL_AFTER), ("PoseNet2D", arch.POSENET2D_POOL_AFTER)):
        pools = 0
        for name, _, stride, _, _, leaky in arch.NETS[scope]:
            k, _, cin, cout = shapes["%s/%s/weights" % (scope, name)]
            out["%s/%s" % (scope, name)] = (B, S >> pools, S >> pools, cin, cout, k, stride, leaky)
            pools += name in pool_after
    return out


def _pixel_blocks_per_cta(shape):
    tile, _, _, splits = wgrad_geometry(shape)
    B, H, W = shape[:3]
    return _cd(_cd(W, tile[0]) * _cd(H, tile[1]) * _cd(B, tile[2]), splits)


def test_training_cases_hold_every_training_layer_geometry():
    layers = _training_layers()
    assert len(layers) == 16 + 31
    missing = {n: s for n, s in layers.items() if s not in Tb.TRAIN_CASES}
    assert not missing, "TRAIN_CASES leaves out %s" % missing
    assert set(Tb.TRAIN_CASES) == set(layers.values()) and len(Tb.TRAIN_CASES) == 19
    # and so every weight-gradient launch of the two graphs (tile, N tile, tiles, splits) runs in a per-layer GPU test
    assert {wgrad_geometry(s) for s in layers.values()} == {wgrad_geometry(s) for s in Tb.TRAIN_CASES}


def test_training_cases_reach_the_longest_weight_gradient_reduction():
    """conv1_x at 256 x 256: 8192 pixel blocks in 44 splits, 187 per CTA (11 fp32 folds per warpgroup in bf16x3), against at most 47
    in the other per-layer cases."""
    layers = _training_layers()
    longest = max(_pixel_blocks_per_cta(s) for s in layers.values())
    assert longest == max(_pixel_blocks_per_cta(s) for s in Tb.TRAIN_CASES)
    assert runtime.conv2d_wgrad_geometry(8, 256, 256, 3, 64, 64) == (8, 8, 1, 64, 9, 44) and longest == 187
    assert longest > max(_pixel_blocks_per_cta(s) for s in Tb.CASES)
