"""Which kernels of csrc/elementwise.cu the tables of tests/test_gpu_postprocess_paths.py reach, and what their rows hold, checked
without a GPU.  Every __global__ of elementwise.cu must be the marked kernel of some table row or be excluded here with the reason and
the test that covers it; every row must take the kernel it is marked with under the launchers' predicates (restated in that module and
checked on the device by its test_dispatch); the tables must reach every instance, store path, grid shape and special value the
module promises."""
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_gpu_postprocess_paths as Tp  # noqa: E402
from oracle import tf1_ops as T  # noqa: E402

SOURCE = os.path.join(os.path.dirname(HERE), "hand3d_b200", "csrc", "elementwise.cu")

# kernel: (why no row of the tables reaches it, the test that covers it)
EXCLUDED = {
    "maxpool_backward_f32_kernel": ("the max-pool's training gradient", "test_gpu_conv_backward.py::test_max_pool_backward_vs_oracle"),
    "maxpool_split_kernel": ("reached only from stage plans, on split planes", "test_gpu_conv_layer_planes.py::test_unfused_pool_equals_fused"),
    "f32_to_split_kernel": ("plane conversion of the tensor-core entries", "test_gpu_tc_conv.py::test_conv2d_tc_vs_oracle"),
    "split_to_f32_kernel": ("plane conversion of the tensor-core entries", "test_gpu_tc_conv.py::test_conv2d_tc_vs_oracle"),
    "f32_to_f8c_kernel": ("plane conversion of the tensor-core entries (fp16_f8c)", "test_gpu_tc_conv.py::test_conv2d_tc_vs_oracle"),
    "f8c_to_f32_kernel": ("plane conversion of the tensor-core entries (fp16_f8c)", "test_gpu_tc_conv.py::test_conv2d_tc_vs_oracle"),
    "copy_channels_kernel": ("reached only from the PoseNet stage plan", "test_gpu_pipeline.py::test_posenet_stage"),
    "mask_grow_kernel": ("the mask grower after seg_prob_kernel (launched, not checked, by the seg rows)",
                         "test_gpu_ops.py::test_seg_postprocess_matches_oracle"),
    "mask_grow_cluster_kernel": ("the mask grower of maps over 512 pixels a side", "test_gpu_native_size.py::test_grower_bit_exact"),
    "rotate_canonical_kernel": ("the lifting stage's epilogue", "test_gpu_ops.py::test_rotate_canonical"),
    "decode_records_kernel": ("the dataset records", "test_gpu_ops.py::test_decode_rhd_and_stb_records"),
    "eval_dist_kernel": ("evaluation", "test_gpu_ops.py::test_eval_util_device_matches_reference_semantics"),
    "gather_records_p2p_kernel": ("the multi-GPU result exchange", "test_gpu_multi.py::test_p2p_gather_matches_nccl_and_single_gpu"),
    "bone_rel_trafo_inv_kernel": ("the lifting stage's forward kinematics", "test_gpu_ops.py::test_bone_rel_trafo_inv"),
    "pack_records_kernel": ("the result records", "test_gpu_ops.py::test_calc_center_bb_leaky_relu_flip_pack"),
    "mask_bbox_kernel": ("calc_center_bb on a given mask", "test_gpu_ops.py::test_calc_center_bb_leaky_relu_flip_pack"),
    "leaky_relu_kernel": ("NetworkOps.leaky_relu", "test_gpu_ops.py::test_calc_center_bb_leaky_relu_flip_pack"),
    "flip_right_hand_kernel": ("the lifting stage's hand flip", "test_gpu_ops.py::test_calc_center_bb_leaky_relu_flip_pack"),
}


def global_kernels():
    src = open(SOURCE).read()
    names = re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", src)
    assert len(names) == src.count("__global__"), "a __global__ the parser does not read"
    return set(names)


def _base(name):
    return name.split("<")[0]


def test_every_kernel_is_reached_or_excluded():
    kernels = global_kernels()
    reached = {_base(k) for k in Tp.expected_kernels() if k != "copy"}
    assert reached <= kernels, "table rows marked with kernels elementwise.cu does not have: %s" % sorted(reached - kernels)
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


def test_rows_take_their_marked_kernel():
    for B, H, W, C, oh, ow, kernel in Tp.RESIZE:
        assert Tp.resize_kernel(H, W, C, oh, ow) == kernel, (B, H, W, C, oh, ow)
    for B, H, W, C, kernel in Tp.MAXPOOL:
        assert Tp.maxpool_kernel(C) == kernel
    for B, H, W, C, crop, _, path in Tp.CROP:
        assert Tp.crop_path(B, C, crop) == path, (B, H, W, C, crop)
    for B, H, W, oh, ow, aligned, kernel in Tp.UPSAMPLE:
        assert Tp.upsample_kernel(H, W, oh, ow, aligned) == kernel, (B, H, W, oh, ow, aligned)


def test_resize_reaches_every_instance_and_store():
    paths = set()
    for B, H, W, C, oh, ow, kernel in Tp.RESIZE:
        store = "float4" if (ow * C) % 4 == 0 else "tail"
        paths.add((kernel, None if kernel == "copy" else store))
        total = B * oh * -(-(ow * C) // 4)
        if -(-total // 256) > 132 * 32:
            paths.add((kernel, "grid-stride"))
    for inst in ("<21>", "<2>", "<0>"):
        assert {("resize_bilinear_tf1_kernel" + inst, "float4"), ("resize_bilinear_tf1_kernel" + inst, "tail")} <= paths, inst
    assert ("copy", None) in paths and ("resize_bilinear_tf1_kernel<21>", "grid-stride") in paths
    rows = [r for r in Tp.RESIZE if r[-1] != "copy"]
    assert any(r[4] > r[1] and r[5] > r[2] for r in rows) and any(r[4] < r[1] and r[5] < r[2] for r in rows)
    assert any(r[4] % r[1] and r[1] % r[4] for r in rows), "a non-integer ratio"
    assert any(r[1] == r[2] == 1 for r in rows) and any(r[4] == r[5] == 1 for r in rows), "1-pixel inputs and outputs"
    assert any(r[1] == r[4] and r[2] != r[5] for r in rows) and any(r[1] != r[4] and r[2] == r[5] for r in rows)


def test_pool_rows():
    kinds = {(k, H % 2 == 1 or W % 2 == 1) for B, H, W, C, k in Tp.MAXPOOL}
    assert kinds == {(k, odd) for k in ("maxpool_f32_kernel", "maxpool_f32_scalar_kernel") for odd in (False, True)}
    for k in ("maxpool_f32_kernel", "maxpool_f32_scalar_kernel"):
        per = 4 if k == "maxpool_f32_kernel" else 1
        assert any(-(-(B * (H // 2) * (W // 2) * C // per) // 256) > 132 * 32 for B, H, W, C, kk in Tp.MAXPOOL if kk == k), \
            "%s: no row runs the grid-stride loop" % k
    assert {C % 4 for *_, C in Tp.AVGPOOL} >= {0, 1, 3}
    assert Tp.GAMMA_63 < 63 * 2.0 ** -24 * 1.0001


def test_crop_rows():
    rows = Tp.CROP
    assert {r[3] for r in rows} >= {1, 2, 3, 4, 21}
    assert {r[4] for r in rows} >= {1, 2, 3, 255, 256, 368}
    assert {p for r in rows for p in r[-1].split("+")} == {"c3", "channels", "single", "loop"}
    assert any(r[0] == 1 and r[4] == 256 and "loop" not in r[-1] for r in rows), "B = 1, one pass"
    assert any(r[0] == 6 and r[4] == 256 and "loop" in r[-1] for r in rows), "B = 6, the grid-stride loop"
    assert any(Tp.crop_grid(r[0], r[4]) == 1 and r[4] * r[4] > 256 for r in rows), "one CTA per image"
    assert any(r[1] == 1 for r in rows) and any(r[2] == 1 for r in rows)
    assert {0.25, 5.0} <= set(Tp.CROP_SCALES) and max(Tp.CROP_SCALES) > 5


def test_crop_edge_rows_hit_the_edges():
    """The edge rows' centres put samples exactly on 0 and n - 1 and just outside, in both axes"""
    for B, H, W, C, crop, boxes, _ in Tp.CROP:
        if boxes != "edge":
            continue
        _, center, scale = Tp.crop_problem(B, H, W, C, crop, boxes)
        hits = set()
        for i in range(B):
            for axis, n in ((0, H), (1, W)):
                s = Tp.crop_samples(center[i, axis], scale[i], n, crop)
                hits |= {(axis, "zero")} if (s == 0).any() else set()
                hits |= {(axis, "top")} if (s == np.float32(n - 1)).any() else set()
                hits |= {(axis, "below")} if ((s < 0) & (s > -1 / 16)).any() else set()
                hits |= {(axis, "above")} if ((s > n - 1) & (s < n - 1 + 1 / 16)).any() else set()
        assert hits == {(a, k) for a in (0, 1) for k in ("zero", "top", "below", "above")}, (B, H, W, C, crop, sorted(hits))


def test_detect_rows():
    assert {r[3] for r in Tp.DETECT} == {1, 2, 21, 64, 255, 256}
    grids = set()
    for B, H, W, C in Tp.DETECT:
        P, gx = Tp.detect_grid(H, W, C)
        assert (H * W) % P or P == 1, (B, H, W, C)
        assert B * C >= len(Tp.PATTERNS), "every pattern on some channel of %s" % ((B, H, W, C),)
        grids.add("one CTA" if gx == 1 else "64 CTAs" if gx == 64 else "several CTAs")
        if gx * P * 16 < H * W:
            grids.add("several steps per thread")
    assert grids == {"one CTA", "several CTAs", "64 CTAs", "several steps per thread"}


def test_detect_maps_carry_the_special_values():
    """np.argmax's answer on each pattern is what the pattern is for: the first of tied maxima (of either zero sign), the first NaN"""
    B, H, W, C = Tp.DETECT[0]
    s = Tp.detect_problem(B, H, W, C).reshape(B, H * W, C)
    for b in range(B):
        m, kind = s[b, :, 0], Tp.PATTERNS[b % len(Tp.PATTERNS)]
        i = int(np.argmax(m))
        if kind.startswith("nan") or kind == "all_nan":
            assert np.isnan(m[i]) and not np.isnan(m[:i]).any()
            if kind == "nan_neg_before":
                assert np.signbit(m[i]) and i < int(np.nanargmax(m))
            if kind == "nan_both":
                assert np.signbit(m[i]) and np.isnan(m[i + 1:]).any()
        if kind in ("neg_zero_first", "pos_zero_first"):
            ties = np.nonzero(m == 0)[0]
            assert m.max() == 0 and ties.size == 2 and i == ties[0] and np.signbit(m[i]) == (kind == "neg_zero_first")
        if kind in ("plateau", "run", "inf"):
            assert (m == m[i]).sum() >= 2
        if kind == "last":
            assert i == H * W - 1


def test_upsample_rows():
    ks = {r[-1] for r in Tp.UPSAMPLE}
    assert ks == {"resize_argmax_pow2_kernel", "resize_argmax_kernel"}
    generic = [r for r in Tp.UPSAMPLE if r[-1] == "resize_argmax_kernel"]
    why = set()
    for B, H, W, oh, ow, aligned, _ in generic:
        s = oh // H
        if not aligned:
            why.add("unaligned")
        elif oh % H or ow % W or oh // H != ow // W:
            why.add("ratio")
        elif s < 2 or s & (s - 1):
            why.add("not a power of two")
        elif ow % 4:
            why.add("out_w % 4")
        else:
            why.add("row too wide")
    assert why == {"unaligned", "ratio", "not a power of two", "out_w % 4", "row too wide"}


def test_upsample_maps_carry_the_special_values():
    """The up-sampled maps carry -0.0 and +0.0 tied at the maximum in both orders and NaNs; and where it fits, the tie that only the
    power-of-two kernel's in-thread tie test resolves (Tp.thread_order_case) and a maximum first reached in its last value slot
    (Tp.last_slot_case)"""
    thread_order = last_slot = 0
    for B, H, W, oh, ow, aligned, kernel in Tp.UPSAMPLE:
        s = Tp.upsample_problem(B, H, W, oh, ow)
        ref = T.resize_bilinear_tf1(s, oh, ow).reshape(B, oh * ow, 21)
        if len(Tp.exact_pixels(H, W, oh, ow)) >= 2:
            for k in range(B * 21):
                kind, m = Tp.PATTERNS[k % len(Tp.PATTERNS)], ref[k // 21, :, k % 21]
                if kernel == "resize_argmax_pow2_kernel" and ((k == 20 and Tp.thread_order_case(H, W, oh // H) is not None) or
                                                              (k == 19 and Tp.last_slot_case(H, W, oh // H) is not None)):
                    continue
                if kind in ("neg_zero_first", "pos_zero_first"):
                    top = np.nonzero(m == m.max())[0]
                    signs = np.signbit(m[top])
                    assert m.max() == 0 and top.size >= 2 and signs.any() and not signs.all(), ((B, H, W, oh, ow), kind)
                    assert signs[0] == (kind == "neg_zero_first"), ((B, H, W, oh, ow), kind)
                if kind.startswith("nan"):
                    assert np.isnan(m).any()
        if kernel == "resize_argmax_pow2_kernel" and Tp.thread_order_case(H, W, oh // H) is not None:
            sf = oh // H
            m = ref[0, :, 20].reshape(oh, ow)
            assert np.argmax(m) == 64 + sf and m[sf // 2, sf] == m.max() == 1.0 and m[0, sf] < 1.0, (B, H, W, oh, ow)
            thread_order += 1
        if kernel == "resize_argmax_pow2_kernel" and Tp.last_slot_case(H, W, oh // H) is not None:
            m = ref[0, :, 19].reshape(oh, ow)
            assert np.argmax(m) == 63 and m[0, 63] == m.max() == 1.0 and m[0, 62] < 1.0, (B, H, W, oh, ow)
            last_slot += 1
    assert thread_order >= 3 and last_slot >= 3
    assert {oh // H for B, H, W, oh, ow, _, k in Tp.UPSAMPLE if k == "resize_argmax_pow2_kernel"} >= {2, 4, 8}


def test_tables_hold_no_duplicates():
    for name in ("RESIZE", "MAXPOOL", "AVGPOOL", "CROP", "DETECT", "UPSAMPLE", "SEG"):
        rows = getattr(Tp, name)
        assert len(set(rows)) == len(rows), name
