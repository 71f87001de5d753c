"""Camera rigs without a GPU: the rig entries are declared, bound and exported; the rig kernels compile for sm_90a without spills while
the single-size frame kernels keep their registers; the host-built rig table (h3d_frame_rig_query) is restated in numpy, each slot's
(slot, band) ranges and coefficient tables checked against Pillow's coefficients (tests/frames_oracle.py); refusals name the slot."""
import os
import re

import numpy as np
import pytest

import frames_oracle as F
from hand3d_b200 import _lib
from hand3d_b200 import frames as FR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "hand3d_b200", "build", "nvcc.log")
SO = os.path.join(ROOT, "hand3d_b200", "libhand3d_b200.so")
ENTRIES = ("h3d_frame_rig_query", "h3d_frame_rig_plan", "h3d_resize_frames_rig")
FORMATS = ("rgb", "bgr", "nv12", "i420", "yuyv")

# rigs of 1..8 slots: mixed sizes (one not a multiple of 8, one above 2048 px), every format, repeated sizes and formats
RIGS = [
    (["rgb", "nv12", "yuyv"], [(1080, 1920), (720, 1280), (480, 640)]),
    (["nv12", "bgr", "i420", "yuyv", "rgb"], [(2160, 3840), (482, 642), (1080, 1920), (100, 78), (243, 321)]),
    (["i420", "i420", "rgb", "bgr", "yuyv", "nv12", "rgb", "yuyv"],
     [(720, 1280), (720, 1280), (240, 320), (4096, 4096), (3, 2050), (2, 2), (1, 1), (720, 1280)]),
    (["yuyv"], [(600, 800)]),
]


def _log_sections():
    if not os.path.exists(LOG):
        pytest.skip("no build log: run python -m hand3d_b200.build first")
    out = {}
    for sec in open(LOG).read().split("Compiling entry function")[1:]:
        name = sec.split("'")[1]
        if "frames_cu" in name:
            out[name] = (sec, int(re.search(r"(\d+) bytes spill stores", sec).group(1)), int(re.search(r"Used (\d+) registers", sec).group(1)))
    return out


def test_rig_entries_are_declared_bound_and_exported():
    main = open(os.path.join(ROOT, "include", "hand3d_b200.h")).read()
    assert '#include "hand3d_b200_rig.h"' in main
    hdr = open(os.path.join(ROOT, "include", "hand3d_b200_rig.h")).read()
    declared = set(re.findall(r"H3D_API\s+[\w\s\*]+?\b(h3d_\w+)\s*\(", hdr))
    assert declared == set(ENTRIES) == set(_lib.RIG_SIGNATURES)
    assert not declared & set(_lib.SIGNATURES)
    for name, value in (("H3D_FRAME_RIG_MAX_SLOTS", _lib.FRAME_RIG_MAX_SLOTS), ("H3D_FRAME_RIG_SLOT_WORDS", _lib.FRAME_RIG_SLOT_WORDS),
                        ("H3D_FRAME_RIG_LAUNCH_WORDS", _lib.FRAME_RIG_LAUNCH_WORDS), ("H3D_RIG_CTA0", _lib.RIG_CTA0),
                        ("H3D_RIG_XB", _lib.RIG_XB), ("H3D_RIG_KY", _lib.RIG_KY), ("H3D_RIG_SIZE", _lib.RIG_SIZE),
                        ("H3D_RIG_LAUNCH_SMEM", _lib.RIG_LAUNCH_SMEM), ("H3D_RIG_SEG_OFF", _lib.RIG_SEG_OFF)):
        assert re.search(r"#define %s %d\b" % (name, value), hdr), name
    src = open(os.path.join(ROOT, "hand3d_b200", "csrc", "api.cu")).read()
    m = re.search(r"int h3d_version\(void\) \{ return (\d+); \}", src)
    assert m and int(m.group(1)) >= 112
    if not os.path.exists(SO):
        pytest.skip("library not built")
    lib = _lib.load()
    for e in ENTRIES:
        assert hasattr(lib, e)
    assert lib.h3d_version() >= 112


def test_every_rig_entry_has_its_launch_count_checked():
    """Every entry bound in _lib.RIG_SIGNATURES is counted by test_gpu_frames_rig.py's launch-count test or excluded with a reason."""
    import test_gpu_frames_rig as G
    assert not set(G.RIG_LAUNCH_CASES) & set(G.RIG_LAUNCH_EXCLUDED)
    assert set(G.RIG_LAUNCH_CASES) | set(G.RIG_LAUNCH_EXCLUDED) == set(_lib.RIG_SIGNATURES)
    assert sorted(G.RIG_LAUNCH_CASES.values()) == ["plan", "resize"]


def test_rig_kernels_compile_for_sm90a_without_spills():
    secs = _log_sections()
    for f in range(5):
        hits = [v for n, v in secs.items() if "resize_frames_rig_kernelILi%dE" % f in n]
        assert len(hits) == 1, f
        sec, spill, regs = hits[0]
        assert "for 'sm_90a'" in sec
        assert spill == 0, "rig instance %d spills %d bytes" % (f, spill)
        assert regs <= 64, "rig instance %d uses %d registers (two 512-thread CTAs per SM need <= 64)" % (f, regs)


def test_single_size_frame_kernels_keep_their_registers():
    # the counts of the single-size instances before the rig kernel shared their band code
    want = {"resize_frames_kernelILi%dE" % f: 64 for f in range(5)}
    want.update({"convert_frames_kernelILi%dE" % f: r for f, r in enumerate((34, 34, 32, 32, 32))})
    secs = _log_sections()
    for k, regs in want.items():
        hits = [v for n, v in secs.items() if k in n]
        assert len(hits) == 1, k
        _, spill, got = hits[0]
        assert spill == 0, "%s spills %d bytes" % (k, spill)
        assert got == regs, "%s uses %d registers, was %d" % (k, got, regs)


def _geometry(fmt, Hf, Wf, h, w, kxs, kys):
    """frames.cu's frame_geometry, restated."""
    def up(v, a):
        return (v + a - 1) // a * a
    w3 = 3 * w
    seg, row_stride, rgb_stride = [0, 0, 0], 0, 0
    if fmt in ("nv12", "i420", "yuyv"):
        n = {"i420": 3, "nv12": 2, "yuyv": 1}[fmt]
        lens = [2 * Wf if fmt == "yuyv" else Wf, Wf if fmt == "nv12" else Wf // 2, Wf // 2]
        for i in range(n):
            seg[i] = row_stride
            row_stride += up(lens[i] + 15, 16)
        rgb_stride = up(Wf * 3, 16)
        chunk = max(1, min(8, 2 * 28 * 1024 // (2 * row_stride + rgb_stride)))
    else:
        row_stride = up(Wf * 3 + 15, 16)
        chunk = max(1, min(8, 28 * 1024 // row_stride))
    band = max(1, min(16, h, 36 * 1024 // (w3 * 4)))
    nbands = -(-h // band)
    acc, inter = up(band * w3 * 4, 16), up(chunk * w3, 16)
    return dict(kxs=kxs, kys=kys, band=band, chunk=chunk, row_stride=row_stride, nbands=nbands, acc=acc, inter=inter,
                smem=acc + inter + 2 * chunk * row_stride + chunk * rgb_stride, seg=seg, rgb_stride=rgb_stride)


def _pillow(in_size, out_size):
    """(bounds [out,2], kk [out,ksize]) as frames.cu builds them: Pillow's, or one tap of weight 1 for an axis that keeps its size."""
    if in_size == out_size:
        return np.stack([np.arange(out_size), np.ones(out_size, np.int64)], 1), np.full((out_size, 1), 1 << F.PRECISION_BITS)
    bounds, kk = F.coeffs(in_size, out_size)
    return np.array(bounds), kk


@pytest.mark.parametrize("size", [(240, 320), (256, 256)], ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("rig", range(len(RIGS)))
def test_rig_table_restated(rig, size):
    fmts, hws = RIGS[rig]
    h, w = size
    B, SW, LW = len(fmts), _lib.FRAME_RIG_SLOT_WORDS, _lib.FRAME_RIG_LAUNCH_WORDS
    table, coef = FR.rig_layout(fmts, hws, size)
    assert table.size == B * SW + B + 5 * LW
    slots = table[:B * SW].reshape(B, SW)
    order = table[B * SW:B * SW + B]
    launches = table[B * SW + B:].reshape(5, LW)
    # the normalisation table: run.py's float32(u / 255.0 - 0.5)
    np.testing.assert_array_equal(coef[:256].view(np.float32), (np.arange(256) / 255.0 - 0.5).astype(np.float32))
    # the order groups the slots by format, in format order and slot order, and each launch record covers its group
    assert sorted(order.tolist()) == list(range(B))
    want_order = [b for f in range(5) for b in range(B) if FORMATS.index(fmts[b]) == f]
    assert order.tolist() == want_order
    sizes = list(dict.fromkeys(hws))
    seen = set()
    for f in range(5):
        first, n, ctas, smem = launches[f]
        group = order[first:first + n].tolist()
        assert group == [b for b in want_order if FORMATS.index(fmts[b]) == f]
        assert ctas == sum(int(slots[b, _lib.RIG_NBANDS]) for b in group)
        assert smem == (max(int(slots[b, _lib.RIG_SMEM]) for b in group) if group else 0)
        for c in range(ctas):                   # the kernel's rule: the last slot of the group whose range starts at or before c
            i = 0
            while i + 1 < n and slots[group[i + 1], _lib.RIG_CTA0] <= c:
                i += 1
            b = group[i]
            band = c - int(slots[b, _lib.RIG_CTA0])
            assert 0 <= band < slots[b, _lib.RIG_NBANDS], (c, b, band)
            assert (b, band) not in seen
            seen.add((b, band))
    # every output row band of every slot exactly once, and the bands cover the output rows
    assert seen == {(b, j) for b in range(B) for j in range(int(slots[b, _lib.RIG_NBANDS]))}
    for b in range(B):
        e = slots[b]
        H, W = hws[b]
        assert (e[_lib.RIG_FORMAT], e[_lib.RIG_H], e[_lib.RIG_W]) == (FORMATS.index(fmts[b]), H, W)
        assert e[_lib.RIG_SIZE] == sizes.index((H, W))
        assert e[22] == 0 and e[23] == 0
        xb, kx = _pillow(W, w)
        yb, ky = _pillow(H, h)
        kxs, kys = kx.shape[1], ky.shape[1]
        np.testing.assert_array_equal(coef[e[_lib.RIG_XB]:e[_lib.RIG_XB] + 2 * w], xb.reshape(-1), err_msg="xb of slot %d" % b)
        np.testing.assert_array_equal(coef[e[_lib.RIG_KX]:e[_lib.RIG_KX] + w * kxs], kx.reshape(-1), err_msg="kx of slot %d" % b)
        np.testing.assert_array_equal(coef[e[_lib.RIG_YB]:e[_lib.RIG_YB] + 2 * h], yb.reshape(-1), err_msg="yb of slot %d" % b)
        np.testing.assert_array_equal(coef[e[_lib.RIG_KY]:e[_lib.RIG_KY] + h * kys], ky.reshape(-1), err_msg="ky of slot %d" % b)
        g = _geometry(fmts[b], H, W, h, w, kxs, kys)
        got = dict(kxs=e[_lib.RIG_KXS], kys=e[_lib.RIG_KYS], band=e[_lib.RIG_BAND], chunk=e[_lib.RIG_CHUNK], row_stride=e[_lib.RIG_ROW_STRIDE],
                   nbands=e[_lib.RIG_NBANDS], acc=e[_lib.RIG_ACC_BYTES], inter=e[_lib.RIG_INTER_BYTES], smem=e[_lib.RIG_SMEM],
                   seg=e[_lib.RIG_SEG_OFF:_lib.RIG_SEG_OFF + 3].tolist(), rgb_stride=e[_lib.RIG_RGB_STRIDE])
        assert {k: (v if isinstance(v, list) else int(v)) for k, v in got.items()} == g, "geometry of slot %d" % b
        assert e[_lib.RIG_NBANDS] * e[_lib.RIG_BAND] >= h > (e[_lib.RIG_NBANDS] - 1) * e[_lib.RIG_BAND]
        assert e[_lib.RIG_SMEM] <= 227 * 1024 - 144
    # one coefficient set per distinct size: slots of one size share their offsets
    for b in range(B):
        for c in range(B):
            if hws[b] == hws[c]:
                assert (slots[b, _lib.RIG_XB:_lib.RIG_KY + 1] == slots[c, _lib.RIG_XB:_lib.RIG_KY + 1]).all()
    assert coef.size == 256 + sum(2 * w + w * _pillow(W, w)[1].shape[1] + 2 * h + h * _pillow(H, h)[1].shape[1] for H, W in sizes)


@pytest.mark.parametrize("fmts,hws,needle", [
    (["nv12", "rgb"], [(1081, 1920), (480, 640)], "slot 0"),
    (["rgb", "i420"], [(480, 640), (480, 641)], "slot 1"),
    (["rgb", "bgr", "yuyv"], [(480, 640), (480, 640), (480, 639)], "slot 2"),
    (["rgb", "bgr"], [(480, 640), (4097, 640)], "slot 1"),
    (["rgb", "bgr"], [(480, 4098), (480, 640)], "slot 0"),
    (["rgb", "bgr"], [(0, 640), (480, 640)], "slot 0"),
    (["rgb", 7], [(480, 640), (480, 640)], "slot 1"),
    ([], [], "1..64 slots"),
    (["rgb"] * 65, [(8, 8)] * 65, "1..64 slots"),
])
def test_refusals_name_the_slot(fmts, hws, needle):
    if not os.path.exists(SO):
        pytest.skip("library not built")
    with pytest.raises(ValueError, match=needle):
        FR.rig_layout(fmts, hws)


def test_refusals_of_lengths_and_output_size():
    if not os.path.exists(SO):
        pytest.skip("library not built")
    with pytest.raises(ValueError, match="pixel formats"):
        FR.rig_layout(["rgb"], [(8, 8), (8, 8)])
    for size in ((0, 320), (240, 513)):
        with pytest.raises(ValueError, match="output"):
            FR.rig_layout(["rgb", "nv12"], [(8, 8), (8, 8)], size)
    # a short table is refused, not overrun
    import ctypes as C
    lib = _lib.load()
    fmts, hw = (C.c_int * 2)(0, 2), (C.c_int * 4)(8, 8, 16, 16)
    tw, cw = C.c_int64(4), C.c_int64(1 << 20)
    buf = np.zeros(4, np.int32)
    assert lib.h3d_frame_rig_query(2, fmts, hw, 240, 320, buf.ctypes.data_as(C.c_void_p), C.byref(tw), None, C.byref(cw)) == _lib.EINVAL
    assert (buf == 0).all()
