"""GPU tests of the RHD reader's training mode: h3d_reader_aug_params against the Philox restatement (tests/reader_train_oracle.py);
each stage teacher-forced with the golden parameters against the oracle and against the reference reader's vectors
(golden_reference_reader_train.npz); hue and dropout bit-exact against their fp32 restatements; the augmented entries with every flag
off against the evaluation entries, bit for bit; reproducibility across runs, batch sizes and the shuffle; the three training demos
with --augment."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import reader_train_oracle as A

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_reference_reader_train as MT  # noqa: E402
import synth_records as SR  # noqa: E402

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(HERE, "golden", "golden_reference_reader_train.npz"))
EXACT = ("image", "image_crop", "hand_parts", "hand_mask", "keypoint_vis21", "keypoint_vis", "hand_side", "crop_scale", "keypoint_uv")


def _np(t):
    return t.detach().cpu().numpy()


def _ctx():
    from hand3d_b200 import runtime
    return runtime.default_context()


@pytest.fixture(scope="module")
def train_db(tmp_path_factory):
    p = tmp_path_factory.mktemp("rhd") / "rhd_training.bin"
    p.write_bytes(b"".join(SR.rhd_records(4)))
    return str(p)


def _reader(path, name, **over):
    from hand3d_b200.data.BinaryDbReader import BinaryDbReader
    kw = dict(MT.CONFIGS[name])
    kw.update(over)
    return BinaryDbReader(mode="training", path_to_db=path, **kw)


def _kw(name):
    kw = dict(MT.CONFIGS[name])
    kw.pop("shuffle")
    return A.flags_of(**kw), {k: kw[k] for k in ("use_wrist_coord", "hand_crop") if k in kw}


# ------------------------------------------------------------------------------------------ the generator
@pytest.mark.parametrize("seed", [0, 7, 20171003, 2 ** 64 - 1])
def test_device_params_against_restatement(seed):
    serials = np.concatenate([np.arange(1000), [41257, 10 ** 9, 2 ** 40 + 5, 2 ** 62]]).astype(np.int64)
    got = _np(_ctx().reader_aug_params(torch.from_numpy(serials), seed, 127))
    ref = A.aug_params(seed, serials, 127)
    exact = [A.SCALE, A.HUE_DELTA, A.WINDOW, A.WINDOW + 1] + list(range(A.KEEP, A.PARAMS))
    np.testing.assert_array_equal(got[:, exact], ref[:, exact])
    normal = list(range(A.UV_NOISE, A.SCALE)) + [A.OFFSET_NOISE, A.OFFSET_NOISE + 1]
    # fp64 log / sincospi on the device against numpy: the same fp32 value almost always, a different accept decision never
    np.testing.assert_allclose(got[:, normal], ref[:, normal], rtol=1e-6, atol=0)
    for flags in (0, A.COORD_UV_NOISE, A.HUE | A.RANDOM_CROP, A.SCOREMAP_DROPOUT):   # other flags leave the values of a flag alone
        sub = _np(_ctx().reader_aug_params(torch.from_numpy(serials[:64]), seed, flags))
        ref = A.aug_params(seed, serials[:64], flags)
        np.testing.assert_array_equal(sub[:, exact], ref[:, exact])
        np.testing.assert_allclose(sub[:, normal], ref[:, normal], rtol=1e-6, atol=0)


# ------------------------------------------------------------------------------------------ teacher-forced stages
def _golden_params(name):
    return torch.from_numpy(np.stack([G["%s/%d/params" % (name, i)] for i in range(4)])).cuda()


@pytest.mark.parametrize("name", list(MT.CONFIGS))
def test_teacher_forced_against_oracle_and_reference(train_db, name):
    recs = SR.rhd_records(4)
    flags, kw = _kw(name)
    rd = _reader(train_db, name, batch_size=4, seed=int(G["seed"]))
    params = _golden_params(name)
    d = rd._get([0, 1, 2, 3], params)
    torch.cuda.synchronize()
    for i in range(4):
        ref = A.rhd_items_train(recs[i], _np(params)[i], flags, **kw)
        assert set(d) == set(ref) - {"crop_center"}, (sorted(d), sorted(ref))
        for k in d:
            v, r = _np(d[k])[i], np.asarray(ref[k])
            if k in EXACT or r.dtype == bool or np.issubdtype(r.dtype, np.integer):
                np.testing.assert_array_equal(v.astype(r.dtype), r, err_msg=k)           # selection, integers, hue, crops: exact
            elif k in ("keypoint_xyz21_can", "rot_mat"):
                np.testing.assert_allclose(v, r, atol=2e-5, err_msg=k)                   # atanf / sinf / cosf chains
            else:
                np.testing.assert_allclose(v, r, atol=2e-6, rtol=2e-6, err_msg=k)
            pre = "%s/%d/%s" % (name, i, k)
            if pre + "/sub8" in G.files:
                np.testing.assert_allclose(v[::8, ::8], G[pre + "/sub8"], atol=2e-6, err_msg=k)
                np.testing.assert_allclose(v.astype(np.float64).sum(), G[pre + "/sums"][0], rtol=1e-5, atol=1e-4, err_msg=k)
            elif k not in ("keypoint_xyz21_can", "rot_mat"):
                np.testing.assert_allclose(v.astype(np.float64), G[pre].astype(np.float64), atol=2e-6, rtol=2e-6, err_msg=k)


def test_hue_and_window_bit_exact():
    rng = np.random.default_rng(3)
    B = 6
    img = (rng.integers(0, 256, size=(B, 320, 320, 3)).astype(np.float32) / np.float32(255.0) - np.float32(0.5)).astype(np.float32)
    img[0, :40] = img[0, :40, :, :1]                                  # grey rows: range 0
    img[1, :40, :, 1] = img[1, :40, :, 0]                            # ties between channels
    parts = rng.integers(0, 34, size=(B, 320, 320)).astype(np.uint8)
    p = A.aug_params(5, np.arange(B), A.HUE | A.RANDOM_CROP)
    p[0, A.HUE_DELTA], p[1, A.HUE_DELTA], p[2, A.WINDOW:A.WINDOW + 2] = -0.1, np.float32(0.1) - np.float32(2 ** -26), (64, 0)
    dp, di, dparts = torch.from_numpy(p).cuda(), torch.from_numpy(img).cuda(), torch.from_numpy(parts).cuda()
    ctx = _ctx()
    hue = _np(ctx.augment_image(di, dp, A.HUE)[0])
    win, wp, wm = [_np(t) for t in ctx.augment_image(di, dp, A.HUE | A.RANDOM_CROP, dparts)]
    plain = _np(ctx.augment_image(di, dp, A.RANDOM_CROP)[0])
    for b in range(B):
        ref = A.adjust_hue(img[b], p[b, A.HUE_DELTA])
        np.testing.assert_array_equal(hue[b], ref)
        oy, ox = int(p[b, A.WINDOW]), int(p[b, A.WINDOW + 1])
        np.testing.assert_array_equal(win[b], ref[oy:oy + 256, ox:ox + 256])
        np.testing.assert_array_equal(plain[b], img[b, oy:oy + 256, ox:ox + 256])
        np.testing.assert_array_equal(wp[b], parts[b, oy:oy + 256, ox:ox + 256])
        np.testing.assert_array_equal(wm[b, ..., 1], parts[b, oy:oy + 256, ox:ox + 256] > 1)
        np.testing.assert_array_equal(wm[b, ..., 0], parts[b, oy:oy + 256, ox:ox + 256] <= 1)
    dark = img.max(-1) <= 0
    assert dark.any() and np.all(hue[dark] == img.max(-1)[dark][:, None])          # the grey collapse of TF 1.3's rgb_to_hsv


def test_dropout_bit_exact():
    rng = np.random.default_rng(4)
    B = 5
    hw = rng.uniform(-10, 266, size=(B, 21, 2)).astype(np.float32)
    vis = (rng.uniform(size=(B, 21)) > 0.2).astype(np.uint8)
    p = A.aug_params(9, np.arange(B), A.SCOREMAP_DROPOUT)
    assert (p[:, A.KEEP:A.KEEP + 21] == 0).any()
    ctx = _ctx()
    dhw, dvis, dp = torch.from_numpy(hw).cuda(), torch.from_numpy(vis).cuda(), torch.from_numpy(p).cuda()
    plain = _np(ctx.gaussian_scoremap(dhw, (256, 256), 25.0, dvis))
    drop = _np(ctx.gaussian_scoremap_dropout(dhw, (256, 256), 25.0, dvis, dp[:, A.KEEP:A.KEEP + 21], 0.8))
    for b in range(B):
        np.testing.assert_array_equal(drop[b], A.dropout(plain[b], p[b, A.KEEP:A.KEEP + 21]))
    kept = np.broadcast_to(p[:, None, None, A.KEEP:A.KEEP + 21] == 1, drop.shape)
    assert (drop[kept] != plain[kept]).any()                 # (x / 0.8) * 0.8 is not always x: the last bit is TF's, not the identity's


# ------------------------------------------------------------------------------------------ flags off = evaluation
@pytest.mark.parametrize("use_wrist,hand_crop", [(False, True), (True, False), (False, False)])
def test_flags_off_equals_evaluation_entries(use_wrist, hand_crop):
    recs = SR.rhd_records(4)
    ctx = _ctx()
    raw = ctx.decode_records(torch.from_numpy(np.frombuffer(b"".join(recs), np.uint8).reshape(4, -1).copy()).cuda(), "rhd", 1)
    a = ctx.rhd_reader_items(raw["header"], raw["mask"], raw["visibility"], use_wrist, hand_crop, 256)
    b = ctx.rhd_reader_items_aug(raw["header"], raw["mask"], raw["visibility"], None, 0, use_wrist, hand_crop, 256)
    for k, v in a.items():
        if v is not None:
            assert torch.equal(v, b[k]), k


def test_reader_without_flags_is_the_evaluation_reader(train_db):
    from hand3d_b200.data.BinaryDbReader import BinaryDbReader
    ev = BinaryDbReader(mode="evaluation", shuffle=False, batch_size=4, use_wrist_coord=False, hand_crop=True, path_to_db=train_db).get()
    tr = BinaryDbReader(mode="training", shuffle=False, batch_size=4, use_wrist_coord=False, hand_crop=True, path_to_db=train_db, seed=1).get()
    assert set(ev) == set(tr) and all(torch.equal(ev[k], tr[k]) for k in ev)
    # an augmented reader's keypoint_uv (palm substituted on the device) equals the evaluation reader's when no noise is drawn
    aug = BinaryDbReader(mode="training", shuffle=False, batch_size=4, use_wrist_coord=False, hand_crop=True, scoremap_dropout=True,
                         path_to_db=train_db, seed=1).get()
    for k in ev:
        if k != "scoremap":
            assert torch.equal(ev[k], aug[k]), k


# ------------------------------------------------------------------------------------------ reproducibility
def _same(a, b):
    assert set(a) == set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_same_seed_same_batches_and_batch_size_independence(train_db):
    r1, r2 = _reader(train_db, "all", batch_size=8, seed=77), _reader(train_db, "all", batch_size=8, seed=77)
    for _ in range(2):
        _same(r1.get(), r2.get())
    r3 = _reader(train_db, "all", batch_size=8, seed=78)
    assert not torch.equal(_reader(train_db, "all", batch_size=8, seed=77).get()["image_crop"], r3.get()["image_crop"])
    big = _reader(train_db, "all", batch_size=8, seed=5).get()
    small = _reader(train_db, "all", batch_size=4, seed=5)
    halves = [small.get(), small.get()]
    for k in big:
        assert torch.equal(big[k], torch.cat([h[k] for h in halves])), k


def test_shuffle_reorders_the_same_per_serial_samples(train_db):
    shuf = _reader(train_db, "lifting", batch_size=8, seed=11)
    serials = A.shuffle_serials(11, 24)
    got = [shuf.get() for _ in range(3)]
    flat = {k: torch.cat([g[k] for g in got]) for k in got[0]}
    seq = _reader(train_db, "lifting", batch_size=16, seed=11, shuffle=False)
    n = int(serials.max()) // 16 + 1
    ordered = [seq.get() for _ in range(n)]
    by_serial = {k: torch.cat([o[k] for o in ordered]) for k in ordered[0]}
    idx = torch.from_numpy(serials).cuda()
    assert len(set(serials.tolist())) == 24 and serials.max() < 124
    for k in flat:
        assert torch.equal(flat[k], by_serial[k][idx]), k


def test_handsegnet_keys_and_shapes(train_db):
    rd = _reader(train_db, "handsegnet", batch_size=8)
    assert isinstance(rd.seed, int)
    d = rd.get()
    assert {k: tuple(v.shape) for k, v in d.items()} == {"image": (8, 256, 256, 3), "hand_parts": (8, 256, 256), "hand_mask": (8, 256, 256, 2)}
    assert d["hand_parts"].dtype == torch.int32 and d["hand_mask"].dtype == torch.int32
    with pytest.raises(NotImplementedError):
        from hand3d_b200.data.BinaryDbReader import BinaryDbReaderSTB
        BinaryDbReaderSTB(mode="training", shuffle=False, hue_aug=True, path_to_db=train_db)


@pytest.mark.parametrize("demo,extra", [("train_handsegnet_demo.py", []), ("train_posenet_demo.py", []),
                                        ("train_lifting_demo.py", ["--variant", "proposed"])])
def test_training_demos_with_augment(tmp_path, demo, extra):
    cmd = [sys.executable, os.path.join(ROOT, "examples", demo), "--augment", "--seed", "3", "--iters", "3", "--show-loss-freq", "1",
           "--snapshot-dir", str(tmp_path / "snap")] + extra
    r = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert r.stdout.count("Iteration") == 3 and "nan" not in r.stdout.lower(), r.stdout
