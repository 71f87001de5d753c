"""DeviceEvalUtil and h3d_eval_feed / h3d_eval_stats on the GPU: the measures equal the unmodified reference's golden and the numpy
restatement (tests/eval_oracle.py) bit for bit; batching, the drop rule and graph capture change nothing; the four evaluation demo
loops replayed from one CUDA graph per batch equal their eager runs and the oracle, with no host synchronisation until get_measures."""
import os
import sys

import numpy as np
import pytest
import torch

import eval_oracle as EO

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from hand3d_b200 import _lib  # noqa: E402
from hand3d_b200.utils.general import DeviceEvalUtil, measures_from_stats  # noqa: E402

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(HERE, "golden", "golden_reference_numpy.npz"))


def _same_measures(got, want):
    for g, w in zip(got, want):
        assert np.asarray(g).dtype == np.asarray(w).dtype
        np.testing.assert_array_equal(g, w)


def _same_stats(got, want):
    """h3d_eval_stats rows: n_k and the counts exactly, the mean and median as float64 values (a NaN's payload is not compared)."""
    np.testing.assert_array_equal(got[:, _lib.EVAL_STAT_N], want[:, _lib.EVAL_STAT_N])
    np.testing.assert_array_equal(got[:, _lib.EVAL_STAT_COUNTS:], want[:, _lib.EVAL_STAT_COUNTS:])
    for c in (_lib.EVAL_STAT_MEAN, _lib.EVAL_STAT_MEDIAN):
        np.testing.assert_array_equal(got[:, c].copy().view(np.float64), want[:, c].copy().view(np.float64))


def _oracle_measures(lists, lo, hi, steps, dtype):
    with np.errstate(invalid="ignore", divide="ignore"):
        return measures_from_stats(EO.stats(lists, np.linspace(lo, hi, steps)), lo, hi, steps, dtype)


def _device_measures(ev, lo, hi, steps):
    with np.errstate(invalid="ignore", divide="ignore"):
        return ev.get_measures(lo, hi, steps)


# ------------------------------------------------------------------------------------------- 1. against the reference's golden
@pytest.mark.parametrize("tag", ["ev2", "ev3"])
def test_device_evalutil_equals_reference_golden(tag):
    ev = DeviceEvalUtil(num_samples=G[tag + "_gt"].shape[0])
    ev.feed(torch.from_numpy(G[tag + "_gt"]).cuda(), torch.from_numpy(G[tag + "_vis"]).cuda(), torch.from_numpy(G[tag + "_pred"]).cuda())
    assert ev.dtype == torch.float64
    lo, hi, steps = G[tag + "_range"]
    mean, median, auc, curve, thr = ev.get_measures(float(lo), float(hi), int(steps))
    np.testing.assert_array_equal(mean, G[tag + "_mean"])
    np.testing.assert_array_equal(median, G[tag + "_median"])
    np.testing.assert_array_equal(auc, G[tag + "_auc"])
    np.testing.assert_array_equal(curve, G[tag + "_curve"])
    np.testing.assert_array_equal(thr, G[tag + "_thr"])
    if tag == "ev2":
        assert len(ev.lists()[13]) == 0


# ------------------------------------------------------------------------------------------- 2. random sets against the oracle
def _random_set(n, D, dtype, seed):
    rng = np.random.default_rng(seed)
    gt = rng.normal(scale=20.0, size=(n, 21, D)).astype(dtype)
    pred = (gt + rng.normal(scale=rng.choice([0.01, 1.0, 10.0], size=(n, 21, 1)), size=gt.shape)).astype(dtype)
    vis = (rng.uniform(size=(n, 21)) > 0.25).astype(np.uint8) * rng.integers(1, 255, size=(n, 21)).astype(np.uint8)
    vis[:, 7] = 0                                           # a key-point that is never visible
    # distances exactly on a threshold: 3-4-5 triangles scaled by powers of two, thresholds at multiples of 1.25
    rows = rng.choice(n, size=max(1, n // 10), replace=False)
    s = 2.0 ** rng.integers(-2, 3, size=len(rows))
    gt[rows, 3] = 0
    pred[rows, 3] = 0
    pred[rows, 3, 0] = 3 * s
    pred[rows, 3, 1] = 4 * s
    # NaN and inf predictions
    pred[rng.choice(n, size=max(1, n // 50)), 5, 0] = np.nan
    pred[rng.choice(n, size=max(1, n // 50)), 9, D - 1] = np.inf
    return gt, vis, pred


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("D,n", [(2, 37), (3, 2728), (2, 41258), (3, 41258), pytest.param(3, 10 ** 6, id="3-1e6"),
                                 pytest.param(2, 10 ** 6, id="2-1e6")])
def test_random_sets_equal_the_oracle(dtype, D, n):
    gt, vis, pred = _random_set(n, D, dtype, seed=n + D)
    ev = DeviceEvalUtil(num_samples=n)
    ev.feed(torch.from_numpy(gt).cuda(), torch.from_numpy(vis).cuda(), torch.from_numpy(pred).cuda())
    with np.errstate(invalid="ignore"):
        lists = EO.feed_lists(gt, vis, pred)
    got_lists = ev.lists()
    for k in range(21):
        np.testing.assert_array_equal(got_lists[k], lists[k])
    for lo, hi, steps in ((0.0, 5.0, 20), (0.0, 40.0, 100), (1.25, 1.25 * 32, 32)):   # the last grid holds every 3-4-5 distance
        want = _oracle_measures(lists, lo, hi, steps, dtype)
        _same_measures(_device_measures(ev, lo, hi, steps), want)
    stats = ev._ctx.eval_stats(ev._store, 21, n, ev.dtype, torch.from_numpy(np.linspace(0.0, 40.0, 100)).cuda()).cpu().numpy()
    _same_stats(stats, EO.stats(lists, np.linspace(0.0, 40.0, 100)))


def test_unsorted_thresholds_are_counted():
    gt, vis, pred = _random_set(3000, 3, np.float32, seed=5)
    ev = DeviceEvalUtil(num_samples=3000)
    ev.feed(torch.from_numpy(gt).cuda(), torch.from_numpy(vis).cuda(), torch.from_numpy(pred).cuda())
    with np.errstate(invalid="ignore"):
        lists = EO.feed_lists(gt, vis, pred)
    thr = np.array([5.0, 0.5, np.nan, 40.0, 2.5, 2.5, 0.0, np.inf], np.float64)
    stats = ev._ctx.eval_stats(ev._store, 21, 3000, torch.float32, torch.from_numpy(thr).cuda()).cpu().numpy()
    _same_stats(stats, EO.stats(lists, thr))
    with np.errstate(invalid="ignore"):
        _same_measures(_device_measures(ev, 30.0, 0.0, 20), _oracle_measures(lists, 30.0, 0.0, 20, np.float32))   # descending grid


# ------------------------------------------------------------------------------------------- 3. batching, the drop rule, capture
def _feed_in_cuts(gt, vis, pred, cuts, n):
    ev = DeviceEvalUtil(num_samples=n)
    lo = 0
    for c in cuts:
        ev.feed(gt[lo:lo + c], vis[lo:lo + c], pred[lo:lo + c])
        lo += c
    assert lo == gt.shape[0]
    return ev


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_batching_changes_nothing(dtype):
    n = 300
    g, v, p = _random_set(n, 3, np.float64, seed=9)
    gt, vis, pred = (torch.from_numpy(g).to(dtype).cuda(), torch.from_numpy(v).cuda(), torch.from_numpy(p).to(dtype).cuda())
    ref = _feed_in_cuts(gt, vis, pred, [n], n)
    ref_lists, ref_m = ref.lists(), _device_measures(ref, 0.0, 30.0, 20)
    single = DeviceEvalUtil(num_samples=n)
    for i in range(n):
        single.feed(gt[i], vis[i], pred[i])                  # [K, D] / [K]: one sample per feed
    for cuts in ([7] * 42 + [6], [32] * 9 + [12], [1, 2, 3, 100, 50, 144], None):
        ev = single if cuts is None else _feed_in_cuts(gt, vis, pred, cuts, n)
        assert ev.kept == n and ev.dropped == 0
        for a, b in zip(ev.lists(), ref_lists):
            np.testing.assert_array_equal(a, b)
        _same_measures(_device_measures(ev, 0.0, 30.0, 20), ref_m)


def test_drop_rule_keeps_each_sample_once():
    g, v, p = _random_set(48, 2, np.float32, seed=4)
    gt, vis, pred = torch.from_numpy(g).cuda(), torch.from_numpy(v).cuda(), torch.from_numpy(p).cuda()
    ev = DeviceEvalUtil(num_samples=37)
    for lo in range(0, 48, 16):                             # 37 samples at B = 16: the last batch wraps around by 11
        ev.feed(gt[lo:lo + 16], vis[lo:lo + 16], pred[lo:lo + 16])
    assert ev.kept == 37 and ev.dropped == 11
    with np.errstate(invalid="ignore"):
        lists = EO.feed_lists(g[:37], v[:37], p[:37])
    for a, b in zip(ev.lists(), lists):
        np.testing.assert_array_equal(a, b)
    ev.reset()
    assert ev.kept == 0 and ev.dropped == 0 and all(len(x) == 0 for x in ev.lists())


def test_captured_feed_replayed_equals_eager_feeds():
    g, v, p = _random_set(16, 3, np.float64, seed=6)
    gt, vis, pred = torch.from_numpy(g).cuda(), torch.from_numpy(v).cuda(), torch.from_numpy(p).cuda()
    eager = DeviceEvalUtil(num_samples=100)
    for _ in range(5):
        eager.feed(gt, vis, pred)
    ev = DeviceEvalUtil(num_samples=100)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ev.feed(gt, vis, pred)                              # eager first feed: allocates the store
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    ev.reset()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ev.feed(gt, vis, pred)
    for _ in range(5):
        graph.replay()
    torch.cuda.synchronize()
    assert ev.kept == 80 == eager.kept
    for a, b in zip(ev.lists(), eager.lists()):
        np.testing.assert_array_equal(a, b)
    _same_measures(_device_measures(ev, 0.0, 30.0, 20), _device_measures(eager, 0.0, 30.0, 20))
    for _ in range(5):                                      # 20 samples fit, 60 are dropped
        graph.replay()
    assert ev.kept == 100 and ev.dropped == 60


def test_refusals():
    gt = torch.zeros((4, 21, 2), device="cuda")
    vis = torch.ones((4, 21), dtype=torch.uint8, device="cuda")
    ev = DeviceEvalUtil(num_samples=10)
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with pytest.raises(RuntimeError, match="eagerly"):
        with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
            ev.feed(gt, vis, gt)
    ev = DeviceEvalUtil(num_samples=10)
    ev.feed(gt, vis, gt)
    with pytest.raises(TypeError, match="float32"):
        ev.feed(gt.double(), vis, gt)                      # float64 after float32
    with pytest.raises(TypeError):
        ev.feed(gt.half(), vis, gt.half())
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="capture"):
        with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
            ev.get_measures(0.0, 1.0, 20)
    with pytest.raises(RuntimeError):
        ev.get_measures(0.0, 1.0, 4097)                    # more thresholds than h3d_eval_stats takes
    with pytest.raises(TypeError):
        ev.feed(gt.cpu(), vis, gt)


# ------------------------------------------------------------------------------------------- 4. the four evaluation loops
class _Recorder:
    """Forwards feeds to a DeviceEvalUtil and keeps host copies of what was fed."""
    def __init__(self, n):
        self.util, self.fed = DeviceEvalUtil(num_samples=n), []

    def feed(self, gt, vis, pred):
        self.fed.append((gt.cpu().numpy(), vis.cpu().numpy(), pred.cpu().numpy()))
        self.util.feed(gt, vis, pred)


def _demo(name):
    import importlib
    return importlib.import_module("examples." + name)


def _loop_parts(name, path, B):
    from hand3d_b200 import runtime
    from hand3d_b200.weights import synthetic_weights
    from hand3d_b200.data.BinaryDbReader import BinaryDbReader, BinaryDbReaderSTB
    ctx = runtime.default_context()
    if name == "eval3d_demo":
        from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
        net = PosePriorNetwork("proposed")
        w = synthetic_weights(0)
        net.init(None, weights={k: v for k, v in w.items() if k.startswith(("PosePrior", "ViewpointNet"))})
        make = lambda: (BinaryDbReader(mode='evaluation', shuffle=False, hand_crop=True, use_wrist_coord=False, batch_size=B, path_to_db=path,  # noqa: E731
                                       device_resident=True), _demo(name).make_step(net))
    else:
        from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
        net = ColorHandPose3DNetwork()
        if name == "eval_full_demo":
            net.init(None, weights=synthetic_weights(0))
            make = lambda: (BinaryDbReaderSTB(mode='evaluation', shuffle=False, use_wrist_coord=False, batch_size=B, path_to_db=path,  # noqa: E731
                                              device_resident=True), _demo(name).make_step(net, ctx))
        else:
            net.init(None, weights=synthetic_weights(0), exclude_var_list=['PosePrior', 'ViewpointNet'])
            if name == "eval2d_demo":
                make = lambda: (BinaryDbReader(mode='evaluation', shuffle=False, use_wrist_coord=True, scale_to_size=True, batch_size=B,  # noqa: E731
                                               path_to_db=path, device_resident=True), _demo(name).make_step(net, True))
            else:
                make = lambda: (BinaryDbReader(mode='evaluation', shuffle=False, hand_crop=True, use_wrist_coord=False, batch_size=B,  # noqa: E731
                                               path_to_db=path, device_resident=True), _demo(name).make_step(net, ctx, True))
    return make


@pytest.mark.parametrize("name,kind,dtype", [("eval2d_demo", "rhd", np.float64), ("eval2d_gt_cropped_demo", "rhd", np.float64),
                                             ("eval3d_demo", "rhd", np.float32), ("eval_full_demo", "stb", np.float32)])
def test_demo_loop_graph_equals_eager_and_oracle(tmp_path, name, kind, dtype):
    from examples._synthetic_db import fake_rhd, fake_stb
    from hand3d_b200.train_loop import GraphedIteration
    n, B = 37, 16
    path = tmp_path / (kind + ".bin")
    path.write_bytes(fake_rhd(n, seed=21) if kind == "rhd" else fake_stb(n, seed=22))
    make = _loop_parts(name, str(path), B)
    steps = [(0.0, 30.0, 20), (0.0, 0.05, 20), (0.0, 200.0, 100)]

    # eager resident loop, recording what is fed
    dataset, step = make()
    rec = _Recorder(n)
    for _ in range(0, n, B):
        step(dataset.get(), rec)
    assert rec.util.kept == n and rec.util.dropped == 3 * B - n
    eager = [_device_measures(rec.util, *s) for s in steps]

    # the oracle fed the same per-sample arrays, the wrapped tail left out
    gt = np.concatenate([f[0] for f in rec.fed])[:n]
    vis = np.concatenate([f[1] for f in rec.fed])[:n]
    pred = np.concatenate([f[2] for f in rec.fed])[:n]
    with np.errstate(invalid="ignore"):
        lists = EO.feed_lists(gt, vis, pred)
    assert lists[0].dtype == dtype and rec.util.dtype == torch.from_numpy(np.zeros(1, dtype)).dtype
    for m, s in zip(eager, steps):
        _same_measures(m, _oracle_measures(lists, *s, dtype))

    # one graph per batch: an eager warm-up batch, then replays with no host synchronisation until get_measures
    dataset, step = make()
    util = DeviceEvalUtil(num_samples=n)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(dataset.get(), util)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step(dataset.get(), util)
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(1, -(-n // B)):
            graph.replay()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert util.kept == n and util.dropped == 3 * B - n
    for m, s in zip(eager, steps):
        _same_measures(_device_measures(util, *s), m)


@pytest.mark.parametrize("demo,kind", [("eval2d_demo.py", "rhd"), ("eval2d_gt_cropped_demo.py", "rhd"), ("eval3d_demo.py", "rhd"),
                                       ("eval_full_demo.py", "stb")])
def test_demo_prints_the_same_lines_with_and_without_graph(tmp_path, demo, kind):
    import subprocess
    base = [sys.executable, os.path.join(ROOT, "examples", demo), "--samples", "37", "--batch", "16"]
    outs = []
    for flags in (["--device-resident"], ["--device-resident", "--graph"]):
        r = subprocess.run(base + flags, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
        outs.append(r.stdout.splitlines())
        print(demo, flags, outs[-1])
    assert outs[0] == outs[1]
    assert any(ln.startswith("Average mean EPE") for ln in outs[0])
    if demo == "eval_full_demo.py":
        assert any(ln.startswith("Area under curve between 20mm - 50mm") for ln in outs[0])
