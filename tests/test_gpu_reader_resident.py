"""GPU tests of device-resident reading (BinaryDbReader / BinaryDbReaderSTB(..., device_resident=True)): the device queue against the
host queue; the fused gather + decode against h3d_decode_records on host-gathered records; every item of resident get() against the
host reader's; get() without a host synchronisation; a captured get() and a captured training iteration (reading, forward, loss,
backward, Adam) against eager runs on the host reader, bit for bit; the stream state across modes; the footprint."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

import reader_train_oracle as A

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, ROOT)
import make_golden_reference_reader_train as MT  # noqa: E402
from examples._synthetic_db import fake_rhd, fake_stb  # noqa: E402

pytestmark = pytest.mark.gpu
RANDOM_SEED = int.from_bytes(os.urandom(8), "little")
EVAL = {"eval2d": dict(shuffle=False, use_wrist_coord=True, scale_to_size=True),                 # eval2d.py
        "eval3d": dict(shuffle=False, hand_crop=True, use_wrist_coord=False)}                    # eval2d_gt_cropped.py, eval3d.py
CONFIGS = {**{k: MT.CONFIGS[k] for k in ("handsegnet", "posenet", "lifting", "all")}, **EVAL}


def _ctx():
    from hand3d_b200 import runtime
    return runtime.default_context()


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("resident")
    out = {}
    for name, data in (("rhd", fake_rhd(130, seed=1)), ("rhd16", fake_rhd(16, seed=2)), ("stb", fake_stb(23, seed=3))):
        p = d / (name + ".bin")
        p.write_bytes(data + (b"\x07" * 1000 if name == "rhd" else b""))       # a trailing partial record is ignored
        out[name] = str(p)
    return out


def _rhd(path, B, seed, resident, **kw):
    from hand3d_b200.data.BinaryDbReader import BinaryDbReader
    return BinaryDbReader(mode="training", batch_size=B, path_to_db=path, seed=seed, device_resident=resident, **kw)


def _stb(path, B, resident):
    from hand3d_b200.data.BinaryDbReader import BinaryDbReaderSTB
    return BinaryDbReaderSTB(mode="evaluation", shuffle=False, batch_size=B, path_to_db=path, device_resident=resident)


def _same(a, b):
    assert set(a) == set(b)
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
        assert torch.equal(a[k], b[k]), k


# ------------------------------------------------------------------------------------------ 1. the serial stream
@pytest.mark.parametrize("B", [1, 7, 8, 32])
@pytest.mark.parametrize("seed", [0, 1, 2 ** 64 - 1, pytest.param(RANDOM_SEED, id="random")])   # the seed is in err_msg
def test_device_serials_equal_host_queue(seed, B):
    from hand3d_b200.data.BinaryDbReader import _DeviceStream, _ShuffleQueue
    steps = -(-2000 // B)
    dev = _DeviceStream(seed, True, _ctx().device)
    got = torch.cat([dev.take(B) for _ in range(steps)]).cpu().numpy()
    want = np.array(_ShuffleQueue(seed).take(steps * B), np.int64)
    np.testing.assert_array_equal(got, want, err_msg="seed %d" % seed)
    np.testing.assert_array_equal(got, A.shuffle_serials(seed, steps * B))
    st = dev.state_dict()
    assert st["count"] == steps * B and st["next"] == 100 + steps * B and sorted(st["slots"]) == sorted(set(st["slots"]))
    seq = _DeviceStream(seed, False, _ctx().device)
    got = torch.cat([seq.take(B) for _ in range(5)]).cpu().numpy()
    np.testing.assert_array_equal(got, np.arange(5 * B))


def test_batch_of_eight_equals_two_of_four():
    from hand3d_b200.data.BinaryDbReader import _DeviceStream
    a, b = _DeviceStream(5, True, _ctx().device), _DeviceStream(5, True, _ctx().device)
    for _ in range(40):
        assert torch.equal(a.take(8), torch.cat([b.take(4), b.take(4)]))
    assert a.state_dict() == b.state_dict()


# ------------------------------------------------------------------------------------------ 2. the fused gather + decode
@pytest.mark.parametrize("name,step", [("rhd", 1), ("rhd", 2), ("rhd16", 1), ("stb", 1), ("stb", 2)])
def test_gather_decode_bit_identical_to_decode_of_host_gathered_records(files, name, step):
    from hand3d_b200.data.BinaryDbReader import _RecordFile, _ResidentFile
    from hand3d_b200.data.records import RHD_RECORD_BYTES, STB_RECORD_BYTES
    ds = "stb" if name == "stb" else "rhd"
    rf = _RecordFile(files[name], STB_RECORD_BYTES if ds == "stb" else RHD_RECORD_BYTES, 10 ** 9)
    res = _ResidentFile(rf, _ctx().device)
    n = rf.available
    assert tuple(res.records.shape) == (n, rf.record_bytes) and res.nbytes == n * rf.record_bytes
    serials = np.array([0, 5, n - 1, n, n + 3, 7 * n + 2, 99, 100, 2 ** 40 + 17, 3, 3], np.int64)
    got = _ctx().decode_records_gather(res.records, torch.from_numpy(serials).cuda(), ds, step)
    want = _ctx().decode_records(rf.gather(serials.tolist()), ds, step)
    for k, v in want.items():
        assert (v is None) == (got[k] is None), k
        if v is not None:
            assert torch.equal(got[k], v), k


# ------------------------------------------------------------------------------------------ 3. the items
@pytest.mark.parametrize("name", list(CONFIGS))
def test_resident_items_equal_host_items(files, name):
    host, res = _rhd(files["rhd"], 8, 17, False, **CONFIGS[name]), _rhd(files["rhd"], 8, 17, True, **CONFIGS[name])
    for _ in range(5):
        _same(res.get(), host.get())
    assert res.state_dict() == host.state_dict()


def test_resident_items_on_a_file_smaller_than_the_queue(files):
    host, res = _rhd(files["rhd16"], 8, 4, False, **MT.CONFIGS["all"]), _rhd(files["rhd16"], 8, 4, True, **MT.CONFIGS["all"])
    for _ in range(5):
        _same(res.get(), host.get())


@pytest.mark.parametrize("with_scoremap", [False, True])
def test_resident_stb_items_equal_host_items(files, with_scoremap):
    host, res = _stb(files["stb"], 6, False), _stb(files["stb"], 6, True)
    host.with_scoremap = res.with_scoremap = with_scoremap
    for _ in range(5):                 # 30 > 23 records: wraps around the file
        _same(res.get(), host.get())
    assert res.state_dict() == host.state_dict()


# ------------------------------------------------------------------------------------------ 4. no host synchronisation
def test_resident_get_runs_under_sync_debug_error(files):
    rd = _rhd(files["rhd"], 8, 3, True, **MT.CONFIGS["all"])
    hs = _rhd(files["rhd"], 8, 3, True, **MT.CONFIGS["handsegnet"])
    stb = _stb(files["stb"], 4, True)
    for r in (rd, hs, stb):
        r.get()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for r in (rd, hs, stb):
            for _ in range(3):
                r.get()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ 5. a captured reader
@pytest.mark.parametrize("name", ["lifting", "handsegnet", "eval3d"])
def test_captured_get_equals_eager_reader_at_the_same_position(files, name):
    rd = _rhd(files["rhd"], 8, 21, True, **CONFIGS[name])
    for _ in range(2):
        rd.get()
    torch.cuda.synchronize()
    start = rd.state_dict()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = rd.get()
    assert rd.state_dict() == start                 # capturing enqueues nothing
    ref = _rhd(files["rhd"], 8, 21, False, **CONFIGS[name])
    ref.load_state_dict(start)
    first = None
    for k in range(4):
        g.replay()
        want = ref.get()
        _same(out, want)
        first = first or {kk: v.clone() for kk, v in out.items()}
    assert rd.state_dict() == ref.state_dict() and rd.state_dict()["count"] == start["count"] + 4 * 8
    rd.load_state_dict(start)                       # rewinds the captured reader
    g.replay()
    _same(out, first)
    del g


# ------------------------------------------------------------------------------------------ 6. a captured training iteration
def _training(case, dataset):
    """(variables, optimiser, iteration) of the demo loop for `case`, from fresh weights."""
    from hand3d_b200 import autograd as AG, weights as Wt
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    from hand3d_b200.optim import Adam
    from hand3d_b200.utils.relative_trafo import bone_rel_trafo_inv
    ctx = _ctx()
    ctx.set_precision("bf16x3")
    if case in ("posenet", "handsegnet"):
        scope = "PoseNet2D" if case == "posenet" else "HandSegNet"
        net = ColorHandPose3DNetwork()
        net.init(weights={k: v for k, v in Wt.synthetic_weights(0).items() if k.startswith(scope + "/")})
        scopes = [scope]
    else:
        ctx.load_weights(Wt.xavier_weights(0))
        net = PosePriorNetwork(case)
        scopes = ["PosePrior", "ViewpointNet"] if case == "proposed" else ["PosePrior"]
    params = [p for s in scopes for p in ctx.variables(s).values()]
    for p in params:
        p.grad = None
    opt = Adam(params, lr=1e-4)

    def iteration():
        d = dataset.get()
        if case == "posenet":
            maps = net.inference_pose2d(d["image_crop"], train=True)
            s = d["scoremap"].shape
            vis = d["keypoint_vis21"].reshape(s[0], s[3]).float()
            loss = sum(AG.scoremap_loss(AG.resize_bilinear(m, s[1], s[2]), d["scoremap"], vis) for m in maps)
        elif case == "handsegnet":
            loss = AG.softmax_xent_loss(net.inference_detection(d["image"], train=True)[0], d["hand_mask"].float())
        else:
            _, coord, R = net.inference(d["scoremap"], d["hand_side"], True, train=True)
            if case == "proposed":
                loss = AG.mse_loss(coord, d["keypoint_xyz21_can"]) + AG.mse_loss(R, d["rot_mat"])
            else:
                loss = AG.mse_loss(bone_rel_trafo_inv(coord), d["keypoint_xyz21_normed"])
        opt.zero_grad()
        loss.backward()
        opt.step()
        return loss.detach()

    return params, iteration


@pytest.mark.parametrize("case,config,B", [("posenet", "posenet", 4), ("handsegnet", "handsegnet", 4), ("proposed", "lifting", 8),
                                           ("local_w_xyz_loss", "lifting", 8)])
def test_captured_iteration_equals_eager_iterations_on_the_host_reader(files, case, config, B):
    from hand3d_b200.train_loop import GraphedIteration
    warmup, k = 2, 10
    params, it = _training(case, _rhd(files["rhd"], B, 9, False, **MT.CONFIGS[config]))
    eager = [it().clone() for _ in range(warmup + k)]
    eager_w = [p.detach().clone() for p in params]
    del it
    gc.collect()
    params, it = _training(case, _rhd(files["rhd"], B, 9, True, **MT.CONFIGS[config]))
    run = GraphedIteration(it, warmup=warmup)
    graphed = [run().clone() for _ in range(warmup + k)]
    torch.cuda.synchronize()
    assert run.graph is not None
    print("%s losses: first %.6e last %.6e" % (case, float(eager[0]), float(eager[-1])))
    for i, (a, b) in enumerate(zip(graphed, eager)):
        assert torch.equal(a, b), (i, float(a), float(b))
    for a, b in zip(params, eager_w):
        assert torch.equal(a.detach(), b)
    del run


# ------------------------------------------------------------------------------------------ 7. state, footprint
def test_state_dict_resumes_the_stream_across_modes(files):
    cfg = MT.CONFIGS["posenet"]
    src = _rhd(files["rhd"], 8, 31, False, **cfg)
    for _ in range(3):
        src.get()
    st = src.state_dict()
    res = _rhd(files["rhd"], 8, 31, True, **cfg)
    res.load_state_dict(st)
    _same(res.get(), src.get())
    st2 = res.state_dict()
    host2 = _rhd(files["rhd"], 8, 31, False, **cfg)
    host2.load_state_dict(st2)
    for _ in range(2):
        _same(host2.get(), res.get())
    assert host2.state_dict() == res.state_dict()


def test_device_bytes_and_release(files):
    from hand3d_b200.data.records import RHD_RECORD_BYTES
    torch.cuda.synchronize()
    gc.collect()
    before = torch.cuda.memory_allocated()
    rd = _rhd(files["rhd"], 8, 1, True, **MT.CONFIGS["lifting"])
    assert rd._file.available == 130 and rd.device_bytes == 130 * RHD_RECORD_BYTES
    assert torch.cuda.memory_allocated() - before >= rd.device_bytes
    assert _stb(files["stb"], 2, True).device_bytes == 23 * 922104
    del rd
    gc.collect()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() - before < 130 * RHD_RECORD_BYTES


@pytest.mark.parametrize("demo,extra", [("train_posenet_demo.py", []), ("train_handsegnet_demo.py", []),
                                        ("train_lifting_demo.py", ["--variant", "proposed"])])
def test_demo_graph_losses_equal_eager_losses(tmp_path, demo, extra):
    import subprocess
    base = [sys.executable, os.path.join(ROOT, "examples", demo), "--augment", "--seed", "3", "--iters", "6", "--show-loss-freq", "1",
            "--snapshot-dir", str(tmp_path / "snap")] + extra
    outs = []
    for flags in ([], ["--device-resident"], ["--device-resident", "--graph"]):
        r = subprocess.run(base + flags, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
        outs.append([ln for ln in r.stdout.splitlines() if ln.startswith("Iteration")])
        print(demo, flags, outs[-1])
    assert len(outs[0]) == 6 and outs[0] == outs[1] == outs[2]
