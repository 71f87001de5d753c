"""HandSegNet and PoseNet2D training at the reference's shapes: B = 8 on 256 x 256 inputs (training_handsegnet.py's random_crop_size,
training_posenet.py's crop_size).  Every variable's gradient against fp64 CPU autograd, teacher-forced with the device's leaky and
max-pool decisions as tests/test_gpu_training.py does at 64 x 64, and one captured training step replayed against eager steps.

At 256 x 256 the trunk ends on 32 x 32 maps, so every tap of PoseNet2D's 7 x 7 recurrent layers reads real pixels, and conv1_x run
the longest weight-gradient reductions of either network (8192 pixel blocks in 44 splits).  The fp64 reference takes half a
minute of CPU per network and a few GB of host memory.

Errors are normwise: max|g - ref| / max|ref|."""
import gc
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_training as Tr  # noqa: E402
import train_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

B, S = 8, 256
# bf16x3: 3x the normwise errors measured on an H100 80GB HBM3 at 700 W (5.6e-5 at PoseNet2D conv6_7/weights, 1.5e-4 at HandSegNet
# conv4_1/biases; DESIGN.md 4.8), within the 1e-3 cap
NET_TOL = {"PoseNet2D": 1.7e-4, "HandSegNet": 4.4e-4}


@pytest.fixture(scope="module")
def ctx():
    from hand3d_b200 import runtime
    c = runtime.default_context()
    c.set_precision("bf16x3")
    return c


@pytest.fixture(scope="module")
def net(ctx):
    from hand3d_b200 import weights as Wt
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    n = ColorHandPose3DNetwork()
    n.init(weights=Wt.synthetic_weights(0))
    return n


def _report(scope, loss, ref_loss, errs):
    worst = max(errs, key=errs.get)
    print("%s at B = %d, %d x %d: loss %.6e (fp64 %.6e), worst gradient error %.3e at %s" % (
        scope, B, S, S, float(loss), float(ref_loss), errs[worst], worst))
    assert abs(float(loss) - float(ref_loss)) <= 1e-4 * abs(float(ref_loss))
    assert errs[worst] <= NET_TOL[scope], errs


def test_pose2d_gradients_at_training_shape_vs_fp64(ctx, net, monkeypatch):
    img, target, vis = Tr._pose_batch(B=B, S=S)
    v, _ = Tr._fresh(ctx, "PoseNet2D")
    assert len(v) == 62
    dec = Tr._Decisions(monkeypatch)
    loss = Tr._pose_loss(net, Tr._cu(img), Tr._cu(target), Tr._cu(vis))[0]
    loss.backward()
    loss = loss.detach()
    grads = {k: p.grad.cpu().numpy() for k, p in v.items()}
    rv = {k: torch.nn.Parameter(p.detach().cpu().double()) for k, p in v.items()}
    t64, vis64 = torch.from_numpy(target).double(), torch.from_numpy(vis).double()
    ref_loss = sum(O.scoremap_loss_torch(O.resize_bilinear_torch(m, S, S), t64, vis64)
                   for m in Tr._ref_pose2d(torch.from_numpy(img).double(), rv, dec))
    ref_loss.backward()
    _report("PoseNet2D", loss, ref_loss, {k: Tr._err(grads[k], rv[k].grad.numpy()) for k in v})


def test_detection_gradients_at_training_shape_vs_fp64(ctx, net, monkeypatch):
    img, lab = Tr._seg_batch(B=B, S=S)
    v, _ = Tr._fresh(ctx, "HandSegNet")
    assert len(v) == 32
    dec = Tr._Decisions(monkeypatch)
    loss = Tr._seg_loss(net, Tr._cu(img), Tr._cu(lab))[0]
    loss.backward()
    loss = loss.detach()
    grads = {k: p.grad.cpu().numpy() for k, p in v.items()}
    rv = {k: torch.nn.Parameter(p.detach().cpu().double()) for k, p in v.items()}
    ref_loss = O.softmax_xent_torch(Tr._ref_detection(torch.from_numpy(img).double(), rv, dec), torch.from_numpy(lab).double())
    ref_loss.backward()
    _report("HandSegNet", loss, ref_loss, {k: Tr._err(grads[k], rv[k].grad.numpy()) for k in v})


@pytest.mark.parametrize("scope", ["PoseNet2D", "HandSegNet"])
def test_cuda_graph_replay_equals_eager_steps_at_training_shape(ctx, net, scope):
    """One captured step (zero grads, forward, loss, backward, Adam) after two eager warm-up steps, replayed k times, equals k more
    eager steps bit for bit."""
    batch = [Tr._cu(a) for a in (Tr._pose_batch(27, B=B, S=S) if scope == "PoseNet2D" else Tr._seg_batch(27, B=B, S=S))]
    k = 2

    def step(opt):
        opt.zero_grad()
        loss = Tr._pose_loss(net, *batch)[0] if scope == "PoseNet2D" else Tr._seg_loss(net, *batch)[0]
        loss.backward()
        opt.step()

    v, opt = Tr._fresh(ctx, scope)
    for _ in range(2 + k):
        step(opt)
    eager = {n: p.detach().clone() for n, p in v.items()}
    # no autograd graph of an earlier step may be alive at capture (see test_gpu_training.test_cuda_graph_replay_equals_eager_steps)
    v, opt = Tr._fresh(ctx, scope)
    gc.collect()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(opt)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step(opt)
    for _ in range(k):
        g.replay()
    torch.cuda.synchronize()
    for n, p in v.items():
        assert torch.equal(p.detach(), eager[n]), n
    del g
