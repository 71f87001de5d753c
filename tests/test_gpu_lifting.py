"""The lifting stage (PosePrior + ViewpointNet: two conv pyramids, their FC stacks, Rodrigues / flip / rotate) across batch sizes,
variants and kernel paths, against the fp64 oracle.

Kernel paths of the stage (api.cu: build_lifting):
  chain_bf16x3, chain_fp16x3   wgmma pyramids + both FC stacks and the rotation as one fc_chain_kernel launch
  layers_bf16x3                fc_chain = 0: one conv_tc_kernel launch per FC layer, CUDA-core view-point heads, rotate_canonical_kernel
  ffma_fp32                    fp32 CUDA-core pyramids and split-K FC (fc_splitk_kernel), as fp16_f8c and lift_direct = 1 run it

The batch sizes reach the FC chain's second 128-row M tile (129: one row, 160: 32 rows), wrap the 12-warp rotation loop (13) and
give fc_splitk_kernel a second 32-row tile (64; there fc_vp0 needs more split-K scratch than fc_rel0, so a reservation sized for
the widest layer alone is rejected with H3D_EINVAL).  Errors are normwise per output: max|g - ref| / max|ref|; with `pytest -s`
each parity case prints its errors, and the module's teardown the largest per path and output against its bound.

The stage runs in a private Context: at B = 160 its workspace (sized for 256x256 PoseNet crops) is several GB, which must not stay
in the process-wide default context.  The tuning switches are process-wide; every call sets all four that the stage reads."""
import gc

import numpy as np
import pytest
import torch

from hand3d_b200 import weights as Wt
from oracle import hand3d_oracle as O

pytestmark = pytest.mark.gpu
f32, f64 = np.float32, np.float64

BATCHES = [1, 13, 64, 128, 129, 160]
BMAX = max(BATCHES)
VARIANTS = ["proposed", "direct", "bottleneck", "local"]
PATHS = {  # path -> (precision, tuning switches)
    "chain_bf16x3": ("bf16x3", {}),
    "chain_fp16x3": ("fp16x3", {}),
    "layers_bf16x3": ("bf16x3", {"fc_chain": 0}),
    "ffma_fp32": ("fp32_ffma", {}),
}
TUNING_DEFAULTS = {"fc_chain": 1, "lift_direct": 0, "pdl": 1, "no_side_stream": 0}
# max|g - ref| / max|ref| per path and output: three times the largest figure one H100 80GB HBM3 (SXM, power limit 700 W) measured
# over the four variants and six batch sizes (DESIGN.md section 6.1)
BOUND = {
    "chain_bf16x3": {"out": 1.8e-4, "can": 8.2e-5, "rot": 1.9e-4},     # measured 6.1e-5, 2.7e-5, 6.3e-5
    "chain_fp16x3": {"out": 1.1e-4, "can": 4.4e-5, "rot": 9.2e-5},     # 3.6e-5, 1.5e-5, 3.1e-5
    "layers_bf16x3": {"out": 1.8e-4, "can": 8.2e-5, "rot": 1.5e-4},    # 6.1e-5, 2.7e-5, 5.0e-5
    "ffma_fp32": {"out": 1.2e-5, "can": 4.1e-6, "rot": 1.5e-5},        # 3.9e-6, 1.4e-6, 4.8e-6
}
MEASURED = {}   # (path, output) -> largest error seen, printed at module teardown


def _inputs():
    rng = np.random.default_rng(2026)
    sm = rng.normal(size=(BMAX, 32, 32, 21)).astype(f32)
    hs = np.zeros((BMAX, 2), f32)
    hs[np.arange(BMAX), rng.integers(0, 2, size=BMAX)] = 1.0
    # edge rows, in the first and in the second M tile: a tie must not flip (argmax picks index 0), (0.3, 0.7) flips, (0, 0) does not
    for rows, v in (((1, 128), (0.5, 0.5)), ((2, 129), (0.3, 0.7)), ((3, 159), (0.0, 0.0))):
        hs[list(rows)] = v
    return sm, hs


SM, HS = _inputs()
W_STD = {k: v for k, v in Wt.synthetic_weights(0).items() if k.startswith(("PosePrior", "ViewpointNet"))}
W_BOTT = {k: v for k, v in Wt.synthetic_weights(0, bottleneck=True).items() if k.startswith("PosePrior")}


@pytest.fixture(scope="module")
def ctx():
    from hand3d_b200 import runtime
    c = runtime.Context()
    try:
        c.ensure_workspace(BMAX, 8, 8)      # once, for the largest batch: no regrowth between tests
        c.load_weights(W_STD)
        c.weight_set = "std"
        yield c
    finally:
        torch.cuda.synchronize()
        for k, v in TUNING_DEFAULTS.items():
            c.set_tuning(k, v)
        c.lib.h3d_destroy(c.h)
        c.h = None
        c._ws = None
        del c
        gc.collect()
        torch.cuda.empty_cache()
        for (path, out), e in sorted(MEASURED.items()):
            print("lifting %-14s %-3s: max normwise error %.2e (bound %.1e)" % (path, out, e, BOUND[path][out]))


@pytest.fixture
def lift(ctx):
    """run(variant, B or row slice, precision, **switches) -> (out, can, rot); restores the default switches afterwards.  hs and wset
    replace the hand_side rows and the weight set (default: the synthetic weights of the variant)."""
    def run(variant, rows, prec, hs=None, wset=None, **switches):
        _weights(ctx, wset or ("bott" if variant == "bottleneck" else "std"))
        ctx.set_precision(prec)
        for k, v in {**TUNING_DEFAULTS, **switches}.items():
            ctx.set_tuning(k, v)
        sl = slice(0, rows) if isinstance(rows, int) else rows
        h = HS[sl] if hs is None else hs
        r = ctx.lifting(_cu(SM[sl]), _cu(h), variant)
        torch.cuda.synchronize()
        return r
    try:
        yield run
    finally:
        for k, v in TUNING_DEFAULTS.items():
            ctx.set_tuning(k, v)
        ctx.set_precision("bf16x3")


def _weights(ctx, name, wd=None):
    """Loads a named weight set into the private context (reloading drops the packed weights and the plans)."""
    if ctx.weight_set == name:
        return
    ctx.load_weights(wd if wd is not None else {"std": W_STD, "bott": W_BOTT}[name])
    ctx.weight_set = name


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


_ORACLE = {}


def oracle(variant):
    """fp64 (out, can, rot or None) for all BMAX rows.  The oracle computes every row on its own, so the rows of a smaller batch are
    a prefix of these."""
    if variant not in _ORACLE:
        if variant == "proposed":
            r = O.inference_pose3d(SM, HS, W_STD, dtype=f64)
        elif variant == "bottleneck":
            c = O.inference_pose3d_can(SM, HS, W_BOTT, dtype=f64, bottleneck=True)
            r = (c, c, None)
        else:
            c = O.inference_pose3d_can(SM, HS, W_STD, dtype=f64)
            r = (O.bone_rel_trafo_inv(c) if variant == "local" else c, c, None)
        _ORACLE[variant] = r
    return _ORACLE[variant]


def _err(g, ref):
    return float(np.abs(g.cpu().numpy().astype(f64) - ref).max() / np.abs(ref).max())


def _outputs(variant):
    return ("out", "can", "rot") if variant == "proposed" else ("out", "can")


# ------------------------------------------------------------------------------------------ (a) parity with the fp64 oracle
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("variant", VARIANTS)
def test_lifting_vs_fp64_oracle(lift, variant, path, B):
    prec, sw = PATHS[path]
    got = dict(zip(("out", "can", "rot"), lift(variant, B, prec, **sw)))
    ref = dict(zip(("out", "can", "rot"), oracle(variant)))
    assert (got["rot"] is None) == (variant != "proposed")
    errs = {}
    for k in _outputs(variant):
        assert tuple(got[k].shape) == ((B, 3, 3) if k == "rot" else (B, 21, 3))
        errs[k] = _err(got[k], ref[k][:B])
        MEASURED[(path, k)] = max(MEASURED.get((path, k), 0.0), errs[k])
    print("%s %s B=%d: %s" % (variant, path, B, " ".join("%s %.2e" % kv for kv in errs.items())))
    for k, e in errs.items():
        assert e < BOUND[path][k], "%s: normwise error %.3e, bound %.1e" % (k, e, BOUND[path][k])


# ------------------------------------------------------------------------------------------ (b) bit-exact equivalences
def _assert_equal(a, b, what):
    for k, x, y in zip(("out", "can", "rot"), a, b):
        assert (x is None) == (y is None), k
        if x is not None:
            assert torch.equal(x, y), "%s: %s differs (max |diff| %.3e)" % (what, k, (x - y).abs().max().item())


@pytest.mark.parametrize("B", [13, 129])
@pytest.mark.parametrize("single,triple", [("fp16", "fp16x3"), ("bf16", "bf16x3")])
@pytest.mark.parametrize("variant", VARIANTS)
def test_single_pass_modes_lift_in_three_passes(lift, variant, single, triple, B):
    """The lifting always runs 3-pass on the tensor path: the single-pass modes give the 3-pass lifting of the same 16-bit type."""
    _assert_equal(lift(variant, B, single), lift(variant, B, triple), "%s vs %s" % (single, triple))


@pytest.mark.parametrize("B", [13, 129])
@pytest.mark.parametrize("variant", VARIANTS)
def test_cuda_core_lifting_paths_agree(lift, variant, B):
    """fp16_f8c, fp32_ffma and lift_direct = 1 (in bf16x3) all run the fp32 CUDA-core kernels: one result, bit for bit."""
    base = lift(variant, B, "fp32_ffma")
    _assert_equal(lift(variant, B, "fp16_f8c"), base, "fp16_f8c vs fp32_ffma")
    _assert_equal(lift(variant, B, "bf16x3", lift_direct=1), base, "lift_direct vs fp32_ffma")


@pytest.mark.parametrize("B", [13, 129])
@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_fc_chain_off_matches_chain(lift, variant, prec, B):
    """fc_chain = 0 runs each FC layer through conv_tc_kernel with the same operands and K chunking as fc_chain_kernel, so the
    canonical coordinates are identical.  For 'proposed' the view-point heads run on the CUDA cores and the rotation in its own kernel
    there: out and rot are held to the layer path's parity bound instead."""
    chain = lift(variant, B, prec)
    layers = lift(variant, B, prec, fc_chain=0)
    assert torch.equal(chain[1], layers[1]), "can differs (max |diff| %.3e)" % (chain[1] - layers[1]).abs().max().item()
    if variant != "proposed":
        assert torch.equal(chain[0], layers[0])
        return
    for i, k in ((0, "out"), (2, "rot")):
        e = float((chain[i] - layers[i]).abs().max() / layers[i].abs().max())
        assert e < BOUND["layers_bf16x3"][k], "%s: chain vs layers %.3e" % (k, e)


@pytest.mark.parametrize("B", [13, 129])
@pytest.mark.parametrize("switch", [{"pdl": 0}, {"no_side_stream": 1}], ids=["pdl0", "no_side_stream"])
@pytest.mark.parametrize("prec", ["bf16x3", "fp32_ffma"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_launch_switches_change_no_bit(lift, variant, prec, switch, B):
    """Programmatic dependent launch off, or both branches on the caller's stream: the same bits as the default."""
    _assert_equal(lift(variant, B, prec, **switch), lift(variant, B, prec), str(switch))


# ------------------------------------------------------------------------------------------ (c) batch independence
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("variant", VARIANTS)
def test_rows_do_not_depend_on_the_batch(lift, variant, path):
    """Rows 0, 127, 128 and 129 of a B = 160 call equal single-image calls: bit for bit on the tensor-core paths (the pyramids'
    arithmetic does not depend on B and the FC chain computes each row on its own); within the parity bound on the CUDA-core path,
    whose split-K count depends on B."""
    prec, sw = PATHS[path]
    full = lift(variant, BMAX, prec, **sw)
    for r in (0, 127, 128, 129):
        one = lift(variant, slice(r, r + 1), prec, **sw)
        for k, a, b in zip(("out", "can", "rot"), full, one):
            if a is None:
                continue
            if path == "ffma_fp32":
                e = float((a[r:r + 1] - b).abs().max() / b.abs().max())
                assert e < BOUND[path][k], "row %d %s: %.3e" % (r, k, e)
            else:
                assert torch.equal(a[r:r + 1], b), "row %d: %s differs (max |diff| %.3e)" % (r, k, (a[r:r + 1] - b).abs().max().item())


# ------------------------------------------------------------------------------------------ (d) exact row canary
# FC weights that make the outputs exact small-integer (PosePrior) and dyadic (ViewpointNet) functions of hand_side: every operand is
# exact in the hi plane of bf16 and fp16, the fp16 weight shift is a power of two, and every partial sum is an integer below 2^24.
# A row mixed up between M tiles, a mis-masked row or a stale tile changes a value.
_A = np.random.default_rng(7).integers(-8, 9, size=(3, 63)).astype(f64)      # can[b, j] = a_j h0 + c_j h1 + d_j
_U = np.array([[1, -2], [3, 1], [-1, 2]], f64) / 64                         # u = _U (h - h_zero): dyadic, zero at h_zero


def _canary_hand_side(B):
    idx = np.random.default_rng(8).choice(100 * 100, size=B, replace=False)
    hs = np.stack([idx // 100 + 1, idx % 100 + 1], 1).astype(f32)            # distinct pairs of integers in 1 ... 100
    return hs


def _canary_weights(hs_zero, bottleneck):
    base = W_BOTT if bottleneck else W_STD
    wd = {k: v.copy() for k, v in base.items()}

    def fc(scope, name, n_in, n_out, pairs, bias=None):
        w = np.zeros((n_in, n_out), f32)
        for (i, j), v in pairs.items():
            w[i, j] = v
        wd["%s/%s/weights" % (scope, name)] = w
        wd["%s/%s/biases" % (scope, name)] = np.zeros(n_out, f32) if bias is None else bias.astype(f32)

    ident = {(0, 0): 1.0, (1, 1): 1.0}
    fc("PosePrior", "fc_rel0", 2050, 512, {(2048, 0): 1.0, (2049, 1): 1.0})
    fc("PosePrior", "fc_rel1", 512, 512, ident)
    if bottleneck:
        fc("PosePrior", "fc_bottleneck", 512, 30, ident)
    xyz = {(i, j): _A[i, j] for i in range(2) for j in range(63)}
    fc("PosePrior", "fc_xyz", 30 if bottleneck else 512, 63, xyz, _A[2])
    if not bottleneck:
        fc("ViewpointNet", "fc_vp0", 4098, 256, {(4096, 0): 1.0, (4097, 1): 1.0})
        fc("ViewpointNet", "fc_vp1", 256, 128, ident)
        d = -_U @ hs_zero.astype(f64)
        for r, name in enumerate(("fc_vp_ux", "fc_vp_uy", "fc_vp_uz")):
            fc("ViewpointNet", name, 128, 1, {(0, 0): _U[r, 0], (1, 0): _U[r, 1]}, d[r:r + 1])
    return wd


@pytest.mark.parametrize("B", [129, 160])
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("variant", ["proposed", "direct", "bottleneck"])
def test_fc_row_canary_is_exact(ctx, lift, variant, path, B):
    hs = _canary_hand_side(B)
    zero_row = B - 20                                                          # in the second M tile
    name = "canary_%s_%d" % (variant, B)
    _weights(ctx, name, _canary_weights(hs[zero_row], variant == "bottleneck"))
    prec, sw = PATHS[path]
    out, can, rot = lift(variant, B, prec, hs=hs, wset=name, **sw)
    h = hs.astype(f64)
    want = (h[:, :1] * _A[0] + h[:, 1:] * _A[1] + _A[2]).astype(f32)
    np.testing.assert_array_equal(can.reshape(B, 63).cpu().numpy(), want)
    if variant != "proposed":
        return
    u = ((h - h[zero_row]) @ _U.T).astype(f32)
    assert not u[zero_row].any()
    rot_ref, out_ref = ctx.rotate_canonical(can, _cu(u), _cu(hs))
    assert torch.equal(rot, rot_ref)
    u64 = u.astype(f64)
    R64 = O.get_rot_mat(u64[:, :1], u64[:, 1:2], u64[:, 2:])
    np.testing.assert_allclose(rot.cpu().numpy(), R64, rtol=0, atol=1e-6)
    out64 = np.matmul(O.flip_right_hand(want.astype(f64).reshape(B, 21, 3), hs), R64)
    assert _err(out, out64) < 1e-6
    assert _err(out_ref, out64) < 1e-6
