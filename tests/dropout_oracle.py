"""numpy restatement of the lifting stage's dropout (csrc/dropout.cu, include/hand3d_b200.h: H3D_DROPOUT_*), bit for bit.

Keep bit of element (row, col) at (seed, draw, layer): word col % 4 of Philox4x64-10 keyed (seed, STREAM) at counter
(draw, layer, row, col // 4), u = (w >> 40) 2^-24, k = floor(keep_prob + u) in fp32.  y = (x / keep_prob) * k and dx = (dy * k) /
keep_prob, each operation rounded to fp32.  The split planes are hi = h16(y), lo = h16(y - hi), zero past `cols`."""
import numpy as np

from reader_train_oracle import philox4x64_10, uniform01

STREAM = 2
LAYER_FC_REL0, LAYER_FC_REL1, LAYER_FC_VP0, LAYER_FC_VP1, LAYER_OP = 0, 1, 2, 3, 4
f32, u64 = np.float32, np.uint64


def words(seed, draw, layer, rows, cols):
    """[rows, cols] uint64: the Philox word each element draws."""
    g = (cols + 3) // 4
    r, q = np.meshgrid(np.arange(rows, dtype=u64), np.arange(g, dtype=u64), indexing="ij")
    ctr = np.stack([np.full_like(r, draw), np.full_like(r, layer), r, q], -1)
    key = np.broadcast_to(np.array([seed & 0xFFFFFFFFFFFFFFFF, STREAM], u64), ctr.shape[:-1] + (2,))
    return philox4x64_10(ctr, key).reshape(rows, 4 * g)[:, :cols]


def keep_bits(seed, draw, layer, rows, cols, keep_prob):
    u = uniform01(words(seed, draw, layer, rows, cols))
    return np.floor(f32(keep_prob) + u).astype(f32)


def forward(x, keep):
    """x, keep [rows, cols] -> y = (x / keep_prob) * k in fp32; keep_prob is passed as `keep[1]` of the (k, keep_prob) pair."""
    k, kp = keep
    return ((np.asarray(x, f32) / f32(kp)).astype(f32) * k).astype(f32)


def backward(dy, keep):
    k, kp = keep
    return ((np.asarray(dy, f32) * k).astype(f32) / f32(kp)).astype(f32)


def dropout(x, seed, draw, layer, keep_prob):
    """-> (y, keep bits uint8) of x [rows, cols]."""
    x = np.asarray(x, f32)
    k = keep_bits(seed, draw, layer, x.shape[0], x.shape[1], keep_prob)
    return forward(x, (k, keep_prob)), k.astype(np.uint8)


def _bf16(v):
    b = np.asarray(v, f32).view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)           # round to nearest even (finite inputs)
    return r


def _from_bf16(h):
    return (np.asarray(h, np.uint16).astype(np.uint32) << 16).view(f32)


def planes(y, stride, half):
    """hi / lo 16-bit planes [rows, stride] of y (half 0 = bf16, 1 = fp16), zeros in the padding columns."""
    rows, cols = y.shape
    full = np.zeros((rows, stride), f32)
    full[:, :cols] = y
    if half == 1:
        with np.errstate(over="ignore", invalid="ignore"):                 # beyond fp16's range: inf, as __float2half_rn gives
            hi = full.astype(np.float16)
            lo = (full - hi.astype(f32)).astype(f32).astype(np.float16)
        return hi.view(np.uint16), lo.view(np.uint16)
    hi = _bf16(full)
    lo = _bf16((full - _from_bf16(hi)).astype(f32))
    return hi, lo
