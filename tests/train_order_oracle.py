"""float32 restatement of the summation order of the training kernels (csrc/train.cu, csrc/train_lift.cu): the resize gradient, the
score-map loss, the cross-entropy and the MSE with their gradients, and the launcher policies that fix each order from the shape.

Every operation of these reductions is written __fadd_rn / __fmul_rn / __fdiv_rn / __fsqrt_rn on the device and its order depends on
the shape alone, so numpy float32 (correctly rounded, never contracted) restates each kernel exactly: its results must equal the
device's bit for bit.  The sums here are plain loops over the kernels' steps, vectorised only across sums that are independent on the
device; np.sum, np.dot and np.mean (pairwise or blocked) are never used.  The cross-entropy's per-row values come from numpy's float32
exp and log, which are not CUDA's expf and logf, so that restatement pins the order only.

tests/test_train_order_oracle.py pins these restatements to the fp64 oracles (train_oracle.py, lift_train_oracle.py);
tests/test_gpu_train_paths.py compares the device with them, and tests/test_train_paths_coverage_cpu.py checks its tables with the
policies below."""
import numpy as np

f32 = np.float32
RED_THREADS = 256                 # block size of every fixed-order reduction (kRedThreads, kMseThreads)
SM_K, SM_GROUPS = 21, 12          # score-map partial kernel: thread t = (pixel group t / 21, key-point t % 21)
GRID_CAP = 132 * 32               # grid_for's cap on the blocks of the grid-stride kernels
ADAM_CHUNK, ADAM_BLOCKS, ADAM_MAX_TENSORS = 8192, 132 * 4, 1024
U = 2.0 ** -24


def cdiv(a, b):
    return -(-a // b)


def gamma(k):
    """gamma_k = k u / (1 - k u): a float32 sum through k roundings is within gamma_k sum |x_i| of the exact sum (Higham, Accuracy and
    Stability of Numerical Algorithms, (4.4))"""
    return k * U / (1 - k * U)


def scoremap_bounds(B, HW):
    """Error bounds of the score-map order against fp64, from the longest chains of roundings: (rms relative, loss relative, gradient
    relative to its largest magnitude).  The sum of squares passes the pixel steps, the 12 groups, the chunks and d, d^2; the vis sums
    their laps and the 8 tree levels."""
    nchunk = scoremap_chunks(B, HW)
    k_ss = cdiv(cdiv(HW, nchunk), SM_GROUPS) + SM_GROUPS + nchunk + 2
    k_n = cdiv(B * SM_K, RED_THREADS) + 8
    return gamma(k_ss) / 2 + gamma(2), gamma(k_n + k_ss) + gamma(k_n + 3), gamma(k_ss) + gamma(k_n + 8)


# ---------------------------------------------------------------------------------------------------------------- launcher policies
def grid_for(work, threads):
    """train.cu grid_for: blocks of a grid-stride kernel"""
    return max(1, min(cdiv(work, threads), GRID_CAP))


def scoremap_chunks(B, HW):
    """train.cu scoremap_chunks: pixel chunks per image, about two blocks per SM over the batch, at least 256 pixels each"""
    return max(1, min(cdiv(HW, 256), cdiv(264, B)))


def reduction_blocks(n):
    """xent_blocks / mse_blocks: (blocks, items per block), at most 1024 blocks of at least 2048 items"""
    nblk = max(1, min(cdiv(n, 2048), 1024))
    per = cdiv(n, nblk)
    return cdiv(n, per), per


xent_blocks = mse_blocks = reduction_blocks


def adam_chunk_prefix(numels):
    """adam_step_kernel's first_chunk: the chunk index each tensor starts at, and the total as the last entry"""
    return np.concatenate([[0], np.cumsum([cdiv(int(n), ADAM_CHUNK) for n in numels], dtype=np.int64)]).astype(np.int64)


def adam_chunks_per_block(numels):
    """chunks each of the ADAM_BLOCKS blocks takes (block b takes chunks b, b + ADAM_BLOCKS, ...)"""
    total = int(adam_chunk_prefix(numels)[-1])
    return np.array([len(range(b, total, ADAM_BLOCKS)) for b in range(ADAM_BLOCKS)])


def resize_grad_passes(H, W, oh, ow):
    """launch_resize_bilinear_tf1_grad: the passes it runs, as (name, outputs of the pass); [] is the copy"""
    if (H, W) == (oh, ow):
        return []
    out = []
    if W != ow:
        out.append(("cols", oh * W))
    if H != oh:
        out.append(("rows", H * W))
    return out


# ---------------------------------------------------------------------------------------------------------------- fixed-order sums
def strided_sum(a, threads=RED_THREADS):
    """Per thread t of a block: 0 + a[t] + a[t + threads] + ... over the last axis of a, in index order -> [..., threads]"""
    a = np.asarray(a, f32)
    n = a.shape[-1]
    s = np.zeros(a.shape[:-1] + (threads,), f32)
    for lap in range(cdiv(n, threads)):
        chunk = a[..., lap * threads:(lap + 1) * threads]
        w = chunk.shape[-1]
        s[..., :w] = s[..., :w] + chunk
    return s


def tree(red):
    """The fixed tree over red[..., 0:256): red[t] += red[t + h] for h = 128 ... 1 -> red[..., 0]"""
    red = np.array(red, f32)
    h = red.shape[-1] // 2
    while h > 0:
        red[..., :h] = red[..., :h] + red[..., h:2 * h]
        h //= 2
    return red[..., 0]


def block_sum_fixed(a):
    """train.cu block_sum_fixed over the last axis: strided partials, then the tree"""
    return tree(strided_sum(a))


def blocked_sum(v, n_blocks, per_block):
    """The partial kernels of the cross-entropy and the MSE: block b sums v[b per_block : min(n, (b + 1) per_block)] by its strided
    partials and the tree -> partial [n_blocks]"""
    v = np.asarray(v, f32)
    pad = np.zeros(n_blocks * per_block, f32)
    pad[:v.size] = v
    blocks = pad.reshape(n_blocks, per_block)
    valid = (np.arange(n_blocks * per_block) < v.size).reshape(n_blocks, per_block)
    s = np.zeros((n_blocks, RED_THREADS), f32)
    for lap in range(cdiv(per_block, RED_THREADS)):
        sl = slice(lap * RED_THREADS, (lap + 1) * RED_THREADS)
        w = blocks[:, sl].shape[1]
        s[:, :w] = np.where(valid[:, sl], s[:, :w] + blocks[:, sl], s[:, :w])
    return tree(s)


# ---------------------------------------------------------------------------------------------------------------- resize gradient
def _axis_terms(n_in, n_out):
    """The terms of one transposed 1-D pass in the kernel's order: for each output o ascending, (i0, o, 1 - l) then (i1, o, l), from
    the forward's fp32 operations: scale = f32(n_in) / f32(n_out), in = f32(o) scale, i0 = floor(in), i1 = min(i0 + 1, n_in - 1)"""
    scale = f32(n_in) / f32(n_out)
    terms = []
    for o in range(n_out):
        x = f32(f32(o) * scale)
        i0 = int(np.floor(x))
        i1 = min(i0 + 1, n_in - 1)
        lam = f32(x - f32(i0))
        terms.append((i0, o, f32(f32(1) - lam)))
        terms.append((i1, o, lam))
    return terms


def _pass(g, axis, n_in):
    """One gather pass along `axis` of g (size n_out there) -> size n_in: input i sums g[o] w over its terms, o ascending"""
    g = np.moveaxis(np.asarray(g, f32), axis, 0)
    acc = np.zeros((n_in,) + g.shape[1:], f32)
    for i, o, w in _axis_terms(n_in, g.shape[0]):
        acc[i] = acc[i] + g[o] * w
    return np.moveaxis(acc, 0, axis)


def resize_grad(dy, H, W):
    """launch_resize_bilinear_tf1_grad: dy [B, oh, ow, C] -> dx [B, H, W, C]; columns first, then rows, a dimension that does not
    change skipped, equal sizes a copy"""
    t = np.asarray(dy, f32)
    if t.shape[2] != W:
        t = _pass(t, 2, W)
    if t.shape[1] != H:
        t = _pass(t, 1, H)
    return t.copy()


# ---------------------------------------------------------------------------------------------------------------- score-map loss
def scoremap_partials(P, T):
    """scoremap_sq_partial_kernel: [B, nchunk, 21]; group j of a chunk sums its pixels p0 + j, p0 + j + 12, ... from 0, then the 12
    groups are added in order"""
    B, H, W, K = P.shape
    HW = H * W
    nchunk = scoremap_chunks(B, HW)
    ppc = cdiv(HW, nchunk)
    d = (np.asarray(P, f32) - np.asarray(T, f32)).reshape(B, HW, K)
    sq = np.concatenate([d * d, np.zeros((B, 1, K), f32)], 1)        # pixel HW: a zero for the idle steps
    steps = cdiv(ppc, SM_GROUPS)
    p0 = (np.arange(nchunk) * ppc)[:, None]
    p1 = np.minimum(HW, p0 + ppc)
    s = np.zeros((B, nchunk, SM_GROUPS, K), f32)
    for m in range(steps):
        p = p0 + np.arange(SM_GROUPS)[None, :] + SM_GROUPS * m      # [nchunk, 12]
        p = np.where(p < p1, p, HW)
        s = s + sq[:, p, :]                                          # adding the zero of an idle step is exact (s >= 0)
    r = s[:, :, 0]
    for j in range(1, SM_GROUPS):
        r = r + s[:, :, j]
    return r


def scoremap_loss(P, T, vis):
    """launch_scoremap_loss -> (loss, rms [B, 21]) in the kernels' order"""
    B, H, W, _ = P.shape
    part = scoremap_partials(P, T)
    ss = np.zeros((B, SM_K), f32)
    for c in range(part.shape[1]):
        ss = ss + part[:, c]
    rms = np.sqrt(ss / f32(H * W)).astype(f32)
    vis = np.asarray(vis, f32).reshape(-1)
    num = tree(strided_sum(vis * rms.reshape(-1)))
    S = f32(block_sum_fixed(vis) + f32(0.001))
    return f32(num / S), rms


def scoremap_loss_grad(P, T, vis, rms, g=None):
    """scoremap_loss_grad_kernel: ((g vis) / S) / (f32(HW) rms) (P - T), 0 where rms == 0; g None is 1"""
    B, H, W, K = P.shape
    g = f32(1) if g is None else f32(g)
    vis = np.asarray(vis, f32).reshape(B, K)
    S = f32(block_sum_fixed(vis.reshape(-1)) + f32(0.001))
    rms = np.asarray(rms, f32).reshape(B, K)
    with np.errstate(divide="ignore", invalid="ignore"):
        coef = np.where(rms != 0, ((g * vis) / S) / (f32(H * W) * rms), f32(0)).astype(f32)
    return (coef[:, None, None, :] * (np.asarray(P, f32) - np.asarray(T, f32))).astype(f32)


# ---------------------------------------------------------------------------------------------------------------- cross-entropy
def xent_rows(logits, labels):
    """Per row as xent_row: m = max, e = exp(x - m), s = e0 + e1, loss = l0 (log s - sh0) + l1 (log s - sh1) -> (loss, e0, e1, s)"""
    x, lab = np.asarray(logits, f32).reshape(-1, 2), np.asarray(labels, f32).reshape(-1, 2)
    m = np.maximum(x[:, 0], x[:, 1])
    sh0, sh1 = x[:, 0] - m, x[:, 1] - m
    e0, e1 = np.exp(sh0), np.exp(sh1)
    s = e0 + e1
    ls = np.log(s)
    return lab[:, 0] * (ls - sh0) + lab[:, 1] * (ls - sh1), e0, e1, s


def xent(logits, labels):
    rows_loss = xent_rows(logits, labels)[0]
    n = rows_loss.size
    nblk, per = xent_blocks(n)
    return f32(block_sum_fixed(blocked_sum(rows_loss, nblk, per)) / f32(n))


def xent_grad(logits, labels, g=None):
    """xent_grad_kernel: (g / f32(rows)) (e / s - labels)"""
    lab = np.asarray(labels, f32).reshape(-1, 2)
    _, e0, e1, s = xent_rows(logits, labels)
    scale = f32((f32(1) if g is None else f32(g)) / f32(lab.shape[0]))
    return np.stack([scale * (e0 / s - lab[:, 0]), scale * (e1 / s - lab[:, 1])], 1).astype(f32)


# ---------------------------------------------------------------------------------------------------------------- MSE
def mse(p, q):
    d = np.asarray(p, f32).reshape(-1) - np.asarray(q, f32).reshape(-1)
    n = d.size
    nblk, per = mse_blocks(n)
    return f32(block_sum_fixed(blocked_sum(d * d, nblk, per)) / f32(n))


def mse_grad(p, q, g=None):
    """mse_grad_kernel: (g / f32(n)) (2 (p - q))"""
    p, q = np.asarray(p, f32), np.asarray(q, f32)
    gn = f32((f32(1) if g is None else f32(g)) / f32(p.size))
    return (gn * (f32(2) * (p - q))).astype(f32)
