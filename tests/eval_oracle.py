"""numpy restatement of what h3d_eval_stats computes per key-point (csrc/eval.cu): np.mean's pairwise summation, np.median and the
threshold counts, written out step by step so that each can be tested against numpy itself and the device against it."""
import numpy as np

from hand3d_b200 import _lib


def _leaf(a):
    t = a.dtype.type
    n = len(a)
    if n < 8:
        r = t(-0.0)
        for x in a:
            r = t(r + x)
        return r
    r = a[:8].copy()
    i = 8
    while i < n - n % 8:
        r += a[i:i + 8]                  # accumulator j gets a[i + j], each add rounded in the array's dtype
        i += 8
    res = t(t(t(r[0] + r[1]) + t(r[2] + r[3])) + t(t(r[4] + r[5]) + t(r[6] + r[7])))
    while i < n:
        res = t(res + a[i])
        i += 1
    return res


def pairwise_sum(a):
    """numpy 2.x pairwise_sum: blocks of at most 128 values with 8 accumulators, split at n/2 - (n/2) % 8 above that."""
    n = len(a)
    if n <= 128:
        return _leaf(a)
    h = n // 2
    h -= h % 8
    return a.dtype.type(pairwise_sum(a[:h]) + pairwise_sum(a[h:]))


def mean(a):
    t = a.dtype.type
    return t(pairwise_sum(a) / t(len(a)))


def median(a):
    t = a.dtype.type
    if np.isnan(a).any():
        return t(np.nan)
    s = np.sort(a)
    n = len(a)
    if n % 2:
        return s[n // 2]
    return t(t(s[n // 2 - 1] + s[n // 2]) / t(2))


def counts(a, thresholds):
    d = a.astype(np.float64)
    return np.array([np.count_nonzero(d <= t) for t in thresholds], np.int64)


def frontier_nodes(n, split=384, leaf=128):
    """Number of subtrees the device cuts pairwise_sum's recursion into (nodes of length <= max(128, ceil(n / split)))."""
    F = max(leaf, -(-n // split))
    stack, count = [n], 0
    while stack:
        L = stack.pop()
        if L <= F:
            count += 1
        else:
            h = L // 2
            h -= h % 8
            stack += [h, L - h]
    return count


def stats(lists, thresholds):
    """The int64 rows h3d_eval_stats writes for these per-key-point lists."""
    out = np.zeros((len(lists), _lib.EVAL_STAT_COUNTS + len(thresholds)), np.int64)
    for k, a in enumerate(lists):
        a = np.asarray(a)
        if len(a) == 0:
            continue
        out[k, _lib.EVAL_STAT_N] = len(a)
        out[k, _lib.EVAL_STAT_MEAN] = np.float64(mean(a)).view(np.int64)
        out[k, _lib.EVAL_STAT_MEDIAN] = np.float64(median(a)).view(np.int64)
        out[k, _lib.EVAL_STAT_COUNTS:] = counts(a, thresholds)
    return out


def feed_lists(gt, vis, pred):
    """The reference's EvalUtil.feed over samples [n, K, D] / [n, K]: per-key-point lists of np.sqrt(np.sum(np.square(gt - pred), axis=1))
    of each sample, in sample order (the sum over D <= 4 coordinates is sequential in both forms)."""
    d = np.sqrt(np.sum(np.square(gt - pred), axis=2))
    v = np.asarray(vis).astype('bool')
    return [d[v[:, k], k] for k in range(d.shape[1])]
