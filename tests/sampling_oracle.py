"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the nucleus and repetition-aware sampler (include/valle_b200.h
vb_sample_logits_ex), built on the hash of tests/test_sampling_gpu.py.

Every fp32 operation the header specifies is done here in float32 with the same association order, so the kept
nucleus and the draw are the device's bit for bit, except for the elementary functions: the device's expf / logf
and numpy's exp / log may differ in the last bit.  `candidates` therefore returns every id a device may return when
such a last-bit difference decides the draw: a near-tie of the best perturbed scores, or a prefix sum within fp32
rounding of top_p * Z at the nucleus boundary."""
import numpy as np

from test_sampling_gpu import NEAR_TIE, _mix64

RAS_STREAM = 2048   # the fallback draw hashes id i at index i + 2^11
BOUNDARY = 1e-5     # relative distance of a prefix sum to top_p * Z below which expf's last bit may decide the cut
F32 = np.float32


def gumbel(seed, step, idx):
    h = _mix64(seed, step, np.asarray(idx))
    u = ((h >> np.uint64(41)).astype(F32) + F32(0.5)) * F32(2.0 ** -23)
    return (-np.log(-np.log(u))).astype(F32)


def scaled(l, T):
    l = np.asarray(l, dtype=F32)
    return l if T == 1.0 else (l / F32(T)).astype(F32)


def top_k_set(x, k):
    n = x.size
    if 0 < k < n:
        return x >= np.partition(x, n - k)[n - k]
    return np.ones(n, dtype=bool)


def float_key(x):
    u = np.asarray(x, dtype=F32).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, (~u) & 0xFFFFFFFF, u | 0x80000000)


def nucleus(x, keep, top_p):
    """(order, j*, slack): the kept ids in nucleus order, the last position of the nucleus, and the smallest relative
    distance |c_j - top_p Z| / Z at positions j* - 1 and j* (how close expf's rounding is to moving the cut)"""
    idx = np.nonzero(keep)[0]
    order = idx[np.lexsort((idx, -float_key(x[idx]).astype(np.int64)))]
    m = order.size
    xs = x[order]
    e = np.zeros(1280, dtype=F32)
    e[:m] = np.exp((xs - xs[0]).astype(F32)).astype(F32)
    run = np.cumsum(e.reshape(256, 5), axis=1, dtype=F32)           # sequential inside each run of 5
    s = run[:, 4].reshape(8, 32).copy()
    for o in (1, 2, 4, 8, 16):                                       # Hillis-Steele inside each group of 32 runs
        s[:, o:] = (s[:, o:] + s[:, :-o]).astype(F32)
    W = s[:, 31]
    O = np.zeros(8, dtype=F32)
    for w in range(1, 8):
        O[w] = F32(O[w - 1] + W[w - 1])
    Z = F32(O[7] + W[7])
    ex = np.zeros_like(s)
    ex[:, 1:] = s[:, :-1]
    base = (O[:, None] + ex).astype(F32).reshape(256)
    c = (base[:, None] + run).astype(F32).reshape(1280)[:m]
    thr = F32(F32(top_p) * Z)
    hits = np.nonzero(c > thr)[0]
    j = int(hits[0]) if hits.size else m - 1
    near = [abs(float(c[i]) - float(thr)) for i in (j - 1, j) if 0 <= i < m]
    return order, j, min(near) / max(float(Z), 1e-30)


def _gumbel_max(x, keep, g):
    sc = np.where(keep, (x + g).astype(F32), F32(-np.inf)).astype(F32)
    best = int(np.argmax(sc))
    near = set(np.nonzero(keep & (sc >= sc[best] - NEAR_TIE * max(1.0, abs(float(sc[best])))))[0].tolist())
    return best, near


def _first(l, seed, step, k, T, top_p, x):
    """the draw before the RAS check and the ids a last-bit difference may give instead"""
    n = x.size
    if k == 1:
        return int(np.argmax(np.asarray(l, dtype=F32))), set()
    keep = top_k_set(x, k)
    g = gumbel(seed, step, np.arange(n))
    alts = [keep]
    if top_p < 1.0:
        order, j, slack = nucleus(x, keep, top_p)
        cut = np.zeros(n, dtype=bool)
        cut[order[: j + 1]] = True
        alts = [cut]
        if slack < BOUNDARY:
            for jj in (j - 1, j + 1):
                if 0 <= jj < order.size:
                    a = np.zeros(n, dtype=bool)
                    a[order[: jj + 1]] = True
                    alts.append(a)
    d, near = _gumbel_max(x, alts[0], g)
    for a in alts[1:]:
        near |= _gumbel_max(x, a, g)[1]
    near.discard(d)
    return d, near


def _ras(d, x, seed, step, window, ras_max, hist):
    if window <= 0:
        return d, set()
    lo = max(0, step - window)
    c = int(np.count_nonzero(np.asarray(hist[lo:step]) == d))
    if c <= ras_max:
        return d, set()
    g = gumbel(seed, step, np.arange(x.size) + RAS_STREAM)
    f, near = _gumbel_max(x, np.ones(x.size, dtype=bool), g)
    near.discard(f)
    return f, near


def draw(l, seed, step, k, T, top_p=1.0, window=0, ras_max=0, hist=()):
    """the id vb_sample_logits_ex returns for one row"""
    return candidates(l, seed, step, k, T, top_p, window, ras_max, hist)[0]


def candidates(l, seed, step, k, T, top_p=1.0, window=0, ras_max=0, hist=()):
    """(id, others): the restated id and the set of ids a device whose expf / logf differ from numpy's in the last bit
    may return instead"""
    x = scaled(l, T)
    d, near = _first(l, seed, step, k, T, top_p, x)
    out, others = _ras(d, x, seed, step, window, ras_max, hist)
    for a in near:                       # a near-tie of the first draw goes through the RAS check on its own
        others |= {_ras(a, x, seed, step, window, ras_max, hist)[0]}
    others.discard(out)
    return out, others


def ras_fallback(d, step, window, ras_max, hist):
    """whether the RAS check replaces the draw d"""
    lo = max(0, step - window)
    return window > 0 and int(np.count_nonzero(np.asarray(hist[lo:step]) == d)) > ras_max
