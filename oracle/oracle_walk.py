"""Two independent numpy statements of the random walks of pgl.sampling (reference pgl/sampling/walk.py:23-183,
graph_kernel.pyx:142-224), written from the rules, not from either implementation:

1. ``replay``: the library's sampling rule (include/pglb.h, csrc/walk.cu) draw for draw -- the same Philox4x32-10
   counters, multiply-high slots, integer acceptance thresholds, trial cap and float64 inverse-CDF fallback -- so it
   matches the kernels and ``pglb_walk_host`` bit for bit.  Membership is a Python set of the successor ids, not a
   binary search in a sorted copy.
2. ``transition_probs``: the exact next-slot distribution of the reference's rules, for goodness-of-fit tests.

The graph is the src-keyed CSR: row u = cols[indptr[u]:indptr[u + 1]], in any order.  Modes: 0 random_walk,
1 node2vec_walk, 2 node2vec_walk_plus (1 and 2 take up to max_depth steps, 0 up to max_depth - 1)."""
import math

import numpy as np

M32 = np.uint64(0xFFFFFFFF)
TRIALS = 16  # a node2vec step takes the exact fallback after max(TRIALS, deg) rejected trials
UNIFORM, NODE2VEC, NODE2VEC_PLUS = 0, 1, 2


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 (Salmon et al., SC 2011) over uint64 arrays holding 32-bit values."""
    c0, c1, c2, c3 = (np.asarray(c, np.uint64) & M32 for c in (c0, c1, c2, c3))
    k0, k1 = np.uint64(k0), np.uint64(k1)
    m0, m1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(0x9E3779B9)) & M32
            k1 = (k1 + np.uint64(0xBB67AE85)) & M32
        p0, p1 = m0 * c0, m1 * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
    return c0, c1, c2, c3


def draw(seed, walkers, step, trial):
    """The four words of (walker, step, trial) for an array of walker indices."""
    w = np.asarray(walkers, np.uint64)
    s = np.full(w.shape, step, np.uint64)
    k = np.full(w.shape, trial, np.uint64)
    return philox4x32_10(w & M32, w >> np.uint64(32), s, k, seed & 0xFFFFFFFF, seed >> 32)


def r64(words):
    return (words[1] << np.uint64(32)) | words[0]


def mulhi64(r, d):
    """floor(r * d / 2^64) for uint64 r and 0 < d < 2^32 (arrays of the same shape)."""
    d = np.asarray(d, np.uint64)
    assert ((d > 0) & (d < np.uint64(2 ** 32))).all()
    hi, lo = r >> np.uint64(32), r & M32
    return (hi * d + ((lo * d) >> np.uint64(32))) >> np.uint64(32)


def thresholds(p, q):
    """(weights, thresholds) of the classes return / near / far: w = 1/p, 1, 1/q; thr = floor(w / w_max * 2^32)."""
    w = (1.0 / p, 1.0, 1.0 / q)
    wmax = max(w)
    return w, tuple(int(math.floor(x / wmax * 4294967296.0)) for x in w)


class _Succ(object):
    def __init__(self, indptr, cols):
        self.indptr, self.cols, self.sets = indptr, cols, {}

    def __call__(self, u):
        s = self.sets.get(u)
        if s is None:
            s = self.sets[u] = set(self.cols[self.indptr[u]:self.indptr[u + 1]].tolist())
        return s


def replay(indptr, cols, nodes, max_depth, mode, seed, p=1.0, q=1.0):
    """(out [n, L] int64 padded with -1, trials, fallbacks) of the library's rule."""
    indptr = np.asarray(indptr, np.int64)
    cols = np.asarray(cols, np.int64)
    nodes = np.asarray(nodes, np.int64).reshape(-1)
    num_nodes = len(indptr) - 1
    n = len(nodes)
    steps, L = (max_depth - 1, max_depth) if mode == UNIFORM else (max_depth, max_depth + 1)
    w, thr = thresholds(p, q)
    succ = _Succ(indptr, cols)
    out = np.full((n, L), -1, np.int64)
    hist = [[int(v)] if 0 <= v < num_nodes else [] for v in nodes]
    near = [set() for _ in range(n)]  # node2vec_plus: successors of v_0 .. v_{t-1}
    alive = np.array([len(h) > 0 for h in hist])
    trials = fallbacks = 0
    for t in range(steps):
        act = [i for i in np.flatnonzero(alive) if indptr[hist[i][-1] + 1] > indptr[hist[i][-1]]]
        alive[:] = False
        if not act:
            break
        alive[act] = True
        ntr = 1 if (mode == UNIFORM or t == 0) else TRIALS
        words = [draw(seed, act, t, k) for k in range(ntr)]   # the first trials of every walker, batched
        rs = [r64(wd) for wd in words]
        degs = np.array([indptr[hist[i][-1] + 1] - indptr[hist[i][-1]] for i in act], np.uint64)
        slots = [mulhi64(r, degs) for r in rs]
        for j, i in enumerate(act):
            h = hist[i]
            cur = h[-1]
            b, d = int(indptr[cur]), int(indptr[cur + 1] - indptr[cur])
            if ntr == 1:
                x = int(cols[b + int(slots[0][j])])
                trials += 1
            else:
                prev = h[-2]
                nb = succ(prev) if mode == NODE2VEC else near[i]

                def cls(y):
                    return 0 if y == prev else (1 if y in nb else 2)
                x = None
                cap = max(TRIALS, d)
                for k in range(cap):
                    if k < TRIALS:
                        y, acc_word = int(cols[b + int(slots[k][j])]), int(words[k][2][j])
                    else:
                        wk = draw(seed, [i], t, k)
                        y, acc_word = int(cols[b + int(mulhi64(r64(wk), [d])[0])]), int(wk[2][0])
                    trials += 1
                    if acc_word < thr[cls(y)]:
                        x = y
                        break
                if x is None:
                    fallbacks += 1
                    row = cols[b:b + d].tolist()
                    W = 0.0
                    for y in row:
                        W += w[cls(y)]
                    u = float(int(r64(draw(seed, [i], t, cap))[0]) >> 11) * 2.0 ** -53
                    target = u * W
                    acc = 0.0
                    for y in row:
                        x = y
                        acc += w[cls(y)]
                        if target < acc:
                            break
            if mode == NODE2VEC_PLUS:
                near[i] |= succ(cur)
            h.append(x)
    for i, h in enumerate(hist):
        out[i, :len(h)] = h
    return out, trials, fallbacks


def as_lists(out):
    """The reference's return value: one list of node ids per walker, without the -1 padding."""
    return [[v for v in row if v >= 0] for row in np.asarray(out).tolist()]


def transition_probs(indptr, cols, walk, mode, p=1.0, q=1.0):
    """Exact P(next slot = s), s over the row of walk[-1], given the walk so far (v_0 .. v_t), under the reference's
    rule: uniform for random_walk and for a first step; otherwise proportional to 1/p (the slot holds v_{t-1}),
    1 (it holds a successor of v_{t-1}; node2vec_plus: of any of v_0 .. v_{t-1}), 1/q (otherwise)."""
    indptr = np.asarray(indptr, np.int64)
    cols = np.asarray(cols, np.int64)
    cur = walk[-1]
    row = cols[indptr[cur]:indptr[cur + 1]]
    if mode == UNIFORM or len(walk) == 1:
        return np.full(len(row), 1.0 / len(row))
    prev = walk[-2]
    earlier = [prev] if mode == NODE2VEC else walk[:-1]
    nb = set()
    for u in earlier:
        nb |= set(cols[indptr[u]:indptr[u + 1]].tolist())
    wt = np.array([1.0 / p if y == prev else (1.0 if y in nb else 1.0 / q) for y in row.tolist()])
    return wt / wt.sum()


def node_probs(indptr, cols, walk, mode, p=1.0, q=1.0):
    """transition_probs summed over the slots that hold the same node: {node: probability}."""
    cur = walk[-1]
    row = np.asarray(cols)[indptr[cur]:indptr[cur + 1]].tolist()
    out = {}
    for y, pr in zip(row, transition_probs(indptr, cols, walk, mode, p, q)):
        out[y] = out.get(y, 0.0) + pr
    return out
