"""numpy statements of the skip-gram pair and alias-sampling rules of include/pglb.h, written from the rules:

* ``replay_skipgram(walks, windows)``: the reference's ``skip_gram_gen_pair`` (graph_kernel.pyx:343-365) over a batch of
  walks with the windows given, its per-walk outputs concatenated.
* ``skipgram_windows``: the library's Philox windows, 1 + mulhi32(word0, win_size) of counter (b, i, TAG).
* ``alias_draws``: the library's alias draws; ``alias_distribution``: the distribution a table implies."""
import numpy as np

from .oracle_walk import M32, mulhi64, philox4x32_10, r64

SKIPGRAM_TAG = 0xFFFFFFFF
ALIAS_TAG = 0xFFFFFFFE


def walk_rows(walks):
    """The walks as a list of int64 arrays: rows of a [B, L] array cut at their first entry < 0, or lists as given."""
    if isinstance(walks, np.ndarray) and walks.ndim == 2:
        out = []
        for row in walks.astype(np.int64):
            neg = np.flatnonzero(row < 0)
            out.append(row[:neg[0]] if len(neg) else row)
        return out
    return [np.asarray(w, np.int64).reshape(-1) for w in walks]


def replay_skipgram(walks, windows):
    """(src, pos) int64: centre i of walk b, with window windows[b][i], pairs with every j in [max(0, i - w),
    min(n - 1, i + w)] whose node differs from the centre's, in walk, centre, j order."""
    src, pos = [], []
    for b, walk in enumerate(walk_rows(walks)):
        w = np.asarray(windows[b], np.int64)
        n = len(walk)
        for i in range(n):
            lo, hi = max(0, i - int(w[i])), min(n - 1, i + int(w[i]))
            seg = walk[lo:hi + 1]
            keep = seg[seg != walk[i]]
            src.append(np.full(len(keep), walk[i], np.int64))
            pos.append(keep)
    if not src:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(src), np.concatenate(pos)


def skipgram_windows(B, L, win_size, seed):
    """[B, L] int64: the window of centre i of walk b under the library's rule (defined for every i < L)."""
    b = np.repeat(np.arange(B, dtype=np.uint64), L)
    i = np.tile(np.arange(L, dtype=np.uint64), B)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    d = philox4x32_10(b & M32, b >> np.uint64(32), i, SKIPGRAM_TAG, seed & 0xFFFFFFFF, seed >> 32)
    return (1 + ((d[0] * np.uint64(win_size)) >> np.uint64(32))).astype(np.int64).reshape(B, L)


def alias_draws(alias, events, count, seed):
    """count int64 draws of the table (alias, events) under the library's rule."""
    alias = np.asarray(alias, np.float64)
    events = np.asarray(events, np.int64)
    n = len(alias)
    k = np.arange(count, dtype=np.uint64)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    d = philox4x32_10(k & M32, k >> np.uint64(32), 0, ALIAS_TAG, seed & 0xFFFFFFFF, seed >> 32)
    slot = mulhi64(r64(d), np.full(count, n, np.uint64)).astype(np.int64)
    u = (((d[2] << np.uint64(32)) | d[3]) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    return np.where(u < alias[slot], slot, events[slot])


def alias_distribution(alias, events):
    """P(draw = i) = min(alias[i], 1) / n + sum over j with events[j] = i and alias[j] < 1 of (1 - alias[j]) / n."""
    alias = np.asarray(alias, np.float64)
    events = np.asarray(events, np.int64)
    n = len(alias)
    p = np.minimum(alias, 1.0) / n
    low = alias < 1
    np.add.at(p, events[low], (1.0 - alias[low]) / n)
    return p
