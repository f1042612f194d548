"""The two ``pgl.graph_kernel`` functions the reference's walk examples import (examples/deepwalk, node2vec,
metapath2vec, graph_based_clustering_demo; apps/Graph4Rec), with the reference's contracts (graph_kernel.pyx:343-393):

* ``skip_gram_gen_pair(walk, win_size=5)``: the skip-gram pairs of one walk, two lists.  The windows are drawn by the
  reference's own call, ``np.random.randint(1, win_size + 1, dtype=np.int64, size=len(walk))``, so under the same
  ``np.random`` state the output is the reference's.  numpy on the host.
* ``alias_sample_build_table(probs)``: the reference's alias table of ``probs`` as given (no normalisation), built by
  ``pglb_alias_build_host``, bit for bit.

No other ``graph_kernel`` function is provided.  For whole batches of walks on the device, use
``pgl.sampling.skip_gram_pairs``, ``alias_table`` and ``alias_sample``."""
import ctypes

import numpy as np

from ._lib import check, lib

__all__ = ["skip_gram_gen_pair", "alias_sample_build_table"]

_CHUNK = 1 << 20   # candidate (centre, offset) cells per vectorised step


def skip_gram_gen_pair(walk, win_size=5):
    """(src, pos) lists: centre i, with window rnd[i] drawn uniformly from [1, win_size], pairs with every j in
    [max(0, i - rnd[i]), min(len(walk) - 1, i + rnd[i])] ascending whose node differs from walk[i]."""
    walk = np.asarray(walk, dtype=np.int64).reshape(-1)
    n = len(walk)
    rnd = np.random.randint(1, win_size + 1, dtype=np.int64, size=n)
    if n == 0:
        return [], []
    D = int(min(win_size, n - 1))
    d = np.arange(-D, D + 1, dtype=np.int64)
    step = max(1, _CHUNK // len(d))
    src, pos = [], []
    for i0 in range(0, n, step):
        i = np.arange(i0, min(n, i0 + step), dtype=np.int64)
        j = i[:, None] + d[None, :]
        ok = (np.abs(d)[None, :] <= rnd[i][:, None]) & (j >= 0) & (j < n)
        jc = np.clip(j, 0, n - 1)
        ok &= walk[jc] != walk[i][:, None]
        src.append(np.broadcast_to(walk[i][:, None], j.shape)[ok])
        pos.append(walk[jc][ok])
    return np.concatenate(src).tolist(), np.concatenate(pos).tolist()


def alias_sample_build_table(probs):
    """(alias float64, events int64) of the 1-D float64 probs, used as given."""
    probs = np.ascontiguousarray(probs, dtype=np.float64)
    if probs.ndim != 1:
        raise ValueError("probs must be 1-D, got shape %s" % (probs.shape,))
    n = len(probs)
    alias = np.empty(n, np.float64)
    events = np.empty(n, np.int64)
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    check(lib.pglb_alias_build_host(ptr(probs), n, ptr(alias), ptr(events)))
    return alias, events
