"""Generate tests/golden/ref_skipgram.npz, and nothing else.

Run in the build container (where /root/reference exists):  python tests/golden/make_skipgram_golden.py

Outputs of the REFERENCE's compiled ``pgl.graph_kernel`` (built by oracle/build.py into oracle/_ref/),
``skip_gram_gen_pair`` and ``alias_sample_build_table`` (pgl/graph_kernel.pyx:343-393):
(a) ``skip_gram_gen_pair`` with its windows injected by replacing ``numpy.random.randint`` for the call (the compiled
    module looks ``np.random.randint`` up at call time, so the replacement reaches it);
(b) a sequence of unpatched calls after ``np.random.seed``;
(c) ``alias_sample_build_table`` on n = 1, uniform n = 7, one-hot, zeros and ties, Dirichlet draws and the normalised
    ``outdegree^0.75`` of a 10^5-node power-law graph.
Each group is stored as flat arrays with ``<name>_off`` offsets (tests/test_skipgram_host.py reads them).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import power_law_edges  # noqa: E402
from oracle import build as obuild  # noqa: E402


def skipgram_walks(rng):
    """The walks of fixture (a): lengths 0, 1, 2, 40 and 130, with revisited nodes and runs of one node (self-loops)."""
    walks = [[], [7], [3, 3], [3, 9]]
    walks.append(rng.integers(0, 1000, 40).tolist())             # mostly distinct
    walks.append(rng.integers(0, 6, 40).tolist())                # many revisits
    w = rng.integers(0, 50, 130)
    w[10:20] = 4                                                # a self-loop run
    w[60:63] = w[59]
    walks.append(w.tolist())
    walks.append([5] * 40)                                      # one node throughout: no pairs
    walks.append(np.tile([1, 2], 65).tolist())                  # 130 nodes, two ids alternating
    return walks


def _flat(out, name, arrays):
    """A list of 1-D arrays as one flat array and its offsets."""
    out[name] = np.concatenate([np.asarray(a).reshape(-1) for a in arrays]) if arrays else np.zeros(0)
    out[name + "_off"] = np.concatenate([[0], np.cumsum([len(a) for a in arrays])]).astype(np.int64)


def ref_skipgram(gk):
    rng = np.random.default_rng(17)
    out = {}
    # (a) injected windows
    walks, wins, windows, srcs, poss = [], [], [], [], []
    real_randint = np.random.randint
    try:
        for walk in skipgram_walks(rng):
            for win_size in (1, 3, 10, 200):
                win = rng.integers(1, win_size + 1, len(walk)).astype(np.int64)
                np.random.randint = lambda lo, hi, dtype=None, size=None, _w=win: _w.copy()
                s, p = gk.skip_gram_gen_pair(list(walk), win_size)
                walks.append(np.asarray(walk, np.int64))
                wins.append(win_size)
                windows.append(win)
                srcs.append(np.asarray(s, np.int64))
                poss.append(np.asarray(p, np.int64))
    finally:
        np.random.randint = real_randint
    _flat(out, "a_walk", walks)
    _flat(out, "a_window", windows)
    _flat(out, "a_src", srcs)
    _flat(out, "a_pos", poss)
    out["a_win_size"] = np.asarray(wins, np.int64)
    # (b) unpatched: np.random.seed(s), then skip_gram_gen_pair walk after walk
    walks, wins, srcs, poss = [], [], [], []
    seed = 2024
    np.random.seed(seed)
    for k in range(24):
        walk = rng.integers(0, 30, int(rng.integers(0, 50))).tolist()
        win_size = (1, 3, 5, 10)[k % 4]
        s, p = gk.skip_gram_gen_pair(walk, win_size)
        walks.append(np.asarray(walk, np.int64))
        wins.append(win_size)
        srcs.append(np.asarray(s, np.int64))
        poss.append(np.asarray(p, np.int64))
    _flat(out, "b_walk", walks)
    _flat(out, "b_src", srcs)
    _flat(out, "b_pos", poss)
    out["b_win_size"] = np.asarray(wins, np.int64)
    out["b_seed"] = np.int64(seed)
    # (c) alias tables
    probs = [np.array([1.0]), np.full(7, 1.0 / 7), np.eye(1, 10, 3)[0],
             np.array([0.0, 0.25, 0.0, 0.25, 0.25, 0.25]), np.array([0.1, 0.2, 0.2, 0.2, 0.3, 0.0])]
    for k, alpha in ((5, 1.0), (100, 1.0), (1000, 0.1), (3000, 0.5)):
        probs.append(rng.dirichlet(np.full(k, alpha)))
    src, _ = power_law_edges(100000, 1000000, 23)
    deg = np.bincount(src, minlength=100000).astype(np.float64)
    pw = deg ** 0.75
    probs.append(pw / pw.sum())
    alias, events = [], []
    for p in probs:
        a, e = gk.alias_sample_build_table(np.ascontiguousarray(p, np.float64))
        alias.append(np.asarray(a))
        events.append(np.asarray(e))
    _flat(out, "c_probs", probs)
    _flat(out, "c_alias", alias)
    _flat(out, "c_events", events)
    return out


def main():
    gk = obuild.load_ref_graph_kernel()
    if gk is None:
        obuild.build_ref()
        gk = obuild.load_ref_graph_kernel()
    if gk is None:
        raise SystemExit("make_skipgram_golden.py: the reference's graph_kernel could not be built "
                         "(set PGL_REFERENCE, install Cython)")
    np.savez_compressed(os.path.join(HERE, "ref_skipgram.npz"), **ref_skipgram(gk))
    print("ref_skipgram.npz written to", HERE)


if __name__ == "__main__":
    main()
