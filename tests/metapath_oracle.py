"""A numpy statement of the metapath walk rule (include/pglb.h, pgl_b200.sampling.metapath_randomwalk), written from
the rule on oracle/oracle_walk.py's Philox draw, and the test graphs the host and device tests share.

The rule: walker i starts at nodes[i]; step t (t = 0, 1, ...) goes from cur to the uniform slot of cur's row in
relation metapath[t % M], slot = mulhi64(r64(draw(seed, i, t, 0)), deg); a walk has at most walk_length nodes and ends
early exactly when cur has no out-edge in the step's relation.  A relation is a src-keyed CSR (indptr, cols)."""
import json
import os

import numpy as np

from oracle import oracle_walk as W

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def replay_metapath(csrs, nodes, metapath_idx, walk_length, seed):
    """[n, walk_length] int64 walks padded with -1.  csrs: list of (indptr, cols) per relation; metapath_idx: the
    relation index of every metapath position."""
    nodes = np.asarray(nodes, np.int64).reshape(-1)
    num_nodes = len(csrs[0][0]) - 1
    out = np.full((len(nodes), walk_length), -1, np.int64)
    ok = (nodes >= 0) & (nodes < num_nodes)
    out[ok, 0] = nodes[ok]
    act, cur = np.flatnonzero(ok), nodes[ok]
    for t in range(walk_length - 1):
        indptr, cols = csrs[metapath_idx[t % len(metapath_idx)]]
        b = np.asarray(indptr, np.int64)[cur]
        deg = np.asarray(indptr, np.int64)[cur + 1] - b
        live = deg > 0
        act, b, deg = act[live], b[live], deg[live]
        if not len(act):
            break
        slot = W.mulhi64(W.r64(W.draw(seed, act, t, 0)), deg.astype(np.uint64)).astype(np.int64)
        cur = np.asarray(cols, np.int64)[b + slot]
        out[act, t + 1] = cur
    return out


def step_probs(csrs, metapath_idx, t, cur):
    """Exact {next node: probability} of step t from cur: the slot counts of cur's row in relation metapath[t % M]
    over its degree (cur must have an out-edge there)."""
    indptr, cols = csrs[metapath_idx[t % len(metapath_idx)]]
    return W.node_probs(indptr, cols, [cur], W.UNIFORM)


def position_probs(csrs, metapath_idx, start, k):
    """Exact {node: probability} of v_k of a walk from start, with key -1 for the walks that ended before step k."""
    dist = {start: 1.0}
    for t in range(k):
        indptr, _ = csrs[metapath_idx[t % len(metapath_idx)]]
        nxt = {}
        for u, p in dist.items():
            if u < 0 or indptr[u + 1] == indptr[u]:
                nxt[-1] = nxt.get(-1, 0.0) + p
                continue
            for y, q in step_probs(csrs, metapath_idx, t, u).items():
                nxt[y] = nxt.get(y, 0.0) + p * q
        dist = nxt
    return dist


def csr(edges, n):
    """src-keyed CSR in edge-id order inside each row (adj_src_index)."""
    e = np.asarray(edges, np.int64).reshape(-1, 2)
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(e[:, 0], minlength=n), out=indptr[1:])
    return indptr, e[np.argsort(e[:, 0], kind="stable"), 1]


def kat_graph():
    """The reference's c / p / a graph (tests/test_hetergraph.py): (edges dict, num_nodes, node_types)."""
    with open(os.path.join(GOLDEN, "kat_hetergraph.json")) as f:
        k = json.load(f)
    edges = {e: np.array(v, np.int64).reshape(-1, 2) for e, v in k["edges"].items()}
    return edges, k["num_nodes"], np.array(k["node_types"])


def typed_graph(seed=7):
    """Six relations over 600 nodes: r0 random with sinks, self-loops and multi-edges; r1 with a hub (node 0) of 10^4
    out-edges; r2 without edges; r3 a sparse random relation; r4 and r5 random with two out-edges per node (no sinks,
    so walks over them run their whole length).  Returns (edges dict, num_nodes, start nodes)."""
    rng = np.random.default_rng(seed)
    n = 600
    r0 = np.stack([rng.integers(0, n // 2, 1500), rng.integers(0, n, 1500)], 1)   # nodes >= 300 are r0 sinks
    r0 = np.concatenate([r0, r0[:200], np.stack([np.arange(0, 40), np.arange(0, 40)], 1)])   # repeats, self-loops
    hub = np.stack([np.zeros(10000, np.int64), rng.integers(1, n, 10000)], 1)
    r1 = np.concatenate([hub, np.stack([rng.integers(1, n, 800), rng.integers(0, n, 800)], 1),
                         np.stack([rng.integers(1, n, 100), np.zeros(100, np.int64)], 1)])
    r3 = np.stack([rng.integers(0, n, 300), rng.integers(0, n, 300)], 1)
    r4, r5 = (np.stack([np.repeat(np.arange(n), 2), rng.integers(0, n, 2 * n)], 1) for _ in range(2))
    edges = {"r0": r0, "r1": r1, "r2": np.zeros((0, 2), np.int64), "r3": r3, "r4": r4, "r5": r5}
    nodes = np.r_[[0] * 30, rng.integers(0, n, 270)]
    return edges, n, nodes
