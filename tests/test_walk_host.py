"""Random walks without a GPU: the library's host entry (the kernels' own step function) against the numpy replay of
oracle/oracle_walk.py bit for bit, the replay's transitions against the exact probabilities of the reference's rules,
walk lengths on the reference's test_sample.py shapes, and the argument checks of the Python layer and the C ABI."""
import ctypes

import numpy as np
import pytest
from scipy import stats

from oracle import oracle_walk as W

EINVAL = -1


@pytest.fixture(scope="module")
def lib():
    from pgl_b200 import _lib
    return _lib


def csr(edges, n):
    """src-keyed CSR in edge-id order inside each row (adj_src_index), and its row-sorted copy."""
    e = np.asarray(edges, np.int64).reshape(-1, 2)
    order = np.argsort(e[:, 0], kind="stable")
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(e[:, 0], minlength=n), out=indptr[1:])
    cols = e[order, 1]
    srt = e[np.lexsort((e[:, 1], e[:, 0])), 1]
    return indptr, cols, srt


def host_walk(lib, g, nodes, max_depth, mode, seed, p=1.0, q=1.0):
    indptr, cols, srt = g
    nodes = np.ascontiguousarray(nodes, np.int64)
    L = max_depth if mode == W.UNIFORM else max_depth + 1
    out = np.full((len(nodes), L), 7, np.int64)
    st = np.zeros(2, np.uint64)
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = lib.lib.pglb_walk_host(ptr(indptr), ptr(cols), ptr(srt), len(indptr) - 1, ptr(nodes), len(nodes), max_depth,
                                p, q, mode, seed, ptr(out), ptr(st))
    assert rc == 0, lib.lib.pglb_last_error()
    return out, int(st[0]), int(st[1])


def small_graph():
    """sinks (5, 6), self-loops (0, 4), multi-edges (0 -> 1 twice, 2 -> 3 three times), a node with no edges at all (6)"""
    edges = [(0, 1), (0, 1), (0, 0), (1, 2), (2, 0), (2, 3), (3, 4), (1, 0), (4, 4), (0, 2), (2, 3), (2, 3), (3, 5),
             (4, 2), (1, 5), (7, 0), (7, 2)]
    return csr(edges, 8), [0, 0, 1, 2, 3, 4, 5, 6, 7, 7, 2]


def hub_graph(seed=3):
    """node 0 has 10^4 out-edges (with repeats) into 300 nodes, whose rows are short and often return to the hub"""
    rng = np.random.default_rng(seed)
    n = 300
    hub = np.stack([np.zeros(10000, np.int64), rng.integers(1, n, 10000)], 1)
    rest = np.stack([rng.integers(1, n, 1500), rng.integers(0, n, 1500)], 1)
    back = np.stack([rng.integers(1, n, 200), np.zeros(200, np.int64)], 1)
    return csr(np.concatenate([hub, rest, back]), n + 5), np.r_[[0] * 40, rng.integers(0, n + 5, 120)]


def random_graph(seed=5):
    rng = np.random.default_rng(seed)
    n = 400
    e = np.stack([rng.integers(0, n, 2500), rng.integers(0, n, 2500)], 1)
    e = np.concatenate([e, e[:300]])  # duplicates
    return csr(e, n), rng.integers(0, n, 300)


GRAPHS = {"small": small_graph, "hub": hub_graph, "random": random_graph}
PQ = [(0.25, 4.0), (4.0, 0.25), (1e-3, 1.0), (2.0, 0.5)]


@pytest.mark.parametrize("name", sorted(GRAPHS))
@pytest.mark.parametrize("mode", [W.UNIFORM, W.NODE2VEC, W.NODE2VEC_PLUS])
def test_host_entry_is_the_replay(lib, name, mode):
    g, nodes = GRAPHS[name]()
    fallbacks = 0
    for seed in (0, 0x0123456789ABCDEF, 2 ** 64 - 1):
        for p, q in (PQ if mode != W.UNIFORM else [(1.0, 1.0)]):
            got, tr, fb = host_walk(lib, g, nodes, 6, mode, seed, p, q)
            want, wtr, wfb = W.replay(g[0], g[1], nodes, 6, mode, seed, p, q)
            assert np.array_equal(got, want), (seed, p, q)
            assert (tr, fb) == (wtr, wfb)
            fallbacks += fb
    if mode != W.UNIFORM:
        assert fallbacks > 0   # p = 1e-3 reaches the exact fallback


def test_walks_are_paths_and_end_at_sinks(lib):
    g, nodes = small_graph()
    indptr, cols, _ = g
    edges = {(u, int(v)) for u in range(len(indptr) - 1) for v in cols[indptr[u]:indptr[u + 1]]}
    for mode in (W.UNIFORM, W.NODE2VEC, W.NODE2VEC_PLUS):
        out, _, _ = host_walk(lib, g, nodes, 8, mode, 11, 0.5, 2.0)
        for start, row in zip(nodes, W.as_lists(out)):
            assert row[0] == start
            assert all((a, b) in edges for a, b in zip(row, row[1:]))
            if len(row) < out.shape[1]:   # a walk stops early only at a node without successors
                assert indptr[row[-1] + 1] == indptr[row[-1]]


def test_start_outside_the_graph_gives_an_empty_row(lib):
    g, _ = small_graph()
    out, _, _ = host_walk(lib, g, [-1, 8, 0], 4, W.NODE2VEC, 1, 0.5, 2.0)
    assert (out[:2] == -1).all() and out[2, 0] == 0


def test_seed_and_walker_index_decide_the_walk(lib):
    g, nodes = random_graph()
    a = host_walk(lib, g, nodes, 10, W.NODE2VEC, 42, 0.5, 2.0)[0]
    assert np.array_equal(a, host_walk(lib, g, nodes, 10, W.NODE2VEC, 42, 0.5, 2.0)[0])
    assert not np.array_equal(a, host_walk(lib, g, nodes, 10, W.NODE2VEC, 43, 0.5, 2.0)[0])
    # a node2vec walk's first step is the random_walk draw of the same walker
    u = host_walk(lib, g, nodes, 10, W.UNIFORM, 42)[0]
    assert np.array_equal(a[:, :2], u[:, :2])


def _chi2(samples, probs):
    keys = sorted(probs)
    obs = np.array([np.sum(samples == k) for k in keys], np.float64)
    assert obs.sum() == len(samples)
    exp = np.array([probs[k] for k in keys]) * len(samples)
    return stats.chisquare(obs, exp).pvalue


def test_first_order_transitions_are_uniform_over_slots():
    g = csr([(0, 1), (0, 2), (0, 2), (0, 3), (0, 0), (0, 4), (0, 4), (0, 4)], 5)
    out, _, _ = W.replay(g[0], g[1], np.zeros(40000, np.int64), 2, W.UNIFORM, 7)
    probs = W.node_probs(g[0], g[1], [0], W.UNIFORM)
    assert probs == {0: 1 / 8, 1: 1 / 8, 2: 2 / 8, 3: 1 / 8, 4: 3 / 8}
    assert _chi2(out[:, 1], probs) > 1e-3


@pytest.mark.parametrize("p,q", [(0.5, 2.0), (2.0, 0.5), (1e-3, 1.0)])
def test_second_order_ratios(p, q):
    """0 -> {1, 2, 3}; the step from 1 after 0 has return 0, near {2, 3} (successors of 0), far {4, 5, 6}:
    probabilities 1/p : 1 : 1/q per slot."""
    g = csr([(0, 1), (0, 2), (0, 3), (1, 0), (1, 2), (1, 3), (1, 4), (1, 5), (1, 6), (1, 6)], 7)
    out, _, fb = W.replay(g[0], g[1], np.zeros(60000, np.int64), 2, W.NODE2VEC, 99, p, q)
    sel = out[out[:, 1] == 1]
    probs = W.node_probs(g[0], g[1], [0, 1], W.NODE2VEC, p, q)
    w = np.array([1 / p, 1, 1, 1 / q, 1 / q, 2 / q])
    assert np.allclose([probs[k] for k in (0, 2, 3, 4, 5, 6)], w / w.sum())
    assert _chi2(sel[:, 2], probs) > 1e-3
    if p == 1e-3:
        assert fb > 0


def test_plus_rule_uses_the_union_of_earlier_successors():
    """Walks that begin 0, 1, 2: the step from 2 has return 1, near {5, 6} under node2vec_plus (successors of 0 and
    of 1) but only {6} under node2vec, far {7, 8}."""
    g = csr([(0, 1), (0, 5), (1, 2), (1, 6), (2, 1), (2, 5), (2, 6), (2, 7), (2, 8), (5, 0), (6, 0), (7, 0), (8, 0)],
            9)
    p, q = 0.5, 4.0
    plus = W.node_probs(g[0], g[1], [0, 1, 2], W.NODE2VEC_PLUS, p, q)
    n2v = W.node_probs(g[0], g[1], [0, 1, 2], W.NODE2VEC, p, q)
    w = np.array([1 / p, 1, 1, 1 / q, 1 / q])
    assert np.allclose([plus[k] for k in (1, 5, 6, 7, 8)], w / w.sum())
    assert plus[5] > n2v[5]
    for mode, probs in ((W.NODE2VEC_PLUS, plus), (W.NODE2VEC, n2v)):
        out, _, _ = W.replay(g[0], g[1], np.zeros(80000, np.int64), 3, mode, 5, p, q)
        sel = out[(out[:, 1] == 1) & (out[:, 2] == 2)]
        assert len(sel) > 15000
        assert _chi2(sel[:, 3], probs) > 1e-3


def test_reference_test_sample_shapes(lib):
    """The graph and calls of the reference's tests/test_sample.py: no node is a sink, so every walk has its full
    length -- max_depth nodes for random_walk and for node2vec with p = q = 1, max_depth + 1 otherwise."""
    from pgl_b200.sampling.walk import walk_mode
    edges = [(0, 1), (1, 2), (3, 4), (1, 0), (2, 1), (4, 3)]
    g = csr(edges, 5)
    for max_depth, p, q, plus, length in ((2, 1.0, 1.0, False, 2), (4, 0.25, 0.25, False, 5),
                                          (4, 0.25, 0.25, True, 5), (4, 1.0, 1.0, False, 4), (4, 1.0, 1.0, True, 4)):
        mode = walk_mode(p, q, plus)
        walks = W.as_lists(host_walk(lib, g, [0, 1], max_depth, mode, 3, p, q)[0])
        assert [len(w) for w in walks] == [length, length], (max_depth, p, q, plus)
        assert [w[0] for w in walks] == [0, 1]


def test_python_layer_refuses_bad_arguments():
    import pgl_b200 as pgl
    from pgl_b200.sampling import node2vec_walk, node2vec_walk_plus, random_walk
    g = pgl.Graph(edges=[(0, 1), (1, 2), (2, 0)], num_nodes=4)
    for bad in (0, -1, 1.5, True):
        with pytest.raises(ValueError):
            random_walk(g, [0], bad)
    for p, q in ((0, 1), (-1, 1), (1, 0), (float("nan"), 1), (1, float("inf")), (1e-320, 1)):
        with pytest.raises(ValueError):
            node2vec_walk(g, [0], 3, p=p, q=q)
        with pytest.raises(ValueError):
            node2vec_walk_plus(g, [0], 3, p=p, q=q)
    for nodes in ([4], [-1], [0, 1, 9], [0.5]):
        with pytest.raises(ValueError):
            random_walk(g, nodes, 3)
        with pytest.raises(ValueError):
            node2vec_walk(g, nodes, 3, p=0.5)


def test_without_cuda_the_walks_raise():
    import torch
    import pgl_b200 as pgl
    from pgl_b200.sampling import random_walk
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    g = pgl.Graph(edges=[(0, 1), (1, 2), (2, 0)], num_nodes=3)
    with pytest.raises(RuntimeError, match="CUDA"):
        random_walk(g, [0, 1], 3)


def test_abi_argument_checks(lib):
    f = lib.lib
    one = ctypes.c_void_p(16)  # non-NULL dummy: must never be dereferenced here
    # pglb_random_walk(indptr, cols, num_nodes, nodes, n, max_depth, seed, out, stream)
    assert f.pglb_random_walk(one, one, 5, one, 3, 0, 1, one, None) == EINVAL
    assert b"max_depth" in f.pglb_last_error()
    assert f.pglb_random_walk(one, one, 5, one, 3, -2, 1, one, None) == EINVAL
    assert f.pglb_random_walk(one, one, 5, None, 3, 4, 1, one, None) == EINVAL
    assert f.pglb_random_walk(None, one, 5, one, 3, 4, 1, one, None) == EINVAL
    assert f.pglb_random_walk(one, one, 5, one, -3, 4, 1, one, None) == EINVAL
    assert f.pglb_random_walk(None, None, 5, None, 0, 4, 1, None, None) == 0
    # pglb_node2vec_walk(indptr, cols, sorted, num_nodes, nodes, n, max_depth, p, q, plus, seed, out, stats, stream)
    for p, q in ((0.0, 1.0), (-1.0, 1.0), (1.0, 0.0), (1.0, -2.0), (float("nan"), 1.0), (1.0, float("inf")),
                 (1e-320, 1.0)):
        for plus in (0, 1):
            assert f.pglb_node2vec_walk(one, one, one, 5, one, 3, 4, p, q, plus, 1, one, None, None) == EINVAL
            assert f.pglb_node2vec_walk(None, None, None, 5, None, 0, 4, p, q, plus, 1, None, None, None) == EINVAL
    assert b"p and q" in f.pglb_last_error()
    assert f.pglb_node2vec_walk(one, one, None, 5, one, 3, 4, 0.5, 2.0, 0, 1, one, None, None) == EINVAL
    assert f.pglb_node2vec_walk(one, one, one, 5, one, 3, 0, 0.5, 2.0, 0, 1, one, None, None) == EINVAL
    assert f.pglb_node2vec_walk(None, None, None, 5, None, 0, 4, 0.5, 2.0, 1, 1, None, None, None) == 0
    # pglb_walk_host(indptr, cols, sorted, num_nodes, nodes, n, max_depth, p, q, mode, seed, out, stats)
    assert f.pglb_walk_host(one, one, one, 5, one, 3, 4, 0.5, 2.0, 3, 1, one, None) == EINVAL
    assert b"mode" in f.pglb_last_error()
    assert f.pglb_walk_host(one, one, one, 5, one, 3, 4, 0.0, 2.0, 1, 1, one, None) == EINVAL
    assert f.pglb_walk_host(one, one, one, 5, one, 3, 0, 0.5, 2.0, 0, 1, one, None) == EINVAL
    assert f.pglb_walk_host(one, one, None, 5, one, 3, 4, 0.5, 2.0, 2, 1, one, None) == EINVAL
    assert f.pglb_walk_host(None, None, None, 5, None, 0, 4, 0.5, 2.0, 1, 1, None, None) == 0
