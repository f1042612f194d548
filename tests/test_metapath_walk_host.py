"""Metapath walks without a GPU: the library's host entry (the kernel's own walk function) against the numpy replay of
tests/metapath_oracle.py bit for bit, the one-relation identity with random_walk's host entry, paths and stops,
node types along the reference's c / p / a walks, a chi-square test out of a 10^4-edge hub, and the argument checks
of the Python layer and of both C entries."""
import ctypes

import numpy as np
import pytest
from scipy import stats

import metapath_oracle as MO
from oracle import oracle_walk as W

EINVAL = -1
SEEDS = (0, 2 ** 64 - 1)


@pytest.fixture(scope="module")
def lib():
    from pgl_b200 import _lib
    return _lib.lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p).value


def host_metapath(lib, csrs, idx, nodes, walk_length, seed):
    """pglb_metapath_walk_host over the relations csrs[idx[k]]; an empty cols is passed as its indptr."""
    csrs = [(np.ascontiguousarray(ip, np.int64), np.ascontiguousarray(c, np.int64)) for ip, c in csrs]
    nodes = np.ascontiguousarray(nodes, np.int64)
    m = len(idx)
    ips = (ctypes.c_void_p * m)(*[_ptr(csrs[r][0]) for r in idx])
    cols = (ctypes.c_void_p * m)(*[_ptr(csrs[r][1] if len(csrs[r][1]) else csrs[r][0]) for r in idx])
    out = np.full((len(nodes), walk_length), 7, np.int64)
    rc = lib.pglb_metapath_walk_host(ips, cols, m, len(csrs[0][0]) - 1, _ptr(nodes), len(nodes), walk_length, seed,
                                     _ptr(out))
    assert rc == 0, lib.pglb_last_error()
    return out


def _csrs(edges, n):
    names = list(edges)
    return names, [MO.csr(edges[e], n) for e in names]


def kat():
    edges, n, types = MO.kat_graph()
    names, csrs = _csrs(edges, n)
    return names, csrs, n, types


def typed():
    edges, n, nodes = MO.typed_graph()
    names, csrs = _csrs(edges, n)
    return names, csrs, n, nodes


def typed_metapaths():
    rng = np.random.default_rng(11)
    long_path = rng.choice(["r0", "r1", "r3"], 64).tolist()
    with_empty = list(long_path)
    with_empty[50] = "r2"
    no_sinks = rng.choice(["r4", "r5"], 64).tolist()
    return [["r0"], ["r1"], ["r2"], ["r0", "r1"], ["r1", "r0", "r1", "r3"], ["r0", "r2", "r1"], ["r1", "r1"],
            ["r4", "r1", "r5"], long_path, with_empty, no_sinks]


@pytest.mark.parametrize("metapath", ["c2p-p2a-a2p-p2c", "p2a-a2p"])
def test_host_entry_is_the_replay_on_the_reference_graph(lib, metapath):
    names, csrs, n, types = kat()
    idx = [names.index(e) for e in metapath.split("-")]
    nodes = np.arange(n)
    for walk_length in (1, 2, 40):
        for seed in SEEDS:
            got = host_metapath(lib, csrs, idx, nodes, walk_length, seed)
            assert np.array_equal(got, MO.replay_metapath(csrs, nodes, idx, walk_length, seed)), (walk_length, seed)
    # node types follow the metapath: v_t has relation t's source type, v_{t+1} its destination type
    etypes = metapath.split("-")
    long_walks = 0
    for row in W.as_lists(got):
        for t in range(len(row) - 1):
            e = etypes[t % len(etypes)]
            assert (types[row[t]], types[row[t + 1]]) == (e[0], e[2]), (row, t)
        long_walks += len(row) == 40
    assert long_walks > 0


def test_host_entry_is_the_replay_on_a_typed_graph(lib):
    names, csrs, n, nodes = typed()
    nodes = np.r_[nodes, [-1, n, 5]]   # starts outside the graph give rows of -1
    for metapath in typed_metapaths():
        idx = [names.index(e) for e in metapath]
        for walk_length in (1, 2, 40) + ((130,) if len(metapath) == 64 else ()):
            for seed in SEEDS:
                got = host_metapath(lib, csrs, idx, nodes, walk_length, seed)
                want = MO.replay_metapath(csrs, nodes, idx, walk_length, seed)
                assert np.array_equal(got, want), (metapath, walk_length, seed)
                assert (got[-3:-1] == -1).all() and got[-1, 0] == 5
    # a 64-relation path without sinks wraps around twice in 130 nodes
    idx = [names.index(e) for e in typed_metapaths()[-1]]
    assert (host_metapath(lib, csrs, idx, nodes[:-3], 130, 3) >= 0).all()


def test_one_relation_is_random_walk(lib):
    for names, csrs, n, nodes in (typed(), kat()[:3] + (np.arange(15),)):
        for r in range(len(names)):
            ip, cols = (np.ascontiguousarray(a, np.int64) for a in csrs[r])
            for walk_length in (1, 2, 40):
                for seed in SEEDS + (0x0123456789ABCDEF,):
                    got = host_metapath(lib, csrs, [r], nodes, walk_length, seed)
                    want = np.full((len(nodes), walk_length), 7, np.int64)
                    nd = np.ascontiguousarray(nodes, np.int64)
                    c = cols if len(cols) else ip
                    assert lib.pglb_walk_host(_ptr(ip), _ptr(c), _ptr(c), n, _ptr(nd), len(nd), walk_length, 1.0, 1.0,
                                              W.UNIFORM, seed, _ptr(want), None) == 0
                    assert np.array_equal(got, want), (names[r], walk_length, seed)


def test_walks_follow_the_relations_and_stop_only_at_their_sinks(lib):
    names, csrs, n, nodes = typed()
    edge_sets = [{(u, int(v)) for u in range(n) for v in cols[ip[u]:ip[u + 1]]} for ip, cols in csrs]
    stopped = 0
    for metapath in typed_metapaths():
        idx = [names.index(e) for e in metapath]
        M = len(idx)
        out = host_metapath(lib, csrs, idx, nodes, 40, 12345)
        for start, row in zip(nodes, W.as_lists(out)):
            assert row[0] == start
            for t in range(len(row) - 1):
                assert (row[t], row[t + 1]) in edge_sets[idx[t % M]], (metapath, row, t)
            if len(row) < 40:
                ip = csrs[idx[(len(row) - 1) % M]][0]
                assert ip[row[-1] + 1] == ip[row[-1]], (metapath, row)
                stopped += 1
    assert stopped > 0


def _chi2(samples, probs):
    """Chi-square p-value of samples against {value: probability}; bins expecting fewer than 5 are pooled."""
    keys = sorted(probs)
    s = np.sort(np.asarray(samples))
    obs = np.array([np.searchsorted(s, k, "right") - np.searchsorted(s, k, "left") for k in keys], np.float64)
    assert obs.sum() == len(s)
    exp = np.array([probs[k] for k in keys]) * len(s)
    small = exp < 5
    if small.any():
        obs = np.r_[obs[~small], obs[small].sum()]
        exp = np.r_[exp[~small], exp[small].sum()]
    return stats.chisquare(obs, exp).pvalue


def test_first_and_second_steps_out_of_the_hub(lib):
    names, csrs, n, _ = typed()
    idx = [names.index("r1"), names.index("r0")]
    out = host_metapath(lib, csrs, idx, np.zeros(200_000, np.int64), 3, 2024)
    first = MO.step_probs(csrs, idx, 0, 0)
    assert abs(sum(first.values()) - 1) < 1e-12 and len(first) > 400
    assert _chi2(out[:, 1], first) > 1e-3
    second = MO.position_probs(csrs, idx, 0, 2)
    assert 0 < second[-1] < 1   # r0 has sinks: some walks end after one step
    assert _chi2(out[:, 2], second) > 1e-3


def test_python_layer_refuses_bad_arguments():
    import pgl_b200 as pgl
    from pgl_b200.sampling import metapath_randomwalk
    edges, n, _ = MO.kat_graph()
    _, _, types = MO.kat_graph()
    hg = pgl.HeterGraph(edges=edges, num_nodes=n, node_types=types)
    before = pgl.ops.launch_count()
    with pytest.raises(TypeError):
        metapath_randomwalk(hg["c2p"], [0], "c2p", 3)
    with pytest.raises(ValueError, match="c2p"):   # names the valid edge types
        metapath_randomwalk(hg, [0], "c2p-x2y", 3)
    for bad in ([], (), "", ["c2p"] * 65, "-".join(["c2p"] * 65)):
        with pytest.raises(ValueError):
            metapath_randomwalk(hg, [0], bad, 3)
    for bad in (0, -1, 1.5, True, 2 ** 31):
        with pytest.raises(ValueError, match="walk_length"):
            metapath_randomwalk(hg, [0], "c2p-p2c", bad)
    for nodes in ([-1], [n], [0, 3, 99], [0.5]):
        with pytest.raises(ValueError):
            metapath_randomwalk(hg, nodes, "c2p-p2c", 3)
    assert pgl.ops.launch_count() == before


def test_without_cuda_the_walks_raise():
    import torch
    import pgl_b200 as pgl
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    edges, n, types = MO.kat_graph()
    hg = pgl.HeterGraph(edges=edges, num_nodes=n, node_types=types)
    with pytest.raises(RuntimeError, match="CUDA"):
        pgl.sampling.metapath_randomwalk(hg, [0, 1], "c2p-p2c", 3)


def test_abi_argument_checks(lib):
    one = ctypes.c_void_p(16)   # non-NULL dummy: must never be dereferenced here
    ptrs = (ctypes.c_void_p * 65)(*([16] * 65))
    holes = (ctypes.c_void_p * 3)(16, None, 16)
    for f, tail in ((lib.pglb_metapath_walk, (None,)), (lib.pglb_metapath_walk_host, ())):
        # (indptrs, cols, m, num_nodes, nodes, n, walk_length, seed, out[, stream])
        for m in (0, 65, -1):
            assert f(ptrs, ptrs, m, 5, one, 3, 4, 1, one, *tail) == EINVAL
            assert b"m must" in lib.pglb_last_error()
        for wl in (0, -2, 2 ** 31 - 1):
            assert f(ptrs, ptrs, 2, 5, one, 3, wl, 1, one, *tail) == EINVAL
            assert b"walk_length" in lib.pglb_last_error()
        assert f(None, ptrs, 2, 5, one, 3, 4, 1, one, *tail) == EINVAL
        assert f(ptrs, None, 2, 5, one, 3, 4, 1, one, *tail) == EINVAL
        assert f(holes, ptrs, 3, 5, one, 3, 4, 1, one, *tail) == EINVAL
        assert f(ptrs, holes, 3, 5, one, 3, 4, 1, one, *tail) == EINVAL
        assert f(ptrs, ptrs, 2, 5, None, 3, 4, 1, one, *tail) == EINVAL
        assert f(ptrs, ptrs, 2, 5, one, 3, 4, 1, None, *tail) == EINVAL
        assert b"NULL" in lib.pglb_last_error()
        assert f(ptrs, ptrs, 2, 5, one, -3, 4, 1, one, *tail) == EINVAL
        assert f(ptrs, ptrs, 2, -5, one, 3, 4, 1, one, *tail) == EINVAL
        assert b"negative" in lib.pglb_last_error()
        assert f(None, None, 2, 5, None, 0, 4, 1, None, *tail) == 0
        assert f(ptrs, ptrs, 64, 5, one, 0, 1, 1, one, *tail) == 0
