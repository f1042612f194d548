"""Skip-gram pairs and alias tables without a GPU: the numpy replay against the compiled reference's outputs
(tests/golden/ref_skipgram.npz), the library's host entries (the kernels' own window, emit and draw functions) against
the replay bit for bit, the pgl.graph_kernel shim against the reference call for call, the alias tables' bits and
implied distributions, the window distribution, and the argument checks of the Python layer and the C ABI."""
import ctypes
import os

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import oracle_skipgram as S
from oracle import oracle_walk as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL = -1
SEEDS = (0, 2 ** 64 - 1)


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


@pytest.fixture(scope="module")
def lib():
    from pgl_b200 import _lib
    return _lib.lib


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "ref_skipgram.npz"))


def unflat(z, name):
    a, off = z[name], z[name + "_off"]
    return [a[off[k]:off[k + 1]] for k in range(len(off) - 1)]


def host_pairs(lib, walks, win_size, seed):
    walks = np.ascontiguousarray(walks, np.int64)
    B, L = walks.shape
    offsets = np.full(B + 1, -7, np.int64)
    assert lib.pglb_skipgram_host(ptr(walks), B, L, win_size, seed, ptr(offsets), None, None) == 0
    src = np.full(offsets[B], -7, np.int64)
    pos = np.full(offsets[B], -7, np.int64)
    rc = lib.pglb_skipgram_host(ptr(walks), B, L, win_size, seed, ptr(offsets), ptr(src), ptr(pos))
    assert rc == 0, lib.pglb_last_error()
    return offsets, src, pos


def replay(walks, win_size, seed):
    """The replay with the library's Philox windows."""
    walks = np.asarray(walks, np.int64)
    return S.replay_skipgram(walks, S.skipgram_windows(walks.shape[0], walks.shape[1], win_size, seed))


def test_replay_is_the_reference(gold):
    walks, windows = unflat(gold, "a_walk"), unflat(gold, "a_window")
    srcs, poss = unflat(gold, "a_src"), unflat(gold, "a_pos")
    assert len(walks) == len(gold["a_win_size"]) == 36
    for walk, win, s, p in zip(walks, windows, srcs, poss):
        rs, rp = S.replay_skipgram([walk], [win])
        np.testing.assert_array_equal(rs, s)
        np.testing.assert_array_equal(rp, p)
    # the batch replay is the per-walk outputs concatenated, in order
    rs, rp = S.replay_skipgram(walks, windows)
    np.testing.assert_array_equal(rs, gold["a_src"])
    np.testing.assert_array_equal(rp, gold["a_pos"])


def test_shim_is_the_reference_with_injected_windows(gold, monkeypatch):
    from pgl_b200 import graph_kernel as gk
    for walk, win_size, win, s, p in zip(unflat(gold, "a_walk"), gold["a_win_size"], unflat(gold, "a_window"),
                                         unflat(gold, "a_src"), unflat(gold, "a_pos")):
        def randint(lo, hi, dtype=None, size=None, _w=win, _ws=int(win_size)):
            assert (lo, hi, dtype, size) == (1, _ws + 1, np.int64, len(_w))
            return _w.copy()
        monkeypatch.setattr(np.random, "randint", randint)
        gs, gp = gk.skip_gram_gen_pair(walk.tolist(), int(win_size))
        assert isinstance(gs, list) and isinstance(gp, list)
        assert gs == s.tolist() and gp == p.tolist()


def test_shim_reproduces_seeded_calls(gold):
    import pgl.graph_kernel as gk
    np.random.seed(int(gold["b_seed"]))
    for walk, win_size, s, p in zip(unflat(gold, "b_walk"), gold["b_win_size"], unflat(gold, "b_src"),
                                    unflat(gold, "b_pos")):
        gs, gp = gk.skip_gram_gen_pair(walk.tolist(), int(win_size))
        assert gs == s.tolist() and gp == p.tolist()


def test_graph_kernel_exports_only_the_two_names():
    import pgl.graph_kernel as gk
    assert sorted(gk.__all__) == ["alias_sample_build_table", "skip_gram_gen_pair"]
    assert "No other" in gk.__doc__


def csr(edges, n):
    e = np.asarray(edges, np.int64).reshape(-1, 2)
    order = np.argsort(e[:, 0], kind="stable")
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(e[:, 0], minlength=n), out=indptr[1:])
    return indptr, e[order, 1]


def host_walks(lib, indptr, cols, nodes, max_depth, seed):
    nodes = np.ascontiguousarray(nodes, np.int64)
    out = np.empty((len(nodes), max_depth), np.int64)
    rc = lib.pglb_walk_host(ptr(indptr), ptr(cols), ptr(cols), len(indptr) - 1, ptr(nodes), len(nodes), max_depth,
                            1.0, 1.0, W.UNIFORM, seed, ptr(out), None)
    assert rc == 0
    return out


def sink_graph(seed=3):
    """400 nodes, a fifth of them sinks, self-loops and repeated edges: walks end early and revisit nodes"""
    rng = np.random.default_rng(seed)
    n = 400
    u = rng.integers(0, n, 1600)
    u = u[u % 5 != 0]
    v = rng.integers(0, n, len(u))
    e = np.concatenate([np.stack([u, v], 1), [[1, 1], [1, 1], [2, 3], [3, 2]]])
    return csr(e, n), n


@pytest.mark.parametrize("L", [1, 2, 7, 40, 130])
@pytest.mark.parametrize("win_size", [1, 3, 10, 200])
def test_host_entry_is_the_replay_on_walks(lib, L, win_size):
    (indptr, cols), n = sink_graph()
    rng = np.random.default_rng(L * 1000 + win_size)
    walks = host_walks(lib, indptr, cols, rng.integers(0, n, 48), L, 11)
    if L > 1:
        assert (walks[:, -1] < 0).any()   # some walks hit a sink and are padded
    for seed in SEEDS:
        offsets, src, pos = host_pairs(lib, walks, win_size, seed)
        rs, rp = replay(walks, win_size, seed)
        np.testing.assert_array_equal(src, rs)
        np.testing.assert_array_equal(pos, rp)
        assert offsets[0] == 0 and offsets[-1] == len(rs) and (np.diff(offsets) >= 0).all()


@pytest.mark.parametrize("win_size", [1, 2, 3, 10, 15, 16, 200])
def test_host_entry_is_the_replay_on_hand_made_walks(lib, win_size):
    """repeats, runs of one node, rows padded at every length, a row of -1 only and a row without padding"""
    rng = np.random.default_rng(win_size)
    L = 60
    walks = rng.integers(0, 5, (40, L))
    walks[3, 10:30] = 2
    for b in range(4, 40):
        walks[b, int(rng.integers(0, L + 1)):] = -1
    walks[5] = -1
    walks[6, 20] = -3   # any negative entry ends the walk
    for seed in SEEDS + (0x0123456789ABCDEF,):
        offsets, src, pos = host_pairs(lib, walks, win_size, seed)
        rs, rp = replay(walks, win_size, seed)
        np.testing.assert_array_equal(src, rs)
        np.testing.assert_array_equal(pos, rp)
        # offsets delimit each walk's own pairs
        for b in range(len(walks)):
            assert np.isin(src[offsets[b]:offsets[b + 1]], walks[b]).all()
        assert offsets[6] == offsets[5]   # the row of -1 only has no pairs


def test_windows_are_uniform_and_centres_emit_2w(lib):
    """Walks of distinct nodes: a centre at least win_size from both ends emits exactly 2w pairs.  Over 10^6 such
    centres w matches the Philox replay and is uniform on [1, win_size] (chi-square)."""
    win_size, L, B = 10, 40, 5000
    inner = np.arange(win_size, L - win_size)
    hist = np.zeros(win_size + 1, np.int64)
    for chunk in range(10):
        walks = np.arange(B * L, dtype=np.int64).reshape(B, L)
        seed = 1000 + chunk
        _, src, _ = host_pairs(lib, walks, win_size, seed)
        cnt = np.bincount(src, minlength=B * L).reshape(B, L)[:, inner]
        w = S.skipgram_windows(B, L, win_size, seed)[:, inner]
        np.testing.assert_array_equal(cnt, 2 * w)
        hist += np.bincount(w.reshape(-1), minlength=win_size + 1)
    assert hist.sum() == 10 ** 6 and hist[0] == 0
    assert stats.chisquare(hist[1:]).pvalue > 1e-4


def test_alias_build_is_the_reference(lib, gold):
    import pgl.graph_kernel as gk
    leftovers = 0
    for p, a, e in zip(unflat(gold, "c_probs"), unflat(gold, "c_alias"), unflat(gold, "c_events")):
        ga, ge = gk.alias_sample_build_table(p)
        np.testing.assert_array_equal(ga.view(np.uint64), a.view(np.uint64))
        np.testing.assert_array_equal(ge, e)
        ca = np.empty(len(p), np.float64)
        ce = np.empty(len(p), np.int64)
        assert lib.pglb_alias_build_host(ptr(np.ascontiguousarray(p)), len(p), ptr(ca), ptr(ce)) == 0
        np.testing.assert_array_equal(ca.view(np.uint64), a.view(np.uint64))
        np.testing.assert_array_equal(ce, e)
        leftovers += int(((a < 1) & (e == 0) & (np.arange(len(a)) != 0)).sum())
    assert leftovers > 0   # the fixture holds rounding leftovers of the reference


def test_alias_table_distribution(gold):
    """alias_table normalises in float64; its table implies the weights' distribution up to the rounding of the
    construction, |p - w| <= 1e-12 w + 1e-15.  Zero weights get up to about 1e-16 of mass.  The error is absolute in
    nature (a few ulps of alias values near 1, over n): the reference's own 10^5-entry table is 5.8e-17 off at a
    weight near 1.4e-5, 4.2e-12 relative, and tiny positive weights need the absolute term as zero weights do."""
    from pgl_b200.sampling import alias_table
    rng = np.random.default_rng(4)
    cases = unflat(gold, "c_probs") + [np.array([0.0, 3.0, 0.0, 1.0, 1.0]), rng.random(1000) * 7,
                                       np.r_[np.zeros(50), rng.pareto(1.5, 5000)]]
    for wts in cases:
        alias, events = alias_table(wts)
        p = S.alias_distribution(alias, events)
        want = wts / wts.sum()
        pos = want > 0
        assert np.all(np.abs(p - want) <= 1e-12 * want + 1e-15)
        assert np.all(p[~pos] <= 1e-15)
    # the reference's own tables sit within the same bound
    for pr, a, e in zip(unflat(gold, "c_probs"), unflat(gold, "c_alias"), unflat(gold, "c_events")):
        p = S.alias_distribution(a, e)
        pos = pr > 0
        assert np.all(np.abs(p - pr) <= 1e-12 * pr + 1e-15) and np.all(p[~pos] <= 1e-15)


def test_alias_table_modes():
    from pgl_b200.sampling import alias_table
    a, e = alias_table([1, 2, 3, 4])
    assert isinstance(a, np.ndarray) and a.dtype == np.float64 and e.dtype == np.int64
    ta, te = alias_table(torch.tensor([1.0, 2.0, 3.0, 4.0]))
    assert isinstance(ta, torch.Tensor) and ta.dtype == torch.float64 and te.dtype == torch.int64
    np.testing.assert_array_equal(ta.numpy(), a)
    np.testing.assert_array_equal(te.numpy(), e)


@pytest.mark.parametrize("n", [1, 2, 7, 1000, 10 ** 5])
def test_alias_sample_host_is_the_replay(lib, gold, n):
    from pgl_b200.sampling import alias_table
    rng = np.random.default_rng(n)
    alias, events = alias_table(rng.pareto(1.0, n) * (rng.random(n) < 0.8) + (np.arange(n) == 0))
    for seed in SEEDS:
        count = 20000
        out = np.full(count, -7, np.int64)
        assert lib.pglb_alias_sample_host(ptr(alias), ptr(events), n, count, seed, ptr(out)) == 0
        np.testing.assert_array_equal(out, S.alias_draws(alias, events, count, seed))
        assert out.min() >= 0 and out.max() < n


def test_alias_sample_host_distribution(lib):
    """host draws of a Pareto-weighted table against its weights (chi-square over 10^6 draws)"""
    rng = np.random.default_rng(8)
    w = rng.pareto(1.2, 300) + 0.01
    from pgl_b200.sampling import alias_table
    alias, events = alias_table(w)
    count = 10 ** 6
    out = np.empty(count, np.int64)
    assert lib.pglb_alias_sample_host(ptr(alias), ptr(events), len(w), count, 5, ptr(out)) == 0
    obs = np.bincount(out, minlength=len(w))
    assert stats.chisquare(obs, w / w.sum() * count).pvalue > 1e-4


def test_c_abi_checks(lib):
    walks = np.zeros((2, 3), np.int64)
    off = np.zeros(3, np.int64)
    ws = ctypes.c_size_t(0)
    assert lib.pglb_skipgram_host(ptr(walks), 2, 3, 0, 0, ptr(off), None, None) == EINVAL
    assert b"win_size" in lib.pglb_last_error()
    assert lib.pglb_skipgram_host(ptr(walks), 2, 3, 2 ** 31, 0, ptr(off), None, None) == EINVAL
    assert lib.pglb_skipgram_host(None, 2, 3, 5, 0, ptr(off), None, None) == EINVAL
    assert lib.pglb_skipgram_host(ptr(walks), 2, 3, 5, 0, None, None, None) == EINVAL
    assert lib.pglb_skipgram_host(ptr(walks), -1, 3, 5, 0, ptr(off), None, None) == EINVAL
    assert lib.pglb_skipgram_host(ptr(walks), 2, -3, 5, 0, ptr(off), None, None) == EINVAL
    assert lib.pglb_skipgram_host(None, 0, 3, 5, 0, None, None, None) == 0   # empty: a no-op
    assert lib.pglb_skipgram_host(None, 2, 0, 5, 0, ptr(off), None, None) == 0 and (off == 0).all()
    # the device entries check before any CUDA call
    assert lib.pglb_skipgram_count(ptr(walks), 2, 3, 0, 0, ptr(off), None, 0, None) == EINVAL
    assert lib.pglb_skipgram_count(None, 2, 3, 1, 0, ptr(off), None, 0, None) == EINVAL
    assert lib.pglb_skipgram_fill(ptr(walks), 2, 3, -5, 0, ptr(off), None, None, None) == EINVAL
    assert lib.pglb_skipgram_fill(ptr(walks), 2, 3, 5, 0, None, None, None, None) == EINVAL
    assert lib.pglb_skipgram_count(None, 0, 3, 5, 0, None, None, 0, None) == 0
    assert lib.pglb_skipgram_count_ws(-1, ctypes.byref(ws)) == EINVAL
    assert lib.pglb_skipgram_count_ws(10 ** 7, ctypes.byref(ws)) == 0 and ws.value > 0
    al = np.ones(4)
    ev = np.zeros(4, np.int64)
    out = np.zeros(4, np.int64)
    for entry in (lambda *a: lib.pglb_alias_sample(*a, None), lib.pglb_alias_sample_host):
        assert entry(ptr(al), ptr(ev), 0, 4, 0, ptr(out)) == EINVAL
        assert b"n must" in lib.pglb_last_error()
        assert entry(ptr(al), ptr(ev), 2 ** 32, 4, 0, ptr(out)) == EINVAL
        assert entry(ptr(al), ptr(ev), 4, -1, 0, ptr(out)) == EINVAL
        assert entry(None, ptr(ev), 4, 4, 0, ptr(out)) == EINVAL
        assert entry(ptr(al), ptr(ev), 4, 4, 0, None) == EINVAL
        assert entry(None, None, 4, 0, 0, None) == 0
    assert lib.pglb_alias_build_host(None, 3, ptr(al), ptr(ev)) == EINVAL
    assert lib.pglb_alias_build_host(ptr(al), -1, ptr(al), ptr(ev)) == EINVAL
    assert lib.pglb_alias_build_host(None, 0, None, None) == 0


def test_value_errors():
    from pgl_b200.sampling import alias_sample, alias_table, skip_gram_pairs
    for bad in (torch.zeros(2, 3), torch.zeros(2, 3, dtype=torch.bool), torch.zeros(6, dtype=torch.int64),
                torch.zeros(1, 2, 3, dtype=torch.int64), np.zeros((2, 3)), np.zeros(3, np.int64),
                [[0, 1.5]], [[[0, 1]]], [[0, -1]]):
        with pytest.raises(ValueError):
            skip_gram_pairs(bad, 3, seed=0)
    for w in (0, -1, 2 ** 31, True, 1.5):
        with pytest.raises(ValueError):
            skip_gram_pairs([[0, 1]], w, seed=0)
    for wts in ([], [1.0, -1.0], [1.0, np.inf], [np.nan, 1.0], [0.0, 0.0], [[1.0, 2.0]]):
        with pytest.raises(ValueError):
            alias_table(wts)
    a, e = alias_table([1.0, 2.0])
    for aa, ee in ((a, e[:1]), (a[:0], e[:0]), (a.reshape(1, 2), e)):
        with pytest.raises(ValueError):
            alias_sample(aa, ee, 5, seed=0)
    with pytest.raises(ValueError):
        alias_sample(a, e, -1, seed=0)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the CPU-only behaviour")
def test_device_functions_raise_without_cuda():
    from pgl_b200.sampling import alias_sample, alias_table, skip_gram_pairs
    with pytest.raises((RuntimeError, AssertionError)):
        skip_gram_pairs([[0, 1, 2]], 2, seed=0)
    with pytest.raises((RuntimeError, AssertionError)):
        skip_gram_pairs(torch.zeros(2, 3, dtype=torch.int64), 2, seed=0)
    a, e = alias_table([1.0, 2.0])
    with pytest.raises((RuntimeError, AssertionError)):
        alias_sample(a, e, 5, seed=0)
