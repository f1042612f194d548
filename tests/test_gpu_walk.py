"""Random walks on the device (csrc/walk.cu through pgl_b200.sampling): bit for bit against the numpy replay of the
library's rule (oracle/oracle_walk.py) on small graphs with sinks, self-loops, multi-edges, duplicate starts and a
10^4-edge hub, for all three rules and through the exact fallback; on RMAT graphs of 2^20 and 10^7 nodes, walks are
paths that stop only at sinks, and fixed-seed chi-square tests hold for first- and second-order transitions over 10^6
walkers; seeds, graph modes and the device cache of a numpy-mode graph."""
import numpy as np
import pytest
import torch
from scipy import stats

from oracle import oracle_walk as W

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    torch.cuda.set_device(0)
    return pgl_b200


def small_edges():
    e = [(0, 1), (0, 1), (0, 0), (1, 2), (2, 0), (2, 3), (3, 4), (1, 0), (4, 4), (0, 2), (2, 3), (2, 3), (3, 5),
         (4, 2), (1, 5), (7, 0), (7, 2)]
    return np.array(e, np.int64), 8, np.array([0, 0, 1, 2, 3, 4, 5, 6, 7, 7, 2])


def hub_edges():
    rng = np.random.default_rng(3)
    n = 300
    hub = np.stack([np.zeros(10000, np.int64), rng.integers(1, n, 10000)], 1)
    rest = np.stack([rng.integers(1, n, 1500), rng.integers(0, n, 1500)], 1)
    back = np.stack([rng.integers(1, n, 200), np.zeros(200, np.int64)], 1)
    return np.concatenate([hub, rest, back]), n + 5, np.r_[[0] * 40, rng.integers(0, n + 5, 120)]


def random_edges():
    rng = np.random.default_rng(5)
    n = 400
    e = np.stack([rng.integers(0, n, 2500), rng.integers(0, n, 2500)], 1)
    return np.concatenate([e, e[:300]]), n, rng.integers(0, n, 300)


GRAPHS = {"small": small_edges, "hub": hub_edges, "random": random_edges}
CALLS = [("random_walk", W.UNIFORM, 1.0, 1.0)] + \
    [(f, m, p, q) for f, m in (("node2vec_walk", W.NODE2VEC), ("node2vec_walk_plus", W.NODE2VEC_PLUS))
     for p, q in ((0.25, 4.0), (4.0, 0.25), (1e-3, 1.0), (2.0, 0.5))]


def _call(pgl, g, name, nodes, depth, p, q, seed):
    f = getattr(pgl.sampling, name)
    if name == "random_walk":
        return f(g, nodes, depth, seed=seed)
    return f(g, nodes, depth, p=p, q=q, seed=seed)


@pytest.mark.parametrize("gname", sorted(GRAPHS))
def test_device_is_the_replay(pgl, gname):
    edges, n, nodes = GRAPHS[gname]()
    g = pgl.Graph(edges=edges, num_nodes=n)
    gt = pgl.Graph(edges=edges, num_nodes=n).tensor()
    indptr, cols = g.adj_src_index._indptr, g.adj_src_index._sorted_v
    fallbacks = 0
    for name, mode, p, q in CALLS:
        for seed in (0, 0x0123456789ABCDEF, 2 ** 64 - 1):
            want, _, fb = W.replay(indptr, cols, nodes, 6, mode, seed, p, q)
            fallbacks += fb
            got = _call(pgl, g, name, nodes, 6, p, q, seed)
            assert got == W.as_lists(want), (name, p, q, seed)
            got_t = _call(pgl, gt, name, torch.as_tensor(nodes).cuda(), 6, p, q, seed)
            assert got_t.dtype == torch.int64 and got_t.is_cuda
            assert np.array_equal(got_t.cpu().numpy(), want), (name, p, q, seed)
    assert fallbacks > 0


def _rmat(scale, e, n, seed):
    """RMAT (0.57, 0.19, 0.19, 0.05) with duplicates and self-loops kept; edges with an id >= n are dropped."""
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    src = torch.zeros(e, dtype=torch.int64, device="cuda")
    dst = torch.zeros(e, dtype=torch.int64, device="cuda")
    for _ in range(scale):
        r = torch.rand(e, generator=gen, device="cuda")
        src = src * 2 + (r >= 0.76).to(torch.int64)
        dst = dst * 2 + (((r >= 0.57) & (r < 0.76)) | (r >= 0.95)).to(torch.int64)
    keep = (src < n) & (dst < n)
    return torch.stack([src[keep], dst[keep]], 1).contiguous()


@pytest.fixture(scope="module", params=["rmat_1m", "rmat_10m"])
def rmat(pgl, request):
    scale, e, n = (20, 10_000_000, 1 << 20) if request.param == "rmat_1m" else (24, 100_000_000, 10_000_000)
    edges = _rmat(scale, e, n, seed=7)
    g = pgl.Graph(edges=edges, num_nodes=n)
    yield request.param, g
    del g, edges
    torch.cuda.empty_cache()


def _edge_keys(g):
    indptr, cols, _ = g._walk_csr()
    n = g._n
    rows = torch.repeat_interleave(torch.arange(n, device="cuda"), indptr[1:] - indptr[:-1])
    return torch.unique(rows * n + cols)


@pytest.mark.parametrize("name,p,q", [("random_walk", 1, 1), ("node2vec_walk", 0.25, 4.0),
                                      ("node2vec_walk", 4.0, 0.25), ("node2vec_walk_plus", 0.5, 2.0)])
def test_rmat_walks_are_paths_that_stop_at_sinks(pgl, rmat, name, p, q):
    _, g = rmat
    n = g._n
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    nodes = torch.randint(0, n, (1_000_000,), device="cuda", generator=gen)
    depth = 20 if name != "node2vec_walk_plus" else 8
    out = _call(pgl, g, name, nodes, depth, p, q, 123)
    assert out.shape == (nodes.numel(), depth if name == "random_walk" else depth + 1)
    assert torch.equal(out[:, 0], nodes)
    valid = out >= 0
    length = valid.sum(1)
    # -1 only as a suffix
    assert torch.equal(valid, torch.arange(out.shape[1], device="cuda")[None, :] < length[:, None])
    keys = _edge_keys(g)
    a, b = out[:, :-1], out[:, 1:]
    pair = valid[:, 1:]
    k = (a * n + b)[pair]
    pos = torch.searchsorted(keys, k).clamp_max(keys.numel() - 1)
    assert torch.equal(keys[pos], k), "a step that is not an edge"
    deg = g._walk_csr()[0].diff()
    last = out.gather(1, (length - 1)[:, None]).squeeze(1)
    short = length < out.shape[1]
    assert torch.equal(short, short & (deg[last] == 0)), "a walk stopped at a node with successors"


def _host_csr(g):
    indptr, cols, _ = g._walk_csr()
    return indptr.cpu().numpy(), cols.cpu().numpy()


def _chi2(samples, probs):
    keys = sorted(probs)
    s = np.sort(samples)
    obs = np.array([np.searchsorted(s, k, "right") - np.searchsorted(s, k, "left") for k in keys], np.float64)
    assert obs.sum() == len(samples)
    exp = np.array([probs[k] for k in keys]) * len(samples)
    return stats.chisquare(obs, exp).pvalue


@pytest.mark.parametrize("rmat", ["rmat_1m"], indirect=True)
def test_rmat_first_and_second_order_transitions(pgl, rmat):
    _, g = rmat
    indptr, cols = _host_csr(g)
    deg = np.diff(indptr)
    # first order: 10^6 walkers out of one node of degree 20..60
    c = int(np.flatnonzero((deg >= 20) & (deg <= 60))[0])
    out = pgl.sampling.random_walk(g, torch.full((1_000_000,), c, device="cuda"), 2, seed=5).cpu().numpy()
    assert _chi2(out[:, 1], W.node_probs(indptr, cols, [c], W.UNIFORM)) > 1e-4
    # second order: start at a (out-degree 2..6), condition on the first step a -> b, where b's row holds a (return),
    # a successor of a (near) and something else (far).  b may be a hub, so the test is over the three classes.
    def pick():
        for a in np.flatnonzero((deg >= 2) & (deg <= 6)):
            row = set(cols[indptr[a]:indptr[a + 1]].tolist())
            for b in row - {int(a)}:
                brow = set(cols[indptr[b]:indptr[b + 1]].tolist())
                if a in brow and brow & row - {a} and brow - row - {a}:
                    return int(a), b
        pytest.fail("no (a, b) pair with return, near and far candidates")
    a, b = pick()
    near = set(cols[indptr[a]:indptr[a + 1]].tolist())
    klass = lambda y: 0 if y == a else (1 if y in near else 2)  # noqa: E731
    for name, mode in (("node2vec_walk", W.NODE2VEC), ("node2vec_walk_plus", W.NODE2VEC_PLUS)):
        for p, q in ((0.25, 4.0), (4.0, 0.25)):
            out = getattr(pgl.sampling, name)(g, torch.full((1_000_000,), a, device="cuda"), 2, p=p, q=q,
                                              seed=17).cpu().numpy()
            sel = out[out[:, 1] == b]
            assert len(sel) > 1_000_000 // 7
            probs = {0: 0.0, 1: 0.0, 2: 0.0}
            for y, pr in W.node_probs(indptr, cols, [a, b], mode, p, q).items():
                probs[klass(y)] += pr
            assert _chi2(np.array([klass(y) for y in sel[:, 2].tolist()]), probs) > 1e-4, (name, p, q)


def test_seeds(pgl):
    edges, n, nodes = random_edges()
    g = pgl.Graph(edges=edges, num_nodes=n)
    a = pgl.sampling.node2vec_walk(g, nodes, 10, p=0.5, q=2.0, seed=1)
    assert a == pgl.sampling.node2vec_walk(g, nodes, 10, p=0.5, q=2.0, seed=1)
    assert a != pgl.sampling.node2vec_walk(g, nodes, 10, p=0.5, q=2.0, seed=2)
    np.random.seed(2024)
    r1 = pgl.sampling.random_walk(g, nodes, 10)
    np.random.seed(2024)
    assert r1 == pgl.sampling.random_walk(g, nodes, 10)
    assert r1 != pgl.sampling.random_walk(g, nodes, 10)


def test_numpy_and_tensor_mode_give_the_same_walks(pgl):
    edges, n, nodes = small_edges()
    g = pgl.Graph(edges=edges, num_nodes=n)
    gt = pgl.Graph(edges=torch.as_tensor(edges).cuda(), num_nodes=n)
    for name, mode, p, q in CALLS:
        lists = _call(pgl, g, name, nodes, 5, p, q, 9)
        t = _call(pgl, gt, name, torch.as_tensor(nodes).cuda(), 5, p, q, 9)
        assert isinstance(lists, list) and all(isinstance(w, list) for w in lists)
        assert all(isinstance(v, int) for w in lists for v in w)
        assert lists == W.as_lists(t.cpu().numpy())
        assert (t.cpu().numpy() == -1).any()   # padded after walks that hit a sink


def test_numpy_graph_uploads_once(pgl):
    edges, n, nodes = hub_edges()
    g = pgl.Graph(edges=edges, num_nodes=n)
    pgl.sampling.node2vec_walk(g, nodes, 4, p=0.5, q=2.0, seed=1)
    cache = dict(g._walk_dev["cuda:0"])
    ptrs = {k: v.data_ptr() for k, v in cache.items()}
    pgl.sampling.node2vec_walk(g, nodes, 4, p=0.5, q=2.0, seed=2)
    pgl.sampling.random_walk(g, nodes, 4, seed=3)
    again = g._walk_dev["cuda:0"]
    assert all(again[k] is cache[k] and again[k].data_ptr() == ptrs[k] for k in cache)
    # the row-sorted copy is the successor columns with every row ascending
    indptr, cols, srt = (t.cpu().numpy() for t in (again["indptr"], again["cols"], again["sorted"]))
    for u in range(n):
        assert np.array_equal(srt[indptr[u]:indptr[u + 1]], np.sort(cols[indptr[u]:indptr[u + 1]]))
    g.tensor()
    assert "_walk_dev" not in g.__dict__
    g.numpy()
    assert pgl.sampling.random_walk(g, nodes, 4, seed=3) == pgl.sampling.random_walk(
        pgl.Graph(edges=edges, num_nodes=n), nodes, 4, seed=3)


def test_pgl_alias_import(pgl):
    from pgl.sampling import node2vec_walk, node2vec_walk_plus, random_walk  # noqa: F401
    edges = [(0, 1), (1, 2), (3, 4), (1, 0), (2, 1), (4, 3)]
    g = pgl.Graph(edges=edges, num_nodes=5)
    assert [len(w) for w in random_walk(g, [0, 1], 2)] == [2, 2]
    assert [len(w) for w in node2vec_walk(g, [0, 1], 4, p=0.25, q=0.25)] == [5, 5]
    assert [len(w) for w in node2vec_walk_plus(g, [0, 1], 4, p=0.25, q=0.25)] == [5, 5]
    assert [len(w) for w in node2vec_walk(g, [0, 1], 4)] == [4, 4]
