"""Metapath walks on the device (csrc/walk.cu through pgl_b200.sampling.metapath_randomwalk): bit for bit against the
numpy replay of tests/metapath_oracle.py on the reference's c / p / a graph and on a typed graph with sinks,
self-loops, multi-edges, an empty relation and a 10^4-edge hub, in both graph modes; the one-relation identity with
random_walk; seeds and the relations' device caches; on a seeded MAG-like graph of 10^6 nodes every step is an edge
of its relation, walks stop only where the next relation has no out-edge, and a chi-square test of the first step out
of a hub holds over 10^6 walkers."""
import importlib.util
import os

import numpy as np
import pytest
import torch
from scipy import stats

import metapath_oracle as MO
from oracle import oracle_walk as W

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEEDS = (0, 0x0123456789ABCDEF, 2 ** 64 - 1)


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    torch.cuda.set_device(0)
    return pgl_b200


def _graphs(pgl):
    """(name, numpy-mode HeterGraph, tensor-mode HeterGraph, start nodes, metapaths)"""
    edges, n, types = MO.kat_graph()
    kat = ("kat", pgl.HeterGraph(edges=edges, num_nodes=n, node_types=types),
           pgl.HeterGraph(edges=edges, num_nodes=n, node_types=types).tensor(), np.arange(n),
           ["c2p-p2a-a2p-p2c", "p2a-a2p", ("a2p",)])
    edges, n, nodes = MO.typed_graph()
    types = np.zeros(n, np.int64)
    rng = np.random.default_rng(11)
    typed = ("typed", pgl.HeterGraph(edges=edges, num_nodes=n, node_types=types),
             pgl.HeterGraph(edges=edges, num_nodes=n, node_types=types).tensor(), nodes,
             [["r0"], ["r1", "r0", "r1", "r3"], ["r0", "r2", "r1"], ["r4", "r1", "r5"],
              rng.choice(["r0", "r1", "r3"], 64).tolist(), rng.choice(["r4", "r5"], 64).tolist()])
    return [kat, typed]


def _host_csrs(hg):
    return {e: (hg[e].adj_src_index._indptr, hg[e].adj_src_index._sorted_v) for e in hg.edge_types}


def _etypes(metapath):
    return metapath.split("-") if isinstance(metapath, str) else list(metapath)


def test_device_is_the_replay(pgl):
    for name, hg, hgt, nodes, metapaths in _graphs(pgl):
        csr = _host_csrs(hg)
        names = list(csr)
        csrs = [csr[e] for e in names]
        nodes_t = torch.as_tensor(nodes).cuda()
        for metapath in metapaths:
            idx = [names.index(e) for e in _etypes(metapath)]
            for walk_length in (1, 2, 40, 130):
                for seed in SEEDS:
                    want = MO.replay_metapath(csrs, nodes, idx, walk_length, seed)
                    got = pgl.sampling.metapath_randomwalk(hgt, nodes_t, metapath, walk_length, seed=seed)
                    assert got.dtype == torch.int64 and got.is_cuda and got.shape == want.shape
                    assert np.array_equal(got.cpu().numpy(), want), (name, metapath, walk_length, seed)
                    lists = pgl.sampling.metapath_randomwalk(hg, nodes, metapath, walk_length, seed=seed)
                    assert lists == W.as_lists(want), (name, metapath, walk_length, seed)
            assert all(isinstance(v, int) for w in lists for v in w)


def test_one_relation_is_random_walk(pgl):
    for name, hg, hgt, nodes, _ in _graphs(pgl):
        nodes_t = torch.as_tensor(nodes).cuda()
        for e in hg.edge_types:
            for walk_length in (1, 2, 40):
                for seed in SEEDS:
                    assert torch.equal(pgl.sampling.metapath_randomwalk(hgt, nodes_t, [e], walk_length, seed=seed),
                                       pgl.sampling.random_walk(hgt[e], nodes_t, walk_length, seed=seed)), (name, e)
                    assert pgl.sampling.metapath_randomwalk(hg, nodes, e, walk_length, seed=seed) == \
                        pgl.sampling.random_walk(hg[e], nodes, walk_length, seed=seed), (name, e)


def test_one_launch_per_call(pgl):
    _, _, hgt, nodes, _ = _graphs(pgl)[1]
    nodes_t = torch.as_tensor(nodes).cuda()
    pgl.sampling.metapath_randomwalk(hgt, nodes_t, "r0-r1-r3", 40, seed=1)   # builds the relations' CSRs
    before = pgl.ops.launch_count()
    pgl.sampling.metapath_randomwalk(hgt, nodes_t, "r0-r1-r3", 40, seed=2)
    assert pgl.ops.launch_count() - before == 1


def test_seeds(pgl):
    _, hg, _, nodes, _ = _graphs(pgl)[1]
    a = pgl.sampling.metapath_randomwalk(hg, nodes, "r1-r0", 20, seed=1)
    assert a == pgl.sampling.metapath_randomwalk(hg, nodes, "r1-r0", 20, seed=1)
    assert a != pgl.sampling.metapath_randomwalk(hg, nodes, "r1-r0", 20, seed=2)
    np.random.seed(2024)
    r1 = pgl.sampling.metapath_randomwalk(hg, nodes, "r1-r0", 20)
    np.random.seed(2024)
    assert r1 == pgl.sampling.metapath_randomwalk(hg, nodes, "r1-r0", 20)
    assert r1 != pgl.sampling.metapath_randomwalk(hg, nodes, "r1-r0", 20)


def test_numpy_graph_uploads_each_relation_once(pgl):
    _, hg, _, nodes, _ = _graphs(pgl)[1]
    used = ["r0", "r1", "r3"]
    first = pgl.sampling.metapath_randomwalk(hg, nodes, "r0-r1-r0-r3", 10, seed=5)
    caches = {e: dict(hg[e]._walk_dev["cuda:0"]) for e in used}
    assert all("_walk_dev" not in hg[e].__dict__ for e in hg.edge_types if e not in used)
    pgl.sampling.metapath_randomwalk(hg, nodes, ["r3", "r1", "r0"], 10, seed=6)
    for e in used:
        again = hg[e]._walk_dev["cuda:0"]
        assert all(again[k] is caches[e][k] for k in caches[e]), e
    hg.tensor()
    assert all("_walk_dev" not in hg[e].__dict__ for e in hg.edge_types)
    got = pgl.sampling.metapath_randomwalk(hg, torch.as_tensor(nodes).cuda(), "r0-r1-r0-r3", 10, seed=5)
    assert W.as_lists(got.cpu().numpy()) == first
    hg.numpy()
    assert all("_walk_dev" not in hg[e].__dict__ for e in hg.edge_types)
    assert pgl.sampling.metapath_randomwalk(hg, nodes, "r0-r1-r0-r3", 10, seed=5) == first


def test_pgl_alias_import(pgl):
    from pgl.sampling import metapath_randomwalk
    edges, n, types = MO.kat_graph()
    hg = pgl.HeterGraph(edges=edges, num_nodes=n, node_types=types)
    csr = _host_csrs(hg)
    names = list(csr)
    idx = [names.index(e) for e in ("c2p", "p2a", "a2p", "p2c")]
    want = MO.replay_metapath([csr[e] for e in names], [0, 1, 2, 3], idx, 5, 3)
    assert metapath_randomwalk(hg, [0, 1, 2, 3], "c2p-p2a-a2p-p2c", 5, seed=3) == W.as_lists(want)


# ---------------------------------------------------------------------------------------------------------------
# a seeded MAG-like graph (scripts/bench_hetero_sampler.py's generator): 10^6 nodes, 10^7 edges, 5 relations
# ---------------------------------------------------------------------------------------------------------------
MAG_METAPATHS = ["rev_writes-writes", "cites-rev_writes-writes"]


@pytest.fixture(scope="module")
def mag(pgl):
    spec = importlib.util.spec_from_file_location("bench_hetero_sampler",
                                                  os.path.join(ROOT, "scripts", "bench_hetero_sampler.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    edges, n, types = mod.mag_like(500_000, 490_000, 10_000, 10_000_000, seed=3)
    hg = pgl.HeterGraph(edges=edges, num_nodes=n, node_types=types)
    yield hg, n
    del hg, edges
    torch.cuda.empty_cache()


def _edge_keys(g, n):
    indptr, cols, _ = g._walk_csr()
    rows = torch.repeat_interleave(torch.arange(n, device="cuda"), indptr[1:] - indptr[:-1])
    return torch.unique(rows * n + cols)


@pytest.mark.parametrize("metapath", MAG_METAPATHS)
def test_mag_walks_follow_the_relations_and_stop_only_at_their_sinks(pgl, mag, metapath):
    hg, n = mag
    etypes = metapath.split("-")
    M = len(etypes)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    nodes = torch.randint(0, 500_000, (1_000_000,), device="cuda", generator=gen)   # papers
    L = 40
    out = pgl.sampling.metapath_randomwalk(hg, nodes, metapath, L, seed=123)
    assert out.shape == (nodes.numel(), L) and torch.equal(out[:, 0], nodes)
    valid = out >= 0
    length = valid.sum(1)
    assert torch.equal(valid, torch.arange(L, device="cuda")[None, :] < length[:, None])   # -1 only as a suffix
    for pos, e in enumerate(etypes):
        keys = _edge_keys(hg[e], n)
        t = torch.arange(pos, L - 1, M, device="cuda")
        a, b = out[:, t], out[:, t + 1]
        k = (a * n + b)[valid[:, t + 1]]
        assert k.numel() > 0
        at = torch.searchsorted(keys, k).clamp_max(keys.numel() - 1)
        assert torch.equal(keys[at], k), "a step of position %d that is not a %s edge" % (pos, e)
    degs = torch.stack([hg[e]._walk_csr()[0].diff() for e in etypes])
    last = out.gather(1, (length - 1)[:, None]).squeeze(1)
    short = length < L
    assert short.any() and not short.all()
    assert torch.equal(short, short & (degs[(length - 1) % M, last] == 0)), "a walk stopped where it could go on"


def _chi2(samples, probs):
    keys = sorted(probs)
    s = np.sort(samples)
    obs = np.array([np.searchsorted(s, k, "right") - np.searchsorted(s, k, "left") for k in keys], np.float64)
    assert obs.sum() == len(samples)
    exp = np.array([probs[k] for k in keys]) * len(samples)
    return stats.chisquare(obs, exp).pvalue


@pytest.mark.parametrize("metapath", MAG_METAPATHS)
def test_mag_first_step_out_of_a_hub(pgl, mag, metapath):
    hg, n = mag
    e = metapath.split("-")[0]
    indptr, cols, _ = hg[e]._walk_csr()
    hub = int(indptr.diff().argmax().item())
    out = pgl.sampling.metapath_randomwalk(hg, torch.full((1_000_000,), hub, device="cuda"), metapath, 2, seed=77)
    row = cols[indptr[hub]:indptr[hub + 1]].cpu().numpy()
    assert len(row) >= 10
    probs = W.node_probs(np.array([0, len(row)]), row, [0], W.UNIFORM)
    assert _chi2(out[:, 1].cpu().numpy(), probs) > 1e-4
