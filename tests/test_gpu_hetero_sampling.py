"""Relation-typed neighbour sampling on the GPU (csrc/sampling.cu: sample_typed_*; pgl_b200.sampling:
sample_typed_neighbors, HeteroNeighborSampler): bit-exact against the CPU models of test_hetero_sampling_model.py,
per-relation properties and uniformity, the one-relation identity with sample_neighbors / NeighborSampler, mini-batch
RGCNConv on the blocks against the full graph, the fused route, empty relations and blocks, and argument checks."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu
FWD_BOUND = 2e-5    # of the output's largest magnitude (test_gpu_rgcn.py)
GRAD_BOUND = 1e-4


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                                     name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


M = _load("test_hetero_sampling_model")
RG = _load("test_gpu_rgcn")


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    return pgl_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def device_csr(pgl, el, n):
    return pgl.heter_graph.typed_in_csr([dev(e) for e in el], n)


def pick_nodes(n, count, seed):
    """The hub (node 3), two empty rows (the last 10% of the nodes) and random others, distinct, shuffled."""
    rng = np.random.default_rng(seed)
    nodes = np.unique(np.concatenate([[3, n - 1, n - 2], rng.permutation(n)[:count]]))
    return nodes[rng.permutation(len(nodes))].astype(np.int64)


def grads_or_zeros(out, inputs, gout):
    """torch.autograd.grad with a zero gradient for an input the output does not use (a graph without edges)."""
    g = torch.autograd.grad(out, inputs, gout, allow_unused=True)
    return [torch.zeros_like(i) if v is None else v for i, v in zip(inputs, g)]


@pytest.mark.parametrize("R", [1, 3, 64])
def test_bit_exact_against_model(pgl, R):
    from pgl_b200.sampling import sample_typed_neighbors
    n = 3000
    el = RG.rel_graph(n, R, 40 + R)
    csr = device_csr(pgl, el, n)
    mcsr = M.typed_in_csr_model(el, n)
    for k in ("indptr", "cols", "rel", "eid"):
        assert np.array_equal(host(csr[k]), mcsr[k]), k
    nodes = pick_nodes(n, 250, R)
    rng = np.random.default_rng(R + 1)
    cases = [[k] * R for k in (-1, 0, 1, 5, 25, 300)] + [[int(v) for v in rng.choice([-1, 0, 1, 5, 25, 300], R)]]
    for sizes in cases:
        for seed in (0, 12345):
            nb, rel, cnt, eids = sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], dev(nodes), sizes,
                                                        eids=csr["eid"], return_eids=True, seed=seed)
            wnb, wrel, wcnt, weid = M.sample_typed_model(mcsr, R, sizes, nodes, seed, eid=mcsr["eid"])
            assert np.array_equal(host(cnt), wcnt), sizes
            assert np.array_equal(host(nb), wnb) and np.array_equal(host(rel), wrel), sizes
            assert np.array_equal(host(eids), weid), sizes


def test_sampler_blocks_match_layer_loop_model(pgl):
    """Per-relation dict fan-outs through HeteroNeighborSampler: every block bit for bit the CPU layer loop's."""
    n, R = 2000, 3
    etypes = ["cites", "writes", "owns"]
    el = RG.rel_graph(n, R, 61, hub_slots=3000)
    g = RG.make_heter(pgl, el, n, etypes)
    layers = [{"cites": 4, "writes": -1, "owns": 0}, {"cites": 2, "writes": 3, "owns": 25}]
    sampler = pgl.sampling.HeteroNeighborSampler(g, layers, seed=5)
    seeds = pick_nodes(n, 60, 8)
    blocks, first = sampler.sample_neighbors(dev(seeds))
    want, wfirst = M.layer_loop_model(el, n, [[d[e] for e in etypes] for d in layers], seeds, seed=5)
    assert np.array_equal(host(first), wfirst)
    for (block, n_target), (parts, index, wt) in zip(blocks, want[::-1]):
        assert n_target == wt and int(block.num_nodes) == len(index)
        assert block.edge_types == etypes and block.is_tensor()
        for e, p in zip(etypes, parts):
            assert np.array_equal(host(block[e].edges).reshape(-1, 2), p.reshape(-1, 2)), e
        assert list(block.node_types) == ["v"] * len(index)


@pytest.mark.parametrize("R", [3, 64])
def test_properties_per_relation(pgl, R):
    from pgl_b200.sampling import sample_typed_neighbors
    n = 3000
    el = RG.rel_graph(n, R, 80 + R)
    csr = device_csr(pgl, el, n)
    nodes = pick_nodes(n, 400, R + 3)
    owner = None
    eoff = np.concatenate([[0], np.cumsum([len(e) for e in el])])
    for k in (-1, 0, 1, 5, 25, 300):
        sizes = [k] * R
        nb, rel, cnt, eids = sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], dev(nodes), sizes,
                                                    eids=csr["eid"], return_eids=True, seed=3)
        nb_h, rel_h, cnt_h, eids_h = host(nb), host(rel), host(cnt), host(eids)
        owner = np.repeat(nodes, cnt_h)
        for r in range(R):
            sel = rel_h == r
            indptr_r, row_r = M.per_relation_csr(el[r], n)
            cnt_r = np.bincount(np.repeat(np.arange(len(nodes)), cnt_h)[sel], minlength=len(nodes))
            assert (cnt_r == np.minimum(np.diff(indptr_r)[nodes], k if k >= 0 else 1 << 40)).all(), (r, k)
            assert O.check_sampled_neighbors(indptr_r, row_r, nodes, k, nb_h[sel], cnt_r) is None, (r, k)
            local = eids_h[sel] - eoff[r]                 # (relation, local eid) of the parent
            assert ((local >= 0) & (local < len(el[r]))).all()
            assert (el[r][local, 0] == nb_h[sel]).all() and (el[r][local, 1] == owner[sel]).all()
        again = sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], dev(nodes), sizes, seed=3)
        assert torch.equal(again[0], nb) and torch.equal(again[1], rel) and torch.equal(again[2], cnt)


def test_uniform_on_the_hub_per_relation(pgl):
    from pgl_b200.sampling import sample_typed_neighbors
    n, R = 3000, 3
    el = RG.rel_graph(n, R, 90)
    csr = device_csr(pgl, el, n)
    indptr_h, rel_h = host(csr["indptr"]), host(csr["rel"])
    s, e = int(indptr_h[3]), int(indptr_h[4])
    k, trials = 8, 4000
    hits = [np.zeros(int((rel_h[s:e] == r).sum())) for r in range(R)]
    lo = [s + int(np.searchsorted(rel_h[s:e], r)) for r in range(R)]
    for t in range(trials // 100):
        _, rel, _, slots = sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], dev(np.full(100, 3)),
                                                  [k] * R, return_eids=True, seed=100 + t)
        rel, slots = host(rel), host(slots)
        for r in range(R):
            np.add.at(hits[r], slots[rel == r] - lo[r], 1)
    for r in range(R):
        deg = len(hits[r])
        assert deg > 1000
        expect = trials * k / deg
        assert abs(hits[r].mean() - expect) < 1e-9 and hits[r].std() < 6 * np.sqrt(expect) + 1, r


def test_one_relation_identity(pgl):
    from pgl_b200.sampling import NeighborSampler, HeteroNeighborSampler, sample_neighbors, sample_typed_neighbors
    n, e = 3000, 120000
    edges = O.chung_lu_edges(n, e, exponent=0.9, seed=711)
    g = pgl.Graph(edges=edges, num_nodes=n).tensor()
    row, colptr, geid = g.adj_dst_index._sorted_v, g.adj_dst_index._indptr, g.adj_dst_index._sorted_eid
    csr = device_csr(pgl, [edges], n)
    assert torch.equal(csr["indptr"], colptr) and torch.equal(csr["cols"], row) and torch.equal(csr["eid"], geid)
    nodes = dev(np.random.default_rng(712).permutation(n)[:700])
    for k in (-1, 0, 1, 5, 25, 40, 300):
        for seed in (3, (1 << 64) - 5):
            nb, cnt, eids = sample_neighbors(row, colptr, nodes, sample_size=k, eids=geid, return_eids=True,
                                             seed=seed)
            tnb, trel, tcnt, teids = sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], nodes, [k],
                                                            eids=csr["eid"], return_eids=True, seed=seed)
            assert torch.equal(nb, tnb) and torch.equal(cnt, tcnt) and torch.equal(eids, teids), k
            assert bool((trel == 0).all())
    # the sampler, block for block
    hg = pgl.HeterGraph(edges={"e": edges}, num_nodes=n, node_types=np.array(["v"] * n)).tensor()
    seeds = dev(np.arange(50, dtype=np.int64) * 7)
    a = NeighborSampler(g, [10, 5, -1], seed=1)
    b = HeteroNeighborSampler(hg, [10, 5, -1], seed=1)
    for _ in range(2):          # the per-call seeds advance alike
        ga, na = a.sample_neighbors(seeds)
        gb, nb_ = b.sample_neighbors(seeds)
        assert torch.equal(na, nb_) and len(ga) == len(gb)
        for (sa, ta), (sb, tb) in zip(ga, gb):
            assert ta == tb and int(sa.num_nodes) == int(sb.num_nodes)
            assert torch.equal(sa.edges, sb["e"].edges)


def ref_two_layers(x64, ws, el, n):
    """Two layers of the reference's op order in float64 (test_gpu_rgcn.ref_torch)."""
    return RG.ref_torch(RG.ref_torch(x64, ws[0], el, n), ws[1], el, n)


def conv_weight(conv, dtype):
    w = conv.weight.detach().to(dtype).requires_grad_()
    if conv.num_bases < conv.num_rels:
        c = conv.w_comp.detach().to(dtype).requires_grad_()
        return (w, c), torch.einsum("rb,bio->rio", c, w)
    return (w,), w


@pytest.mark.parametrize("num_bases", [0, 8])
def test_exact_receptive_field_matches_full_graph(pgl, num_bases, monkeypatch):
    n, R, D = 3000, 10, 64
    etypes = ["r%d" % r for r in range(R)]
    el = RG.rel_graph(n, R, 33, hub_slots=3000)
    g = RG.make_heter(pgl, el, n, etypes)
    torch.manual_seed(4)
    convs = [pgl.nn.RGCNConv(D, D, etypes, num_bases=num_bases).cuda() for _ in range(2)]
    x = torch.randn((n, D), generator=torch.Generator().manual_seed(9)).cuda()
    seeds = pick_nodes(n, 100, 21)
    gout = torch.randn((len(seeds), D), generator=torch.Generator().manual_seed(10)).cuda()

    routed = []
    real = pgl.ops.rgcn_aggregate

    def record(*a, **k):
        out = real(*a, **k)
        routed.append(out is not None)
        return out
    monkeypatch.setattr(pgl.ops, "rgcn_aggregate", record)

    sampler = pgl.sampling.HeteroNeighborSampler(g, [-1, -1], seed=2)
    blocks, nodes = sampler.sample_neighbors(dev(seeds))
    h = x[nodes]
    for conv, (block, n_target) in zip(convs, blocks):
        h = conv(block, h)[:n_target]
    assert routed == [True, True]                       # both blocks on the fused kernel
    with torch.no_grad():
        full = convs[1](g, convs[0](g, x))[dev(seeds)]
    assert RG.maxerr(h, full) <= FWD_BOUND
    grads = torch.autograd.grad(h, [p for c in convs for p in c.parameters()], gout)

    x64 = x.double()
    leaves, ws = zip(*[conv_weight(c, torch.float64) for c in convs])
    ref = ref_two_layers(x64, ws, el, n)[dev(seeds)]
    assert RG.maxerr(h, ref) <= FWD_BOUND
    want = torch.autograd.grad(ref, [p for lv in leaves for p in lv], gout.double())
    assert len(grads) == len(want)
    for a, b in zip(grads, want):
        assert a.shape == b.shape and RG.maxerr(a, b) <= GRAD_BOUND


def test_empty_relation_and_empty_block(pgl, monkeypatch):
    n, R, D = 2000, 4, 32
    etypes = ["a", "b", "c", "d"]
    el = RG.rel_graph(n, R, 55, hub_slots=800)
    g = RG.make_heter(pgl, el, n, etypes)
    conv = pgl.nn.RGCNConv(D, D, etypes).cuda()
    x = torch.randn((n, D), device="cuda")
    routed = []
    real = pgl.ops.rgcn_aggregate

    def record(*a, **k):
        out = real(*a, **k)
        routed.append(out is not None)
        return out
    monkeypatch.setattr(pgl.ops, "rgcn_aggregate", record)

    def both_routes(block, h):
        """The block on the fused route and on the per-relation route (a dict of its Graphs)."""
        hf = h.clone().requires_grad_()
        hd = h.clone().requires_grad_()
        a = conv(block, hf)
        b = conv({e: block[e] for e in etypes}, hd)
        gout = torch.randn_like(a)
        ga = grads_or_zeros(a, [hf] + list(conv.parameters()), gout)
        gb = grads_or_zeros(b, [hd] + list(conv.parameters()), gout)
        return a, b, ga, gb

    # a block whose relation "b" got no edges (fan-out 0), and "d" only some
    sampler = pgl.sampling.HeteroNeighborSampler(g, [{"a": 5, "b": 0, "c": -1, "d": 1}], seed=3)
    blocks, nodes = sampler.sample_neighbors(dev(pick_nodes(n, 80, 2)))
    (block, nt), = blocks
    assert block.edge_types == etypes and int(block["b"].num_edges) == 0 and int(block["a"].num_edges) > 0
    a, b, ga, gb = both_routes(block, x[nodes])
    assert routed == [True]
    assert RG.maxerr(a, b) <= 1e-4 and all(RG.maxerr(u, v) <= 1e-4 for u, v in zip(ga, gb))
    # targets without in-edges (the last 10% of the nodes receive nothing): a block with no edges at all
    empty = np.arange(n - 50, n, dtype=np.int64)
    sampler = pgl.sampling.HeteroNeighborSampler(g, [5, -1], seed=3)
    blocks, nodes = sampler.sample_neighbors(dev(empty))
    assert torch.equal(nodes.cpu(), torch.from_numpy(empty))
    for block, nt in blocks:
        assert nt == 50 and int(block.num_nodes) == 50 and block.edge_types == etypes
        assert all(int(block[e].num_edges) == 0 for e in etypes)
        routed.clear()
        a, b, ga, gb = both_routes(block, x[nodes])
        assert routed == [True]
        assert bool((a == 0).all()) and torch.equal(a, b)
        for u, v in zip(ga, gb):
            assert bool((u == 0).all()) and bool((v == 0).all())


def test_validation_before_any_launch(pgl):
    from pgl_b200.sampling import HeteroNeighborSampler, sample_typed_neighbors
    n, R = 500, 3
    etypes = ["a", "b", "c"]
    el = RG.rel_graph(n, R, 7, hub_slots=300)
    g = RG.make_heter(pgl, el, n, etypes)
    csr = device_csr(pgl, el, n)
    ok = dev(np.arange(10))
    hs = HeteroNeighborSampler(g, [5])
    bad_calls = [
        lambda: sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], dev(np.array([0, n])), [1] * R),
        lambda: sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], dev(np.array([-1, 0])), [1] * R),
        lambda: sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], ok, [1, 4097, 1]),
        lambda: sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], ok, [1, -2, 1]),
        lambda: sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], ok, [1, 1.5, 1]),
        lambda: sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], ok, [1, True, 1]),
        lambda: sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], ok, 5),
        lambda: sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], ok, [1, 1], num_rels=R),
        lambda: sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], ok, [1] * 32768),
        lambda: sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], ok, []),
        lambda: sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"].long(), ok, [1] * R),
        lambda: HeteroNeighborSampler(g, [5], uva=True),
        lambda: HeteroNeighborSampler(g, [5, "x"]),
        lambda: HeteroNeighborSampler(g, [5, 4097]),
        lambda: HeteroNeighborSampler(g, [{"a": 1, "b": 1}]),
        lambda: HeteroNeighborSampler(g, [{"a": 1, "b": 1, "c": 1, "z": 1}]),
        lambda: HeteroNeighborSampler(g, 5),
        lambda: HeteroNeighborSampler(g, [5], etypes=["a", "zz"]),
        lambda: hs.sample_neighbors(dev(np.array([1, 2, 1]))),
        lambda: hs.sample_neighbors(dev(np.array([1, n]))),
    ]
    for i, call in enumerate(bad_calls):
        torch.cuda.synchronize()
        l0 = pgl.ops.launch_count()
        with pytest.raises(ValueError):
            call()
        assert pgl.ops.launch_count() == l0, i
    # a sampler over a subset of the relations, in another order, with a dict naming exactly those
    s = HeteroNeighborSampler(g, [{"c": 2, "a": -1}], etypes=["c", "a"])
    (block, nt), = s.sample_neighbors(ok)[0]
    assert block.edge_types == ["c", "a"] and nt == 10
