"""CPU models of the relation-typed sampling kernels (csrc/sampling.cu: sample_typed_count_kernel,
sample_typed_fill_kernel) and of HeteroNeighborSampler's layer loop, statement by statement, checked without a GPU:

* count: per relation min(deg_r, k_r) over the runs found by binary search, and the exclusive scan;
* fill: the lane chunks of 32 relations, the scan over the lanes, the binary-search run lookup, and Floyd's selection
  with the kernel's hash (mix64), its draw counter base(seed, i) + r 2^32 + c and the multiply-high reduction;
* against oracle.check_sampled_neighbors applied per relation, against the existing Floyd model with one relation,
  and the layer loop's node order against a plain-Python first-appearance reindex.

tests/test_gpu_hetero_sampling.py checks the device output against these models bit for bit."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import oracle as O

M64 = (1 << 64) - 1
EMPTY = np.iinfo(np.int64).max


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                                     name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def mix64(z):
    z = (z + 0x9e3779b97f4a7c15) & M64
    z = ((z ^ (z >> 30)) * 0xbf58476d1ce4e5b9) & M64
    z = ((z ^ (z >> 27)) * 0x94d049bb133111eb) & M64
    return z ^ (z >> 31)


def draw_base(seed, i):                                  # draw_base
    return mix64((seed & M64) ^ mix64(i))


def floyd_subset(deg, k, base):                          # floyd_subset (the warp's any-hit is `t in chosen`)
    chosen = []
    for c in range(k):
        j = deg - k + c
        r = mix64((base + c) & M64)
        t = (r * (j + 1)) >> 64                          # __umul64hi
        if t in chosen:
            t = j
        chosen.append(t)
    return chosen


def rel_lower_bound(rel, lo, hi, r):                     # rel_lower_bound
    while lo < hi:
        mid = (lo + hi) >> 1
        if int(rel[mid]) < r:
            lo = mid + 1
        else:
            hi = mid
    return lo


def typed_run(rel, start, end, r, k):                    # typed_run: (lo relative to start, deg, take)
    b = rel_lower_bound(rel, start, end, r)
    deg = rel_lower_bound(rel, b, end, r + 1) - b
    return b - start, deg, (deg if (k < 0 or deg <= k) else k)


def typed_count_model(indptr, rel, R, sizes, nodes):
    """sample_typed_count_kernel + small_exclusive_scan_kernel: (count, offsets[n + 1])."""
    count = np.zeros(len(nodes), np.int64)
    for i, v in enumerate(nodes):
        start, end = int(indptr[v]), int(indptr[v + 1])
        total = 0
        if end > start:
            r1 = min(R - 1, int(rel[end - 1]))
            for r in range(max(0, int(rel[start])), r1 + 1):     # the lanes' relations, in any order
                k = sizes[r]
                if k != 0:
                    total += typed_run(rel, start, end, r, k)[2]
        count[i] = total
    return count, np.concatenate([[0], np.cumsum(count)]).astype(np.int64)


def typed_fill_model(indptr, cols, rel, eid, R, sizes, nodes, seed, offsets):
    """sample_typed_fill_kernel: (neighbors, rel, eids) of offsets[-1] slots."""
    m = int(offsets[-1])
    nb, orel, oeid = np.full(m, -1, np.int64), np.full(m, -1, np.int16), np.full(m, -1, np.int64)
    for i, v in enumerate(nodes):
        start, end = int(indptr[v]), int(indptr[v + 1])
        if end == start:
            continue
        base = draw_base(seed, i)
        o = int(offsets[i])
        r1 = min(R - 1, int(rel[end - 1]))
        for r0 in range(max(0, int(rel[start])), r1 + 1, 32):
            lanes = []
            for lane in range(32):                        # a lane per relation
                r = r0 + lane
                lo = deg = take = 0
                if r <= r1 and sizes[r] != 0:
                    lo, deg, take = typed_run(rel, start, end, r, sizes[r])
                lanes.append((lo, deg, take))
            incl = np.cumsum([t for _, _, t in lanes])     # __shfl_up_sync scan
            for src in range(32):                          # the ballot's lanes in order
                lo, deg, take = lanes[src]
                if take <= 0:
                    continue
                s0 = start + lo
                ro = o + int(incl[src]) - take
                rr = r0 + src
                pos = range(deg) if take == deg else floyd_subset(deg, take, (base + (rr << 32)) & M64)
                for c, q in enumerate(pos):
                    nb[ro + c] = cols[s0 + q]
                    orel[ro + c] = rr
                    oeid[ro + c] = eid[s0 + q] if eid is not None else s0 + q
            o += int(incl[-1])
    return nb, orel, oeid


def sample_typed_model(csr, R, sizes, nodes, seed, eid=None):
    """sample_typed_neighbors on the CPU: (neighbors, rel, count, eids)."""
    count, offsets = typed_count_model(csr["indptr"], csr["rel"], R, sizes, nodes)
    nb, rel, eids = typed_fill_model(csr["indptr"], csr["cols"], csr["rel"], eid, R, sizes, nodes, seed, offsets)
    return nb, rel, count, eids


def typed_in_csr_model(edge_lists, n):
    """heter_graph.typed_in_csr: relations concatenated, stably sorted by dst."""
    src = np.concatenate([np.asarray(e, np.int64).reshape(-1, 2)[:, 0] for e in edge_lists])
    dst = np.concatenate([np.asarray(e, np.int64).reshape(-1, 2)[:, 1] for e in edge_lists])
    rel_e = np.concatenate([np.full(len(np.asarray(e).reshape(-1, 2)), r, np.int16) for r, e in enumerate(edge_lists)])
    o = np.argsort(dst, kind="stable")
    return {"indptr": np.concatenate([[0], np.cumsum(np.bincount(dst, minlength=n))]).astype(np.int64),
            "cols": src[o], "rel": rel_e[o], "eid": o.astype(np.int64)}


def layer_loop_model(edge_lists, n, layer_sizes, nodes, seed, calls=0):
    """HeteroNeighborSampler.sample_neighbors: per layer one typed sampling (seed + calls), the kernels' reindex
    (test_sampling_model.reindex_model) and a stable partition per relation.  Returns [(per-relation [E_r, 2] block
    edges, block nodes, n_target)] outermost first, and the first layer's input nodes."""
    rx = _load("test_sampling_model").reindex_model
    csr = typed_in_csr_model(edge_lists, n)
    R = len(edge_lists)
    table = np.full(n, EMPTY, np.int64)
    out = []
    nodes = np.asarray(nodes, np.int64)
    for sizes in layer_sizes:
        calls += 1
        nb, rel, count, _ = sample_typed_model(csr, R, sizes, nodes, seed + calls)
        src, dst, index = rx(nodes, nb, count, n, table)
        order = np.argsort(rel, kind="stable")
        e = np.stack([src, dst], 1)[order]
        per = np.bincount(rel.astype(np.int64), minlength=R)
        out.append(([p for p in np.split(e, np.cumsum(per)[:-1])], index, len(nodes)))
        nodes = index
    return out, nodes


def rel_graph(n, R, seed, hub_slots=2000):
    """tests/test_gpu_rgcn.py's graph shape: empty rows (the last 10% of nodes), partial relation sets, multi-edges,
    self-loops and a hub row (node 3) whose in-edges are spread over the relations."""
    return _load("test_gpu_rgcn").rel_graph(n, R, seed, hub_slots=hub_slots)


def per_relation_csr(edges, n):
    o = np.argsort(edges[:, 1], kind="stable")
    return np.concatenate([[0], np.cumsum(np.bincount(edges[:, 1], minlength=n))]), edges[o, 0]


def test_binary_search_run_lookup():
    rel = np.array([0, 0, 2, 2, 2, 5, 7, 7], np.int16)
    assert typed_run(rel, 0, 8, 0, -1) == (0, 2, 2)
    assert typed_run(rel, 0, 8, 1, 3) == (2, 0, 0)
    assert typed_run(rel, 0, 8, 2, 1) == (2, 3, 1)
    assert typed_run(rel, 0, 8, 7, 5) == (6, 2, 2)
    assert typed_run(rel, 0, 8, 8, -1) == (8, 0, 0)
    assert typed_run(rel, 2, 5, 2, 4) == (0, 3, 3)      # a row [2, 5) of a longer slot array


@pytest.mark.parametrize("R", [1, 3, 40])
def test_model_against_oracle_per_relation(R):
    n = 600
    el = rel_graph(n, R, 100 + R)
    csr = typed_in_csr_model(el, n)
    rng = np.random.default_rng(R)
    nodes = np.concatenate([[3], rng.permutation(n)[:150]])        # the hub, empty rows, partial relation sets
    nodes = np.unique(nodes)[rng.permutation(len(np.unique(nodes)))]
    for sizes in ([-1] * R, [0] * R, [1] * R, [5] * R, [25] * R, list(rng.integers(-1, 30, R))):
        sizes = [int(k) for k in sizes]
        nb, rel, count, eids = sample_typed_model(csr, R, sizes, nodes, seed=7, eid=csr["eid"])
        count2, offsets = typed_count_model(csr["indptr"], csr["rel"], R, sizes, nodes)
        assert (count == count2).all() and offsets[-1] == len(nb)
        assert (np.diff(offsets) == count).all()
        # node-major, ascending relation inside a node
        for i in range(len(nodes)):
            assert (np.diff(rel[offsets[i]:offsets[i + 1]]) >= 0).all()
        owner = np.repeat(np.arange(len(nodes)), count)
        for r in range(R):
            sel = rel == r
            indptr_r, row_r = per_relation_csr(el[r], n)
            cnt_r = np.bincount(owner[sel], minlength=len(nodes))
            msg = O.check_sampled_neighbors(indptr_r, row_r, nodes, sizes[r], nb[sel], cnt_r)
            assert msg is None, (r, sizes[r], msg)
        # eids point back at an edge of the concatenation: (neighbour -> node) in relation rel
        src = np.concatenate([e[:, 0] for e in el])
        dst = np.concatenate([e[:, 1] for e in el])
        rel_e = np.concatenate([np.full(len(e), r) for r, e in enumerate(el)])
        assert (src[eids] == nb).all() and (dst[eids] == nodes[owner]).all() and (rel_e[eids] == rel).all()
        # a pure function of the seed; another seed draws another subset
        assert all((a == b).all() for a, b in zip((nb, rel, count), sample_typed_model(csr, R, sizes, nodes, 7)[:3]))
    nb7 = sample_typed_model(csr, R, [5] * R, nodes, 7)[0]
    nb8 = sample_typed_model(csr, R, [5] * R, nodes, 8)[0]
    assert not (nb7 == nb8).all()


def floyd_model_existing(deg, k, seed, i):
    """tests/test_sampling_model.py's model of sample_fill_kernel's Floyd, restated."""
    base = mix64(seed ^ mix64(i))
    chosen = []
    for c in range(k):
        j = deg - k + c
        r = mix64((base + c) & M64)
        t = (r * (j + 1)) >> 64
        if t in chosen:
            t = j
        chosen.append(t)
    return chosen


def test_one_relation_is_sample_fill():
    n = 400
    el = rel_graph(n, 1, 5)
    csr = typed_in_csr_model(el, n)
    nodes = np.random.default_rng(3).permutation(n)[:120]
    for k in (-1, 0, 1, 5, 25, 300):
        for seed in (0, 11, (1 << 64) - 3):
            nb, rel, count, eids = sample_typed_model(csr, 1, [k], nodes, seed)
            want, wcnt = [], []
            for i, v in enumerate(nodes):
                s, e = int(csr["indptr"][v]), int(csr["indptr"][v + 1])
                deg = e - s
                pos = range(deg) if (k < 0 or deg <= k) else floyd_model_existing(deg, k, seed, i)
                want += [csr["cols"][s + t] for t in pos]
                wcnt.append(len(pos))
            assert nb.tolist() == want and count.tolist() == wcnt and (rel == 0).all()


def test_relations_draw_independent_streams():
    """The same run length and fan-out in two relations of one row draw different subsets (counter r 2^32 + c)."""
    el = [np.stack([np.arange(100), np.zeros(100, np.int64)], 1) for _ in range(2)]
    csr = typed_in_csr_model(el, 100)
    nb, rel, count, eids = sample_typed_model(csr, 2, [10, 10], np.array([0]), seed=1)
    a, b = eids[rel == 0], eids[rel == 1] - 100
    assert count.tolist() == [20] and sorted(a.tolist()) != sorted(b.tolist())


def test_layer_loop_node_order():
    """The layer loop's blocks: node order = plain-Python first appearance (seeds first), edges = the sampled
    neighbour -> target pairs of each relation in node-major order."""
    n, R = 500, 4
    el = rel_graph(n, R, 9)
    seeds = np.random.default_rng(4).permutation(n)[:40]
    layers = [[5, 0, -1, 2], [3] * R]
    blocks, first = layer_loop_model(el, n, layers, seeds, seed=13)
    csr = typed_in_csr_model(el, n)
    nodes, calls = seeds, 0
    for (parts, index, n_target), sizes in zip(blocks, layers):
        calls += 1
        nb, rel, count, _ = sample_typed_model(csr, R, sizes, nodes, 13 + calls)
        order = {}
        for v in list(nodes) + list(nb):                  # first appearance
            order.setdefault(int(v), len(order))
        assert index.tolist() == list(order.keys()) and n_target == len(nodes)
        owner = np.repeat(nodes, count)
        for r in range(R):
            got = index[parts[r]]                         # block ids -> global ids
            assert got[:, 0].tolist() == nb[rel == r].tolist()
            assert got[:, 1].tolist() == owner[rel == r].tolist()
        assert len(parts) == R and (sizes[1] != 0 or len(parts[1]) == 0)   # fan-out 0: empty, still present
        nodes = index
    assert (first == nodes).all()
