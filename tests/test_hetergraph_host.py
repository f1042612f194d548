"""pgl.HeterGraph on the host (numpy mode): the reference's known answers (tests/golden/kat_hetergraph.json), node
batches by type, dump / load in the reference's directory layout, the deliberate differences from the reference, and a
numpy model of the relation-typed CSRs that RGCNConv's fused aggregation runs on (heter_graph.typed_csr; the GPU test
checks the device build against this model)."""
import json
import os
import pickle

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    return pgl_b200


@pytest.fixture(scope="module")
def kat():
    with open(os.path.join(GOLDEN, "kat_hetergraph.json")) as f:
        return json.load(f)


def build(pgl, kat, with_feat=True):
    rng = np.random.default_rng(1)
    n = kat["num_nodes"]
    edges = {t: [tuple(e) for e in v] for t, v in kat["edges"].items()}
    node_types = [(i, t) for i, t in enumerate(kat["node_types"])]
    nfeat = {"nfeat": rng.standard_normal((n, 4))} if with_feat else None
    efeat = {t: {"efeat": rng.standard_normal((len(v), 4))} for t, v in edges.items()} if with_feat else None
    return pgl.HeterGraph(edges=edges, node_types=node_types, node_feat=nfeat, edge_feat=efeat)


def test_reference_known_answers(pgl, kat):
    """With one node id the per-type degree is a scalar, as in the reference (whose test compares it to [n])."""
    hg = build(pgl, kat)
    a = kat["answers"]
    assert not hg.is_tensor()
    assert np.atleast_1d(hg.indegree(5)).tolist() == a["indegree_5"]
    assert np.atleast_1d(hg.outdegree(4)).tolist() == a["outdegree_4"]
    assert np.atleast_1d(hg.outdegree(4, "c2p")).tolist() == a["outdegree_4_c2p"]
    assert np.atleast_1d(hg.indegree(5, "c2p")).tolist() == a["indegree_5_c2p"]
    assert np.atleast_1d(hg.outdegree(4, "p2a")).tolist() == a["outdegree_4_p2a"]
    assert [list(s) for s in hg.successor("c2p", [4])] == a["successor_c2p_4"]
    assert [list(p) for p in hg.predecessor("a2p", [4])] == a["predecessor_a2p_4"]


def test_basic_information(pgl, kat):
    hg = build(pgl, kat)
    assert hg.edge_types == ["c2p", "p2c", "p2a", "a2p"] == hg.edge_types_info()
    assert hg.num_nodes == 15
    assert hg.num_edges == {"c2p": 10, "p2c": 10, "p2a": 12, "a2p": 12}
    assert list(hg.node_types) == kat["node_types"]
    assert hg.num_nodes_by_type("p") == 6 and hg.num_nodes_by_type("a") == 5
    assert np.array_equal(hg.nodes, np.arange(15))
    assert hg["p2a"].num_edges == 12
    assert set(hg.edge_feat) == set(hg.edge_types) and hg.edge_feat["c2p"]["efeat"].shape == (10, 4)
    # summed over types when edge_type is None
    want = sum(hg.indegree(edge_type=t) for t in hg.edge_types)
    assert np.array_equal(hg.indegree(), want)


def test_node_batch_iter_by_type(pgl, kat):
    hg = build(pgl, kat)
    batches = list(hg.node_batch_iter(3, n_type="p"))
    assert [b.tolist() for b in batches] == [[4, 5, 6], [7, 8, 9]]
    assert sum(len(b) for b in hg.node_batch_iter(4)) == 15
    np.random.seed(0)
    got = np.concatenate(list(hg.node_batch_iter(2, shuffle=True, n_type="a")))
    assert sorted(got.tolist()) == [10, 11, 12, 13, 14]
    assert list(hg.node_batch_iter(2, n_type="a"))[0].tolist() == [10, 11]   # the type's node list is not shuffled


def test_node_feat_shared_not_copied(pgl, kat):
    hg = build(pgl, kat)
    arrays = [hg[t].node_feat["nfeat"] for t in hg.edge_types]
    dicts = [hg[t].node_feat for t in hg.edge_types]
    assert all(a is arrays[0] for a in arrays)
    assert len({id(d) for d in dicts}) == len(dicts)
    assert hg.node_feat["nfeat"] is arrays[0]


def test_deliberate_differences(pgl, kat):
    hg = build(pgl, kat)
    with pytest.raises(ValueError):
        hg.num_nodes_by_type("x")
    with pytest.raises(NotImplementedError):
        hg.sample_successor("c2p", [1], 2)
    with pytest.raises(NotImplementedError):
        hg.sample_predecessor("c2p", [4], 2)


def test_dump_load_round_trip(pgl, kat, tmp_path):
    hg = build(pgl, kat)
    hg.dump(str(tmp_path / "hg"), indegree=True, outdegree=True)
    assert sorted(os.listdir(tmp_path / "hg")) == sorted(["node_types.npy", "edge_types.pkl"] + hg.edge_types)
    for mmap in ("r", None):
        lg = pgl.HeterGraph.load(str(tmp_path / "hg"), mmap_mode=mmap)
        assert lg.edge_types == hg.edge_types and list(lg.node_types) == list(hg.node_types)
        for t in hg.edge_types:
            assert np.array_equal(lg[t].edges, hg[t].edges)
            assert np.array_equal(lg[t].edge_feat["efeat"], hg[t].edge_feat["efeat"])
        assert np.array_equal(lg.node_feat["nfeat"], hg.node_feat["nfeat"])
        assert lg.indegree(5).tolist() == [2] and lg.num_nodes_by_type("c") == 4


def test_load_reference_layout(pgl, kat, tmp_path):
    """A directory as the reference's HeterGraph.dump writes it: node_types.npy (object array), edge_types.pkl and
    per edge type Graph.dump's files (num_nodes.npy, edges.npy, num_graph.npy, graph_*_index.npy, node_feat/)."""
    root = tmp_path / "ref"
    root.mkdir()
    np.save(root / "node_types.npy", np.array([(i, t) for i, t in enumerate(kat["node_types"])], dtype=object)[:, 1])
    etypes = list(kat["edges"])
    with open(root / "edge_types.pkl", "wb") as f:
        pickle.dump(etypes, f)
    feat = np.arange(15 * 2, dtype=np.float64).reshape(15, 2)
    for t in etypes:
        d = root / t
        (d / "node_feat").mkdir(parents=True)
        e = np.asarray(kat["edges"][t], np.int64)
        np.save(d / "num_nodes.npy", np.int64(15))
        np.save(d / "edges.npy", e)
        np.save(d / "num_graph.npy", np.int64(1))
        np.save(d / "graph_node_index.npy", np.array([0, 15], np.int64))
        np.save(d / "graph_edge_index.npy", np.array([0, len(e)], np.int64))
        np.save(d / "node_feat" / "nfeat.npy", feat)
    hg = pgl.HeterGraph.load(str(root))
    assert hg.edge_types == etypes and hg.num_nodes == 15
    assert np.atleast_1d(hg.outdegree(4)).tolist() == [7]
    assert [list(p) for p in hg.predecessor("a2p", [4])] == [[10, 11, 12, 14, 13]]
    assert np.array_equal(hg.node_feat["nfeat"], feat)


@pytest.mark.gpu
def test_tensor_numpy_conversions(pgl, kat):
    import torch
    hg = build(pgl, kat)
    t = hg.tensor(inplace=False)
    assert t.is_tensor() and not hg.is_tensor()
    assert isinstance(t.node_feat["nfeat"], torch.Tensor) and t.node_feat["nfeat"].is_cuda
    assert all(t[e].node_feat["nfeat"] is t.node_feat["nfeat"] for e in t.edge_types)   # one device copy
    assert int(t.indegree(torch.tensor([5]).cuda())[0]) == 2
    assert int(t.outdegree(torch.tensor([4]).cuda(), "p2a")[0]) == 5
    assert [b.tolist() for b in t.node_batch_iter(3, n_type="c")] == [[0, 1, 2], [3]]
    back = t.numpy(inplace=False)
    assert not back.is_tensor() and t.is_tensor()
    assert np.array_equal(back.node_feat["nfeat"], hg.node_feat["nfeat"])
    assert hg.tensor() is hg and hg.is_tensor() and hg["c2p"].is_tensor()
    assert all(hg[e].node_feat["nfeat"] is hg.node_feat["nfeat"] for e in hg.edge_types)
    assert hg.numpy() is hg and not hg.is_tensor() and not hg["a2p"].is_tensor()
    assert np.atleast_1d(hg.indegree(5)).tolist() == [2]


# ---- the relation-typed CSRs (heter_graph.typed_csr), modelled in numpy -------------------------------------------

def typed_csr_model(edge_lists, n):
    """Relations' edges concatenated in order, stably sorted by dst (fwd) / src (bwd): every row's slots grouped by
    relation in relation order, ascending eid inside a group; the (row, relation) runs sorted by relation (stable);
    the bwd slot weight 1 / cnt_r(dst)."""
    src = np.concatenate([np.asarray(e, np.int64).reshape(-1, 2)[:, 0] for e in edge_lists])
    dst = np.concatenate([np.asarray(e, np.int64).reshape(-1, 2)[:, 1] for e in edge_lists])
    rel_e = np.concatenate([np.full(len(np.asarray(e).reshape(-1, 2)), r, np.int16) for r, e in enumerate(edge_lists)])
    R = len(edge_lists)
    o = np.argsort(dst, kind="stable")
    rows, rel = dst[o], rel_e[o]
    indptr = np.concatenate([[0], np.cumsum(np.bincount(dst, minlength=n))])
    runs = []
    for j in range(len(o)):
        if j == 0 or rows[j] != rows[j - 1] or rel[j] != rel[j - 1]:
            runs.append([int(rel[j]), int(rows[j]), j, j + 1])
        else:
            runs[-1][3] = j + 1
    runs.sort(key=lambda q: q[0])       # list.sort is stable
    runs = np.asarray(runs, np.int64).reshape(-1, 4)
    cnt = {}
    for d, r in zip(dst, rel_e):
        cnt[(d, r)] = cnt.get((d, r), 0) + 1
    ob = np.argsort(src, kind="stable")
    fwd = {"indptr": indptr, "cols": src[o], "rel": rel, "run_row": runs[:, 1], "run_beg": runs[:, 2],
           "run_end": runs[:, 3],
           "run_off": np.concatenate([[0], np.cumsum(np.bincount(runs[:, 0], minlength=R))]).astype(np.int64)}
    bwd = {"indptr": np.concatenate([[0], np.cumsum(np.bincount(src, minlength=n))]), "cols": dst[ob],
           "rel": rel_e[ob], "w": np.array([np.float32(1) / np.float32(cnt[(dst[e], rel_e[e])]) for e in ob],
                                           np.float32)}
    return {"fwd": fwd, "bwd": bwd}


def test_typed_csr_model():
    # relation 0: multi-edge 0->2 twice, self-loop 2->2; relation 1 empty; relation 2: 1->2, 0->0
    el = [np.array([[0, 2], [2, 2], [0, 2], [1, 0]]), np.zeros((0, 2), np.int64), np.array([[1, 2], [0, 0]])]
    m = typed_csr_model(el, 4)
    f, b = m["fwd"], m["bwd"]
    assert f["indptr"].tolist() == [0, 2, 2, 6, 6]                  # row 1 and row 3 empty
    assert f["cols"].tolist() == [1, 0, 0, 2, 0, 1] and f["rel"].tolist() == [0, 2, 0, 0, 0, 2]
    # runs: (row 0, rel 0), (row 0, rel 2), (row 2, rel 0) [3 slots], (row 2, rel 2); sorted by relation
    assert f["run_row"].tolist() == [0, 2, 0, 2]
    assert list(zip(f["run_beg"].tolist(), f["run_end"].tolist())) == [(0, 1), (2, 5), (1, 2), (5, 6)]
    assert f["run_off"].tolist() == [0, 2, 2, 4]
    # src-keyed: node 0 -> [2 (r0), 2 (r0), 0 (r2)], node 1 -> [0 (r0), 2 (r2)], node 2 -> [2 (r0)]
    assert b["cols"].tolist() == [2, 2, 0, 0, 2, 2] and b["rel"].tolist() == [0, 0, 2, 0, 2, 0]
    assert np.allclose(b["w"], [1 / 3, 1 / 3, 1, 1, 1, 1 / 3])
    # a reordering only permutes relation ids and the groups inside every row
    m2 = typed_csr_model([el[2], el[1], el[0]], 4)
    assert m2["fwd"]["cols"].tolist() == [0, 1, 1, 0, 2, 0] and m2["fwd"]["rel"].tolist() == [0, 2, 0, 2, 2, 2]
    assert m2["fwd"]["run_off"].tolist() == [0, 2, 2, 4]
