"""HeterGraph: PGL's heterogeneous graph (mirror of reference pgl/heter_graph.py) -- one homogeneous ``Graph`` per
edge type over a shared node set, plus the relation-typed CSRs that RGCNConv's fused aggregation runs on.

What differs from the reference by design (DESIGN.md section 7):
 * every relation Graph gets its own ``node_feat`` dict, but the dicts share the arrays (the reference deep-copies
   node_feat into every relation: R copies of [N, D]);
 * ``num_nodes_by_type`` with an unknown type raises ValueError (the reference raises a str, a TypeError);
 * ``sample_successor`` / ``sample_predecessor`` raise NotImplementedError: Graph has no samplers here.
"""
import os
import pickle as pkl

import numpy as np
import torch

from . import ops
from .graph import Graph
from .utils.helper import to_tensor

__all__ = ["HeterGraph"]


class HeterGraph(object):
    """Heterogeneous graph (reference pgl/heter_graph.py:33-511).

    Args:
        edges: dict etype -> list of (u, v) tuples, [E, 2] numpy.ndarray or torch.Tensor.
        num_nodes: optional node count (default len(node_types)).
        node_types: list of (node id, type) tuples, or an array of the type of every node.
        node_feat: optional dict name -> [num_nodes, ...] array, shared by every relation.
        edge_feat: optional dict etype -> dict name -> array.
        multi_graph: (keyword) dict etype -> Graph, used instead of ``edges``.
    """

    def __init__(self, edges, num_nodes=None, node_types=None, node_feat=None, edge_feat=None, **kwargs):
        self._edges_dict = edges
        if isinstance(node_types, list):
            self._node_types = np.array(node_types, dtype=object)[:, 1]
        else:
            self._node_types = node_types
        self._num_nodes = len(node_types) if num_nodes is None else num_nodes
        self._nodes_type_dict = {}
        for ntype in np.unique(self._node_types):
            self._nodes_type_dict[ntype] = np.where(self._node_types == ntype)[0]
        self._node_feat = node_feat if node_feat is not None else {}
        self._edge_feat = edge_feat if edge_feat is not None else {}

        if "multi_graph" in kwargs:
            self._multi_graph = kwargs["multi_graph"]
        else:
            self._multi_graph = {}
            for etype, _edges in self._edges_dict.items():
                efeat = self._edge_feat[etype] if self._edge_feat else None
                self._multi_graph[etype] = Graph(edges=_edges, num_nodes=self._num_nodes,
                                                 node_feat=dict(self._node_feat), edge_feat=efeat)
            self._share_node_feat()

        self._edge_types = self.edge_types_info()
        self._nodes = None
        first = next(iter(self._multi_graph.values()))
        self._is_tensor = first.is_tensor()

    def _share_node_feat(self, feat=None):
        """Give every relation Graph its own dict over the same arrays (the first relation's by default)."""
        graphs = list(self._multi_graph.values())
        if not graphs:
            return
        feat = graphs[0]._node_feat if feat is None else feat
        for g in graphs:
            g._node_feat = dict(feat)

    def is_tensor(self):
        return self._is_tensor

    @property
    def edge_types(self):
        return self._edge_types

    @property
    def num_nodes(self):
        return self._multi_graph[self._edge_types[0]].num_nodes

    @property
    def num_edges(self):
        return {etype: self._multi_graph[etype].num_edges for etype in self._edge_types}

    @property
    def node_types(self):
        return self._node_types

    @property
    def edge_feat(self):
        return {etype: g.edge_feat for etype, g in self._multi_graph.items()}

    @property
    def node_feat(self):
        return self._multi_graph[self._edge_types[0]].node_feat

    @property
    def nodes(self):
        if self._nodes is None:
            g = self._multi_graph[self._edge_types[0]]
            self._nodes = g.nodes
        return self._nodes

    def __getitem__(self, edge_type):
        return self._multi_graph[edge_type]

    def num_nodes_by_type(self, n_type=None):
        if n_type not in self._nodes_type_dict:
            raise ValueError("%s is not in valid node type" % n_type)
        return len(self._nodes_type_dict[n_type])

    def _sum_over_types(self, degs):
        if self.is_tensor():
            return torch.stack(degs).sum(0)
        return np.sum(np.vstack(degs), axis=0)

    def indegree(self, nodes=None, edge_type=None):
        """In-degree of ``nodes`` (all nodes when None) in ``edge_type``, or summed over every type."""
        if edge_type is None:
            return self._sum_over_types([self._multi_graph[e].indegree(nodes) for e in self._edge_types])
        return self._multi_graph[edge_type].indegree(nodes)

    def outdegree(self, nodes=None, edge_type=None):
        """Out-degree of ``nodes`` (all nodes when None) in ``edge_type``, or summed over every type."""
        if edge_type is None:
            return self._sum_over_types([self._multi_graph[e].outdegree(nodes) for e in self._edge_types])
        return self._multi_graph[edge_type].outdegree(nodes)

    def successor(self, edge_type, nodes=None, return_eids=False):
        return self._multi_graph[edge_type].successor(nodes, return_eids)

    def predecessor(self, edge_type, nodes=None, return_eids=False):
        return self._multi_graph[edge_type].predecessor(nodes, return_eids)

    def sample_successor(self, edge_type, nodes, max_degree, return_eids=False, shuffle=False):
        raise NotImplementedError("HeterGraph.sample_successor: Graph has no neighbour samplers in pgl_b200 "
                                  "(DESIGN.md section 7)")

    def sample_predecessor(self, edge_type, nodes, max_degree, return_eids=False, shuffle=False):
        raise NotImplementedError("HeterGraph.sample_predecessor: Graph has no neighbour samplers in pgl_b200 "
                                  "(DESIGN.md section 7)")

    def node_batch_iter(self, batch_size, shuffle=False, n_type=None):
        """Batches of node ids, all nodes or those of type ``n_type``; reference heter_graph.py:349-378."""
        if n_type is None:
            nodes = np.arange(int(self._multi_graph[self._edge_types[0]]._n), dtype="int64")
        else:
            nodes = self._nodes_type_dict[n_type].copy()
        if shuffle:
            np.random.shuffle(nodes)
        if self.is_tensor():
            nodes = to_tensor(nodes)
        start = 0
        while start < len(nodes):
            yield nodes[start:start + batch_size]
            start += batch_size

    def edge_types_info(self):
        return list(self._multi_graph.keys())

    def _convert(self, to_t, inplace):
        feat = self.node_feat
        conv = (lambda v: to_tensor(v)) if to_t else \
            (lambda v: v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v))
        shared = {k: conv(v) for k, v in feat.items()}
        new_multi = {}
        for etype in self._edge_types:
            g = self._multi_graph[etype]
            kept = g._node_feat
            g._node_feat = {}         # the shared arrays are converted once, above
            new_multi[etype] = g.tensor(inplace) if to_t else g.numpy(inplace)
            if not inplace:
                g._node_feat = kept
        if inplace:
            self._is_tensor = to_t
            self._nodes = None
            self.__dict__.pop("_typed_csr", None)
            self._share_node_feat(shared)
            return self
        new = self.__class__(edges=None, node_types=self._node_types, multi_graph=new_multi)
        new._share_node_feat(shared)
        return new

    def tensor(self, inplace=True):
        """Tensor (CUDA) mode; reference heter_graph.py:393-423."""
        if self._is_tensor:
            return self
        return self._convert(True, inplace)

    def numpy(self, inplace=True):
        """numpy mode; reference heter_graph.py:425-454."""
        if not self._is_tensor:
            return self
        return self._convert(False, inplace)

    def dump(self, path, indegree=False, outdegree=False):
        """The reference's layout: node_types.npy, edge_types.pkl and one Graph.dump directory per edge type."""
        if indegree:
            for g in self._multi_graph.values():
                g.indegree()
        if outdegree:
            for g in self._multi_graph.values():
                g.outdegree()
        if not os.path.exists(path):
            os.makedirs(path)
        np.save(os.path.join(path, "node_types.npy"), self._node_types)
        with open(os.path.join(path, "edge_types.pkl"), "wb") as f:
            pkl.dump(self._edge_types, f)
        for etype, g in self._multi_graph.items():
            g.dump(os.path.join(path, etype))

    @classmethod
    def load(cls, path, mmap_mode="r"):
        """A numpy-mode HeterGraph from a directory written by ``dump`` (or the reference's)."""
        node_types = np.load(os.path.join(path, "node_types.npy"), allow_pickle=True)
        with open(os.path.join(path, "edge_types.pkl"), "rb") as f:
            edge_types = pkl.load(f)
        multi = {etype: Graph.load(os.path.join(path, etype), mmap_mode) for etype in edge_types}
        new = cls(edges=None, node_types=node_types, multi_graph=multi)
        new._share_node_feat()
        return new

    # ------------------------------------------------------------------
    # relation-typed CSRs of RGCNConv's fused aggregation (ops.rgcn_aggregate)
    # ------------------------------------------------------------------
    def typed_csr(self, etypes, device):
        """(fwd, bwd) of ``ops.rgcn_aggregate`` for the relations ``etypes`` (any subset or order of the edge types;
        relation r is etypes[r]), built once per (etypes, device) and cached here.  See ``typed_csr``."""
        key = (tuple(etypes), str(torch.device(device)))
        cache = self.__dict__.setdefault("_typed_csr", {})
        if key not in cache:
            n = int(self._multi_graph[self._edge_types[0]]._n)
            cache[key] = typed_csr([to_tensor(self._multi_graph[e].edges, device).to(device) for e in etypes], n)
        return cache[key]


def typed_in_csr(edge_lists, num_nodes):
    """The dst-keyed CSR of all relations together: the edges of ``edge_lists[r]`` ([E_r, 2] int64 CUDA tensors,
    (src, dst) rows) concatenated in order and run through the stable ``ops.csr_build``, so the slots of every row
    come out grouped by relation in ascending relation id, ascending eid inside a group.  Returns a dict: indptr,
    cols (src), rows (dst), eid (index into the concatenation), rel (int16 relation per slot), and per edge of the
    concatenation src, dst, rel_e.  The typed sampler (sampling.sample_typed_neighbors) reads indptr / cols / rel."""
    dev = edge_lists[0].device
    src = torch.cat([e.reshape(-1, 2)[:, 0] for e in edge_lists])
    dst = torch.cat([e.reshape(-1, 2)[:, 1] for e in edge_lists])
    rel_e = torch.cat([torch.full((int(e.reshape(-1, 2).shape[0]),), r, dtype=torch.int16, device=dev)
                       for r, e in enumerate(edge_lists)])
    _, cols, rows, eid, indptr = ops.csr_build(dst, src, num_nodes)
    return {"indptr": indptr, "cols": cols, "rows": rows, "eid": eid, "rel": rel_e.index_select(0, eid),
            "src": src, "dst": dst, "rel_e": rel_e}


def typed_csr(edge_lists, num_nodes):
    """The relation-typed CSRs of edge lists ``edge_lists[r]`` ([E_r, 2] int64 CUDA tensors, (src, dst) rows) over
    ``num_nodes`` nodes, on ``typed_in_csr``'s layout.

    fwd (dst-keyed): indptr, cols (src), rel (int16 relation per slot); the run list of the weight gradient --
    run_row / run_beg / run_end of every (row, relation) group, sorted by relation (stable), run_off [R + 1] --
    and its work items: chunk runs per item, item_off [R + 1], n_items; tile_rels, the number of distinct
    (64-row tile, relation) pairs, each of which stages one W_r in the forward kernel.
    bwd (src-keyed): indptr, cols (dst), rel, w = 1 / cnt_r(dst) per slot."""
    R = len(edge_lists)
    dev = edge_lists[0].device
    t = typed_in_csr(edge_lists, num_nodes)
    src, dst, rel_e = t["src"], t["dst"], t["rel_e"]
    cols, rows, eid, indptr, rel = t["cols"], t["rows"], t["eid"], t["indptr"], t["rel"]
    E = int(src.shape[0])
    brk = torch.ones(E, dtype=torch.bool, device=dev)
    if E > 1:
        brk[1:] = (rel[1:] != rel[:-1]) | (rows[1:] != rows[:-1])
    beg = torch.nonzero(brk).reshape(-1)
    end = torch.cat([beg[1:], torch.full((1,), E, dtype=torch.int64, device=dev)])[:beg.shape[0]]
    run_rel = rel.index_select(0, beg).long()
    order = torch.sort(run_rel, stable=True).indices
    counts = torch.bincount(run_rel, minlength=R)
    run_off = torch.zeros(R + 1, dtype=torch.int64, device=dev)
    run_off[1:] = torch.cumsum(counts, 0)

    # work items of the weight gradient: about two per SM over all runs, at least 64 runs each
    T = int(beg.shape[0])
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    chunk = max(64, -(-T // (2 * sms)))
    chunk = -(-chunk // 64) * 64
    items = (counts + chunk - 1) // chunk
    item_off = torch.zeros(R + 1, dtype=torch.int64, device=dev)
    item_off[1:] = torch.cumsum(items, 0)
    tile_rels = int(torch.unique(rows.index_select(0, beg) // 64 * R + run_rel).shape[0]) if T else 0
    fwd = {"indptr": indptr, "cols": cols, "rel": rel, "run_row": rows.index_select(0, beg).index_select(0, order),
           "run_beg": beg.index_select(0, order), "run_end": end.index_select(0, order), "run_off": run_off,
           "item_off": item_off, "n_items": int(item_off[-1].item()), "chunk": chunk, "num_rels": R,
           "n_rows": int(num_nodes), "tile_rels": tile_rels}

    # 1 / cnt_r(dst) per edge (cnt = the length of the edge's run), then per src-CSR slot
    run_of = torch.cumsum(brk.to(torch.int64), 0) - 1
    cnt_slot = (end - beg).index_select(0, run_of)
    cnt_e = torch.empty(E, dtype=torch.int64, device=dev)
    cnt_e[eid] = cnt_slot
    _, scols, _, seid, sindptr = ops.csr_build(src, dst, num_nodes)
    bwd = {"indptr": sindptr, "cols": scols, "rel": rel_e.index_select(0, seid),
           "w": 1.0 / cnt_e.index_select(0, seid).to(torch.float32), "num_rels": R, "n_rows": int(num_nodes)}
    return fwd, bwd
