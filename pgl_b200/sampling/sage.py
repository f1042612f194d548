"""NeighborSampler: layer-wise uniform neighbour sampling on the device for mini-batch GraphSAGE
(reference pgl/sampling/sage.py:130-155).  ``sample_neighbors`` / ``reindex_graph`` stand in for
``paddle.geometric.sample_neighbors`` / ``paddle.geometric.reindex_graph`` on the sm_90a kernels of
csrc/sampling.cu (validated on hardware in round 2: tests/test_gpu_sampling.py).

HeteroNeighborSampler: the same on a HeterGraph, every relation in one ``sample_typed_neighbors`` pass over the typed
in-CSR (DESIGN.md section 4.14); its blocks feed RGCNConv's fused aggregation."""
import ctypes

import numpy as np
import torch

from .. import ops
from .._lib import check, lib
from ..graph import Graph
from ..heter_graph import HeterGraph, typed_in_csr
from ..utils.helper import to_tensor

__all__ = ["NeighborSampler", "HeteroNeighborSampler", "sample_neighbors", "sample_typed_neighbors",
           "reindex_graph"]

MAX_FANOUT = 4096     # the kernels' cap: Floyd's chosen positions live in shared memory


def sample_neighbors(row, colptr, input_nodes, sample_size=-1, eids=None, return_eids=False, seed=0):
    """paddle.geometric.sample_neighbors: for every node of ``input_nodes`` up to ``sample_size``
    in-neighbours drawn uniformly without replacement from ``row[colptr[v]:colptr[v+1]]`` (all of them
    when sample_size is -1 or the degree is not larger).  Returns (neighbors, count[, eids])."""
    ops.require_cuda(row, colptr, input_nodes)
    nodes = input_nodes.reshape(-1).to(torch.int64).contiguous()
    n = int(nodes.shape[0])
    dev = nodes.device
    count = torch.empty(n, dtype=torch.int64, device=dev)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    with torch.cuda.device(dev):
        check(lib.pglb_sample_count(p(colptr), p(nodes), n, int(sample_size), p(count), p(offsets), stream))
    total = int(offsets[n].item())
    neighbors = torch.empty(total, dtype=torch.int64, device=dev)
    out_eids = torch.empty(total, dtype=torch.int64, device=dev) if return_eids else None
    if total > 0:  # sample_size == 0 (or no neighbours at all): nothing to fill, and an empty tensor has no address
        with torch.cuda.device(dev):
            check(lib.pglb_sample_fill(p(colptr), p(row), p(eids), p(nodes), n, int(sample_size),
                                       int(seed) & 0xFFFFFFFFFFFFFFFF, p(offsets), p(neighbors), p(out_eids),
                                       stream))
    neighbors._pglb_offsets = offsets  # rides along for reindex_graph (saves a scan)
    if return_eids:
        return neighbors, count, out_eids
    return neighbors, count


def _fanout(k):
    if isinstance(k, (bool, np.bool_)) or not isinstance(k, (int, np.integer)) or not -1 <= int(k) <= MAX_FANOUT:
        raise ValueError("a fan-out must be an int in [-1, %d] (-1: all neighbours), got %r" % (MAX_FANOUT, k))
    return int(k)


def sample_typed_neighbors(indptr, cols, rel, input_nodes, sample_sizes, eids=None, return_eids=False, seed=0,
                           num_rels=None):
    """Relation-typed ``sample_neighbors`` on a typed in-CSR (``heter_graph.typed_in_csr``: the slots of every row
    grouped by relation in ascending relation id; ``rel`` the int16 relation of every slot).  For every node of
    ``input_nodes`` and every relation r, up to ``sample_sizes[r]`` in-neighbours are drawn uniformly without
    replacement from the node's r-run (all of them when the fan-out is -1 or the run is not longer, none when it is 0),
    in one pass over all relations.  ``num_rels`` (default len(sample_sizes)) is R.

    Returns (neighbors, rel, count[, eids]): node-major, relation by relation in ascending order inside a node; rel is
    each sampled slot's relation, count the number per input node, eids ``eids[slot]`` (the slot when eids is None).
    The draws are a pure function of (seed, input position, relation, draw); with one relation they, and the output,
    equal ``sample_neighbors``'.  Raises ValueError, before any launch, for a node outside [0, N), a fan-out that is
    not an int in [-1, 4096], a number of fan-outs other than R, or R outside [1, 32767]."""
    ops.require_cuda(indptr, cols, rel, input_nodes, eids)
    if not isinstance(sample_sizes, (list, tuple)):
        raise ValueError("sample_sizes must be a list of per-relation fan-outs, got %r" % (sample_sizes,))
    sizes = [_fanout(k) for k in sample_sizes]
    R = len(sizes) if num_rels is None else int(num_rels)
    if not 1 <= R <= 32767:
        raise ValueError("the number of relations must lie in [1, 32767] (relations are int16), got %d" % R)
    if len(sizes) != R:
        raise ValueError("%d fan-outs given for %d relations" % (len(sizes), R))
    if rel.dtype != torch.int16:
        raise ValueError("rel must be int16 (heter_graph.typed_in_csr), got %s" % rel.dtype)
    nodes = input_nodes.reshape(-1).to(torch.int64).contiguous()
    n = int(nodes.shape[0])
    num_nodes = int(indptr.shape[0]) - 1
    if n and bool(((nodes < 0) | (nodes >= num_nodes)).any()):
        raise ValueError("input_nodes holds ids outside [0, %d)" % num_nodes)
    dev = nodes.device
    count = torch.empty(n, dtype=torch.int64, device=dev)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    sizes_h = (ctypes.c_int64 * R)(*sizes)
    sizes_d = torch.empty(R, dtype=torch.int32, device=dev)
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    hp = ctypes.cast(sizes_h, ctypes.c_void_p)
    with torch.cuda.device(dev):
        check(lib.pglb_sample_typed_count(p(indptr), p(rel), R, hp, p(sizes_d), p(nodes), n, p(count), p(offsets),
                                          stream))
    total = int(offsets[n].item())
    neighbors = torch.empty(total, dtype=torch.int64, device=dev)
    out_rel = torch.empty(total, dtype=torch.int16, device=dev)
    out_eids = torch.empty(total, dtype=torch.int64, device=dev) if return_eids else None
    if total > 0:  # nothing sampled: nothing to fill, and an empty tensor has no address
        with torch.cuda.device(dev):
            check(lib.pglb_sample_typed_fill(p(indptr), p(cols), p(rel), p(eids), R, hp, p(sizes_d), p(nodes), n,
                                             int(seed) & 0xFFFFFFFFFFFFFFFF, p(offsets), p(neighbors), p(out_rel),
                                             p(out_eids), stream))
    neighbors._pglb_offsets = offsets  # rides along for reindex_graph (saves a scan)
    if return_eids:
        return neighbors, out_rel, count, out_eids
    return neighbors, out_rel, count


_tables = {}


def _table(dev, num_nodes):
    key = (str(dev), int(num_nodes))
    t = _tables.get(key)
    if t is None:
        t = torch.empty(int(num_nodes), dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            check(lib.pglb_reindex_table_init(ctypes.c_void_p(t.data_ptr()), int(num_nodes),
                                              ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        _tables[key] = t
    return t


def reindex_graph(x, neighbors, count, num_nodes=None):
    """paddle.geometric.reindex_graph: compact ids in first-appearance order (``x`` first).
    Returns (reindex_src, reindex_dst, out_nodes).  ``num_nodes`` bounds the ids (size of the dense
    lookup table, cached per device); default max id + 1."""
    ops.require_cuda(x, neighbors, count)
    x = x.reshape(-1).to(torch.int64).contiguous()
    offsets = getattr(neighbors, "_pglb_offsets", None)  # set by sample_neighbors (saves a scan)
    neighbors = neighbors.reshape(-1)
    nb = neighbors.to(torch.int64).contiguous()
    n, m = int(x.shape[0]), int(nb.shape[0])
    dev = x.device
    if offsets is None or int(offsets.shape[0]) != n + 1:
        offsets = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        torch.cumsum(count.reshape(-1).to(torch.int64), 0, out=offsets[1:])
    if num_nodes is None:
        num_nodes = int(max(int(x.max().item()) if n else -1, int(nb.max().item()) if m else -1)) + 1
    table = _table(dev, num_nodes)
    src = torch.empty(m, dtype=torch.int64, device=dev)
    dst = torch.empty(m, dtype=torch.int64, device=dev)
    out_nodes = torch.empty(n + m, dtype=torch.int64, device=dev)
    num_out = torch.zeros(1, dtype=torch.int64, device=dev)
    need = ctypes.c_size_t(0)
    check(lib.pglb_reindex_graph_ws(m, ctypes.byref(need)))
    ws = ops.workspace(dev, need.value)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    with torch.cuda.device(dev):
        check(lib.pglb_reindex_graph(p(x), n, p(nb), p(offsets), m, p(table), p(src), p(dst), p(out_nodes),
                                     p(num_out), p(ws), ws.numel(),
                                     ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return src, dst, out_nodes[: int(num_out.item())]


class NeighborSampler(object):
    """reference pgl/sampling/sage.py:130-155: ``samples`` = fan-out per layer (outermost first);
    ``sample_neighbors(nodes)`` returns ``(graph_list[::-1], nodes)`` where every entry is
    ``(subgraph, number of target nodes)`` and the returned nodes are the input nodes of the first
    layer (gather the features with them)."""

    def __init__(self, graph, samples, uva=False, seed=0):
        if uva:
            raise ValueError("uva mode is not supported by pgl_b200")
        if not graph.is_tensor():
            graph = graph.tensor(inplace=False)
        self.graph = graph
        self.samples = samples
        self.row = graph.adj_dst_index._sorted_v
        self.colptr = graph.adj_dst_index._indptr
        self.num_nodes = graph._n
        self.seed = int(seed)
        self._calls = 0

    def sample_neighbors(self, nodes):
        graph_list = []
        for size in self.samples:
            self._calls += 1
            neighbors, neighbors_count = sample_neighbors(self.row, self.colptr, nodes, sample_size=size,
                                                          seed=self.seed + self._calls)
            edge_src, edge_dst, sample_index = reindex_graph(nodes, neighbors, neighbors_count,
                                                             num_nodes=self.num_nodes)
            subgraph = Graph(num_nodes=int(sample_index.shape[0]),
                             edges=torch.stack([edge_src, edge_dst], dim=1))
            graph_list.append((subgraph, int(nodes.shape[0])))
            nodes = sample_index
        return graph_list[::-1], nodes


class HeteroNeighborSampler(object):
    """``NeighborSampler`` on a ``HeterGraph``: every layer is one ``sample_typed_neighbors`` pass over all relations
    of the graph's typed in-CSR (built once here) and one ``reindex_graph`` over all of them jointly.

    ``samples``: one entry per layer (outermost first), each an int applied to every relation or a dict etype -> int
    naming exactly the sampler's relations; fan-outs in [-1, 4096].  ``etypes`` (default ``graph.edge_types``) are the
    sampler's relations in order.  The reference's stub takes ``(graph_list, sample_list, uva)`` and raises
    NotImplementedError; this signature follows NeighborSampler's instead (DESIGN.md section 4.14).

    ``sample_neighbors(nodes)`` returns ``(blocks[::-1], nodes)`` like NeighborSampler: every block is
    ``(HeterGraph, number of target nodes)``, a tensor-mode HeterGraph over the block's nodes with every relation of
    ``etypes`` (empty ones too) and the parent's node types; the returned nodes are the global ids of the first
    layer's inputs (gather the features with them)."""

    def __init__(self, graph, samples, uva=False, seed=0, etypes=None):
        if uva:
            raise ValueError("uva mode is not supported by pgl_b200")
        if not isinstance(graph, HeterGraph):
            raise ValueError("HeteroNeighborSampler needs a HeterGraph, got %s" % type(graph).__name__)
        if not graph.is_tensor():
            graph = graph.tensor(inplace=False)
        self.graph = graph
        self.etypes = list(graph.edge_types if etypes is None else etypes)
        unknown = [e for e in self.etypes if e not in graph.edge_types]
        if not self.etypes or unknown or len(set(self.etypes)) != len(self.etypes):
            raise ValueError("etypes must be distinct edge types of the graph, got %r" % (self.etypes,))
        if len(self.etypes) > 32767:
            raise ValueError("at most 32767 relations (relations are int16), got %d" % len(self.etypes))
        if not isinstance(samples, (list, tuple)):
            raise ValueError("samples must be a list with one fan-out per layer, got %r" % (samples,))
        self.samples = samples
        self._sizes = [self._layer_sizes(s) for s in samples]
        self.num_nodes = int(graph[self.etypes[0]]._n)
        dev = graph[self.etypes[0]].edges.device
        csr = typed_in_csr([to_tensor(graph[e].edges, dev) for e in self.etypes], self.num_nodes)
        self.csr = {k: csr[k] for k in ("indptr", "cols", "rel")}     # what the sampler reads
        self._node_types = np.asarray(graph.node_types)
        self.seed = int(seed)
        self._calls = 0

    def _layer_sizes(self, size):
        if isinstance(size, dict):
            if set(size.keys()) != set(self.etypes):
                raise ValueError("a per-relation fan-out dict must name exactly the relations %r, got %r"
                                 % (self.etypes, sorted(size.keys(), key=str)))
            return [_fanout(size[e]) for e in self.etypes]
        return [_fanout(size)] * len(self.etypes)

    def sample_neighbors(self, nodes):
        nodes = to_tensor(nodes).reshape(-1).to(torch.int64)
        if int(torch.unique(nodes).shape[0]) != int(nodes.shape[0]):
            raise ValueError("the seed nodes must be distinct")
        R = len(self.etypes)
        blocks = []
        for sizes in self._sizes:
            self._calls += 1
            neighbors, rel, count = sample_typed_neighbors(self.csr["indptr"], self.csr["cols"], self.csr["rel"],
                                                           nodes, sizes, seed=self.seed + self._calls, num_rels=R)
            edge_src, edge_dst, sample_index = reindex_graph(nodes, neighbors, count, num_nodes=self.num_nodes)
            # the node-major output split per relation by a stable partition
            order = torch.sort(rel, stable=True).indices
            per = torch.bincount(rel.to(torch.int64), minlength=R).tolist()
            edges = torch.stack([edge_src, edge_dst], dim=1).index_select(0, order)
            parts = torch.split(edges, per)
            types = self._node_types[sample_index.cpu().numpy()]    # the one device-to-host copy of the block
            block = HeterGraph(edges=dict(zip(self.etypes, parts)), num_nodes=int(sample_index.shape[0]),
                               node_types=types)
            blocks.append((block, int(nodes.shape[0])))
            nodes = sample_index
        return blocks[::-1], nodes
