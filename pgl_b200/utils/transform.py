"""Graph transforms (mirror of reference pgl/utils/transform.py).  to_undirected / add_self_loops work on numpy-mode
graphs as in the reference; to_dense_batch runs on the pad kernel (pglb_segment_pad) and filter_adj on
pglb_map_edges."""
import numpy as np
import torch

from .. import ops
from .helper import maybe_num_nodes

__all__ = ["to_undirected", "add_self_loops", "to_dense_batch", "filter_adj"]


def _copy_feats(graph, g, copy_node_feat, copy_edge_feat, what):
    if copy_node_feat:
        for k, v in graph._node_feat.items():
            g._node_feat[k] = v
    if copy_edge_feat:
        raise NotImplementedError("The copy of edge feature is not implemented for %s." % what)
    return g


def to_undirected(graph, copy_node_feat=True, copy_edge_feat=False):
    """reference transform.py:25-61: the edges and their reverses, deduplicated and sorted (np.unique); numpy mode."""
    from ..graph import Graph
    if graph.is_tensor():
        raise TypeError("The input graph should be numpy format.")
    edges = np.asarray(graph.edges)
    edges = np.unique(np.vstack((edges, edges[:, ::-1])), axis=0)
    g = Graph(num_nodes=graph.num_nodes, edges=edges)
    return _copy_feats(graph, g, copy_node_feat, copy_edge_feat, "to_undirected")


def add_self_loops(graph, copy_node_feat=True, copy_edge_feat=False):
    """reference transform.py:64-98: the edges followed by one self-loop per node; numpy mode."""
    from ..graph import Graph
    if graph.is_tensor():
        raise TypeError("The input graph should be numpy format.")
    loops = np.repeat(np.arange(graph.num_nodes, dtype=np.int64)[:, None], 2, axis=1)
    g = Graph(num_nodes=graph.num_nodes, edges=np.vstack((np.asarray(graph.edges).reshape(-1, 2), loops)))
    return _copy_feats(graph, g, copy_node_feat, copy_edge_feat, "add_self_loops")


def to_dense_batch(x, graph, fill_value=0, max_num_nodes=None):
    """reference transform.py:101-135: (out [B, L, *F], mask [B, L]) with B = graph_node_id.max() + 1, row p of block b
    = node p of graph b, padding = fill_value, mask True at padding.  out keeps x's dtype (the reference returns the
    default float dtype).  A max_num_nodes below the largest graph raises ValueError (the reference scatters out of
    range)."""
    ids = graph.graph_node_id
    ops.require_cuda(x, ids)
    n = int(ids.shape[0])
    B = int(ids.max().item()) + 1 if n else 0
    indptr = ops.segment_indptr(ids, B)
    longest = ops.segment_max_len(indptr)
    if max_num_nodes is None:
        max_num_nodes = longest
    elif int(max_num_nodes) < longest:
        raise ValueError("to_dense_batch: max_num_nodes=%d is smaller than the largest graph (%d nodes)"
                         % (int(max_num_nodes), longest))
    L = int(max_num_nodes)
    out = ops.segment_pad(x, indptr, L, fill_value)
    counts = indptr[1:] - indptr[:-1]
    mask = torch.arange(L, device=counts.device).unsqueeze(0) >= counts.unsqueeze(1)
    return out, mask


def filter_adj(edge_index, perm, edge_attr=None, num_nodes=None):
    """reference transform.py:138-168: keep the edges whose ends are both in perm, relabelled to positions in perm, in
    their original order.  The position table is int64 (the reference's float32 table is wrong above 2^24 nodes) and
    num_nodes is honoured when given; without it the table covers every id of the edges and of perm.  A perm id
    outside [0, num_nodes) raises ValueError."""
    ops.require_cuda(edge_index, perm)
    perm = ops._i64(perm).reshape(-1)
    lo, hi = (int(v) for v in torch.stack([perm.min(), perm.max()]).tolist()) if perm.numel() else (0, -1)
    if num_nodes is None:
        num_nodes = max(int(maybe_num_nodes(edge_index)), hi + 1)
    if lo < 0 or hi >= int(num_nodes):
        raise ValueError("filter_adj: perm holds node ids outside [0, %d)" % int(num_nodes))
    table = torch.full((int(num_nodes),), -1, dtype=torch.int64, device=perm.device)
    table[perm] = torch.arange(perm.shape[0], dtype=torch.int64, device=perm.device)
    mapped = ops.map_edges(None, edge_index.reshape(-1, 2), table, strict=False)
    keep = ((mapped[:, 0] >= 0) & (mapped[:, 1] >= 0)).nonzero().reshape(-1)
    if edge_attr is not None:
        edge_attr = edge_attr[keep]
    return mapped[keep], edge_attr
