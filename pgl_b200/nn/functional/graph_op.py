"""Graph functional ops on the send/recv path (mirror of reference
pgl/nn/functional/graph_op.py:29-123)."""

from ... import math, ops

import torch

__all__ = ["degree_norm", "graph_pool", "graph_norm", "edge_softmax"]


def degree_norm(graph, mode="indegree"):
    """clip(float(degree), 1) ** -0.5 as [num_nodes, 1]; reference graph_op.py:29-55.
    Cached on the graph (the degree vector is immutable)."""
    assert mode in ["indegree", "outdegree"], \
        "The degree_norm mode should be in ['indegree', 'outdegree']. But recieve mode=%s" % mode
    key = "_norm_" + mode
    cached = graph.__dict__.get(key)
    if cached is not None:
        return cached
    degree = graph.indegree() if mode == "indegree" else graph.outdegree()
    norm = ops.degree_norm(degree)
    if type(graph).__name__ == "Graph":
        graph.__dict__[key] = norm
    return norm


def graph_pool(graph, feature, pool_type):
    """reference graph_op.py:58-76: segment pool over graph_node_id."""
    return math.segment_pool(feature, graph.graph_node_id, pool_type)


def graph_norm(graph, feature):
    """reference graph_op.py:78-98: every node's feature divided by sqrt(number of nodes of its graph), in the
    reference's op order (segment_sum of ones, sqrt, gather, divide) so the result is the same bit for bit.  A
    bfloat16 / float16 feature is divided in fp32 and rounded once back to its own dtype."""
    nodes = torch.ones((graph._n, 1), dtype=torch.float32, device=feature.device)
    norm = graph_pool(graph, nodes, pool_type="sum")
    norm = torch.sqrt(norm)
    norm = ops.gather_rows(norm, graph.graph_node_id)
    if feature.dtype in ops.HALF_DTYPES:
        return (feature.float() / norm).to(feature.dtype)
    return feature / norm


def edge_softmax(graph, logits, norm_by="dst"):
    """Softmax over the incoming (norm_by='dst') or outgoing ('src') edges of every node, in
    the ORIGINAL edge order; reference graph_op.py:101-123 (gather by eid + 7-op
    segment_softmax + scatter) fused into one launch over the cached CSR."""
    if norm_by not in ("src", "dst"):
        raise ValueError("sort_by should be in 'src' or 'dst'.")
    index = graph.adj_dst_index if norm_by == "dst" else graph.adj_src_index
    return ops.edge_softmax_csr(index._indptr, index._sorted_eid, logits, int(graph.num_edges))
