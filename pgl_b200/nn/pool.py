"""Graph-level pooling (mirror of reference pgl/nn/pool.py) as torch.nn.Modules over tensor-mode batched graphs.
GlobalAttention and Set2Set run their softmax readout on the fused kernel (ops.attn_readout); SAGPool runs on the
segmented top-k kernels (math.segment_topk) and filter_adj."""
import warnings

import torch
import torch.nn as nn

from .. import math, ops
from ..utils.transform import filter_adj
from . import functional as GF
from .conv import GCNConv

__all__ = ["GraphPool", "GraphNorm", "Set2Set", "GlobalAttention", "SAGPool"]


def _graph_indptr(graph):
    """Segment CSR of the batch for the readouts, taken from the graph's own _graph_node_index (no ids regenerated,
    no segment_indptr launch).  It keeps the reference's segment count -- last graph_node_id + 1, so trailing empty
    graphs get no output row -- and the longest graph; both come from one 16-byte read back on the first call and are
    cached on the graph for as long as it holds the same _graph_node_index."""
    gni = graph._graph_node_index
    cached = graph.__dict__.get("_pglb_readout_csr")
    if cached is not None and cached[0] is gni:
        return cached[1]
    index = ops._i64(gni).reshape(-1)
    counts = index[1:] - index[:-1]
    last = torch.arange(1, counts.numel() + 1, device=index.device) * (counts > 0)
    k, longest = (int(v) for v in torch.stack([last.max(), counts.max()]).tolist()) if counts.numel() else (0, 0)
    indptr = index[:k + 1].contiguous()
    indptr._pglb_max_len = longest
    graph.__dict__["_pglb_readout_csr"] = (gni, indptr)
    return indptr


class GraphPool(nn.Module):
    """reference pool.py:30-62: segment pool ("sum", "mean", "max", "min") of the node features of every graph."""

    def __init__(self, pool_type=None):
        super().__init__()
        self.pool_type = pool_type

    def forward(self, graph, feature, pool_type=None):
        if pool_type is not None:
            warnings.warn("The pool_type (%s) argument in forward function will be discarded in the future, "
                          "please initialize it when creating a GraphPool instance." % pool_type)
        else:
            pool_type = self.pool_type
        return math.segment_pool(feature, graph.graph_node_id, pool_type)


class GraphNorm(nn.Module):
    """reference pool.py:65-93: every node's features divided by sqrt(number of nodes of its graph)."""

    def forward(self, graph, feature):
        return GF.graph_norm(graph, feature)


class Set2Set(nn.Module):
    """reference pool.py:96-145.  As in the reference, the LSTM input q_star is never updated (the loop assigns
    ``q_start``), so the LSTM always reads zeros, its state carries the iterations, and the layer returns
    concat(q, r) of the last iteration, [num_graph, 2 * input_dim]."""

    def __init__(self, input_dim, n_iters, n_layers=1):
        super().__init__()
        self.input_dim = input_dim
        self.output_dim = 2 * input_dim
        self.n_iters = n_iters
        self.n_layers = n_layers
        self.lstm = nn.LSTM(input_size=self.output_dim, hidden_size=self.input_dim, num_layers=n_layers)

    def forward(self, graph, x):
        indptr = _graph_indptr(graph)
        batch_size = int(indptr.numel()) - 1
        zeros = torch.zeros((self.n_layers, batch_size, self.input_dim), dtype=x.dtype, device=x.device)
        h = (zeros, zeros.clone())
        q_star = torch.zeros((batch_size, self.output_dim), dtype=x.dtype, device=x.device)
        q_start = None
        for _ in range(self.n_iters):
            q, h = self.lstm(q_star.unsqueeze(0), h)
            q = q.reshape(batch_size, self.input_dim)
            r = ops.attn_readout(x, indptr, query=q)
            q_start = torch.cat([q, r], dim=-1)
        return q_start


class GlobalAttention(nn.Module):
    """reference pool.py:148-179: out[g] = sum_{i in g} softmax_g(gate(x))_i * nn(x)_i."""

    def __init__(self, gate, nn=None):
        super().__init__()
        self.gate = gate
        self.nn = nn

    def forward(self, graph, x):
        gate_x = self.gate(x).reshape(-1, 1)
        x = self.nn(x) if self.nn else x
        assert x.dim() == gate_x.dim() and x.shape[0] == gate_x.shape[0]
        return ops.attn_readout(x, _graph_indptr(graph), gate=gate_x)


class SAGPool(nn.Module):
    """reference pool.py:182-252.  gnn=None uses GCNConv (the reference names it without importing it).  Returns
    (kept node features scaled by their score, their graph ids, the pooled Graph)."""

    def __init__(self, input_dim, ratio=0.5, gnn=None, min_score=None, nonlinearity=None):
        super().__init__()
        self.input_dim = input_dim
        self.ratio = ratio
        self.gnn = (GCNConv if gnn is None else gnn)(input_dim, 1)
        self.min_score = min_score
        self.nonlinearity = torch.tanh if nonlinearity is None else nonlinearity

    def forward(self, graph, x):
        from ..graph import Graph
        batch = graph.graph_node_id
        attn_score = self.gnn(graph, x).reshape(-1)
        if self.min_score is None:
            attn_score = self.nonlinearity(attn_score)
        else:
            attn_score = math.segment_softmax(attn_score, batch)
        out, rank = math.segment_topk(x, attn_score, batch, self.ratio, self.min_score, return_index=True)
        x = out * ops.gather_rows(attn_score.reshape(-1, 1), rank)
        batch = batch[rank]
        edge_index, _ = filter_adj(graph.edges, rank, num_nodes=attn_score.shape[0])
        ng = graph.num_graph
        batch_size = int(ng.reshape(-1)[0].item()) if isinstance(ng, torch.Tensor) else int(ng)
        counts = torch.bincount(batch.to(torch.int64), minlength=batch_size)[:batch_size]
        graph_node_index = torch.zeros(batch_size + 1, dtype=torch.int64, device=x.device)
        graph_node_index[1:] = counts.cumsum(0)
        g = Graph(num_nodes=int(x.shape[0]), edges=edge_index, node_feat={"attr": x},
                  _graph_node_index=graph_node_index,
                  _num_graph=int(batch.max().item()) + 1 if batch.numel() else 0)
        return x, batch, g
