"""Graph Multiset Transformer pooling (mirror of reference pgl/nn/gmt_pool.py) as torch.nn.Modules.  Dense layers
follow the paddle.nn.Linear layout of nn.conv.Linear; node sets are batched densely by to_dense_batch (the pad
kernel).  Kept as the reference computes it: the padding mask is ``batch_x.sum(-1) == 0`` (a real node whose features
sum to 0 is masked too) scaled by -1e9, the attention softmax is over axis 1 (the queries), and with layer_norm the
block applies ln0 twice and never ln1."""
import math as _math

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..utils.transform import to_dense_batch
from .conv import GCNConv, Linear

__all__ = ["GraphMultisetTransformer", "MAB", "SAB", "PMA"]


class MAB(nn.Module):
    """reference gmt_pool.py:27-109: multi-head attention block; conv (a graph conv class) computes K and V from the
    graph when the block is called with graph=(graph, x)."""

    def __init__(self, dim_Q, dim_K, dim_V, num_heads, conv=None, layer_norm=False):
        super().__init__()
        self.dim_V = dim_V
        self.num_heads = num_heads
        self.layer_norm = layer_norm
        self.proj_q = Linear(dim_K, dim_V)
        if conv is None:
            self.layer_k = Linear(dim_K, dim_V)
            self.layer_v = Linear(dim_K, dim_V)
        else:
            self.layer_k = conv(dim_K, dim_V)
            self.layer_v = conv(dim_K, dim_V)
        if layer_norm:
            self.ln0 = nn.LayerNorm(dim_V)
            self.ln1 = nn.LayerNorm(dim_V)
        self.proj_o = Linear(dim_V, dim_V)

    def forward(self, Q, K, graph=None, mask=None):
        Q = self.proj_q(Q)
        if graph is not None:
            graph, x = graph
            K, V = self.layer_k(graph, x), self.layer_v(graph, x)
            K, _ = to_dense_batch(K, graph)
            V, _ = to_dense_batch(V, graph)
        else:
            K, V = self.layer_k(K), self.layer_v(K)
        Q_ = torch.cat(Q.chunk(self.num_heads, 2), 0)
        K_ = torch.cat(K.chunk(self.num_heads, 2), 0)
        V_ = torch.cat(V.chunk(self.num_heads, 2), 0)
        score = Q_.bmm(K_.transpose(1, 2)) / _math.sqrt(self.dim_V)
        if mask is not None:
            mask = torch.cat([mask for _ in range(self.num_heads)], 0)
            mask = mask.reshape(K_.shape[0], K_.shape[1]).unsqueeze(1)
            score = mask + score
        A = F.softmax(score, 1)
        output = torch.cat((Q_ + A.bmm(V_)).chunk(self.num_heads, 0), 2)
        if self.layer_norm:
            output = self.ln0(output)
        output = output + F.relu(self.proj_o(output))
        if self.layer_norm:
            output = self.ln0(output)
        return output


class SAB(nn.Module):
    """reference gmt_pool.py:115-152: self-attention block."""

    def __init__(self, input_dim, output_dim, num_heads, conv=None, layer_norm=False):
        super().__init__()
        self.mab = MAB(input_dim, input_dim, output_dim, num_heads, conv=conv, layer_norm=layer_norm)

    def forward(self, x, graph, mask):
        return self.mab(x, x, graph, mask)


class PMA(nn.Module):
    """reference gmt_pool.py:155-195: pooling by multi-head attention over num_seeds learned seeds (Kaiming uniform,
    fan_in = num_seeds * dim as paddle's KaimingUniform computes it)."""

    def __init__(self, dim, num_heads, num_seeds, conv=None, layer_norm=False):
        super().__init__()
        self.Q_S = nn.Parameter(torch.empty(1, num_seeds, dim))
        nn.init.kaiming_uniform_(self.Q_S, a=0.0)
        self.dim = dim
        self.num_seeds = num_seeds
        self.mab = MAB(dim, dim, dim, num_heads, conv=conv, layer_norm=layer_norm)

    def forward(self, x, graph, mask):
        return self.mab(self.Q_S.expand(x.shape[0], self.num_seeds, self.dim), x, graph, mask)


class GraphMultisetTransformer(nn.Module):
    """reference gmt_pool.py:198-291: lin1 -> dense batch -> the pool sequence (GMPool_G / SelfAtt / GMPool_I) ->
    lin2, one output row per graph."""

    def __init__(self, input_dim, hidden_dim, output_dim, conv=None, num_nodes=30, pooling_ratio=0.25,
                 pool_sequences=None, num_heads=4, layer_norm=False):
        super().__init__()
        self.input_dim = input_dim
        self.hidden_dim = hidden_dim
        self.output_dim = output_dim
        self.conv = conv or GCNConv
        self.num_nodes = num_nodes
        self.pooling_ratio = pooling_ratio
        self.pool_sequences = ["GMPool_G", "SelfAtt", "GMPool_I"] if pool_sequences is None else pool_sequences
        self.num_heads = num_heads
        self.layer_norm = layer_norm
        self.pools = nn.ModuleList()
        num_out_nodes = _math.ceil(num_nodes * pooling_ratio)
        self.lin1 = Linear(input_dim, hidden_dim)
        self.lin2 = Linear(hidden_dim, output_dim)
        for i, pool_type in enumerate(self.pool_sequences):
            if pool_type not in ["GMPool_G", "GMPool_I", "SelfAtt"]:
                raise ValueError("Elements in 'pool_sequences' should be one of 'GMPool_G', 'GMPool_I', or 'SelfAtt'")
            if i == len(self.pool_sequences) - 1:
                num_out_nodes = 1
            if pool_type == "GMPool_G":
                self.pools.append(PMA(hidden_dim, num_heads, num_out_nodes, conv=self.conv, layer_norm=layer_norm))
                num_out_nodes = _math.ceil(num_out_nodes * self.pooling_ratio)
            elif pool_type == "GMPool_I":
                self.pools.append(PMA(hidden_dim, num_heads, num_out_nodes, conv=None, layer_norm=layer_norm))
                num_out_nodes = _math.ceil(num_out_nodes * self.pooling_ratio)
            else:
                self.pools.append(SAB(hidden_dim, hidden_dim, num_heads, conv=None, layer_norm=layer_norm))

    def forward(self, graph, x):
        x = self.lin1(x)
        batch_x, _ = to_dense_batch(x, graph)
        mask = (batch_x.sum(-1) == 0).to(batch_x.dtype).unsqueeze(0) * -1e9
        for name, pool in zip(self.pool_sequences, self.pools):
            g = (graph, x) if name == "GMPool_G" else None
            batch_x = pool(batch_x, g, mask)
            mask = None
        return self.lin2(batch_x.squeeze(1))
