"""The reference's conv layers (pgl/nn/conv.py) re-hosted on torch.nn.Module over the sm_90a
send/recv kernels.  GCNConv / GATConv / GraphSageConv are the hot-path rows (SURVEY 8a17-19); the
others are compositions of the same primitives (SURVEY 8f rank 2).  Wherever the reference wraps an
aggregation in two ``* norm`` multiplies, both ride inside the aggregation kernel (``_propagate``).

Parameter layout follows paddle.nn.Linear: ``weight`` is [in, out] and y = x @ weight + bias,
so reference checkpoints map one to one.
"""
import functools
import math as _math

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..heter_graph import HeterGraph
from . import functional as GF

__all__ = ["GCNConv", "GATConv", "GraphSageConv", "Linear", "PinSageConv", "GATv2Conv", "APPNP",
           "GPRConv", "GCNII", "TransformerConv", "GINConv", "RGCNConv", "SGCConv", "SSGCConv",
           "NGCFConv", "LightGCNConv", "FAConv"]


class Linear(nn.Module):
    """paddle.nn.Linear semantics: weight [in_features, out_features]."""

    def __init__(self, in_features, out_features, bias=True):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(in_features, out_features))
        self.bias = nn.Parameter(torch.zeros(out_features)) if bias else None
        bound = _math.sqrt(6.0 / (in_features + out_features))  # paddle default: Xavier uniform
        nn.init.uniform_(self.weight, -bound, bound)

    def forward(self, x, act=None):
        """act (None | "relu") is applied after the bias; on the tensor-core path it is fused into
        the GEMM epilogue (ops.linear_tc), elsewhere it is a separate op."""
        from .. import ops
        if ops.linear_tc_ok(x, self.weight):
            return ops.linear_tc(x, self.weight, self.bias, act)
        y = x @ self.weight
        if self.bias is not None:
            y = y + self.bias
        if act == "relu":
            y = F.relu(y)
        return y


def _activation(act):
    if isinstance(act, str):
        return getattr(F, act)
    return act


def _propagate(graph, feature, norm):
    """``(feature * norm) -> send_recv(sum) -> * norm`` -- the step the reference spells as three
    ops in GCN/APPNP/GPR/GCNII/SGC/SSGC/LightGCN (e.g. conv.py:491-493).  On a plain Graph with a
    per-node norm the two multiplies are the kernel's scale_src / scale_dst operands."""
    if norm is not None and type(graph).__name__ == "Graph" and feature.dim() == 2 \
            and norm.numel() == feature.shape[0] and graph._n == feature.shape[0]:
        nv = norm.reshape(-1)
        return graph._send_u_recv(feature, "sum", None, scale_src=nv, scale_dst=nv)
    if norm is not None:
        feature = feature * norm
    feature = graph.send_recv(feature, "sum")
    if norm is not None:
        feature = feature * norm
    return feature


def _propagate_fused(graph, feature, norm, fallback, **kw):
    """One K-hop step ``a * _propagate(graph, feature, norm) (+ b * h)`` (and ``acc + c * y``) as one aggregation with a
    row epilogue (``ops.propagate``): bit for bit the op-by-op hop in float32.  Where that route declines (not a plain
    Graph, a feature or norm it does not take), ``fallback()`` runs the layer's op-by-op hop unchanged."""
    out = None
    if type(graph).__name__ == "Graph" and norm is not None and isinstance(feature, torch.Tensor) \
            and feature.dim() == 2 and graph._n == feature.shape[0]:
        out = ops.propagate(feature, graph._fwd_csr(), graph._bwd_csr, norm, **kw)
    return fallback() if out is None else out


def _with_self_loops(graph):
    """reference conv.py:474-484: drop the existing self loops, prepend one per node."""
    edges = graph.edges
    n = graph._n
    index = torch.arange(n, dtype=torch.int64, device=edges.device)
    keep = edges[edges[:, 0] != edges[:, 1]]
    return type(graph)(num_nodes=n, edges=torch.cat([torch.stack([index, index], 1), keep], 0))


class GraphSageConv(nn.Module):
    """reference pgl/nn/conv.py:46-115."""

    def __init__(self, input_size, hidden_size, aggr_func="sum", normalize=True):
        super().__init__()
        assert aggr_func in ["sum", "mean", "max", "min"], \
            "Only support 'sum', 'mean', 'max', 'min'."
        self.aggr_func = aggr_func
        self.normalize = normalize
        self.self_linear = Linear(input_size, hidden_size)
        self.neigh_linear = Linear(input_size, hidden_size)

    def forward(self, graph, feature, act=None):
        if isinstance(feature, torch.Tensor):
            feature = (feature, feature)
        neigh_feature = graph.send_recv(feature[0], self.aggr_func, out_size=feature[1].shape[0])
        neigh_feature = self.neigh_linear(neigh_feature)
        self_feature = self.self_linear(feature[1])
        output = self_feature + neigh_feature
        if act is not None:
            output = getattr(F, act)(output)
        if self.normalize:
            output = F.normalize(output, dim=1)
        return output


class GCNConv(nn.Module):
    """reference pgl/nn/conv.py:189-254.  The two ``* norm`` multiplies around the aggregation
    (conv.py:242,250) are fused into the aggregation kernel (scale_src / scale_dst)."""

    def __init__(self, input_size, output_size, activation=None, norm=True):
        super().__init__()
        self.input_size = input_size
        self.output_size = output_size
        self.linear = Linear(input_size, output_size, bias=False)
        self.bias = nn.Parameter(torch.zeros(output_size))
        self.norm = norm
        self.activation = _activation(activation)

    def forward(self, graph, feature, norm=None):
        if self.norm and norm is None:
            norm = GF.degree_norm(graph)
        if self.input_size > self.output_size:
            feature = self.linear(feature)
        fused = norm is not None and type(graph).__name__ == "Graph" and \
            norm.numel() == feature.shape[0]
        if fused:
            # both norm multiplies ride inside the aggregation kernel.  When the linear comes
            # second the reference scales after it (conv.py:246-251); row scaling commutes with
            # the right-multiplication, so only the rounding differs (within the 1e-4 bar).
            nv = norm.reshape(-1)
            output = graph._send_u_recv(feature, "sum", None, scale_src=nv, scale_dst=nv)
            if self.input_size <= self.output_size:
                from .. import ops
                if ops.linear_tc_ok(output, self.linear.weight):
                    # 3xTF32 tensor-core GEMM with bias + ReLU in its epilogue: one read, one write
                    relu = self.activation is F.relu
                    output = ops.linear_tc(output, self.linear.weight, self.bias,
                                           "relu" if relu else None)
                    if self.activation is not None and not relu:
                        output = self.activation(output)
                    return output
                output = torch.addmm(self.bias, output, self.linear.weight)
            else:
                output = output + self.bias
            if self.activation is not None:
                output = self.activation(output)
            return output
        if norm is not None:
            feature = feature * norm
        output = graph.send_recv(feature, "sum")
        if self.input_size <= self.output_size:
            output = self.linear(output)
        if norm is not None:
            output = output * norm
        output = output + self.bias
        if self.activation is not None:
            output = self.activation(output)
        return output


# feature dtypes of GATConv's fused training path (16-bit: the *_x16 kernels)
_FUSED_TRAIN_DTYPES = (torch.float32, torch.bfloat16, torch.float16)


class GATConv(nn.Module):
    """reference pgl/nn/conv.py:257-346."""

    def __init__(self, input_size, hidden_size, feat_drop=0.6, attn_drop=0.6, num_heads=1,
                 concat=True, activation=None):
        super().__init__()
        self.hidden_size = hidden_size
        self.num_heads = num_heads
        self.feat_drop = feat_drop
        self.attn_drop = attn_drop
        self.concat = concat
        self.linear = Linear(input_size, num_heads * hidden_size)
        self.weight_src = nn.Parameter(torch.empty(num_heads, hidden_size))
        self.weight_dst = nn.Parameter(torch.empty(num_heads, hidden_size))
        bound = _math.sqrt(6.0 / (num_heads + hidden_size))
        nn.init.uniform_(self.weight_src, -bound, bound)
        nn.init.uniform_(self.weight_dst, -bound, bound)
        self.feat_dropout = nn.Dropout(p=feat_drop)
        self.attn_dropout = nn.Dropout(p=attn_drop)
        self.leaky_relu = nn.LeakyReLU(negative_slope=0.2)
        self.activation = _activation(activation)

    def forward(self, graph, feature):
        if self.feat_drop > 1e-15:
            feature = self.feat_dropout(feature)
        feature = self.linear(feature)
        feature = feature.reshape(-1, self.num_heads, self.hidden_size)
        from .. import ops as _ops
        # the dtype of the attention logits and of the layer's output: torch's promotion of the features' and the
        # attention weights' dtypes (a bf16 module gives bf16, bf16 features under fp32 weights give fp32)
        out_dtype = functools.reduce(torch.promote_types, (feature.dtype, self.weight_src.dtype, self.weight_dst.dtype))
        dots = _ops.head_dots(feature, self.weight_src, self.weight_dst) if feature.is_cuda else None
        if dots is not None:      # both projections in one pass over the features (float32 logits)
            attn_src, attn_dst = dots
        else:
            attn_src = torch.sum(feature * self.weight_src, dim=-1)
            attn_dst = torch.sum(feature * self.weight_dst, dim=-1)

        def unfused_attn():
            # the op-by-op paths take the logits in the layer's dtype, as the two torch expressions give them
            return attn_src.to(out_dtype), attn_dst.to(out_dtype)
        no_attn_drop = self.attn_drop <= 1e-15 or not self.training
        if not torch.is_grad_enabled() and no_attn_drop and type(graph).__name__ == "Graph":
            # inference: send_uv + LeakyReLU + edge_softmax in one kernel (logits never stored),
            # alpha kept in CSR slot order so the aggregation reads it sequentially
            from .. import ops
            csr = graph._fwd_csr()
            # one pass when the row fits the wide-row kernel (H*Dh in (64, 128]); otherwise the
            # fused attention kernel + slot-ordered aggregation
            output = ops.gat_fused(csr, feature, attn_src, attn_dst, self.leaky_relu.negative_slope,
                                   out_dtype=out_dtype)
            if output is None:
                attn_src, attn_dst = unfused_attn()
                alpha = ops.gat_attention_csr(csr, attn_src, attn_dst, self.leaky_relu.negative_slope)
                output = ops.aggregate_ue_slots(feature, alpha.reshape(-1, self.num_heads, 1), csr,
                                                int(feature.shape[0]), "mul", "sum")
            if self.concat:
                output = output.reshape(-1, self.num_heads * self.hidden_size)
            else:
                output = torch.mean(output, dim=1)
            if self.activation is not None:
                output = self.activation(output)
            return output
        output = None
        if type(graph).__name__ == "Graph" and feature.dtype in _FUSED_TRAIN_DTYPES:
            # training: the same single-pass kernel, which keeps the rows' log-sum-exp, and a fused backward
            # (ops._GatFused), with the attention dropout inside both; None when the shape is outside them
            from .. import ops
            output = ops.gat_fused_train(graph._fwd_csr(), graph._bwd_csr, feature, attn_src, attn_dst,
                                         self.leaky_relu.negative_slope, out_dtype=out_dtype,
                                         attn_drop=0.0 if no_attn_drop else self.attn_drop)
        if output is None:
            attn_src, attn_dst = unfused_attn()
            alpha = graph.send_uv(attn_src, attn_dst, "add")
            alpha = self.leaky_relu(alpha)
            alpha = GF.edge_softmax(graph, alpha)
            alpha = alpha.reshape(-1, self.num_heads, 1)
            if self.attn_drop > 1e-15:
                alpha = self.attn_dropout(alpha)
            output = graph.send_ue_recv(feature, alpha, "mul", "sum")
        if self.concat:
            output = output.reshape(-1, self.num_heads * self.hidden_size)
        else:
            output = torch.mean(output, dim=1)
        if self.activation is not None:
            output = self.activation(output)
        return output


class PinSageConv(nn.Module):
    """reference pgl/nn/conv.py:118-186.  The reference's UDF pair (send ``h[src] * w`` ->
    recv ``reduce_*``) is exactly ``send_ue_recv(nfeat, efeat, "mul", aggr)``: one fused kernel, no
    [E, D] message."""

    def __init__(self, input_size, hidden_size, aggr_func="sum"):
        super().__init__()
        assert aggr_func in ["sum", "mean", "max", "min"], \
            "Only support 'sum', 'mean', 'max', 'min' built-in receive function."
        self.aggr_func = aggr_func
        self.self_linear = Linear(input_size, hidden_size)
        self.neigh_linear = Linear(input_size, hidden_size)

    def forward(self, graph, nfeat, efeat, act=None):
        neigh_feature = graph.send_ue_recv(nfeat, efeat, "mul", self.aggr_func)
        output = self.self_linear(nfeat) + self.neigh_linear(neigh_feature)
        if act is not None:
            output = getattr(F, act)(output)
        return F.normalize(output, dim=1)


class GATv2Conv(nn.Module):
    """reference pgl/nn/conv.py:349-435.  On a ``Graph`` the attention (send_uv(add), LeakyReLU, the sum with attn,
    edge_softmax, dropout, send_ue_recv) is one fused pass with a fused backward (``ops.gatv2_attention``); shapes
    those kernels refuse keep the op-by-op route."""

    def __init__(self, input_size, hidden_size, feat_drop=0.6, attn_drop=0.6, num_heads=1,
                 concat=True, activation=None):
        super().__init__()
        self.hidden_size = hidden_size
        self.num_heads = num_heads
        self.feat_drop = feat_drop
        self.attn_drop = attn_drop
        self.concat = concat
        self.linear = Linear(input_size, num_heads * hidden_size)
        self.attn = nn.Parameter(torch.empty(1, num_heads, hidden_size))
        bound = _math.sqrt(6.0 / (num_heads + hidden_size))
        nn.init.uniform_(self.attn, -bound, bound)
        self.feat_dropout = nn.Dropout(p=feat_drop)
        self.attn_dropout = nn.Dropout(p=attn_drop)
        self.leaky_relu = nn.LeakyReLU(negative_slope=0.2)
        self.activation = _activation(activation)

    def forward(self, graph, feature):
        if self.feat_drop > 1e-15:
            feature = self.feat_dropout(feature)
        feature = self.linear(feature).reshape(-1, self.num_heads, self.hidden_size)
        output = None
        if type(graph).__name__ == "Graph" and feature.is_cuda:
            # score, softmax, dropout and weighted sum in one pass with a fused backward (ops._GatV2): no [E, H*Dh]
            # tensor; None when the call is outside the kernels
            from .. import ops
            drop = self.attn_drop if self.attn_drop > 1e-15 and self.training else 0.0
            output = ops.gatv2_attention(graph._fwd_csr(), graph._bwd_csr, feature, self.attn,
                                         self.leaky_relu.negative_slope, attn_drop=drop)
        if output is None:
            alpha = graph.send_uv(feature, feature, "add")
            alpha = self.leaky_relu(alpha)
            alpha = torch.sum(alpha * self.attn, dim=-1)
            alpha = GF.edge_softmax(graph, alpha)
            alpha = alpha.reshape(-1, self.num_heads, 1)
            if self.attn_drop > 1e-15:
                alpha = self.attn_dropout(alpha)
            output = graph.send_ue_recv(feature, alpha, "mul", "sum")
        if self.concat:
            output = output.reshape(-1, self.num_heads * self.hidden_size)
        else:
            output = torch.mean(output, dim=1)
        if self.activation is not None:
            output = self.activation(output)
        return output


class APPNP(nn.Module):
    """reference pgl/nn/conv.py:438-497."""

    def __init__(self, alpha=0.2, k_hop=10, self_loop=False):
        super().__init__()
        self.alpha = alpha
        self.k_hop = k_hop
        self.self_loop = self_loop

    def forward(self, graph, feature, norm=None):
        if self.self_loop:
            graph = _with_self_loops(graph)
        if norm is None:
            norm = GF.degree_norm(graph)
        h0 = feature

        def hop(feature):
            feature = _propagate(graph, feature, norm)
            return self.alpha * h0 + (1 - self.alpha) * feature

        for _ in range(self.k_hop):
            feature = _propagate_fused(graph, feature, norm, functools.partial(hop, feature),
                                       a=1 - self.alpha, b=self.alpha, h=h0)
        return feature


class GPRConv(nn.Module):
    """reference pgl/nn/conv.py:500-642."""

    def __init__(self, input_size, hidden_size, output_size, drop=0.5, dprate=0.5,
                 activation="relu", self_loop=False, alpha=0.1, k_hop=10, init_method="PPR",
                 gamma=None):
        super().__init__()
        import numpy as np
        self.alpha = alpha
        self.k_hop = k_hop
        self.init_method = init_method
        self.gamma = gamma
        self.self_loop = self_loop
        assert init_method in ["SGC", "PPR", "NPPR", "Random", "WS"]
        if init_method == "SGC":  # alpha is the (integer) position of the peak
            temp = np.zeros(k_hop + 1)
            temp[alpha] = 1.0
        elif init_method == "PPR":
            temp = alpha * (1 - alpha) ** np.arange(k_hop + 1)
            temp[-1] = (1 - alpha) ** k_hop
        elif init_method == "NPPR":
            temp = alpha ** np.arange(k_hop + 1)
            temp = temp / np.sum(np.abs(temp))
        elif init_method == "Random":
            bound = np.sqrt(3 / (k_hop + 1))
            temp = np.random.uniform(-bound, bound, k_hop + 1)
            temp = temp / np.sum(np.abs(temp))
        else:
            temp = np.asarray(gamma)
        self.temp = nn.Parameter(torch.as_tensor(np.asarray(temp), dtype=torch.float32))
        self.linear_1 = Linear(input_size, hidden_size)
        self.linear_2 = Linear(hidden_size, output_size)
        self.drop = drop
        self.dprate = dprate
        self.feat_dropout_1 = nn.Dropout(p=drop)
        self.feat_dropout_2 = nn.Dropout(p=dprate)
        self.activation = _activation(activation)

    def forward(self, graph, feature, norm=None):
        if self.self_loop:
            graph = _with_self_loops(graph)
        feature = self.feat_dropout_1(feature)
        feature = self.activation(self.linear_1(feature))
        feature = self.feat_dropout_1(feature)
        feature = self.linear_2(feature)
        if self.dprate > 0.0:
            feature = self.feat_dropout_2(feature)
        if norm is None:
            norm = GF.degree_norm(graph)
        hidden = feature * self.temp[0]

        def hop(feature, hidden, k):
            feature = _propagate(graph, feature, norm)
            return feature, hidden + self.temp[k + 1] * feature

        for k in range(self.k_hop):
            # temp[k + 1] is read on the device: no host sync per hop
            feature, hidden = _propagate_fused(graph, feature, norm, functools.partial(hop, feature, hidden, k),
                                               acc=hidden, c=self.temp[k + 1])
        return hidden


class GCNII(nn.Module):
    """reference pgl/nn/conv.py:645-721."""

    def __init__(self, hidden_size, activation=None, lambda_l=0.5, alpha=0.2, k_hop=10,
                 dropout=0.6):
        super().__init__()
        self.hidden_size = hidden_size
        self.lambda_l = lambda_l
        self.alpha = alpha
        self.k_hop = k_hop
        self.dropout = dropout
        self.drop_fn = nn.Dropout(dropout)
        self.mlps = nn.ModuleList([Linear(hidden_size, hidden_size) for _ in range(k_hop)])
        self.activation = _activation(activation)

    def forward(self, graph, feature, norm=None):
        if norm is None:
            norm = GF.degree_norm(graph)
        h0 = feature
        for i in range(self.k_hop):
            beta_i = _math.log(1.0 * self.lambda_l / (i + 1) + 1)
            feature = self.drop_fn(feature)
            feature = _propagate_fused(graph, feature, norm, functools.partial(self._hop, graph, feature, norm, h0),
                                       a=1 - self.alpha, b=self.alpha, h=h0)
            feature_transed = self.mlps[i](feature)
            feature = beta_i * feature_transed + (1 - beta_i) * feature
            if self.activation is not None:
                feature = self.activation(feature)
        return feature

    def _hop(self, graph, feature, norm, h0):
        feature = _propagate(graph, feature, norm)
        return self.alpha * h0 + (1 - self.alpha) * feature


class TransformerConv(nn.Module):
    """reference pgl/nn/conv.py:724-885.  On a ``Graph`` the reference's UDF pair (send
    q[dst]*(k[src] + e) summed over the head dim -> recv softmax, dropout, weight v[src] + e, reduce)
    is one fused pass with a fused backward (``ops.dot_attention``), with or without edge features e.
    Shapes those kernels refuse are lowered, without edge features, to ``send_uv(mul)`` -> sum ->
    ``edge_softmax`` -> ``send_ue_recv(mul, sum)`` (no second gather of v by edge id, no
    zero+scatter); with edge features they run the send/recv pair like the reference."""

    def __init__(self, input_size, hidden_size, num_heads=4, feat_drop=0.6, attn_drop=0.6,
                 concat=True, skip_feat=True, gate=False, layer_norm=True, activation="relu"):
        super().__init__()
        self.hidden_size = hidden_size
        self.num_heads = num_heads
        self.feat_drop = feat_drop
        self.attn_drop = attn_drop
        self.concat = concat
        self.q = Linear(input_size, num_heads * hidden_size)
        self.k = Linear(input_size, num_heads * hidden_size)
        self.v = Linear(input_size, num_heads * hidden_size)
        self.feat_dropout = nn.Dropout(p=feat_drop)
        self.attn_dropout = nn.Dropout(p=attn_drop)
        width = num_heads * hidden_size if concat else hidden_size
        self.skip_feat = Linear(input_size, width) if skip_feat else None
        self.gate = Linear(3 * width, 1) if gate else None
        self.layer_norm = nn.LayerNorm(width) if layer_norm else None
        self.activation = _activation(activation)

    def send_attention(self, src_feat, dst_feat, edge_feat):
        if "edge_feat" in edge_feat:
            alpha = dst_feat["q"] * (src_feat["k"] + edge_feat["edge_feat"])
            v = src_feat["v"] + edge_feat["edge_feat"]
        else:
            alpha = dst_feat["q"] * src_feat["k"]
            v = src_feat["v"]
        return {"alpha": torch.sum(alpha, dim=-1), "v": v}

    def reduce_attention(self, msg):
        alpha = msg.reduce_softmax(msg["alpha"])
        alpha = alpha.reshape(-1, self.num_heads, 1)
        if self.attn_drop > 1e-15:
            alpha = self.attn_dropout(alpha)
        feature = msg["v"] * alpha
        if self.concat:
            feature = feature.reshape(-1, self.num_heads * self.hidden_size)
        else:
            feature = torch.mean(feature, dim=1)
        return msg.reduce(feature, pool_type="sum")

    def send_recv(self, graph, q, k, v, edge_feat):
        q = q / (self.hidden_size ** 0.5)
        output = None
        if type(graph).__name__ == "Graph" and q.is_cuda:
            # score, softmax, dropout and weighted sum in one pass with a fused backward (ops._DotAttn): no [E, H*Dh]
            # product; None when the shape is outside the kernels
            from .. import ops
            drop = self.attn_drop if self.attn_drop > 1e-15 and self.training else 0.0
            output = ops.dot_attention(graph._fwd_csr(), graph._bwd_csr, q, k, v, attn_drop=drop,
                                       edge_feat=edge_feat)
        if output is None and edge_feat is not None:
            msg = graph.send(self.send_attention, src_feat={"k": k, "v": v}, dst_feat={"q": q},
                             edge_feat={"edge_feat": edge_feat})
            return graph.recv(reduce_func=self.reduce_attention, msg=msg)
        if output is None:
            alpha = torch.sum(graph.send_uv(k, q, "mul"), dim=-1)
            alpha = GF.edge_softmax(graph, alpha).reshape(-1, self.num_heads, 1)
            if self.attn_drop > 1e-15:
                alpha = self.attn_dropout(alpha)
            output = graph.send_ue_recv(v, alpha, "mul", "sum")
        if self.concat:
            return output.reshape(-1, self.num_heads * self.hidden_size)
        return torch.mean(output, dim=1)

    def forward(self, graph, feature, edge_feat=None):
        if self.feat_drop > 1e-5:
            feature = self.feat_dropout(feature)
        q = self.q(feature).reshape(-1, self.num_heads, self.hidden_size)
        k = self.k(feature).reshape(-1, self.num_heads, self.hidden_size)
        v = self.v(feature).reshape(-1, self.num_heads, self.hidden_size)
        if edge_feat is not None:
            if self.feat_drop > 1e-5:
                edge_feat = self.feat_dropout(edge_feat)
            edge_feat = edge_feat.reshape(-1, self.num_heads, self.hidden_size)
        output = self.send_recv(graph, q, k, v, edge_feat=edge_feat)
        if self.skip_feat is not None:
            skip_feat = self.skip_feat(feature)
            if self.gate is not None:
                gate = torch.sigmoid(
                    self.gate(torch.cat([skip_feat, output, skip_feat - output], dim=-1)))
                output = gate * skip_feat + (1 - gate) * output
            else:
                output = skip_feat + output
        if self.layer_norm is not None:
            output = self.layer_norm(output)
        if self.activation is not None:
            output = self.activation(output)
        return output


class GINConv(nn.Module):
    """reference pgl/nn/conv.py:888-958."""

    def __init__(self, input_size, output_size, activation=None, init_eps=0.0, train_eps=False):
        super().__init__()
        self.input_size = input_size
        self.output_size = output_size
        self.linear1 = Linear(input_size, output_size)
        self.linear2 = Linear(output_size, output_size)
        self.layer_norm = nn.LayerNorm(output_size)
        if train_eps:
            self.epsilon = nn.Parameter(torch.full((1, 1), float(init_eps)))
        else:
            self.epsilon = init_eps
        self.activation = _activation(activation)

    def forward(self, graph, feature):
        neigh_feature = graph.send_recv(feature, reduce_func="sum")
        output = neigh_feature + feature * (self.epsilon + 1.0)
        output = self.linear1(output)
        output = self.layer_norm(output)
        if self.activation is not None:
            output = self.activation(output)
        return self.linear2(output)


class RGCNConv(nn.Module):
    """reference pgl/nn/conv.py:961-1024.  ``graph[etype]`` must give the homogeneous Graph of
    that relation (a HeterGraph in the reference; any mapping of Graphs here).  On a tensor-mode
    ``HeterGraph`` the layer runs as one relation-typed aggregation (``ops.rgcn_aggregate``) over the
    graph's typed CSR of ``etypes``; every other input, and every call that path declines, keeps the
    reference's per-relation loop."""

    def __init__(self, in_dim, out_dim, etypes, num_bases=0):
        super().__init__()
        self.in_dim = in_dim
        self.out_dim = out_dim
        self.etypes = etypes
        self.num_rels = len(self.etypes)
        self.num_bases = num_bases
        if self.num_bases <= 0 or self.num_bases >= self.num_rels:
            self.num_bases = self.num_rels
        self.weight = nn.Parameter(torch.empty(self.num_bases, in_dim, out_dim))
        nn.init.xavier_uniform_(self.weight)
        if self.num_bases < self.num_rels:
            self.w_comp = nn.Parameter(torch.empty(self.num_rels, self.num_bases))
            nn.init.xavier_uniform_(self.w_comp)

    def forward(self, graph, feat):
        if self.num_bases < self.num_rels:
            weight = torch.einsum("rb,bio->rio", self.w_comp, self.weight)
        else:
            weight = self.weight
        if isinstance(graph, HeterGraph) and graph.is_tensor() and isinstance(feat, torch.Tensor) and feat.is_cuda:
            fwd, bwd = graph.typed_csr(self.etypes, feat.device)
            out = ops.rgcn_aggregate(fwd, bwd, feat, weight)
            if out is not None:
                return out
        out = None
        for idx, etype in enumerate(self.etypes):
            h = graph[etype].send_recv(feat @ weight[idx], reduce_func="mean")
            out = h if out is None else out + h
        return out


class _KHopCached(nn.Module):
    def _smooth(self, graph, feature):
        raise NotImplementedError

    def _features(self, graph, feature):
        if not self.cached:
            return self._smooth(graph, feature)
        if self.cached_output is None:
            self.cached_output = self._smooth(graph, feature)
        return self.cached_output

    def _head(self, feature):
        output = self.linear(feature)
        if self.bias is not None:
            output = output + self.bias
        if self.activation is not None:
            output = self.activation(output)
        return output


class SGCConv(_KHopCached):
    """reference pgl/nn/conv.py:1027-1101."""

    def __init__(self, input_size, output_size, k_hop=2, cached=True, activation=None, bias=False):
        super().__init__()
        self.input_size = input_size
        self.output_size = output_size
        self.k_hop = k_hop
        self.linear = Linear(input_size, output_size, bias=False)
        self.bias = nn.Parameter(torch.zeros(output_size)) if bias else None
        self.cached = cached
        self.cached_output = None
        self.activation = _activation(activation)

    def _smooth(self, graph, feature):
        norm = GF.degree_norm(graph)
        for _ in range(self.k_hop):
            feature = _propagate(graph, feature, norm)
        return feature

    def forward(self, graph, feature):
        return self._head(self._features(graph, feature))


class SSGCConv(_KHopCached):
    """reference pgl/nn/conv.py:1104-1199 (the paper's formula: the running sum is accumulated out
    of place, it never aliases the caller's feature tensor)."""

    def __init__(self, input_size, output_size, k_hop=16, alpha=0.05, cached=True,
                 activation=None, bias=False):
        super().__init__()
        self.input_size = input_size
        self.output_size = output_size
        self.k_hop = k_hop
        self.alpha = alpha
        self.linear = Linear(input_size, output_size, bias=False)
        self.bias = nn.Parameter(torch.zeros(output_size)) if bias else None
        self.cached = cached
        self.cached_output = None
        self.activation = _activation(activation)

    def _smooth(self, graph, feature):
        norm = GF.degree_norm(graph)
        ori_feature = feature
        sum_feature = feature

        def hop(feature, sum_feature):
            feature = (1 - self.alpha) * _propagate(graph, feature, norm)
            return feature, sum_feature + feature

        for k in range(self.k_hop):
            # after the first hop the running sum is a buffer of this call's own, updated in place
            feature, sum_feature = _propagate_fused(graph, feature, norm, functools.partial(hop, feature, sum_feature),
                                                    a=1 - self.alpha, acc=sum_feature, inplace_acc=k > 0)
        return sum_feature / self.k_hop + self.alpha * ori_feature

    def forward(self, graph, feature):
        return self._head(self._features(graph, feature))


class NGCFConv(nn.Module):
    """reference pgl/nn/conv.py:1202-1249."""

    def __init__(self, input_size, output_size):
        super().__init__()
        self.input_size = input_size
        self.output_size = output_size
        self.linear = Linear(input_size, output_size)
        self.linear2 = Linear(input_size, output_size)
        for lin in (self.linear, self.linear2):
            bound = _math.sqrt(6.0 / (1 + output_size))
            nn.init.uniform_(lin.bias, -bound, bound)
        self.leaky_relu = nn.LeakyReLU(negative_slope=0.2)

    def forward(self, graph, feature):
        norm = GF.degree_norm(graph)
        neigh_feature = graph.send_recv(feature, "sum")
        output = (neigh_feature + feature) * norm
        output = self.linear(output) + self.linear2(feature * output)
        return self.leaky_relu(output)


class LightGCNConv(nn.Module):
    """reference pgl/nn/conv.py:1252-1284."""

    def forward(self, graph, feature):
        return _propagate(graph, feature, GF.degree_norm(graph))


class FAConv(nn.Module):
    """reference pgl/nn/conv.py:1287-1341.  The gate ``tanh(Linear([h_src ; h_dst]))`` splits into
    ``send_uv(h W_top, h W_bot, add)`` (two [N,1] projections instead of an [E, 2D] concat) and the
    weighted sum is ``send_ue_recv(mul, sum)``; the UDF spelling of the reference materialises
    [E, 2D] + [E, D].  On a ``Graph`` with CUDA features the gate, the norms, the dropout and the weighted sum are one
    fused pass with a fused backward (``ops.fa_attention``): no [E] tensor; calls those kernels refuse keep the op-by-op
    route.  The fused route returns the op-by-op route's dtype (torch's promotion of the feature, gate and norm dtypes);
    16-bit features are aggregated by the 16-bit kernel, whose result is rounded once to the feature dtype first."""

    def __init__(self, hidden_size, drop=0.5):
        super().__init__()
        self.hidden_size = hidden_size
        self.dropout = nn.Dropout(p=drop)
        self.gate = Linear(2 * hidden_size, 1)

    def forward(self, graph, feature):
        norm = GF.degree_norm(graph)
        d = self.hidden_size
        g_src = feature @ self.gate.weight[:d]
        g_dst = feature @ self.gate.weight[d:] + self.gate.bias
        if type(graph).__name__ == "Graph" and feature.is_cuda:
            drop = self.dropout.p if self.training else 0.0
            output = ops.fa_attention(graph._fwd_csr(), graph._bwd_csr, feature, g_src, g_dst, norm, attn_drop=drop)
            if output is not None:
                want = functools.reduce(torch.promote_types, (feature.dtype, g_src.dtype, g_dst.dtype, norm.dtype))
                return output if output.dtype == want else output.to(want)
        h = torch.tanh(graph.send_uv(g_src, g_dst, "add"))
        alpha = h * graph.send_uv(norm, norm, "mul")
        alpha = self.dropout(alpha)
        return graph.send_ue_recv(feature, alpha, "mul", "sum")
