"""pgl_b200 -- PGL's send/recv message-passing path on H100 (sm_90a).

Drop-in for the hot path of PaddlePaddle/PGL (``import pgl_b200 as pgl``): Graph.send / recv /
send_recv / send_u_recv / send_ue_recv / send_uv, Message.reduce_*, pgl.math.segment_*,
GF.degree_norm / edge_softmax, GCNConv / GATConv / GraphSageConv, pgl.partition -- with torch
CUDA tensors as the device container and hand-written CUDA kernels behind a C-ABI
(include/pglb.h, libpglb.so).  Importing this package fails if libpglb.so has not been built.
"""
from . import _lib  # noqa: F401  (raises ImportError when the native library is missing)
from . import bigraph, graph, heter_graph, math, message, nn, ops, partition, sampling, utils  # noqa: F401
from .bigraph import BiGraph  # noqa: F401
from .graph import DistGPUGraph, Graph  # noqa: F401
from .heter_graph import HeterGraph  # noqa: F401

__version__ = "0.1.0"
