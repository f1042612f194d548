"""Random walks (mirror of reference pgl/sampling/walk.py:23-183) on the sm_90a kernels of csrc/walk.cu: one walker
per thread, the whole walk in one launch, on the graph's src-keyed CSR (successors = out-edges; a duplicate edge counts
once per slot, self-loops are allowed).

* ``random_walk``: at most ``max_depth`` nodes; each step takes a successor slot uniformly.
* ``node2vec_walk``: with ``p == q == 1`` it is ``random_walk``; otherwise up to ``max_depth`` steps, so at most
  ``max_depth + 1`` nodes (the reference's count).  A step from ``cur`` after ``prev`` takes a slot with probability
  proportional to 1/p (it holds ``prev``), 1 (a successor of ``prev``) or 1/q (anything else).
* ``node2vec_walk_plus``: the same, with "near" meaning a successor of any earlier node of the walk.
* ``metapath_randomwalk``: on a ``HeterGraph`` (the reference's examples/metapath2vec), at most ``walk_length``
  nodes; step t takes a successor slot uniformly in relation ``metapath[t % len(metapath)]``, by the draw of a
  ``random_walk`` step, so a one-relation metapath ``[r]`` gives ``random_walk(graph[r], ...)`` exactly.

A walk ends early exactly when its current node has no successors (in the step's relation).  Return type by graph mode: a numpy-mode graph
gives a list of ``len(nodes)`` lists of ints (the reference's contract); a tensor-mode graph gives one int64 CUDA
tensor ``[len(nodes), L]`` padded with -1 (L = max_depth or walk_length, or max_depth + 1 for the node2vec rules).  ``seed=None``
draws a 64-bit seed from ``np.random``, so ``np.random.seed`` makes the walks reproducible; the walks are a pure
function of (graph, nodes, seed)."""
import math

import numpy as np
import torch

from .. import ops

__all__ = ["random_walk", "node2vec_walk", "node2vec_walk_plus", "metapath_randomwalk"]

UNIFORM, NODE2VEC, NODE2VEC_PLUS = 0, 1, 2   # the modes of pglb_walk_host
METAPATH_MAX = 64   # relations per metapath (the kernel's parameter bank)


def walk_mode(p, q, plus):
    """The rule a call runs: p == q == 1 is random_walk (at most max_depth nodes), as in the reference."""
    if p == 1.0 and q == 1.0:
        return UNIFORM
    return NODE2VEC_PLUS if plus else NODE2VEC


def check_args(num_nodes, nodes, max_depth, p=1.0, q=1.0, depth_name="max_depth"):
    """ValueError for arguments the walks refuse, before any device work.  Returns nodes as a 1-D int64 array or
    tensor."""
    if isinstance(max_depth, bool) or int(max_depth) != max_depth or not 1 <= int(max_depth) < 2 ** 31 - 1:
        raise ValueError("%s must be an integer >= 1, got %r" % (depth_name, max_depth))
    for name, v in (("p", p), ("q", q)):
        v = float(v)
        if not (v > 0 and math.isfinite(v) and math.isfinite(1.0 / v)):
            raise ValueError("%s must be positive and finite, got %r" % (name, v))
    if isinstance(nodes, torch.Tensor):
        if nodes.dtype.is_floating_point or nodes.dtype == torch.bool:
            raise ValueError("nodes must hold integer ids")
        nodes = nodes.reshape(-1).to(torch.int64)
        lo, hi = (int(nodes.min().item()), int(nodes.max().item())) if nodes.numel() else (0, -1)
    else:
        arr = np.asarray(nodes)
        if arr.size and arr.dtype.kind not in "iu":
            raise ValueError("nodes must hold integer ids")
        nodes = arr.astype(np.int64).reshape(-1)
        lo, hi = (int(nodes.min()), int(nodes.max())) if nodes.size else (0, -1)
    if nodes.shape[0] and (lo < 0 or hi >= num_nodes):
        raise ValueError("start node %d outside [0, %d)" % (lo if lo < 0 else hi, num_nodes))
    return nodes


def _seed(seed):
    if seed is None:
        return int(np.random.randint(0, 2 ** 64, dtype=np.uint64))
    return int(seed) & 0xFFFFFFFFFFFFFFFF


def _walk(graph, nodes, max_depth, p, q, plus, seed):
    nodes = check_args(graph._n, nodes, max_depth, p, q)
    mode = walk_mode(float(p), float(q), plus)
    seed = _seed(seed)
    indptr, cols, sorted_cols = graph._walk_csr(row_sorted=mode != UNIFORM)
    nodes = torch.as_tensor(nodes).to(indptr.device)
    if mode == UNIFORM:
        out = ops.random_walk(indptr, cols, graph._n, nodes, max_depth, seed)
    else:
        out = ops.node2vec_walk(indptr, cols, sorted_cols, graph._n, nodes, max_depth, p, q, mode == NODE2VEC_PLUS,
                                seed)
    return _by_mode(graph, out)


def _by_mode(graph, out):
    """The padded [n, L] walks as the graph's mode returns them: the tensor itself, or lists without the padding."""
    if graph.is_tensor():
        return out
    rows = out.cpu().numpy()
    lengths = (rows >= 0).sum(1).tolist()
    return [r[:k] for r, k in zip(rows.tolist(), lengths)]


def random_walk(graph, nodes, max_depth, seed=None):
    """Uniform random walks from ``nodes`` with at most ``max_depth`` nodes each (reference walk.py:23-64)."""
    return _walk(graph, nodes, max_depth, 1.0, 1.0, False, seed)


def node2vec_walk(graph, nodes, max_depth, p=1.0, q=1.0, seed=None):
    """node2vec walks (Grover & Leskovec, KDD'16; reference walk.py:67-122): return parameter p, in-out parameter q."""
    return _walk(graph, nodes, max_depth, p, q, False, seed)


def node2vec_walk_plus(graph, nodes, max_depth, p=1.0, q=1.0, seed=None):
    """node2vec walks whose "near" set is the successors of every earlier node of the walk (reference
    walk.py:125-183)."""
    return _walk(graph, nodes, max_depth, p, q, True, seed)


def metapath_randomwalk(graph, start_nodes, metapath, walk_length, seed=None):
    """Metapath walks on a ``HeterGraph`` (the reference's examples/metapath2vec/datasets/sampling.py
    ``metapath_randomwalk``), all walkers and steps in one launch.

    Args:
        graph: a ``HeterGraph``, numpy or tensor mode.
        start_nodes: the start node of every walk.
        metapath: ``"c2p-p2a-a2p-p2c"`` (split on ``-``) or a list / tuple of edge types, 1 to 64 of them; a relation
            may repeat.  Step t follows ``metapath[t % len(metapath)]``.  Nothing checks that the relations chain by
            node type.
        walk_length: at most this many nodes per walk.  A walk ends early exactly when its node has no out-edge in
            the step's relation; a start without one in ``metapath[0]`` gives a walk of one node.
        seed: 64-bit seed; None draws one from ``np.random``.

    Returns a list of lists of node ids (numpy mode) or an int64 CUDA tensor ``[len(start_nodes), walk_length]``
    padded with -1 (tensor mode)."""
    from ..heter_graph import HeterGraph
    if not isinstance(graph, HeterGraph):
        raise TypeError("metapath_randomwalk needs a HeterGraph, got %s" % type(graph).__name__)
    etypes = metapath.split("-") if isinstance(metapath, str) else list(metapath)
    if not etypes:
        raise ValueError("metapath is empty")
    if len(etypes) > METAPATH_MAX:
        raise ValueError("a metapath has at most %d relations, got %d" % (METAPATH_MAX, len(etypes)))
    valid = graph.edge_types
    for e in etypes:
        if e not in valid:
            raise ValueError("unknown edge type %r in the metapath; the graph has %s" % (e, valid))
    num_nodes = int(graph[etypes[0]]._n)
    nodes = check_args(num_nodes, start_nodes, walk_length, depth_name="walk_length")
    seed = _seed(seed)
    csr = {}
    for e in etypes:
        if e not in csr:
            csr[e] = graph[e]._walk_csr()[:2]
    indptrs, cols = zip(*[csr[e] for e in etypes])
    nodes = torch.as_tensor(nodes).to(indptrs[0].device)
    return _by_mode(graph, ops.metapath_walk(indptrs, cols, num_nodes, nodes, walk_length, seed))
