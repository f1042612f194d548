"""numpy restatement of the graph-level readouts (reference pgl/math.py:227-364, pgl/utils/transform.py:101-168,
pgl/nn/functional/graph_op.py:78-98, pgl/nn/pool.py:121-179) in the reference's op order, quirks included.
segment_topk is stated by np.lexsort under the library's total order (score descending, -0.0 == +0.0, NaN after every
number, ties by ascending node index), with every score ranked (the reference's -1e20 padding is a defect, not a rule).
"""
import numpy as np


def indptr_of(segment_ids, num_segments=None):
    ids = np.asarray(segment_ids, np.int64)
    k = (int(ids[-1]) + 1 if ids.size else 0) if num_segments is None else int(num_segments)
    return np.searchsorted(ids, np.arange(k + 1), side="left").astype(np.int64)


def segment_padding(data, segment_ids):
    """math.py:254-272: (out [K, max_len, D], seq_len int32 [K], index int64 [N, 2]), K = last id + 1."""
    data = np.asarray(data)
    ids = np.asarray(segment_ids, np.int64)
    ip = indptr_of(ids)
    seq_len = np.diff(ip).astype(np.int32)
    max_len = int(seq_len.max()) if seq_len.size else 0
    pos = np.arange(ids.size, dtype=np.int64) - ip[ids]
    out = np.zeros((seq_len.size, max_len) + data.shape[1:], data.dtype)
    out[ids, pos] = data
    return out, seq_len, np.stack([ids, pos], 1)


def topk_k(n, ratio):
    """k of a segment of n nodes: min(ratio, n) for an int ratio, ceil(fp32(ratio) * fp32(n)) in fp32 otherwise
    (math.py:348-353: the float32 count tensor times the ratio, ceil)."""
    n = np.asarray(n)
    if isinstance(ratio, (int, np.integer)):
        return np.minimum(int(ratio), n).astype(np.int64)
    return np.ceil(np.float32(ratio) * n.astype(np.float32)).astype(np.int64)


def rank_order(scores):
    """Node order of one segment under the total order (scores as float32)."""
    s = np.asarray(scores, np.float32).astype(np.float64)
    nan = np.isnan(s)
    key = np.where(nan, 0.0, -s) + 0.0          # -0.0 -> +0.0; descending via the negation
    return np.lexsort((np.arange(s.size), key, nan))


def segment_topk_perm(scores, segment_ids, ratio):
    ids = np.asarray(segment_ids, np.int64)
    ip = indptr_of(ids)
    ks = topk_k(np.diff(ip), ratio)
    s = np.asarray(scores, np.float32).reshape(-1)
    parts = [ip[g] + rank_order(s[ip[g]:ip[g + 1]])[:ks[g]] for g in range(ip.size - 1)]
    return np.concatenate(parts).astype(np.int64) if parts else np.zeros(0, np.int64)


def segment_topk(x, scores, segment_ids, ratio, min_score=None):
    """math.py:336-364 -> (x[perm], perm).  min_score: keep i iff scores[i] > min(fp32(segmax - 1e-7), min_score),
    ascending node order."""
    x = np.asarray(x)
    if min_score is not None:
        s = np.asarray(scores, np.float32).reshape(-1)
        ids = np.asarray(segment_ids, np.int64)
        ip = indptr_of(ids)
        smax = np.array([s[ip[g]:ip[g + 1]].max() if ip[g + 1] > ip[g] else 0 for g in range(ip.size - 1)],
                        np.float32)
        thresh = np.minimum(smax[ids] - np.float32(1e-7), np.float32(min_score))
        perm = np.nonzero(s > thresh)[0].astype(np.int64)
    else:
        perm = segment_topk_perm(scores, segment_ids, ratio)
    return x[perm], perm


def to_dense_batch(x, graph_node_id, fill_value=0, max_num_nodes=None):
    """transform.py:120-135 -> (out [B, L, *F], mask [B, L], True at padding), B = max id + 1, out in x's dtype."""
    x = np.asarray(x)
    ids = np.asarray(graph_node_id, np.int64)
    B = int(ids.max()) + 1 if ids.size else 0
    ip = indptr_of(ids, B)
    counts = np.diff(ip)
    L = int(counts.max()) if max_num_nodes is None else int(max_num_nodes)
    pos = np.arange(ids.size) - ip[ids]
    out = np.full((B, L) + x.shape[1:], fill_value, x.dtype)
    out[ids, pos] = x
    mask = np.arange(L)[None, :] >= counts[:, None]
    return out, mask


def filter_adj(edge_index, perm, num_nodes=None):
    """transform.py:156-168 with an int64 position table: edges whose ends are both kept, relabelled, in order."""
    e = np.asarray(edge_index, np.int64).reshape(-1, 2)
    n = (int(e.max()) + 1 if e.size else 0) if num_nodes is None else int(num_nodes)
    table = np.full(n, -1, np.int64)
    table[np.asarray(perm, np.int64)] = np.arange(len(perm))
    m = table[e]
    return m[(m[:, 0] >= 0) & (m[:, 1] >= 0)]


def graph_norm(graph_node_id, feature):
    """graph_op.py:94-98 in float32: segment_sum(ones) -> sqrt -> gather -> divide."""
    ids = np.asarray(graph_node_id, np.int64)
    counts = np.bincount(ids).astype(np.float32).reshape(-1, 1)
    norm = np.sqrt(counts)[ids]
    return (np.asarray(feature, np.float32) / norm).astype(np.float32)


def attn_readout(x, segment_ids_or_indptr, gate=None, query=None, indptr=False):
    """pool.py:139-142 / 173-178 in float64: s = gate, or s_i = <x_i, q_g>; a = segment_softmax(s) (exp(s - max) /
    sum); out = segment_sum(a * x).  Returns (out [B, D], lse [B]); an empty segment gives 0 and -inf."""
    x = np.asarray(x, np.float64)
    ip = np.asarray(segment_ids_or_indptr, np.int64) if indptr else indptr_of(segment_ids_or_indptr)
    B, D = ip.size - 1, x.shape[1]
    out = np.zeros((B, D))
    lse = np.full(B, -np.inf)
    for g in range(B):
        rows = x[ip[g]:ip[g + 1]]
        if rows.shape[0] == 0:
            continue
        s = np.asarray(gate, np.float64).reshape(-1)[ip[g]:ip[g + 1]] if gate is not None else \
            rows @ np.asarray(query, np.float64)[g]
        m = s.max()
        e = np.exp(s - m)
        out[g] = (e / e.sum()) @ rows
        lse[g] = m + np.log(e.sum())
    return out, lse
