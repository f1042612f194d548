"""Segment operators (mirror of reference pgl/math.py:30-224) on the sm_90a kernels.

``paddle.geometric.segment_*`` -> ``pglb_spmm_csr_f32`` with identity columns (a sorted-segment
reduce is a CSR row reduce whose slot j reads row j); ``segment_softmax`` (7 Paddle ops in the
reference, math.py:216-224) -> one fused ``pglb_edge_softmax_csr_f32`` launch.
``segment_padding`` / ``segment_topk`` (math.py:227-364) -> ``pglb_segment_pad`` and
``pglb_segment_topk_count`` / ``_fill`` (csrc/readout.cu).
"""
import torch

from . import ops

__all__ = [
    "segment_pool", "segment_sum", "segment_mean", "segment_max", "segment_min",
    "segment_softmax", "segment_padding", "segment_topk",
]


def _indptr_of(segment_ids):
    """Compact CSR over the segments.  Graph.get_segment_ids attaches the cached one so the
    UDF recv path never re-derives it (and never syncs)."""
    cached = getattr(segment_ids, "_pglb_indptr", None)
    if cached is not None:
        return cached, getattr(segment_ids, "_pglb_max_degree", -1)
    ids = segment_ids if segment_ids.dtype == torch.int64 else segment_ids.to(torch.int64)
    n = int(ids.shape[0])
    k = int(ids[-1].item()) + 1 if n else 0
    return ops.segment_indptr(ids, k), -1


def segment_pool(data, segment_ids, pool_type, name=None):
    """reference pgl/math.py:30-46."""
    pool_type = pool_type.upper()
    if pool_type not in ("SUM", "MEAN", "MAX", "MIN"):
        raise ValueError(
            "We only support sum, mean, max, min pool types in segment_pool function.")
    ops.require_cuda(data, segment_ids)
    indptr, maxdeg = _indptr_of(segment_ids)
    from .utils.op import LazyRows
    if isinstance(data, LazyRows) and data.is_lazy():
        # untouched message rows: fuse the gather into the reduce (no [E, D] materialisation)
        return ops.segment_reduce(data._lz_base, None, pool_type.lower(), indptr=indptr,
                                  cols=data._lz_index.contiguous(), max_degree=maxdeg)
    return ops.segment_reduce(data, None, pool_type.lower(), indptr=indptr, max_degree=maxdeg)


def segment_sum(data, segment_ids, name=None):
    """reference pgl/math.py:49-79: out_i = sum_j data_j over segment_ids[j] == i."""
    return segment_pool(data, segment_ids, "sum")


def segment_mean(data, segment_ids, name=None):
    """reference pgl/math.py:82-113."""
    return segment_pool(data, segment_ids, "mean")


def segment_min(data, segment_ids, name=None):
    """reference pgl/math.py:116-145."""
    return segment_pool(data, segment_ids, "min")


def segment_max(data, segment_ids, name=None):
    """reference pgl/math.py:148-178."""
    return segment_pool(data, segment_ids, "max")


def segment_softmax(data, segment_ids):
    """reference pgl/math.py:181-224: exp(x - segmax) / segsum, fused into one kernel."""
    ops.require_cuda(data, segment_ids)
    indptr, _ = _indptr_of(segment_ids)
    return ops.edge_softmax_csr(indptr, None, data, int(data.shape[0]))


def segment_padding(data, segment_ids):
    """reference pgl/math.py:227-272: (out [K, max_len, D], seq_len int32 [K], index int64 [N, 2]) with K = last id + 1;
    ids that do not appear get zero blocks.  out is written once by the pad kernel, in data's dtype; index[i] =
    (segment_ids[i], position of row i inside its segment)."""
    ops.require_cuda(data, segment_ids)
    ids = segment_ids if segment_ids.dtype == torch.int64 else segment_ids.to(torch.int64)
    n = int(ids.shape[0])
    k = int(ids[-1].item()) + 1 if n else 0
    indptr = ops.segment_indptr(ids, k)
    seq_len = (indptr[1:] - indptr[:-1]).to(torch.int32)
    out = ops.segment_pad(data, indptr, ops.segment_max_len(indptr), 0)
    pos = torch.arange(n, dtype=torch.int64, device=ids.device) - indptr[ids]
    return out, seq_len, torch.stack([ids, pos], 1)


def segment_topk(x, scores, segment_ids, ratio, min_score=None, return_index=False):
    """reference pgl/math.py:299-364.  Without min_score: the first k_g ranks of every segment (``ops.segment_topk_perm``:
    score descending, ties by ascending node index, every score ranks -- no -1e20 padding), k_g = ceil(fp32(ratio) *
    n_g) for a float ratio in (0, 1], min(ratio, n_g) for an int ratio >= 1; anything else raises ValueError.  With
    min_score: the reference's arithmetic -- keep node i iff scores[i] > min(fp32(segmax_g - 1e-7), min_score), in
    ascending node order.  x[perm] is a row gather, so gradients reach x."""
    if min_score is None:
        if isinstance(ratio, int):
            if ratio < 1:
                raise ValueError("segment_topk: an int ratio must be at least 1, got %d" % ratio)
        elif not 0.0 < float(ratio) <= 1.0:
            raise ValueError("segment_topk: a float ratio must lie in (0, 1], got %r" % (ratio,))
    ops.require_cuda(x, scores, segment_ids)
    if min_score is not None:
        smax = segment_max(scores, segment_ids)
        thresh = (ops.gather_rows(smax.reshape(-1, 1), segment_ids).reshape(-1) - 1e-7).clamp(max=min_score)
        perm = (scores.reshape(-1) > thresh).nonzero().reshape(-1)
    else:
        indptr, _ = _indptr_of(segment_ids)
        perm = ops.segment_topk_perm(scores, indptr, ratio)
    out = ops.gather_rows(x, perm)
    if return_index:
        return out, perm
    return out
