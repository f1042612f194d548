"""Torch-tensor front end of the C-ABI (include/pglb.h): allocates outputs / workspaces with
torch, passes raw device pointers + the current CUDA stream to libpglb.  CUDA tensors only --
every function raises on CPU tensors; there is no eager / CPU fallback on this path.
"""
import ctypes
import functools
import os

import torch

from . import _lib
from ._lib import BCAST_FULL, BCAST_HEAD, BCAST_SCALAR, MSG, REDUCE, check, lib

_ws_cache = {}


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                "pgl_b200: tensor-mode ops run on CUDA tensors only (got a %s tensor); "
                "there is no CPU fallback on the send/recv path" % t.device)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def workspace(device, nbytes):
    """Per-(device, stream) scratch buffer, grown geometrically; stream-ordered reuse."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        n = max(int(nbytes), 1 << 20)
        if buf is not None:
            n = max(n, int(buf.numel() * 1.5))
        buf = torch.empty(n, dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


def _i64(t):
    if t.dtype != torch.int64:
        t = t.to(torch.int64)
    return t


HALF_DTYPES = (torch.bfloat16, torch.float16)
_DTYPE16 = {torch.bfloat16: _lib.DTYPE_BF16, torch.float16: _lib.DTYPE_F16}


def _cast_through(fn, native16):
    """Run fp32 kernels for callers in other float dtypes; autograd flows through every cast.
    float64 anywhere in the arguments: every float64 and 16-bit tensor is rounded / widened to float32 on the way in
    and the float32 results are widened to float64 on the way out.  Otherwise, unless `native16` (fn has 16-bit kernels
    of its own and takes such tensors as they are), 16-bit tensors are widened to float32 exactly, the fp32 kernels
    run, and float32 results are rounded to the promoted dtype of the floating-point tensor arguments (torch
    promotion: bf16 with fp32 gives fp32)."""

    def dtype_of(v):
        return v.dtype if isinstance(v, torch.Tensor) or hasattr(v, "materialize") else None

    def dtypes(v):
        d = dtype_of(v)
        if d is not None:
            return [d] if d.is_floating_point else []
        if isinstance(v, (list, tuple)):
            return [x for a in v for x in dtypes(a)]
        return []

    def to32(v, widen):
        if dtype_of(v) in widen:
            mat = getattr(v, "materialize", None)
            return (mat() if mat is not None else v).to(torch.float32)
        if isinstance(v, (list, tuple)):
            return type(v)(to32(a, widen) for a in v)
        return v

    def back(v, dtype):
        if isinstance(v, torch.Tensor) and v.dtype == torch.float32:
            return v.to(dtype)
        if isinstance(v, tuple):
            return tuple(back(a, dtype) for a in v)
        return v

    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        found = [d for a in list(args) + list(kwargs.values()) for d in dtypes(a)]
        if torch.float64 in found:
            widen, result = (torch.float64,) + HALF_DTYPES, torch.float64
        elif not native16 and any(d in HALF_DTYPES for d in found):
            widen, result = HALF_DTYPES, functools.reduce(torch.promote_types, found)
        else:
            return fn(*args, **kwargs)
        out = fn(*[to32(a, widen) for a in args], **{k: to32(a, widen) for k, a in kwargs.items()})
        return back(out, result) if result != torch.float32 else out
    return wrapper


def f64_through(fn):
    """float64 in -> float64 out for the public feature ops (the reference's tests/test_conv.py:43-71 runs GCN,
    GraphSage and GAT in float64), and bfloat16 / float16 in -> the same dtype out for ops without 16-bit kernels.
    The kernels are fp32: float64 tensors are rounded to float32 on the way in and the result is widened on the way
    out, so a float64 caller gets fp32-accurate values in its own dtype -- within the path's stated 1e-4 relative
    tolerance, not fp64 accuracy (INTEGRATION.md).  16-bit tensors are widened exactly and the result rounded once
    (see _cast_through)."""
    return _cast_through(fn, native16=False)


def native16_through(fn):
    """f64_through for the ops with 16-bit kernels of their own (copy aggregation, segment_*): bfloat16 / float16
    features reach them unchanged; float64 follows f64_through."""
    return _cast_through(fn, native16=True)


def _f32_2d(t, allow16=False):
    """[n, d1, d2, ...] -> contiguous [n, D] float32 view (no copy when already so).  A lazy row
    gather (utils.op.LazyRows) is resolved to its plain tensor first: the wrapper itself carries no
    autograd state, so requires_grad must be read from the gathered result.  allow16: bfloat16 / float16 pass
    too (the copy aggregation's 16-bit route)."""
    mat = getattr(t, "materialize", None)
    if mat is not None:
        t = mat()
    if t.dtype != torch.float32 and not (allow16 and t.dtype in HALF_DTYPES):
        raise TypeError("pgl_b200: float32 features expected on the CUDA path, got %s" % t.dtype)
    t2 = t.reshape(t.shape[0], -1) if t.dim() != 2 else t
    if not t2.is_contiguous():
        t2 = t2.contiguous()
    return t2


# ------------------------------------------------------------------------------------------
# index construction
# ------------------------------------------------------------------------------------------


def csr_build(u, v, num_nodes):
    """Device twin of graph_kernel.build_index (reference pgl/graph_kernel.pyx:59-88).
    u, v: 1-D int64 CUDA tensors (strided views such as edges[:, 1] are read in place).
    Returns (degree, sorted_v, sorted_u, sorted_eid, indptr) like the reference."""
    require_cuda(u, v)
    u = _i64(u)
    v = _i64(v)
    E = int(u.shape[0])
    N = int(num_nodes)
    dev = u.device
    degree = torch.empty(N, dtype=torch.int64, device=dev)
    indptr = torch.empty(N + 1, dtype=torch.int64, device=dev)
    su = torch.empty(E, dtype=torch.int64, device=dev)
    sv = torch.empty(E, dtype=torch.int64, device=dev)
    se = torch.empty(E, dtype=torch.int64, device=dev)
    need = ctypes.c_size_t(0)
    check(lib.pglb_csr_build_ws(E, N, ctypes.byref(need)))
    ws = workspace(dev, need.value)
    us = u.stride(0) if E > 0 else 1
    vs = v.stride(0) if E > 0 else 1
    with torch.cuda.device(dev):
        check(lib.pglb_csr_build(_ptr(u), max(us, 1), _ptr(v), max(vs, 1), E, N, _ptr(degree),
                                 _ptr(indptr), _ptr(su), _ptr(sv), _ptr(se), _ptr(ws),
                                 ws.numel(), _stream()))
    return degree, sv, su, se, indptr


# random walks (csrc/walk.cu)
# ------------------------------------------------------------------------------------------


def _walk_args(indptr, cols, nodes):
    require_cuda(indptr, cols, nodes)
    nodes = _i64(nodes).reshape(-1).contiguous()
    # a graph without edges has an empty cols tensor (no address); the kernels never read it then
    cols_p = _ptr(cols) if cols.numel() else _ptr(indptr)
    return nodes, cols_p


def random_walk(indptr, cols, num_nodes, nodes, max_depth, seed):
    """pglb_random_walk: [len(nodes), max_depth] int64 walks over the src-keyed CSR (indptr, cols), -1 after a walk
    ends."""
    nodes, cols_p = _walk_args(indptr, cols, nodes)
    out = torch.empty((nodes.numel(), int(max_depth)), dtype=torch.int64, device=nodes.device)
    with torch.cuda.device(nodes.device):
        check(lib.pglb_random_walk(_ptr(indptr), cols_p, int(num_nodes), _ptr(nodes), nodes.numel(), int(max_depth),
                                   int(seed), _ptr(out), _stream()))
    return out


def node2vec_walk(indptr, cols, sorted_cols, num_nodes, nodes, max_depth, p, q, plus, seed, stats=None):
    """pglb_node2vec_walk: [len(nodes), max_depth + 1] int64 walks, -1 after a walk ends.  sorted_cols: cols with every
    row ascending by id.  stats: optional int64 CUDA tensor of 2, incremented by (candidate draws, fallback steps)."""
    nodes, cols_p = _walk_args(indptr, cols, nodes)
    out = torch.empty((nodes.numel(), int(max_depth) + 1), dtype=torch.int64, device=nodes.device)
    with torch.cuda.device(nodes.device):
        check(lib.pglb_node2vec_walk(_ptr(indptr), cols_p, _ptr(sorted_cols) if sorted_cols.numel() else cols_p,
                                     int(num_nodes), _ptr(nodes), nodes.numel(), int(max_depth), float(p), float(q),
                                     int(bool(plus)), int(seed), _ptr(out), _ptr(stats), _stream()))
    return out


def metapath_walk(indptrs, cols_list, num_nodes, nodes, walk_length, seed):
    """pglb_metapath_walk: [len(nodes), walk_length] int64 walks, -1 after a walk ends.  Step t follows the src-keyed
    CSR (indptrs[t % m], cols_list[t % m]); the m CSRs share num_nodes and one device."""
    nodes, _ = _walk_args(indptrs[0], cols_list[0], nodes)
    cols_p = [_walk_args(ip, c, nodes)[1].value for ip, c in zip(indptrs, cols_list)]
    if any(t.device != nodes.device for t in list(indptrs) + list(cols_list)):
        raise ValueError("metapath_walk: the CSRs and the start nodes must be on one device")
    m = len(cols_p)
    indptr_arr = (ctypes.c_void_p * m)(*[ip.data_ptr() for ip in indptrs])
    cols_arr = (ctypes.c_void_p * m)(*cols_p)
    out = torch.empty((nodes.numel(), int(walk_length)), dtype=torch.int64, device=nodes.device)
    with torch.cuda.device(nodes.device):
        check(lib.pglb_metapath_walk(indptr_arr, cols_arr, m, int(num_nodes), _ptr(nodes), nodes.numel(),
                                     int(walk_length), int(seed), _ptr(out), _stream()))
    return out


# skip-gram pairs and alias sampling (csrc/skipgram.cu)
# ------------------------------------------------------------------------------------------


def skip_gram_pairs(walks, win_size, seed):
    """pglb_skipgram_count + pglb_skipgram_fill: (src, pos) int64 pairs of the padded [B, L] int64 walks.  One count,
    the scan, one device-to-host read of the total and one fill."""
    require_cuda(walks)
    walks = _i64(walks).contiguous()
    B, L = walks.shape
    dev = walks.device
    if B == 0 or L == 0:
        return (torch.empty(0, dtype=torch.int64, device=dev), torch.empty(0, dtype=torch.int64, device=dev))
    offsets = torch.empty(B + 1, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        need = ctypes.c_size_t(0)
        check(lib.pglb_skipgram_count_ws(B, ctypes.byref(need)))
        ws = workspace(dev, need.value)
        check(lib.pglb_skipgram_count(_ptr(walks), B, L, int(win_size), int(seed), _ptr(offsets), _ptr(ws),
                                      ws.numel(), _stream()))
        total = int(offsets[B].item())
        src = torch.empty(total, dtype=torch.int64, device=dev)
        pos = torch.empty(total, dtype=torch.int64, device=dev)
        if total:
            check(lib.pglb_skipgram_fill(_ptr(walks), B, L, int(win_size), int(seed), _ptr(offsets), _ptr(src),
                                         _ptr(pos), _stream()))
    return src, pos


def alias_sample(alias, events, count, seed):
    """pglb_alias_sample: count int64 draws of the table (alias float64 [n], events int64 [n]) on their device."""
    require_cuda(alias, events)
    alias = alias.to(torch.float64).contiguous()
    events = _i64(events).contiguous()
    out = torch.empty(int(count), dtype=torch.int64, device=alias.device)
    with torch.cuda.device(alias.device):
        check(lib.pglb_alias_sample(_ptr(alias), _ptr(events), alias.numel(), int(count), int(seed), _ptr(out),
                                    _stream()))
    return out


# skip-gram negative-sampling loss (csrc/sgns.cu forward; the backward on csr_build and the aggregation)
# ------------------------------------------------------------------------------------------


def _sgns_check_ids(src, dsts):
    """The id checks that need no device: dtype, rank, K >= 1 and matching P."""
    for name, t in (("src", src), ("dsts", dsts)):
        if not isinstance(t, torch.Tensor) or t.dtype not in (torch.int32, torch.int64):
            raise ValueError("skip_gram_loss: %s must be an int32 or int64 tensor, got %s"
                             % (name, getattr(t, "dtype", type(t).__name__)))
    if not (src.dim() == 1 or (src.dim() == 2 and src.shape[1] == 1)):
        raise ValueError("skip_gram_loss: src must be [P] or [P, 1], got %s" % (tuple(src.shape),))
    if dsts.dim() != 2 or dsts.shape[1] < 2:
        raise ValueError("skip_gram_loss: dsts must be [P, 1 + K] with K >= 1, got %s" % (tuple(dsts.shape),))
    P = int(src.shape[0])
    if P < 1 or int(dsts.shape[0]) != P:
        raise ValueError("skip_gram_loss: src has %d pairs and dsts %d; both need at least one" % (P, dsts.shape[0]))


def _sgns_ids(src, dsts, n_emb, n_ctx):
    """src / dsts as contiguous int64 [P] / [P, 1 + K], after one read-back of the ids' extremes: IndexError outside
    the tables, before any kernel dereferences a row."""
    lo_s, hi_s = torch.aminmax(src)
    lo_d, hi_d = torch.aminmax(dsts)
    lo_s, hi_s, lo_d, hi_d = torch.stack([lo_s.long(), hi_s.long(), lo_d.long(), hi_d.long()]).tolist()
    if lo_s < 0 or hi_s >= n_emb:
        raise IndexError("skip_gram_loss: src ids span [%d, %d], outside the centre table of %d rows"
                         % (lo_s, hi_s, n_emb))
    if lo_d < 0 or hi_d >= n_ctx:
        raise IndexError("skip_gram_loss: dsts ids span [%d, %d], outside the context table of %d rows"
                         % (lo_d, hi_d, n_ctx))
    return _i64(src).reshape(-1).contiguous(), _i64(dsts).contiguous()


def _sgns_table(t):
    """t as rows of unit column stride that do not overlap (ld >= D), copied only when it is not already so: an
    expanded or otherwise overlapping view is read from a contiguous copy."""
    return t if t.stride(1) == 1 and t.stride(0) >= t.shape[1] else t.contiguous()


def _sgns_fwd_raw(emb, ctx, src, dsts, train):
    """pglb_sgns_fwd_f32: (loss, c, w); c [P, 1 + K] and w [P, D] only when train."""
    P, J = dsts.shape
    D = int(emb.shape[1])
    dev = emb.device
    loss = torch.empty((), dtype=torch.float32, device=dev)
    c = torch.empty((P, J), dtype=torch.float32, device=dev) if train else None
    w = torch.empty((P, D), dtype=torch.float32, device=dev) if train else None
    need = ctypes.c_size_t(0)
    check(lib.pglb_sgns_fwd_ws(P, ctypes.byref(need)))
    ws = workspace(dev, need.value)
    with torch.cuda.device(dev):
        check(lib.pglb_sgns_fwd_f32(_ptr(emb), int(emb.shape[0]), emb.stride(0), _ptr(ctx), int(ctx.shape[0]),
                                    ctx.stride(0), _ptr(src), _ptr(dsts), P, J - 1, D, _ptr(loss), _ptr(c), _ptr(w),
                                    D, _ptr(ws), ws.numel(), _stream()))
    return loss, c, w


def _touched(indptr, num_edges):
    """Rows of a key-sorted CSR that hold a slot, and the CSR compacted to them: (rows [R], indptr [R + 1])."""
    rows, _ = segment_ids_from_indptr(indptr, num_edges)
    return rows, torch.cat([indptr[rows], indptr[-1:]])


def _sgns_grads(g, emb, src, dsts, c, w, n_emb, n_ctx, shared, sparse, need_emb, need_ctx):
    """d loss / d emb and d ctx (one tensor for a shared table) as segment sums by node id:
    d emb[n] = g sum_{p: src[p] = n} w[p] over the CSR of the P keys src (slots -> pairs);
    d ctx[m] = g sum_{(p, j): dsts[p, j] = m} c[p, j] emb[src[p]] over the CSR of the P (1 + K) keys dsts, with the
    edge operand g c.  csr_build is stable and the aggregation sums every row in slot order: no atomics, so the
    gradients are bit-identical run to run.  sparse: coalesced COO gradients over the touched rows only."""
    P, J = dsts.shape
    D = int(emb.shape[1])
    dev = emb.device
    E = P * J
    ge = gc = None
    if need_emb or shared:
        _, _, _, pair, ip_e = csr_build(src, src, n_emb)
        # the upstream scalar as a per-slot operand of stride 0: stays on the device
        g_slot = g.reshape(1, 1).expand(P, 1)
    if need_ctx or shared:
        _, col_c, _, slot_c, ip_c = csr_build(dsts.reshape(-1), src.repeat_interleave(J), n_ctx)
        gcoef = (c.reshape(-1) * g).reshape(E, 1)

    def emb_part(indptr, rows, out, acc):
        return _spmm_raw(indptr, pair, w, rows, "sum", y2=g_slot, y_bcast=BCAST_SCALAR, msg_op="mul", num_edges=P,
                         out=out, accumulate=acc)

    def ctx_part(indptr, rows, out, acc):
        return _spmm_raw(indptr, col_c, emb, rows, "sum", eid=slot_c, y2=gcoef, y_bcast=BCAST_SCALAR, msg_op="mul",
                         num_edges=E, out=out, accumulate=acc)

    if shared:
        if not sparse:
            out = emb_part(ip_e, n_emb, None, False)
            return ctx_part(ip_c, n_emb, out, True), None
        rows, _ = segment_ids_from_indptr(ip_e + ip_c, P + E)     # rows touched in either role
        cip_e = torch.cat([ip_e[rows], ip_e[-1:]])
        cip_c = torch.cat([ip_c[rows], ip_c[-1:]])
        vals = emb_part(cip_e, int(rows.numel()), None, False)
        vals = ctx_part(cip_c, int(rows.numel()), vals, True)
        return torch.sparse_coo_tensor(rows[None], vals, (n_emb, D), is_coalesced=True, check_invariants=False), None
    if need_emb:
        if sparse:
            rows, cip = _touched(ip_e, P)
            ge = torch.sparse_coo_tensor(rows[None], emb_part(cip, int(rows.numel()), None, False), (n_emb, D),
                                         is_coalesced=True, check_invariants=False)
        else:
            ge = emb_part(ip_e, n_emb, None, False)
    if need_ctx:
        if sparse:
            rows, cip = _touched(ip_c, E)
            gc = torch.sparse_coo_tensor(rows[None], ctx_part(cip, int(rows.numel()), None, False), (n_ctx, D),
                                         is_coalesced=True, check_invariants=False)
        else:
            gc = ctx_part(ip_c, n_ctx, None, False)
    return ge, gc


class _SkipGramLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, emb, ctx_table, src, dsts, sparse, train):
        shared = ctx_table is None
        table = emb if shared else ctx_table
        loss, c, w = _sgns_fwd_raw(emb, table, src, dsts, train)
        if train:
            ctx.save_for_backward(emb, src, dsts, c, w)
            ctx.meta = (int(emb.shape[0]), int(table.shape[0]), shared, bool(sparse))
        return loss

    @staticmethod
    def backward(ctx, g):
        emb, src, dsts, c, w = ctx.saved_tensors
        n_emb, n_ctx, shared, sparse = ctx.meta
        ge, gc = _sgns_grads(g, emb, src, dsts, c, w, n_emb, n_ctx, shared, sparse,
                             ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        return ge, gc, None, None, None, None


@f64_through
def _skip_gram_loss_f32(emb, ctx, src, dsts, sparse):
    # training writes c and w for the backward; inside torch.no_grad(), or when no table needs a gradient, the kernel
    # writes the loss only (needs_input_grad inside forward follows requires_grad, not grad mode)
    train = torch.is_grad_enabled() and (emb.requires_grad or (ctx is not None and ctx.requires_grad))
    return _SkipGramLoss.apply(_sgns_table(emb), None if ctx is None else _sgns_table(ctx), src, dsts, sparse, train)


def skip_gram_loss(emb, ctx, src, dsts, sparse=False):
    """The skip-gram negative-sampling loss of the reference's SkipGramModel on the fused kernel (pglb_sgns_fwd_f32):
    (BCEWithLogits(<emb[src], ctx[dsts[:, 0]]>, 1) + BCEWithLogits(<emb[src], ctx[dsts[:, 1:]]>, 0)) / 2, mean
    reduction.  ``ctx is emb`` is a shared table, which receives both roles' gradients.  float32 tables (float64
    through f64_through); int32 / int64 CUDA ids.  sparse: the gradients are coalesced sparse COO tensors over the
    touched rows (for torch.optim.SparseAdam, SGD, Adagrad), else dense [N, D].  Every check precedes any launch:
    16-bit or other non-float32/64 tables raise TypeError; float or bool ids, wrong ranks and K = 0 raise ValueError;
    ids outside their table raise IndexError (one read-back of the ids' extremes)."""
    shared = ctx is emb
    for name, t in (("emb", emb), ("ctx", ctx)):
        if t.dtype not in (torch.float32, torch.float64):
            raise TypeError("skip_gram_loss: float32 or float64 tables, got %s for %s" % (t.dtype, name))
        if t.dim() != 2:
            raise ValueError("skip_gram_loss: %s must be a 2-D table, got %s" % (name, tuple(t.shape)))
    if emb.shape[1] != ctx.shape[1] or emb.shape[1] < 1:
        raise ValueError("skip_gram_loss: the tables' widths differ or are 0 (%d, %d)" % (emb.shape[1], ctx.shape[1]))
    _sgns_check_ids(src, dsts)
    require_cuda(emb, ctx, src, dsts)
    if len({emb.device, ctx.device, src.device, dsts.device}) != 1:
        raise ValueError("skip_gram_loss: the tables and ids must be on one device")
    src, dsts = _sgns_ids(src, dsts, int(emb.shape[0]), int(ctx.shape[0]))
    return _skip_gram_loss_f32(emb, None if shared else ctx, src, dsts, sparse)


# graph-level readouts (csrc/readout.cu)
# ------------------------------------------------------------------------------------------


def segment_max_len(indptr):
    """Longest segment of a segment CSR: one 8-byte read back, cached on the indptr tensor so repeated readouts over
    the same batch (Set2Set's iterations) read it once.  The value only picks the kernels' work layout: a stale one
    (an indptr refilled in place) still gives correct results (DESIGN section 4.10)."""
    cached = getattr(indptr, "_pglb_max_len", None)
    if cached is None:
        B = int(indptr.numel()) - 1
        cached = int((indptr[1:] - indptr[:-1]).max().item()) if B > 0 else 0
        indptr._pglb_max_len = cached
    return cached


def _readout_ws(B, N, D, max_len, dev):
    need = ctypes.c_size_t(0)
    check(lib.pglb_attn_readout_ws(B, N, D, max_len, ctypes.byref(need)))
    return workspace(dev, need.value) if need.value else None


def _attn_readout_raw(x2, indptr, gate, query, max_len):
    N, D = int(x2.shape[0]), int(x2.shape[1])
    B = int(indptr.numel()) - 1
    out = torch.empty((B, D), dtype=torch.float32, device=x2.device)
    lse = torch.empty(B, dtype=torch.float32, device=x2.device)
    ws = _readout_ws(B, N, D, max_len, x2.device)
    with torch.cuda.device(x2.device):
        check(lib.pglb_attn_readout_f32(_ptr(x2), N, D, _ptr(indptr), B, max_len, _ptr(gate), _ptr(query), _ptr(out),
                                        _ptr(lse), _ptr(ws), ws.numel() if ws is not None else 0, _stream()))
    return out, lse


class _AttnReadout(torch.autograd.Function):
    """Fused attention readout; saves lse and the output r for the one-launch backward."""

    @staticmethod
    def forward(ctx, x2, gate, query, indptr, max_len):
        out, lse = _attn_readout_raw(x2, indptr, gate, query, max_len)
        ctx.meta = (indptr, max_len)
        ctx.save_for_backward(x2, gate, query, out, lse)
        return out

    @staticmethod
    def backward(ctx, g):
        indptr, max_len = ctx.meta
        x2, gate, query, out, lse = ctx.saved_tensors
        g = g.contiguous()
        N, D = int(x2.shape[0]), int(x2.shape[1])
        B = int(indptr.numel()) - 1
        gx = torch.empty_like(x2)
        gg = torch.empty_like(gate) if gate is not None else None
        gq = torch.empty_like(query) if query is not None else None
        ws = _readout_ws(B, N, D, max_len, x2.device)
        with torch.cuda.device(x2.device):
            check(lib.pglb_attn_readout_bwd_f32(_ptr(x2), N, D, _ptr(indptr), B, max_len, _ptr(gate), _ptr(query),
                                                _ptr(out), _ptr(lse), _ptr(g), _ptr(gx), _ptr(gg), _ptr(gq), _ptr(ws),
                                                ws.numel() if ws is not None else 0, _stream()))
        return gx, gg, gq, None, None


@f64_through
def attn_readout(x, indptr, gate=None, query=None, return_lse=False):
    """out[g] = sum_{i in g} softmax_g(s)_i * x_i over the segments of indptr (int64 [B + 1]), with s = gate ([N] or
    [N, 1]: GlobalAttention) or s_i = <x_i, query[g]> (query [B, D]: Set2Set) -- the reference's gather, multiply,
    reduce, 7-op segment_softmax, multiply and segment_sum (pgl/nn/pool.py:139-142, 177-178) in one pass over x.
    Gradients reach x, gate and query."""
    if (gate is None) == (query is None):
        raise ValueError("attn_readout: pass exactly one of gate and query")
    require_cuda(x, indptr, gate, query)
    x2 = _f32_2d(x)
    if x.dim() != 2:
        raise ValueError("attn_readout: x must be [N, D]")
    indptr = _i64(indptr).contiguous()
    B, N, D = int(indptr.numel()) - 1, int(x2.shape[0]), int(x2.shape[1])
    if gate is not None:
        if gate.numel() != N:
            raise ValueError("attn_readout: gate must hold one score per row of x")
        gate = _f32_2d(gate.reshape(N, 1)).reshape(N)
    else:
        if tuple(query.shape) != (B, D):
            raise ValueError("attn_readout: query must be [num_segments, D]")
        query = _f32_2d(query)
    max_len = segment_max_len(indptr)
    grad = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x2, gate, query))
    if grad and not return_lse:
        return _AttnReadout.apply(x2, gate, query, indptr, max_len)
    out, lse = _attn_readout_raw(x2, indptr, gate, query, max_len)
    return (out, lse) if return_lse else out


def segment_topk_perm(scores, indptr, ratio):
    """perm of segment_topk (reference pgl/math.py:342-359): for every segment g of indptr, the nodes of its first
    k_g ranks (score descending, -0.0 == +0.0, NaN last, ties by ascending node index), segments in order.
    Scores outside [indptr[0], indptr[B]) belong to no segment and are never ranked, on either kernel path.
    k_g = ceil(fp32(ratio) * fp32(n_g)) for a float ratio in (0, 1], min(ratio, n_g) for an int ratio >= 1.  Scores
    are ranked in float32, as the reference's dense score matrix holds them.  One 16-byte read back (the total and the
    longest segment), as the reference also synchronises here."""
    if isinstance(ratio, int):
        if ratio < 1:
            raise ValueError("segment_topk: an int ratio must be at least 1, got %d" % ratio)
        k, r = int(ratio), 0.0
    else:
        r = float(ratio)
        if not 0.0 < r <= 1.0:
            raise ValueError("segment_topk: a float ratio must lie in (0, 1], got %r" % ratio)
        k = 0
    require_cuda(scores, indptr)
    s = scores.reshape(-1).to(torch.float32).contiguous()
    indptr = _i64(indptr).contiguous()
    B, N = int(indptr.numel()) - 1, int(s.numel())
    dev = s.device
    offsets = torch.empty(B + 1, dtype=torch.int64, device=dev)
    info = torch.empty(2, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        check(lib.pglb_segment_topk_count(_ptr(indptr), B, r, k, _ptr(offsets), _ptr(info), _stream()))
        total, max_len = (int(v) for v in info.tolist())
        perm = torch.empty(total, dtype=torch.int64, device=dev)
        need = ctypes.c_size_t(0)
        check(lib.pglb_segment_topk_ws(B, N, max_len, ctypes.byref(need)))
        ws = workspace(dev, need.value) if need.value else None
        check(lib.pglb_segment_topk_fill(_ptr(s), N, _ptr(indptr), B, _ptr(offsets), max_len, _ptr(perm), _ptr(ws),
                                         ws.numel() if ws is not None else 0, _stream()))
    return perm


_BITS_VIEW = {2: torch.int16, 4: torch.int32, 8: torch.int64}


def _fill_bits(value, dtype):
    t = torch.tensor([value], dtype=dtype)
    size = t.element_size()
    return int(t.view(_BITS_VIEW[size]).item()) & ((1 << (8 * size)) - 1)


def _rows_of(t):
    if t.element_size() not in _BITS_VIEW:
        raise TypeError("pgl_b200: segment padding copies elements of 2, 4 or 8 bytes, got %s" % t.dtype)
    t2 = t.reshape(t.shape[0], -1) if t.dim() != 2 else t
    return t2.contiguous()


def _segment_pad_raw(x2, indptr, max_len, fill_bits):
    N, D = int(x2.shape[0]), int(x2.shape[1])
    B = int(indptr.numel()) - 1
    out = torch.empty((B, max_len, D), dtype=x2.dtype, device=x2.device)
    with torch.cuda.device(x2.device):
        check(lib.pglb_segment_pad(_ptr(x2), N, D, x2.element_size(), _ptr(indptr), B, max_len, fill_bits, _ptr(out),
                                   _stream()))
    return out


def _segment_unpad_raw(p3, indptr, num_rows):
    B, L, D = int(p3.shape[0]), int(p3.shape[1]), int(p3.shape[2])
    out = torch.empty((int(num_rows), D), dtype=p3.dtype, device=p3.device)
    with torch.cuda.device(p3.device):
        check(lib.pglb_segment_unpad(_ptr(p3), B, L, D, p3.element_size(), _ptr(indptr), int(num_rows), _ptr(out),
                                     _stream()))
    return out


class _SegmentPad(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x2, indptr, max_len, fill_bits):
        ctx.meta = (indptr, int(x2.shape[0]))
        return _segment_pad_raw(x2, indptr, max_len, fill_bits)

    @staticmethod
    def backward(ctx, g):
        indptr, n = ctx.meta
        return _segment_unpad_raw(g.contiguous(), indptr, n), None, None, None


class _SegmentUnpad(torch.autograd.Function):
    @staticmethod
    def forward(ctx, p3, indptr, num_rows):
        ctx.meta = (indptr, int(p3.shape[1]))
        return _segment_unpad_raw(p3, indptr, num_rows)

    @staticmethod
    def backward(ctx, g):
        indptr, max_len = ctx.meta
        return _segment_pad_raw(g.contiguous(), indptr, max_len, 0), None, None


def segment_pad(x, indptr, max_len, fill_value=0):
    """[N, *F] -> [B, max_len, *F]: row p of block b is x[indptr[b] + p] for p < n_b, else fill_value.  Native in
    every dtype of 2, 4 or 8 bytes (a copy, so exact); max_len must be at least the longest segment.  The gradient is
    segment_unpad."""
    require_cuda(x, indptr)
    indptr = _i64(indptr).contiguous()
    x2 = _rows_of(x)
    bits = _fill_bits(fill_value, x2.dtype)
    if x2.requires_grad and torch.is_grad_enabled():
        out = _SegmentPad.apply(x2, indptr, int(max_len), bits)
    else:
        out = _segment_pad_raw(x2, indptr, int(max_len), bits)
    return out.reshape(out.shape[:2] + tuple(x.shape[1:]))


def segment_unpad(padded, indptr, num_rows):
    """The adjoint gather of segment_pad: [B, max_len, *F] -> [num_rows, *F], row i = padded[b, i - indptr[b]]."""
    require_cuda(padded, indptr)
    indptr = _i64(indptr).contiguous()
    if padded.element_size() not in _BITS_VIEW:
        raise TypeError("pgl_b200: segment padding copies elements of 2, 4 or 8 bytes, got %s" % padded.dtype)
    p3 = padded.reshape(padded.shape[0], padded.shape[1], -1).contiguous()
    if p3.requires_grad and torch.is_grad_enabled():
        out = _SegmentUnpad.apply(p3, indptr, int(num_rows))
    else:
        out = _segment_unpad_raw(p3, indptr, int(num_rows))
    return out.reshape((int(num_rows),) + tuple(padded.shape[2:]))


# partition -> local graph (csrc/localgraph.cu)
# ------------------------------------------------------------------------------------------


def map_nodes(nodes, table, strict=True):
    """graph_kernel.map_nodes on the device: table[nodes] for a dense table new_id[old_id] (int64 CUDA tensors).
    strict: ids outside the table raise (one 4-byte read back); otherwise they map to -1."""
    require_cuda(nodes, table)
    nodes = _i64(nodes).contiguous()
    table = _i64(table).contiguous()
    out = torch.empty_like(nodes)
    bad = torch.zeros(1, dtype=torch.int32, device=nodes.device)
    with torch.cuda.device(nodes.device):
        check(lib.pglb_map_nodes(_ptr(nodes), nodes.numel(), _ptr(table), table.numel(), _ptr(out), _ptr(bad),
                                 _stream()))
    if strict and int(bad.item()):
        raise IndexError("pgl_b200.map_nodes: node id outside the relabelling table")
    return out


def map_edges(eid, edges, table, strict=True):
    """graph_kernel.map_edges on the device: table[edges[eid]] (eid None = every edge in order)."""
    require_cuda(edges, table)
    edges = _i64(edges).contiguous()
    table = _i64(table).contiguous()
    if edges.dim() != 2 or edges.shape[1] != 2:
        raise ValueError("pgl_b200.map_edges: edges must be [E, 2]")
    if eid is not None:
        eid = _i64(eid).contiguous()
    n = int(eid.numel()) if eid is not None else int(edges.shape[0])
    out = torch.empty((n, 2), dtype=torch.int64, device=edges.device)
    bad = torch.zeros(1, dtype=torch.int32, device=edges.device)
    with torch.cuda.device(edges.device):
        check(lib.pglb_map_edges(_ptr(eid), n, _ptr(edges), int(edges.shape[0]), _ptr(table), table.numel(),
                                 _ptr(out), _ptr(bad), _stream()))
    if strict and int(bad.item()):
        raise IndexError("pgl_b200.map_edges: edge or node id outside its table")
    return out


def partition_relabel(part, num_parts):
    """part[N] (int64 CUDA tensor, values in [0, num_parts)) -> (new_id[N], offsets[num_parts + 1]) such that every
    part is a contiguous range of new ids, stable inside a part (reference apps/GNNAutoScale/graph_partition.py:94-101:
    ``permutation = argsort(part)`` + offsets).  The stable sort is pglb_csr_build's radix sort with u = part."""
    require_cuda(part)
    part = _i64(part).contiguous()
    n = int(part.numel())
    deg, sv, su, perm, offsets = csr_build(part, part, int(num_parts))
    new_id = torch.empty(n, dtype=torch.int64, device=part.device)
    with torch.cuda.device(part.device):
        check(lib.pglb_invert_perm(_ptr(perm), n, _ptr(new_id), _stream()))
    return new_id, offsets


def halo_plan(edges, num_nodes, lo, hi, offsets):
    """One rank's local graph of a contiguous 1-D node partition (pglb_halo_plan_count / _fill).
    edges [E, 2] int64 CUDA (global ids), this rank owns [lo, hi), offsets = python list / tensor of K + 1 part
    starts.  Returns (eid, dst_local, col_local, halo_ids, recv_counts) -- all int64 CUDA tensors."""
    require_cuda(edges)
    edges = _i64(edges).contiguous()
    dev = edges.device
    E, N = int(edges.shape[0]), int(num_nodes)
    off_t = torch.as_tensor(offsets, dtype=torch.int64).to(dev).contiguous()
    K = int(off_t.numel()) - 1
    need = ctypes.c_size_t(0)
    check(lib.pglb_halo_plan_ws(E, N, ctypes.byref(need)))
    ws = torch.empty(max(need.value, 1), dtype=torch.uint8, device=dev)  # private: must survive between the two calls
    counts = torch.zeros(2, dtype=torch.int64, device=dev)
    bad = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        check(lib.pglb_halo_plan_count(_ptr(edges), E, N, int(lo), int(hi), _ptr(counts), _ptr(bad), _ptr(ws),
                                       ws.numel(), _stream()))
        e_loc, n_halo = (int(v) for v in counts.tolist())
        if int(bad.item()):
            raise IndexError("pgl_b200.halo_plan: edge endpoint outside [0, num_nodes)")
        eid = torch.empty(e_loc, dtype=torch.int64, device=dev)
        dst_local = torch.empty(e_loc, dtype=torch.int64, device=dev)
        col_local = torch.empty(e_loc, dtype=torch.int64, device=dev)
        halo_ids = torch.empty(n_halo, dtype=torch.int64, device=dev)
        recv_counts = torch.zeros(K, dtype=torch.int64, device=dev)
        check(lib.pglb_halo_plan_fill(_ptr(edges), E, N, int(lo), int(hi), _ptr(off_t), K, _ptr(eid),
                                      _ptr(dst_local), _ptr(col_local), _ptr(halo_ids), _ptr(recv_counts), _ptr(ws),
                                      ws.numel(), _stream()))
    return eid, dst_local, col_local, halo_ids, recv_counts


def segment_ids_from_indptr(indptr, num_edges):
    """(uniq_ind, segment_ids) of a CSR == paddle.unique(sorted_key, return_inverse=True)
    (reference pgl/utils/helper.py:156-160).  One D2H read of K (the reference's unique syncs too)."""
    require_cuda(indptr)
    N = int(indptr.shape[0]) - 1
    E = int(num_edges)
    dev = indptr.device
    uniq = torch.empty(max(N, 0), dtype=torch.int64, device=dev)
    seg = torch.empty(E, dtype=torch.int64, device=dev)
    k = torch.zeros(1, dtype=torch.int64, device=dev)
    need = ctypes.c_size_t(0)
    check(lib.pglb_segment_ids_ws(N, ctypes.byref(need)))
    ws = workspace(dev, need.value)
    with torch.cuda.device(dev):
        check(lib.pglb_segment_ids(_ptr(indptr), N, E, _ptr(uniq), _ptr(seg), _ptr(k), _ptr(ws),
                                   ws.numel(), _stream()))
    return uniq[: int(k.item())], seg


def segment_indptr(segment_ids, num_segments):
    require_cuda(segment_ids)
    ids = _i64(segment_ids).contiguous()
    E = int(ids.shape[0])
    K = int(num_segments)
    indptr = torch.empty(K + 1, dtype=torch.int64, device=ids.device)
    with torch.cuda.device(ids.device):
        check(lib.pglb_segment_indptr(_ptr(ids), E, K, _ptr(indptr), _stream()))
    return indptr


# ------------------------------------------------------------------------------------------
# aggregation
# ------------------------------------------------------------------------------------------


def _spmm_raw(indptr, cols, x2, n_dst, reduce_op, eid=None, y2=None, y_bcast=BCAST_FULL,
              head_dim=1, msg_op="copy", scale_src=None, scale_dst=None, max_degree=-1,
              num_edges=None, out=None, packed=None, accumulate=False):
    """float32 x: pglb_spmm_csr_slot_scale_f32, or pglb_spmm_narrow_f32 with a NarrowPlan.  bfloat16 / float16 x:
    copy messages through pglb_spmm_csr_x16; a per-head or scalar float32 edge operand with mul / add messages and sum
    (the fused GAT backward's grad f) through pglb_spmm_csr_ue_x16.  The output has x's dtype."""
    half = x2.dtype in HALF_DTYPES
    half_ue = (half and y2 is not None and msg_op in ("mul", "add") and reduce_op == "sum" and not accumulate
               and y_bcast in (BCAST_HEAD, BCAST_SCALAR))
    if half and not half_ue and (msg_op != "copy" or y2 is not None or accumulate):
        raise TypeError("pgl_b200: 16-bit features aggregate copy messages, or mul / add messages with a per-head or "
                        "scalar edge operand into a sum (got msg_op=%s, reduce_op=%s%s%s)"
                        % (msg_op, reduce_op, ", an edge operand" if y2 is not None else "",
                           ", accumulate" if accumulate else ""))
    if half_ue and y2.dtype != torch.float32:
        y2 = y2.float()
    dev = x2.device
    D = int(x2.shape[1])
    E = int(num_edges if num_edges is not None else (cols.shape[0] if cols is not None else 0))
    # the norms are fp32 on every route (an N-sized cast for a 16-bit norm)
    if scale_src is not None and scale_src.dtype != torch.float32:
        scale_src = scale_src.float()
    if scale_dst is not None and scale_dst.dtype != torch.float32:
        scale_dst = scale_dst.float()
    if out is None:
        out = torch.empty((n_dst, D), dtype=x2.dtype, device=dev)
    if isinstance(packed, NarrowPlan):
        if (not half and reduce_op in ("sum", "mean") and msg_op == "copy" and y2 is None and not accumulate
                and E > 0 and n_dst > 0 and x2.data_ptr() % 16 == 0 and x2.stride(0) % 4 == 0 and x2.stride(1) == 1
                and out.data_ptr() % 16 == 0 and out.stride(0) % 4 == 0 and int(x2.shape[0]) < (1 << 30)):
            need = ctypes.c_size_t(0)
            check(lib.pglb_spmm_narrow_ws(E, D, ctypes.byref(need)))
            ws = workspace(dev, need.value)
            sval = None
            if scale_src is not None and NARROW_SLOT_SCALE and packed.slot_scale is not None:
                sval = packed.slot_scale(scale_src)     # scale_src[cols[j]] per slot, cached per scale tensor
            with torch.cuda.device(dev):
                check(lib.pglb_spmm_narrow_f32(_ptr(packed.plan), _ptr(packed.nz_row), _ptr(packed.blk_k),
                                               _ptr(indptr), _ptr(x2), x2.stride(0), _ptr(out), out.stride(0),
                                               n_dst, int(x2.shape[0]), E, D, REDUCE[reduce_op], _ptr(scale_src),
                                               _ptr(sval), _ptr(scale_dst), 2 if packed.hints else 0, _ptr(ws),
                                               ws.numel(), _stream()))
            return out
        packed = None
    need = ctypes.c_size_t(0)
    check(lib.pglb_spmm_csr_ws(n_dst, E, D, ctypes.byref(need)))
    ws = workspace(dev, need.value)
    sslot = None
    if (scale_src is not None and reduce_op in ("sum", "mean") and msg_op == "copy"
            and getattr(packed, "slot_scale", None) is not None):
        # scale_src[cols[j]] per slot (None before the scale's second call) for spmm_v5, the kernel of these calls
        sslot = packed.slot_scale(scale_src)
    ids = _ptr(packed[0]) if packed is not None else None
    flags = (1 if accumulate else 0) | (2 if (packed is not None and packed[1]) else 0)
    with torch.cuda.device(dev):
        if half_ue:
            check(lib.pglb_spmm_csr_ue_x16(
                _ptr(indptr), _ptr(cols), _ptr(eid), _ptr(x2), x2.stride(0), _ptr(y2), y2.stride(0), y_bcast,
                _ptr(out), out.stride(0), n_dst, int(x2.shape[0]), E, D, head_dim, _DTYPE16[x2.dtype], MSG[msg_op],
                REDUCE[reduce_op], _ptr(scale_src), _ptr(scale_dst), int(max_degree), 0, _ptr(ws), ws.numel(),
                _stream()))
        elif half:
            check(lib.pglb_spmm_csr_x16(
                _ptr(indptr), _ptr(cols), _ptr(x2), x2.stride(0), _ptr(out), out.stride(0), n_dst, int(x2.shape[0]),
                E, D, _DTYPE16[x2.dtype], REDUCE[reduce_op], _ptr(scale_src), _ptr(sslot), _ptr(scale_dst), ids,
                int(max_degree), flags, _ptr(ws), ws.numel(), _stream()))
        else:
            check(lib.pglb_spmm_csr_slot_scale_f32(
                _ptr(indptr), _ptr(cols), _ptr(eid), _ptr(x2), x2.stride(0), _ptr(y2),
                (y2.stride(0) if y2 is not None else 0), y_bcast, _ptr(out), out.stride(0), n_dst,
                int(x2.shape[0]), E, D, head_dim, MSG[msg_op], REDUCE[reduce_op], _ptr(scale_src), _ptr(sslot),
                _ptr(scale_dst), ids, int(max_degree), flags, _ptr(ws), ws.numel(), _stream()))
    return out


def _copy2d(dst_ptr, dpitch, src_ptr, spitch, width, height, kind, stream):
    """kind 1: host -> device, 2: device -> host (pglb_memcpy2d_async's convention)."""
    check(lib.pglb_memcpy2d_async(ctypes.c_void_p(dst_ptr), dpitch, ctypes.c_void_p(src_ptr), spitch,
                                  width, height, kind, ctypes.c_void_p(stream)))


class HostAggregator(object):
    """send_u_recv for features that live in (pinned) HOST memory: out_host = aggregate(x_host).

    The graph stays resident on the GPU; per call the [N, D] float32 matrix is streamed through the GPU
    in `chunks` column blocks on three streams -- upload of block c+1, aggregation of block c and
    download of block c-1 run concurrently (PCIe is full duplex, and the columns of a copy-message
    aggregation are independent).

    Two ways to call it:

    * ``agg(x_host, out_host, ...)``  BLOCKING: returns when ``out_host`` holds the result (the host
      thread has waited for the last device-to-host copy), so the caller may read ``out_host`` and
      rewrite ``x_host`` immediately.
    * ``t = agg.submit(x_host, out_host, ...)`` ... ``agg.wait(t)``  PIPELINED across calls: the
      aggregator owns ``depth`` device buffer sets, so the upload of call i+1 overlaps the kernel and
      the download of call i (a stream of feature matrices costs one direction of PCIe traffic per
      matrix).  Contract: ``x_host`` must not be written and ``out_host`` must not be read until
      ``wait(t)`` (or ``t.synchronize()``) has returned."""

    def __init__(self, fwd, n_src, n_dst, dim, device, chunks=2, depth=2):
        self.fwd, self.n_src, self.n_dst, self.dim = fwd, int(n_src), int(n_dst), int(dim)
        self.device = device
        chunks = max(1, min(int(chunks), self.dim // 4 if self.dim >= 4 else 1))
        w = -(-self.dim // chunks)
        w = (w + 3) // 4 * 4
        self.bounds = [(c, min(c + w, self.dim)) for c in range(0, self.dim, w)]
        self.depth = max(1, int(depth))
        self.sets = [None] * self.depth       # device buffer sets, allocated on first use
        self.count = 0
        self.s_in = torch.cuda.Stream(device=device)
        self.s_k = torch.cuda.Stream(device=device)
        self.s_out = torch.cuda.Stream(device=device)

    def _set(self, i):
        st = self.sets[i]
        if st is None:
            st = {"xd": torch.empty((self.n_src, self.dim), dtype=torch.float32, device=self.device),
                  "od": torch.empty((self.n_dst, self.dim), dtype=torch.float32, device=self.device),
                  "kernel_done": None, "d2h_done": None}
            self.sets[i] = st
        return st

    def submit(self, x_host, out_host, reduce_op="sum", scale_src=None, scale_dst=None):
        assert x_host.dtype == torch.float32 and out_host.dtype == torch.float32
        assert tuple(x_host.shape) == (self.n_src, self.dim) and x_host.is_contiguous()
        assert tuple(out_host.shape) == (self.n_dst, self.dim) and out_host.is_contiguous()
        st = self._set(self.count % self.depth)
        self.count += 1
        main = torch.cuda.current_stream(self.device)
        self.s_k.wait_stream(main)  # the scale vectors may have been produced on the caller's stream
        if st["kernel_done"] is not None:
            self.s_in.wait_event(st["kernel_done"])   # the previous user of this xd has been aggregated
        if st["d2h_done"] is not None:
            self.s_k.wait_event(st["d2h_done"])       # the previous result has left this od
        xd, od = st["xd"], st["od"]
        pitch = self.dim * 4
        full = len(self.bounds) == 1
        with torch.cuda.device(self.device):
            ev_in = []
            for lo, hi in self.bounds:
                if full:
                    with torch.cuda.stream(self.s_in):
                        xd.copy_(x_host, non_blocking=True)
                else:
                    _copy2d(xd.data_ptr() + lo * 4, pitch, x_host.data_ptr() + lo * 4, pitch,
                            (hi - lo) * 4, self.n_src, 1, self.s_in.cuda_stream)
                e = torch.cuda.Event()
                e.record(self.s_in)
                ev_in.append(e)
            for i, (lo, hi) in enumerate(self.bounds):
                self.s_k.wait_event(ev_in[i])
                with torch.cuda.stream(self.s_k):
                    _spmm_raw(self.fwd["indptr"], self.fwd["cols"], xd[:, lo:hi], self.n_dst, reduce_op,
                              scale_src=scale_src, scale_dst=scale_dst,
                              max_degree=self.fwd.get("max_degree", -1), out=od[:, lo:hi],
                              packed=_packed_of(self.fwd, xd[:, lo:hi]))
                e = torch.cuda.Event()
                e.record(self.s_k)
                self.s_out.wait_event(e)
                if full:
                    with torch.cuda.stream(self.s_out):
                        out_host.copy_(od, non_blocking=True)
                else:
                    _copy2d(out_host.data_ptr() + lo * 4, pitch, od.data_ptr() + lo * 4, pitch,
                            (hi - lo) * 4, self.n_dst, 2, self.s_out.cuda_stream)
                st["kernel_done"] = e
        done = torch.cuda.Event()
        done.record(self.s_out)
        st["d2h_done"] = done
        return done

    def wait(self, ticket):
        ticket.synchronize()

    def __call__(self, x_host, out_host, reduce_op="sum", scale_src=None, scale_dst=None):
        t = self.submit(x_host, out_host, reduce_op, scale_src, scale_dst)
        torch.cuda.current_stream(self.device).wait_event(t)
        t.synchronize()  # the host may touch out_host / x_host as soon as this returns
        return out_host


class IpcBuffer(object):
    """A cudaMalloc'ed float32 [rows, cols] buffer with a CUDA IPC handle (pglb_ipc_alloc), exposed
    to torch zero-copy through __cuda_array_interface__.  Used for the multi-GPU feature buffer
    whose rows peers pull over NVLink."""

    def __init__(self, rows, cols, device):
        self.shape = (int(rows), int(cols))
        self.device = device
        nbytes = max(self.shape[0] * self.shape[1] * 4, 256)
        ptr = ctypes.c_void_p()
        self.handle = ctypes.create_string_buffer(64)
        with torch.cuda.device(device):
            check(lib.pglb_ipc_alloc(nbytes, ctypes.byref(ptr), self.handle))
        self.ptr = int(ptr.value)
        self.__cuda_array_interface__ = {"shape": self.shape, "typestr": "<f4",
                                         "data": (self.ptr, False), "version": 2, "strides": None}
        self.tensor = torch.as_tensor(self, device=device)

    def handle_bytes(self):
        return bytes(self.handle.raw)

    def close(self):
        if self.ptr:
            self.tensor = None
            lib.pglb_ipc_free(ctypes.c_void_p(self.ptr))
            self.ptr = 0


def ipc_open(handle_bytes, device):
    """Map a peer's IpcBuffer under `device`; returns the raw device pointer (int)."""
    ptr = ctypes.c_void_p()
    buf = ctypes.create_string_buffer(handle_bytes, 64)
    with torch.cuda.device(device):
        check(lib.pglb_ipc_open(buf, ctypes.byref(ptr)))
    return int(ptr.value)


def gather_rows_ptr(src_ptr, ld, index, out):
    """out[i] = src[index[i]] where src is a raw (possibly peer-mapped) float32 pointer."""
    n = int(index.shape[0])
    if n == 0:
        return out
    D = int(out.shape[1])
    with torch.cuda.device(out.device):
        check(lib.pglb_gather_rows_f32(ctypes.c_void_p(src_ptr), int(ld), _ptr(index),
                                       max(index.stride(0), 1), n, D, _ptr(out), out.stride(0),
                                       _stream()))
    return out


# Share of the device's L2 given to the rows marked evict_last (the "hot set") of the wide-row kernel: 32 MB of an
# H100's 50 MB.  The rest of the cache holds what streams past it: packed ids, per-slot norms, output write-back and
# the cold rows in flight.  scripts/l2_sweep.py on cfg5 (DESIGN.md section 6) found the step time flat within 0.1 %
# from 24 to 64 MB with streamed norms and 32 MB the lowest median; no budget at all costs about 1 %.
HOT_L2_FRACTION = 0.64


@functools.lru_cache(maxsize=None)
def _l2_bytes(device_index):
    return int(torch.cuda.get_device_properties(device_index).L2_cache_size)


def hot_l2_bytes(device):
    """L2 budget of the wide-row hot set on `device`: PGLB_HOT_MB when set (0 = no hints), else HOT_L2_FRACTION of
    the device's L2."""
    env = os.environ.get("PGLB_HOT_MB")
    if env is not None:
        return int(float(env) * (1 << 20))
    dev = torch.device(device)
    return int(HOT_L2_FRACTION * _l2_bytes(dev.index if dev.index is not None else torch.cuda.current_device()))


class PackedCols(tuple):
    """(packed uint32 column ids, has_hints) of pack_cols for the wide-row kernel, plus `slot_scale(scale_src)`: the
    EdgeIndex's per-slot source scale (None until a scale tensor's second call), which the kernel streams instead
    of gathering scale_src per edge."""

    def __new__(cls, packed, slot_scale=None):
        self = tuple.__new__(cls, packed)
        self.slot_scale = slot_scale
        return self


def pack_cols(cols, n_src, row_bytes, budget_bytes=None):
    """(packed uint32 column ids, has_hints) for the wide-row aggregation kernel, or None when
    ids do not fit 31 bits.  With a budget (default hot_l2_bytes(cols.device); 0 = no hints) bit 31 marks the
    most frequently gathered sources, as many as fit in the budget, for an evict_last L2 policy.
    One-off per graph; cached by EdgeIndex."""
    budget = hot_l2_bytes(cols.device) if budget_bytes is None else int(budget_bytes)
    n_src = int(n_src)
    E = int(cols.shape[0])
    if n_src >= (1 << 31) - 1 or E == 0 or n_src == 0:
        return None
    dev = cols.device
    count = torch.empty(n_src, dtype=torch.int32, device=dev)
    packed = torch.empty(E, dtype=torch.int32, device=dev)  # uint32 payload
    k = budget // max(int(row_bytes), 1)
    thr = (1 << 62)
    hints = budget > 0 and 0 < k < n_src
    if hints:
        with torch.cuda.device(dev):
            check(lib.pglb_pack_cols(_ptr(cols), E, n_src, _ptr(count), 1 << 62, _ptr(packed), _stream()))
        thr = max(int(torch.topk(count, k, sorted=True).values[-1].item()), 2)
    with torch.cuda.device(dev):
        check(lib.pglb_pack_cols(_ptr(cols), E, n_src, _ptr(count), thr, _ptr(packed), _stream()))
    return packed, hints


class _CopyAgg(torch.autograd.Function):
    """out[d] = reduce_{e -> d} scale_src[src] * x[src]  (* scale_dst[d]); sum / mean.
    Backward is the same kernel on the reverse (src-keyed) CSR."""

    @staticmethod
    def forward(ctx, x2, fwd, bwd, n_dst, reduce_op, scale_src, scale_dst):
        ctx.bwd = bwd
        ctx.reduce_op = reduce_op
        ctx.n_src = int(x2.shape[0])
        ctx.scales = (scale_src, scale_dst)
        ctx.fwd = fwd
        return _spmm_raw(fwd["indptr"], fwd["cols"], x2, n_dst, reduce_op, scale_src=scale_src,
                         scale_dst=scale_dst, max_degree=fwd.get("max_degree", -1),
                         packed=_packed_of(fwd, x2))

    @staticmethod
    def backward(ctx, g):
        bwd = ctx.bwd() if callable(ctx.bwd) else ctx.bwd
        if bwd is None:
            raise RuntimeError("pgl_b200: backward of this aggregation needs the reverse CSR")
        g = g.contiguous()
        scale_src, scale_dst = ctx.scales
        s_in = scale_dst
        if ctx.reduce_op == "mean":
            inv = 1.0 / torch.clamp(ctx.fwd["degree"].to(torch.float32), min=1.0)
            s_in = inv if s_in is None else s_in * inv
        # the reverse CSR has one row per graph node; a feature matrix with MORE rows than the graph has nodes
        # (legal in the forward: the extra rows are never gathered) gets zero gradient rows, never an indptr over-read
        nb = int(bwd["indptr"].shape[0]) - 1
        rows = min(ctx.n_src, nb)
        sdst = scale_src[:rows] if (scale_src is not None and int(scale_src.shape[0]) > rows) else scale_src
        gx = _spmm_raw(bwd["indptr"][: rows + 1] if rows < nb else bwd["indptr"], bwd["cols"], g, rows, "sum",
                       scale_src=s_in, scale_dst=sdst, max_degree=bwd.get("max_degree", -1),
                       packed=_packed_of(bwd, g) if rows == nb else None)
        if ctx.n_src > rows:
            gx = torch.cat([gx, gx.new_zeros((ctx.n_src - rows, gx.shape[1]))], 0)
        return gx, None, None, None, None, None, None


class _MaxMinAgg(torch.autograd.Function):
    """send_u_recv(max|min); backward routes the gradient to every source entry that equals the
    reduced value (pglb_maxmin_bwd_f32 on the reverse CSR)."""

    @staticmethod
    def forward(ctx, x2, fwd, bwd, n_dst, reduce_op):
        out = _spmm_raw(fwd["indptr"], fwd["cols"], x2, n_dst, reduce_op,
                        max_degree=fwd.get("max_degree", -1), packed=_packed_of(fwd, x2))
        ctx.bwd = bwd
        ctx.save_for_backward(x2, out)
        return out

    @staticmethod
    def backward(ctx, g):
        bwd = ctx.bwd() if callable(ctx.bwd) else ctx.bwd
        if bwd is None:
            raise RuntimeError("pgl_b200: backward of this aggregation needs the reverse CSR")
        x2, out = ctx.saved_tensors
        dtype = x2.dtype
        if dtype in HALF_DTYPES:
            # widening is exact, so the fp32 kernel's equality test x == out picks the same entries
            x2, out, g = x2.float(), out.float(), g.float()
        g = g.contiguous()
        # as in _CopyAgg.backward: feature rows past the graph's nodes are never gathered, so they get zero gradient;
        # the kernel only walks the rows the reverse CSR has
        n_src = int(x2.shape[0])
        rows = min(n_src, int(bwd["indptr"].shape[0]) - 1)
        gx = torch.zeros_like(x2) if rows < n_src else torch.empty_like(x2)
        with torch.cuda.device(x2.device):
            check(lib.pglb_maxmin_bwd_f32(_ptr(bwd["indptr"]), _ptr(bwd["cols"]), _ptr(x2), _ptr(out),
                                          _ptr(g), _ptr(gx), rows, int(x2.shape[1]), _stream()))
        return gx.to(dtype), None, None, None, None


# rows of <= 64 floats: spmm_narrow2_kernel for copy-sum / mean
NARROW_HOT_BYTES = int(float(os.environ.get("PGLB_NARROW_HOT_MB", "64")) * (1 << 20))   # L2 residency budget, narrow rows
NARROW_SLOT_SCALE = os.environ.get("PGLB_NARROW_SLOT_SCALE", "1") != "0"                 # stream cached per-slot norms


class NarrowPlan(object):
    """What pglb_spmm_narrow_f32 streams instead of cols / indptr (see include/pglb.h).  `hints`: bit 31 of the plan
    carries an L2 residency hint.  `slot_scale(scale_src)`: the source scale laid out per CSR slot (cached per scale
    tensor by the EdgeIndex).  Calls the narrow kernel does not take run without packed ids."""
    __slots__ = ("plan", "nz_row", "blk_k", "hints", "slot_scale")

    def __init__(self, plan, nz_row, blk_k, hints=False, slot_scale=None):
        self.plan, self.nz_row, self.blk_k, self.hints = plan, nz_row, blk_k, bool(hints)
        self.slot_scale = slot_scale


def narrow_plan(indptr, cols, n_src, row_bytes=64):
    """Build the plan of a dst-CSR once (cached by the EdgeIndex).  Returns (plan, nz_row, blk_k, hints)."""
    require_cuda(indptr, cols)
    dev = indptr.device
    n_dst = int(indptr.shape[0]) - 1
    E = int(cols.shape[0])
    pk = pack_cols(cols, n_src, row_bytes, NARROW_HOT_BYTES) if NARROW_HOT_BYTES > 0 else None
    hints = bool(pk is not None and pk[1])
    plan = torch.empty(E, dtype=torch.int32, device=dev)
    nz_row = torch.empty(n_dst + 2, dtype=torch.int32, device=dev)
    blk_k = torch.empty((E + 31) // 32, dtype=torch.int32, device=dev)
    need = ctypes.c_size_t(0)
    check(lib.pglb_narrow_plan_ws(n_dst, ctypes.byref(need)))
    ws = workspace(dev, need.value)
    with torch.cuda.device(dev):
        check(lib.pglb_narrow_plan(_ptr(indptr), _ptr(cols), _ptr(pk[0]) if hints else None, n_dst, int(n_src), E,
                                   _ptr(plan), _ptr(nz_row), _ptr(blk_k), _ptr(ws), ws.numel(), _stream()))
    return plan, nz_row, blk_k, hints


def _packed_of(csr, x2):
    """Per-(graph, row width) index data from the EdgeIndex cache: packed column ids (+ optional L2 hints, the hot set
    chosen for the real row size) for the wide-row kernels (64 < D <= 128), the narrow plan for float32 rows of
    D <= 64.  Only rows of at most 128 elements and a multiple of 16 bytes get either; the others get None."""
    fn = csr.get("packed")
    D = int(x2.shape[1])
    row_bytes = D * x2.element_size()
    if fn is None or D > 128 or row_bytes % 16:
        return None
    n_src = int(x2.shape[0])
    if D <= 64:
        if x2.dtype == torch.float32 and csr.get("plan") is not None and 0 < n_src < (1 << 30) and \
                csr["cols"] is not None and int(csr["cols"].shape[0]) > 0:
            plan, nz_row, blk_k, hints = csr["plan"](n_src, row_bytes)
            return NarrowPlan(plan, nz_row, blk_k, hints, slot_scale=csr.get("slot_scale"))
        return None
    pk = fn(n_src, row_bytes)
    return PackedCols(pk, csr.get("slot_scale")) if pk is not None else None


@native16_through
def aggregate_copy(x, fwd, n_dst, reduce_op="sum", bwd=None, scale_src=None, scale_dst=None):
    """send_u_recv on a cached dst-CSR.  fwd/bwd: dicts {indptr, cols, degree, max_degree}.  float32, bfloat16 or
    float16 x; the output has x's dtype."""
    require_cuda(x)
    shape = x.shape
    x2 = _f32_2d(x, allow16=True)
    needs_grad = x2.requires_grad and torch.is_grad_enabled()
    if reduce_op in ("sum", "mean") and needs_grad:
        out = _CopyAgg.apply(x2, fwd, bwd, n_dst, reduce_op, scale_src, scale_dst)
    elif needs_grad and scale_src is None and scale_dst is None:
        out = _MaxMinAgg.apply(x2, fwd, bwd, n_dst, reduce_op)
    elif needs_grad:
        # max / min with fused scales has no backward kernel: do not hand back a silently detached result (ADVICE r1)
        raise NotImplementedError("pgl_b200: send_u_recv(%s) with fused scale vectors is not differentiable; apply the "
                                  "scales outside the aggregation" % reduce_op)
    else:
        out = _spmm_raw(fwd["indptr"], fwd["cols"], x2, n_dst, reduce_op, scale_src=scale_src,
                        scale_dst=scale_dst, max_degree=fwd.get("max_degree", -1),
                        packed=_packed_of(fwd, x2))
    return out.reshape((n_dst,) + tuple(shape[1:]))


_EUNSUPPORTED = -4   # PGLB_EUNSUPPORTED


def _rows16(t):
    return t.data_ptr() % 16 == 0 and t.stride(0) % 4 == 0


def _propagate_raw(csr, x2, scale, a, b, h, acc, c, acc_out):
    """One pglb_propagate_*_f32 call on the route _spmm_raw takes for x2 with scale_src = scale_dst = scale: the
    narrow plan when _spmm_raw would use it, else pglb_propagate_f32 with the same packed ids and per-slot scale.
    c: a float, or a one-element float32 CUDA tensor read on the device.  acc_out: None, acc itself (in place) or a
    fresh [N, D] tensor.  Returns the output, or None when the entry refuses the call (PGLB_EUNSUPPORTED)."""
    dev = x2.device
    n, D = int(x2.shape[0]), int(x2.shape[1])
    E = int(csr["cols"].shape[0])
    out = torch.empty((n, D), dtype=torch.float32, device=dev)
    c_dev = c if isinstance(c, torch.Tensor) else None
    c_val = 0.0 if c_dev is not None else float(c)
    epi = (ctypes.c_float(a), ctypes.c_float(b), _ptr(h), h.stride(0) if h is not None else 0, _ptr(acc),
           acc.stride(0) if acc is not None else 0, _ptr(acc_out), acc_out.stride(0) if acc_out is not None else 0,
           ctypes.c_float(c_val), _ptr(c_dev))
    packed = _packed_of(csr, x2)
    indptr = csr["indptr"]
    if isinstance(packed, NarrowPlan):
        if _rows16(x2) and n < (1 << 30):
            need = ctypes.c_size_t(0)
            check(lib.pglb_spmm_narrow_ws(E, D, ctypes.byref(need)))
            ws = workspace(dev, need.value)
            sval = packed.slot_scale(scale) if (NARROW_SLOT_SCALE and packed.slot_scale is not None) else None
            with torch.cuda.device(dev):
                rc = lib.pglb_propagate_narrow_f32(_ptr(packed.plan), _ptr(packed.nz_row), _ptr(packed.blk_k),
                                                   _ptr(indptr), _ptr(x2), x2.stride(0), _ptr(out), out.stride(0), n,
                                                   n, E, D, _ptr(scale), _ptr(sval), _ptr(scale), *epi,
                                                   2 if packed.hints else 0, _ptr(ws), ws.numel(), _stream())
            if rc == _EUNSUPPORTED:
                return None
            check(rc)
            return out
        packed = None
    need = ctypes.c_size_t(0)
    check(lib.pglb_spmm_csr_ws(n, E, D, ctypes.byref(need)))
    ws = workspace(dev, need.value)
    sslot = packed.slot_scale(scale) if getattr(packed, "slot_scale", None) is not None else None
    flags = 2 if (packed is not None and packed[1]) else 0
    with torch.cuda.device(dev):
        rc = lib.pglb_propagate_f32(_ptr(indptr), _ptr(csr["cols"]), _ptr(x2), x2.stride(0), _ptr(out),
                                    out.stride(0), n, n, E, D, _ptr(scale), _ptr(sslot), _ptr(scale), *epi,
                                    _ptr(packed[0]) if packed is not None else None,
                                    int(csr.get("max_degree", -1)), flags, _ptr(ws), ws.numel(), _stream())
    if rc == _EUNSUPPORTED:
        return None
    check(rc)
    return out


class _Propagate(torch.autograd.Function):
    """y = a * (scale * A (scale * x)) (+ b * h), acc_out = acc + c * y as one aggregation (pglb_propagate_f32).
    Backward: g_tot = g_y + c g_acc; g_x is one pglb_propagate_f32 call on the reverse CSR with a and the scales
    swapped (one shared scale here); g_h = b g_tot; g_acc passes through; g_c = sum(g_acc * y).  No atomics: the
    gradients are the same from run to run."""

    @staticmethod
    def forward(ctx, x2, h, acc, c, fwd, bwd, scale, a, b):
        acc_out = torch.empty_like(acc) if acc is not None else None
        y = _propagate_raw(fwd, x2, scale, a, b, h, acc, c, acc_out)
        if y is None:
            raise RuntimeError("pgl_b200: pglb_propagate_f32 refused a call ops.propagate accepted")
        ctx.bwd, ctx.scale, ctx.a, ctx.b, ctx.c = bwd, scale, a, b, c
        ctx.c_grad = isinstance(c, torch.Tensor) and ctx.needs_input_grad[3]
        if ctx.c_grad:
            ctx.save_for_backward(y)
        return y if acc is None else (y, acc_out)

    @staticmethod
    def backward(ctx, g_y, g_acc=None):
        c = ctx.c
        g_tot = g_y
        if g_acc is not None:
            g_tot = torch.addcmul(g_y, g_acc, c) if isinstance(c, torch.Tensor) else torch.add(g_y, g_acc, alpha=c)
        g_tot = g_tot.contiguous()
        g_x = g_h = g_c = None
        if ctx.needs_input_grad[0]:
            bwd = ctx.bwd() if callable(ctx.bwd) else ctx.bwd
            if bwd is None:
                raise RuntimeError("pgl_b200: backward of this propagation needs the reverse CSR")
            g_x = _propagate_raw(bwd, g_tot, ctx.scale, ctx.a, 0.0, None, None, 1.0, None)
            if g_x is None:
                raise RuntimeError("pgl_b200: pglb_propagate_f32 refused the backward of an accepted call")
        if ctx.needs_input_grad[1]:
            g_h = torch.mul(g_tot, ctx.b)
        if ctx.c_grad:
            (y,) = ctx.saved_tensors
            g_c = (g_acc * y).sum().reshape(c.shape) if g_acc is not None else torch.zeros_like(c)
        return g_x, g_h, g_acc, g_c, None, None, None, None, None


def _propagate_declines(x, n, others, scale):
    if not isinstance(x, torch.Tensor) or not x.is_cuda or x.dtype != torch.float32 or x.dim() != 2:
        return True
    if int(x.shape[0]) != n:
        return True
    for t in others:
        if t is not None and (not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32
                              or tuple(t.shape) != tuple(x.shape) or t.device != x.device):
            return True
    return (not isinstance(scale, torch.Tensor) or not scale.is_cuda or scale.dtype != torch.float32
            or scale.numel() != n or scale.requires_grad or scale.device != x.device)


def propagate(x, fwd, bwd, scale, a=1.0, b=0.0, h=None, acc=None, c=1.0, inplace_acc=False):
    """One K-hop propagation step of APPNP / GCNII / SSGCConv / GPRConv on a graph's dst-CSR `fwd` (reverse CSR
    `bwd`, a dict or a callable returning one, needed for the gradient of x) as one aggregation with a row epilogue:
        t = scale * sum_{j -> d} scale[j] * x[j]      (the rows send_u_recv with scale_src = scale_dst = scale gives)
        y = a * t + b * h                              (b * h only when h is given; h may be x itself)
        acc_out = acc + c * y                          (only when acc is given)
    Every product and sum is rounded on its own, so y and acc_out are bit for bit torch's op-by-op hop on the same
    aggregation route.  a, b: floats (rounded to float32).  c: a float, or a one-element float32 CUDA tensor (GPRConv's
    temp[k + 1]) read on the device, whose gradient is sum(g_acc * y).  inplace_acc: write acc_out into acc when no
    gradient is recorded (acc must then be a buffer the caller owns).
    Returns y, or (y, acc_out) when acc is given, or None when the call is outside the fused route: x, h, acc or the
    norm not float32 CUDA tensors of [N, D] / N elements (N = the graph's node count), a norm that requires grad, a
    graph without edges, or a shape the kernels refuse (PGLB_EUNSUPPORTED: 16-byte rows of D > 128 elements, which the
    copy aggregation sends to spmm_stream).  Callers then run the op-by-op hop."""
    n = int(fwd["indptr"].shape[0]) - 1
    if fwd.get("cols") is None or int(fwd["cols"].shape[0]) == 0:
        return None
    if _propagate_declines(x, n, (h, acc), scale):
        return None
    if isinstance(c, torch.Tensor) and (not c.is_cuda or c.dtype != torch.float32 or c.numel() != 1
                                        or c.device != x.device):
        return None
    scale = scale.reshape(-1)
    if not scale.is_contiguous():
        scale = scale.contiguous()
    x2 = x if x.is_contiguous() else x.contiguous()
    h2 = None if h is None else (x2 if h is x else h.contiguous())
    acc2 = None if acc is None else acc.contiguous()
    # the vector kernels read h / acc rows 16 bytes at a time: a row-offset view is copied to a fresh allocation
    if int(x.shape[1]) % 4 == 0:
        h2 = h2 if h2 is None or _rows16(h2) else h2.clone()
        acc2 = acc2 if acc2 is None or _rows16(acc2) else acc2.clone()
    D = int(x.shape[1])
    if D % 4 == 0 and D > 128 and _rows16(x2):
        return None   # the wide-row shapes past spmm_v5 (spmm_stream) have no epilogue
    grad = torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in (x, h, acc, c))
    if grad:
        return _Propagate.apply(x2, h2, acc2, c, fwd, bwd, scale, float(a), float(b))
    acc_out = None
    if acc2 is not None:
        acc_out = acc2 if (inplace_acc and acc2 is acc) else torch.empty_like(acc2)
    y = _propagate_raw(fwd, x2, scale, float(a), float(b), h2, acc2, c, acc_out)
    if y is None:
        return None
    return y if acc is None else (y, acc_out)


def classify_bcast(x_shape, y_shape):
    """Map (x feature dims, y feature dims) to a kernel broadcast mode.
    Returns (mode, head_dim) or None when y must be materialised by expand()."""
    xf = tuple(x_shape[1:])
    yf = tuple(y_shape[1:])
    D = 1
    for s in xf:
        D *= s
    ny = 1
    for s in yf:
        ny *= s
    if ny == 1:
        return BCAST_SCALAR, 1
    if len(yf) < len(xf):
        yf = (1,) * (len(xf) - len(yf)) + yf
    if len(yf) != len(xf):
        return None
    if yf == xf:
        return BCAST_FULL, 1
    # [.., H, 1, 1] against [.., H, a, b]: leading dims equal, trailing dims of y all 1
    k = len(xf)
    while k > 0 and yf[k - 1] == 1:
        k -= 1
    if yf[:k] == xf[:k]:
        hd = 1
        for s in xf[k:]:
            hd *= s
        return BCAST_HEAD, hd
    return None


def sddmm_dot(a2, b2, ia, ib, H, Dh):
    """out[e,h] = <a2[ia[e], h, :], b2[ib[e], h, :]>; a2, b2 are [n, H*Dh]."""
    E = int(ia.shape[0])
    out = torch.empty((E, H), dtype=torch.float32, device=a2.device)
    with torch.cuda.device(a2.device):
        check(lib.pglb_sddmm_dot_f32(_ptr(a2), _ptr(b2), _ptr(ia), max(ia.stride(0), 1) if E else 1,
                                     _ptr(ib), max(ib.stride(0), 1) if E else 1, E, H, Dh, _ptr(out),
                                     _stream()))
    return out


class _UeAgg(torch.autograd.Function):
    """send_ue_recv with reduce sum and message mul / add, differentiable in x and y."""

    @staticmethod
    def forward(ctx, x2, y2, fwd, bwd, edges, n_dst, mode, hd, msg_op):
        ctx.meta = (fwd, bwd, edges, mode, hd, msg_op)
        ctx.save_for_backward(x2, y2)
        return _spmm_raw(fwd["indptr"], fwd["cols"], x2, n_dst, "sum", eid=fwd["eid"], y2=y2,
                         y_bcast=mode, head_dim=hd, msg_op=msg_op, max_degree=fwd.get("max_degree", -1))

    @staticmethod
    def backward(ctx, g):
        fwd, bwd, edges, mode, hd, msg_op = ctx.meta
        bwd = bwd() if callable(bwd) else bwd
        x2, y2 = ctx.saved_tensors
        g = g.contiguous()
        n_src, D = int(x2.shape[0]), int(x2.shape[1])
        src, dst = edges[:, 0], edges[:, 1]
        gx = gy = None
        if msg_op == "mul":
            if ctx.needs_input_grad[0]:
                gx = _spmm_raw(bwd["indptr"], bwd["cols"], g, n_src, "sum", eid=bwd["eid"], y2=y2,
                               y_bcast=mode, head_dim=hd, msg_op="mul",
                               max_degree=bwd.get("max_degree", -1))
            if ctx.needs_input_grad[1]:
                if mode == BCAST_FULL:
                    gy = send_uv(x2, g, src, dst, "mul")
                elif mode == BCAST_HEAD:
                    gy = sddmm_dot(x2, g, src, dst, D // hd, hd)
                else:
                    gy = sddmm_dot(x2, g, src, dst, 1, D)
        else:  # add
            if ctx.needs_input_grad[0]:
                gx = _spmm_raw(bwd["indptr"], bwd["cols"], g, n_src, "sum",
                               max_degree=bwd.get("max_degree", -1))
            if ctx.needs_input_grad[1]:
                ge = gather_rows(g, dst)
                if mode == BCAST_FULL:
                    gy = ge
                elif mode == BCAST_HEAD:
                    gy = ge.reshape(ge.shape[0], D // hd, hd).sum(-1)
                else:
                    gy = ge.sum(-1, keepdim=True)
        return gx, gy, None, None, None, None, None, None, None


def _ue_with_grad(x2, y2, fwd, bwd, edges, n_dst, mode, hd, message_op, reduce_op):
    """Differentiable send_ue_recv for every (message_op, reduce_op) of the reference (pgl/graph.py:889-937).
    add / mul with sum run on the fused kernels (_UeAgg: transpose-SpMM for the node operand, SDDMM / gather for
    the edge operand).  The rest is composed from those and from pieces that already carry a backward:
      sub  = add with -y,   div = mul with 1 / y   (autograd differentiates the negation / reciprocal),
      mean = sum / in-degree,
      max / min: the [E, D] message is materialised like the reference does (gather_rows(x, src) op y) and reduced
      by the segment kernel over the dst-CSR slots, whose backward routes the gradient to the selected entries."""
    if message_op == "sub":
        return _ue_with_grad(x2, -y2, fwd, bwd, edges, n_dst, mode, hd, "add", reduce_op)
    if message_op == "div":
        return _ue_with_grad(x2, 1.0 / y2, fwd, bwd, edges, n_dst, mode, hd, "mul", reduce_op)
    if reduce_op == "sum":
        return _UeAgg.apply(x2, y2, fwd, bwd, edges, n_dst, mode, hd, message_op)
    if reduce_op == "mean":
        total = _UeAgg.apply(x2, y2, fwd, bwd, edges, n_dst, mode, hd, message_op)
        deg = (fwd["indptr"][1:] - fwd["indptr"][:-1])[:n_dst].clamp(min=1).to(total.dtype)
        return total / deg.unsqueeze(1)
    # max / min
    D = int(x2.shape[1])
    xe = gather_rows(x2, edges[:, 0])                                     # [E, D], differentiable
    if mode == BCAST_FULL:
        ye = y2
    elif mode == BCAST_HEAD:
        ye = y2.reshape(y2.shape[0], D // hd, 1).expand(-1, -1, hd).reshape(y2.shape[0], D)
    else:
        ye = y2.reshape(-1, 1).expand(-1, D)
    msg = xe * ye if message_op == "mul" else xe + ye
    return segment_reduce(msg, None, reduce_op, indptr=fwd["indptr"][: n_dst + 1], cols=fwd["eid"],
                          max_degree=fwd.get("max_degree", -1))


@f64_through
def aggregate_ue(x, y, fwd, n_dst, message_op="add", reduce_op="sum", bwd=None, edges=None):
    """send_ue_recv on a cached dst-CSR: y is in original edge order, read through eid."""
    require_cuda(x, y)
    xs = tuple(x.shape)
    y_shape_in = tuple(y.shape)
    if y.dim() == 1:
        y = y.reshape(-1, 1)
    out_feat = torch.broadcast_shapes(tuple(x.shape[1:]) if x.dim() > 1 else (1,), tuple(y.shape[1:]))
    if tuple(out_feat) != tuple(xs[1:]):
        x = x.reshape((xs[0],) + (1,) * (len(out_feat) - len(xs[1:])) + tuple(xs[1:]))
        x = x.expand((xs[0],) + tuple(out_feat)).contiguous()
    cls = classify_bcast(x.shape, y.shape)
    if cls is None:
        y = y.expand((y.shape[0],) + tuple(out_feat)).contiguous()
        cls = (BCAST_FULL, 1)
    mode, hd = cls
    x2 = _f32_2d(x)
    y2 = _f32_2d(y)
    needs_grad = torch.is_grad_enabled() and (x2.requires_grad or y2.requires_grad)
    if needs_grad:
        if bwd is None or edges is None:
            raise NotImplementedError("pgl_b200: a differentiable send_ue_recv needs the reverse CSR and the edge list")
        out = _ue_with_grad(x2, y2, fwd, bwd, edges, n_dst, mode, hd, message_op, reduce_op)
    else:
        out = _spmm_raw(fwd["indptr"], fwd["cols"], x2, n_dst, reduce_op, eid=fwd["eid"], y2=y2,
                        y_bcast=mode, head_dim=hd, msg_op=message_op,
                        max_degree=fwd.get("max_degree", -1))
    return out.reshape((n_dst,) + tuple(out_feat))


class _SegmentReduce(torch.autograd.Function):
    """Row reduce over a compact CSR (segment_* / fused gather+segment).  Backward: sum / mean
    expand the gradient back over the slots (then scatter-add through `cols` if the forward
    gathered); max / min route it to the entries equal to the reduced value."""

    @staticmethod
    def forward(ctx, d2, indptr, cols, pool_type, max_degree, n_slots):
        K = int(indptr.shape[0]) - 1
        out = _spmm_raw(indptr, cols, d2, K, pool_type, num_edges=n_slots, max_degree=max_degree)
        ctx.meta = (indptr, cols, pool_type, n_slots)
        ctx.save_for_backward(d2, out)
        return out

    @staticmethod
    def backward(ctx, g):
        indptr, cols, pool_type, n_slots = ctx.meta
        d2, out = ctx.saved_tensors
        dtype = d2.dtype
        if dtype in HALF_DTYPES:
            # the gradient is formed in fp32 (counts exact, sums over out-edges accumulated in fp32) and rounded once;
            # widening is exact, so max / min select the same entries
            d2, out, g = d2.float(), out.float(), g.float()
        g = g.contiguous()
        K = int(indptr.shape[0]) - 1
        counts = indptr[1:] - indptr[:-1]
        seg = torch.repeat_interleave(torch.arange(K, device=g.device), counts)  # slot -> row
        ge = gather_rows(g, seg)  # [n_slots, D]
        if pool_type == "mean":
            ge = ge / counts.clamp(min=1).to(ge.dtype)[seg].unsqueeze(1)
        elif pool_type in ("max", "min"):
            src_rows = d2 if cols is None else gather_rows(d2, cols)
            ge = ge * (src_rows == gather_rows(out, seg)).to(ge.dtype)
        if cols is None:
            return ge.to(dtype), None, None, None, None, None
        gd = torch.zeros_like(d2).index_add_(0, cols, ge)
        return gd.to(dtype), None, None, None, None, None


@native16_through
def segment_reduce(data, segment_ids, pool_type, num_segments=None, indptr=None, cols=None,
                   max_degree=-1):
    """paddle.geometric.segment_* over sorted ids (reference pgl/math.py:36-42).
    `cols` (optional) fuses a row gather: slot j reads data[cols[j]] (lazy messages).  float32, bfloat16 or float16
    data; the output has data's dtype."""
    require_cuda(data)
    d2 = _f32_2d(data, allow16=True)
    if indptr is None:
        ids = _i64(segment_ids)
        E = int(ids.shape[0])
        if num_segments is None:
            num_segments = int(ids[-1].item()) + 1 if E > 0 else 0
        indptr = segment_indptr(ids, num_segments)
    else:
        E = int(cols.shape[0]) if cols is not None else int(d2.shape[0])
        num_segments = int(indptr.shape[0]) - 1
    if d2.requires_grad and torch.is_grad_enabled():
        out = _SegmentReduce.apply(d2, indptr, cols, pool_type, max_degree, E)
    else:
        out = _spmm_raw(indptr, cols, d2, int(num_segments), pool_type, num_edges=E,
                        max_degree=max_degree)
    feat = tuple(data.shape[1:])
    return out.reshape((int(num_segments),) + feat)


def _send_uv_raw(x2, y2, src, dst, message_op):
    E = int(src.shape[0])
    D = int(x2.shape[1])
    out = torch.empty((E, D), dtype=torch.float32, device=x2.device)
    with torch.cuda.device(x2.device):
        check(lib.pglb_send_uv_f32(_ptr(x2), _ptr(y2), _ptr(src), max(src.stride(0), 1) if E else 1,
                                   _ptr(dst), max(dst.stride(0), 1) if E else 1, E, D,
                                   MSG[message_op], _ptr(out), _stream()))
    return out


class _SendUV(torch.autograd.Function):
    """send_uv (add / sub / mul) with gradients reduced over the cached src- and dst-CSR."""

    @staticmethod
    def forward(ctx, x2, y2, src, dst, message_op, src_csr, dst_csr):
        ctx.meta = (message_op, src_csr, dst_csr)
        ctx.save_for_backward(x2, y2)
        return _send_uv_raw(x2, y2, src, dst, message_op)

    @staticmethod
    def backward(ctx, g):
        op_, src_csr, dst_csr = ctx.meta
        x2, y2 = ctx.saved_tensors
        g = g.contiguous()
        gx = gy = None
        sc = src_csr() if callable(src_csr) else src_csr
        dc = dst_csr() if callable(dst_csr) else dst_csr
        if op_ in ("add", "sub"):
            if ctx.needs_input_grad[0]:   # sum of g over the out-edges of every source
                gx = _spmm_raw(sc["indptr"], sc["eid"], g, int(x2.shape[0]), "sum",
                               max_degree=sc.get("max_degree", -1))
            if ctx.needs_input_grad[1]:
                gy = _spmm_raw(dc["indptr"], dc["eid"], g, int(y2.shape[0]), "sum",
                               max_degree=dc.get("max_degree", -1))
                if op_ == "sub":
                    gy = -gy
        elif op_ == "mul":
            if ctx.needs_input_grad[0]:   # gx[s] = sum_e g[e] * y[dst[e]]
                gx = _spmm_raw(sc["indptr"], sc["cols"], y2, int(x2.shape[0]), "sum", eid=sc["eid"],
                               y2=g, y_bcast=BCAST_FULL, msg_op="mul", max_degree=sc.get("max_degree", -1))
            if ctx.needs_input_grad[1]:
                gy = _spmm_raw(dc["indptr"], dc["cols"], x2, int(y2.shape[0]), "sum", eid=dc["eid"],
                               y2=g, y_bcast=BCAST_FULL, msg_op="mul", max_degree=dc.get("max_degree", -1))
        else:
            raise NotImplementedError("pgl_b200: send_uv(div) has no backward yet")
        return gx, gy, None, None, None, None, None


@f64_through
def send_uv(x, y, src, dst, message_op="add", src_csr=None, dst_csr=None):
    require_cuda(x, y, src, dst)
    xf = tuple(x.shape[1:]) if x.dim() > 1 else (1,)
    yf = tuple(y.shape[1:]) if y.dim() > 1 else (1,)
    of = tuple(torch.broadcast_shapes(xf, yf))
    if xf != of:
        x = x.reshape((x.shape[0],) + (1,) * (len(of) - len(xf)) + xf).expand((x.shape[0],) + of)
    if yf != of:
        y = y.reshape((y.shape[0],) + (1,) * (len(of) - len(yf)) + yf).expand((y.shape[0],) + of)
    x2 = _f32_2d(x.reshape(x.shape[0], -1) if x.dim() != 2 else x)
    y2 = _f32_2d(y.reshape(y.shape[0], -1) if y.dim() != 2 else y)
    E = int(src.shape[0])
    if torch.is_grad_enabled() and (x2.requires_grad or y2.requires_grad) and src_csr is not None:
        out = _SendUV.apply(x2, y2, src, dst, message_op, src_csr, dst_csr)
    else:
        out = _send_uv_raw(x2, y2, src, dst, message_op)
    return out.reshape((E,) + of)


def _gather_rows_raw(x2, index, out2=None):
    n = int(index.shape[0])
    D = int(x2.shape[1])
    dev = index.device
    if out2 is None:
        out2 = torch.empty((n, D), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(lib.pglb_gather_rows_f32(_ptr(x2), x2.stride(0), _ptr(index),
                                       max(index.stride(0), 1) if n else 1, n, D, _ptr(out2),
                                       out2.stride(0), _stream()))
    return out2


class _GatherRows(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x2, index):
        ctx.meta = (index, int(x2.shape[0]))
        return _gather_rows_raw(x2, index)

    @staticmethod
    def backward(ctx, g):
        index, n = ctx.meta
        gx = torch.zeros((n, g.shape[1]), dtype=g.dtype, device=g.device)
        gx.index_add_(0, index.contiguous(), g.contiguous())
        return gx, None


@f64_through
def gather_rows(x, index, out=None):
    """paddle.gather(x, index, axis=0).  The kernel is launched on the device of ``index`` /
    ``out``; ``x`` may live on a peer GPU mapped into this process (NVLink P2P pull)."""
    require_cuda(x, index)
    index = _i64(index)
    n = int(index.shape[0])
    if x.dtype != torch.float32:
        return x.index_select(0, index.contiguous())  # integer gathers (degree subsets): torch device op
    x2 = _f32_2d(x)
    D = int(x2.shape[1])
    if out is None and x2.requires_grad and torch.is_grad_enabled():
        return _GatherRows.apply(x2, index).reshape((n,) + tuple(x.shape[1:]))
    out2 = None
    if out is not None:
        out2 = out.reshape(n, D) if out.dim() != 2 else out
    res = _gather_rows_raw(x2, index, out2)
    if out is not None:
        return out
    return res.reshape((n,) + tuple(x.shape[1:]))


class _ScatterRows(torch.autograd.Function):
    @staticmethod
    def forward(ctx, init, index, updates):
        out = init.clone()
        o2 = out.reshape(out.shape[0], -1) if out.dim() != 2 else out
        u2 = _f32_2d(updates)
        n = int(index.shape[0])
        with torch.cuda.device(out.device):
            check(lib.pglb_scatter_rows_f32(_ptr(u2), u2.stride(0), _ptr(index), n, int(u2.shape[1]),
                                            _ptr(o2), o2.stride(0), _stream()))
        ctx.index = index
        return out

    @staticmethod
    def backward(ctx, g):
        index = ctx.index
        g = g.contiguous()
        gu = _gather_rows_raw(g.reshape(g.shape[0], -1), index).reshape((index.shape[0],) + tuple(g.shape[1:]))
        gi = g.clone()
        gi.index_fill_(0, index, 0)
        return gi, None, gu


@f64_through
def scatter_rows(init, index, updates):
    """paddle.scatter(init, index, updates, overwrite=True) for unique indices (out-of-place)."""
    require_cuda(init, index, updates)
    index = _i64(index).contiguous()
    return _ScatterRows.apply(init, index, updates)


def _edge_softmax_raw(indptr, eid, l2, E):
    H = int(l2.shape[1])
    out = torch.empty_like(l2)
    need = ctypes.c_size_t(0)
    check(lib.pglb_edge_softmax_csr_ws(E, ctypes.byref(need)))
    ws = workspace(l2.device, need.value)
    with torch.cuda.device(l2.device):
        check(lib.pglb_edge_softmax_csr_f32(_ptr(indptr), _ptr(eid), _ptr(l2), _ptr(out),
                                            int(indptr.shape[0]) - 1, E, H, _ptr(ws), ws.numel(),
                                            _stream()))
    return out


class _EdgeSoftmax(torch.autograd.Function):
    @staticmethod
    def forward(ctx, l2, indptr, eid, E):
        out = _edge_softmax_raw(indptr, eid, l2, E)
        ctx.meta = (indptr, eid, E)
        ctx.save_for_backward(out)
        return out

    @staticmethod
    def backward(ctx, g):
        indptr, eid, E = ctx.meta
        (alpha,) = ctx.saved_tensors
        g = g.contiguous()
        gl = torch.zeros_like(alpha)
        with torch.cuda.device(alpha.device):
            check(lib.pglb_edge_softmax_bwd_csr_f32(_ptr(indptr), _ptr(eid), _ptr(alpha), _ptr(g),
                                                    _ptr(gl), int(indptr.shape[0]) - 1, E,
                                                    int(alpha.shape[1]), _stream()))
        return gl, None, None, None


@f64_through
def edge_softmax_csr(indptr, eid, logits, num_edges):
    """Fused per-row softmax; eid=None -> rows are contiguous slots (segment_softmax)."""
    require_cuda(indptr, logits)
    shape = logits.shape
    l2 = logits.reshape(shape[0], -1) if logits.dim() != 2 else logits
    l2 = _f32_2d(l2)
    E = int(num_edges)
    if l2.requires_grad and torch.is_grad_enabled():
        out = _EdgeSoftmax.apply(l2, indptr, eid, E)
    else:
        out = _edge_softmax_raw(indptr, eid, l2, E)
    return out.reshape(shape)


@f64_through
def gat_attention_csr(csr, attn_src, attn_dst, negative_slope=0.2):
    """alpha[slot, h] = softmax over the dst row of leaky_relu(attn_src[src] + attn_dst[dst]) in CSR
    SLOT order (send_uv + LeakyReLU + edge_softmax fused; inference only)."""
    require_cuda(attn_src, attn_dst)
    a_s = _f32_2d(attn_src)
    a_d = _f32_2d(attn_dst)
    H = int(a_s.shape[1])
    E = int(csr["cols"].shape[0])
    out = torch.empty((E, H), dtype=torch.float32, device=a_s.device)
    need = ctypes.c_size_t(0)
    check(lib.pglb_edge_softmax_csr_ws(E, ctypes.byref(need)))
    ws = workspace(a_s.device, need.value)
    with torch.cuda.device(a_s.device):
        check(lib.pglb_gat_attention_csr_f32(_ptr(csr["indptr"]), _ptr(csr["cols"]), _ptr(a_s), _ptr(a_d),
                                             float(negative_slope), _ptr(out),
                                             int(csr["indptr"].shape[0]) - 1, E, H, _ptr(ws), ws.numel(),
                                             _stream()))
    return out


def _result_dtype(out_dtype, *tensors):
    """out_dtype, or torch's promotion of the tensors' dtypes when it is None."""
    if out_dtype is not None:
        return out_dtype
    return functools.reduce(torch.promote_types, [t.dtype for t in tensors])


def _att32(a):
    """Attention logits of the 16-bit GAT routes as a float32 [N, H] tensor (an N x H cast for 16-bit ones)."""
    mat = getattr(a, "materialize", None)
    a = mat() if mat is not None else a
    return _f32_2d(a.float() if a.dtype in HALF_DTYPES else a)


def _gat_fused_x16(csr, f, attn_src, attn_dst, negative_slope):
    """pglb_gat_fused_csr_x16 on 16-bit f; None when the kernel does not take the shape or layout."""
    n, H, Dh = int(f.shape[0]), int(f.shape[1]), int(f.shape[2])
    f2 = _f32_2d(f, allow16=True)
    a_s, a_d = _att32(attn_src), _att32(attn_dst)
    E = int(csr["cols"].shape[0])
    n_dst = int(csr["indptr"].shape[0]) - 1
    out = torch.empty((n_dst, H * Dh), dtype=f2.dtype, device=f2.device)
    need = ctypes.c_size_t(0)
    check(lib.pglb_spmm_csr_ws(n_dst, E, H * Dh, ctypes.byref(need)))
    ws = workspace(f2.device, need.value)
    try:
        with torch.cuda.device(f2.device):
            check(lib.pglb_gat_fused_csr_x16(_ptr(csr["indptr"]), _ptr(csr["cols"]), _ptr(f2), f2.stride(0),
                                             _ptr(a_s), _ptr(a_d), float(negative_slope), _ptr(out),
                                             out.stride(0), n_dst, n, E, H, Dh, _DTYPE16[f2.dtype], _ptr(ws),
                                             ws.numel(), _stream()))
    except _lib.PglbError as ex:
        if ex.code in (-2, -4):   # PGLB_ESHAPE / PGLB_EUNSUPPORTED: checked before any device work
            return None
        raise
    return out.reshape(n_dst, H, Dh)


def gat_fused(csr, f, attn_src, attn_dst, negative_slope=0.2, out_dtype=None):
    """Single-pass GAT aggregation (online softmax in the wide-row kernel).  f [N, H, Dh] with
    H*Dh <= 128 and Dh % 4 == 0; returns [N, H, Dh], or None when the shape is not supported.
    The result has dtype ``out_dtype``, or by default torch's promotion of f's and the attention's dtypes.  When f is
    bfloat16 / float16 and the result has f's dtype, the 16-bit kernel runs on f as it is (attention widened to
    float32): the result equals the float32 kernel's on the widened f, rounded once.  Other calls, and 16-bit shapes
    that kernel does not take, run the float32 kernel on widened inputs and round its result to the result dtype."""
    require_cuda(f, attn_src, attn_dst)
    n, H, Dh = int(f.shape[0]), int(f.shape[1]), int(f.shape[2])
    if H * Dh > 128 or Dh % 4 or H * Dh <= 64:
        return None
    res = _result_dtype(out_dtype, f, attn_src, attn_dst)
    if f.dtype in HALF_DTYPES and res == f.dtype and torch.float64 not in (attn_src.dtype, attn_dst.dtype):
        out = _gat_fused_x16(csr, f, attn_src, attn_dst, negative_slope)
        if out is not None:
            return out
    out = _gat_fused_f32(csr, f, attn_src, attn_dst, negative_slope)
    return out if out_dtype is None or out.dtype == out_dtype else out.to(out_dtype)


@f64_through
def _gat_fused_f32(csr, f, attn_src, attn_dst, negative_slope=0.2):
    """gat_fused on the float32 kernel (other float dtypes through f64_through)."""
    n, H, Dh = int(f.shape[0]), int(f.shape[1]), int(f.shape[2])
    f2 = _f32_2d(f)
    a_s, a_d = _f32_2d(attn_src), _f32_2d(attn_dst)
    E = int(csr["cols"].shape[0])
    n_dst = int(csr["indptr"].shape[0]) - 1
    out = torch.empty((n_dst, H * Dh), dtype=torch.float32, device=f2.device)
    need = ctypes.c_size_t(0)
    check(lib.pglb_spmm_csr_ws(n_dst, E, H * Dh, ctypes.byref(need)))
    ws = workspace(f2.device, need.value)
    with torch.cuda.device(f2.device):
        check(lib.pglb_gat_fused_csr_f32(_ptr(csr["indptr"]), _ptr(csr["cols"]), _ptr(f2), f2.stride(0),
                                         _ptr(a_s), _ptr(a_d), float(negative_slope), _ptr(out),
                                         out.stride(0), n_dst, n, E, H, Dh, _ptr(ws), ws.numel(),
                                         _stream()))
    return out.reshape(n_dst, H, Dh)


class _HeadDots(torch.autograd.Function):
    """attn_src / attn_dst of GATConv in one pass over the features (pglb_head_dots_f32, or pglb_head_dots_x16 for
    16-bit f); the backward is three elementwise / reduce torch ops on the gradient path, formed in float32 and
    returned in each input's dtype."""

    @staticmethod
    def forward(ctx, f3, w_src, w_dst):
        n, H, Dh = (int(v) for v in f3.shape)
        f2 = f3.reshape(n, H * Dh)
        a_s = torch.empty((n, H), dtype=torch.float32, device=f3.device)
        a_d = torch.empty((n, H), dtype=torch.float32, device=f3.device)
        ws, wd = w_src.float().contiguous(), w_dst.float().contiguous()   # an H x Dh cast for 16-bit weights
        with torch.cuda.device(f3.device):
            if f3.dtype in HALF_DTYPES:
                check(lib.pglb_head_dots_x16(_ptr(f2), f2.stride(0), n, H, Dh, _DTYPE16[f3.dtype], _ptr(ws),
                                             _ptr(wd), _ptr(a_s), _ptr(a_d), _stream()))
            else:
                check(lib.pglb_head_dots_f32(_ptr(f2), f2.stride(0), n, H, Dh, _ptr(ws), _ptr(wd), _ptr(a_s),
                                             _ptr(a_d), _stream()))
        ctx.save_for_backward(f3, w_src, w_dst)
        return a_s, a_d

    @staticmethod
    def backward(ctx, g_s, g_d):
        f3, w_src, w_dst = ctx.saved_tensors
        gf = gw_s = gw_d = None
        if ctx.needs_input_grad[0]:
            gf = (g_s.unsqueeze(-1) * w_src.float() + g_d.unsqueeze(-1) * w_dst.float()).to(f3.dtype)
        if ctx.needs_input_grad[1]:
            gw_s = (g_s.unsqueeze(-1) * f3.float()).sum(0).reshape(w_src.shape).to(w_src.dtype)
        if ctx.needs_input_grad[2]:
            gw_d = (g_d.unsqueeze(-1) * f3.float()).sum(0).reshape(w_dst.shape).to(w_dst.dtype)
        return gf, gw_s, gw_d


def head_dots(f, w_src, w_dst):
    """(sum(f * w_src, -1), sum(f * w_dst, -1)) for f [N, H, Dh], w [H, Dh] (or [1, H, Dh]) -- GATConv's attention
    projections, reference pgl/nn/conv.py:323-326 -- or None when the shape is outside the kernel (the caller keeps
    the two torch expressions).  f float32 with float32 weights, or bfloat16 / float16 f with weights in float32 or
    f's dtype; the projections are float32 (for 16-bit f: the float32 kernel's result on the widened f and weights)."""
    if f.dim() != 3 or not f.is_cuda:
        return None
    if not (f.dtype == torch.float32 or f.dtype in HALF_DTYPES):
        return None
    if any(w.dtype not in (torch.float32, f.dtype) for w in (w_src, w_dst)):
        return None
    n, H, Dh = (int(v) for v in f.shape)
    lph = Dh // 4
    if H * Dh > 128 or Dh % 4 or (lph & (lph - 1)) or w_src.numel() != H * Dh or w_dst.numel() != H * Dh:
        return None
    if (H * Dh * f.element_size()) % 16:
        return None     # the kernel reads 16-byte rows: a 16-bit row needs H*Dh % 8 == 0 (e.g. not 3 heads x 4)
    if not f.is_contiguous():
        f = f.contiguous()
    # float32 weights reach the kernel as they are (16-bit ones are widened into a fresh, aligned copy)
    if f.data_ptr() % 16 or any(w.dtype == torch.float32 and w.data_ptr() % 16 for w in (w_src, w_dst)):
        return None
    return _HeadDots.apply(f, w_src, w_dst)


class _GatFused(torch.autograd.Function):
    """The single-pass GAT aggregation under autograd (reference pgl/nn/conv.py:333-339 differentiated by Paddle over
    four ops).  Forward = pglb_gat_fused_train_csr_f32 (one launch; keeps only lse[N, H]).  Backward = one edge kernel
    (pglb_gat_bwd_edge_f32: alpha rebuilt, SDDMM dot, softmax and LeakyReLU backward) + three reverse-CSR aggregations
    on the existing kernels.  16-bit f2: the *_x16 entries; out and grad f in f2's dtype, lse, alpha, dz and the
    attention and its gradients float32 (a_s / a_d are float32 here).  drop = (p, seed, offset): attention dropout on
    the *_drop_* entries, which recompute the keep mask from (seed, offset) in the forward and in the backward; the
    edge kernel then returns the dropped attention, with which grad f is aggregated as before."""

    @staticmethod
    def forward(ctx, f2, a_s, a_d, fwd, bwd, slope, H, Dh, drop=None):
        n = int(f2.shape[0])
        E = int(fwd["cols"].shape[0])
        n_dst = int(fwd["indptr"].shape[0]) - 1
        out = torch.empty((n_dst, H * Dh), dtype=f2.dtype, device=f2.device)
        lse = torch.zeros((n_dst, H), dtype=torch.float32, device=f2.device)
        need = ctypes.c_size_t(0)
        check(lib.pglb_spmm_csr_ws(n_dst, E, H * Dh, ctypes.byref(need)))
        ws = workspace(f2.device, need.value)
        with torch.cuda.device(f2.device):
            if drop is not None and f2.dtype in HALF_DTYPES:
                check(lib.pglb_gat_fused_train_drop_csr_x16(
                    _ptr(fwd["indptr"]), _ptr(fwd["cols"]), _ptr(f2), f2.stride(0), _ptr(a_s), _ptr(a_d), float(slope),
                    _ptr(out), out.stride(0), _ptr(lse), n_dst, n, E, H, Dh, _DTYPE16[f2.dtype], *drop, _ptr(ws),
                    ws.numel(), _stream()))
            elif drop is not None:
                check(lib.pglb_gat_fused_train_drop_csr_f32(
                    _ptr(fwd["indptr"]), _ptr(fwd["cols"]), _ptr(f2), f2.stride(0), _ptr(a_s), _ptr(a_d), float(slope),
                    _ptr(out), out.stride(0), _ptr(lse), n_dst, n, E, H, Dh, *drop, _ptr(ws), ws.numel(), _stream()))
            elif f2.dtype in HALF_DTYPES:
                check(lib.pglb_gat_fused_train_csr_x16(
                    _ptr(fwd["indptr"]), _ptr(fwd["cols"]), _ptr(f2), f2.stride(0), _ptr(a_s), _ptr(a_d), float(slope),
                    _ptr(out), out.stride(0), _ptr(lse), n_dst, n, E, H, Dh, _DTYPE16[f2.dtype], _ptr(ws), ws.numel(),
                    _stream()))
            else:
                check(lib.pglb_gat_fused_train_csr_f32(
                    _ptr(fwd["indptr"]), _ptr(fwd["cols"]), _ptr(f2), f2.stride(0), _ptr(a_s), _ptr(a_d), float(slope),
                    _ptr(out), out.stride(0), _ptr(lse), n_dst, n, E, H, Dh, _ptr(ws), ws.numel(), _stream()))
        ctx.meta = (fwd, bwd, float(slope), H, Dh, drop)
        ctx.save_for_backward(f2, a_s, a_d, out, lse)
        return out

    @staticmethod
    def backward(ctx, g):
        fwd, bwd, slope, H, Dh, drop = ctx.meta
        bwd = bwd() if callable(bwd) else bwd
        f2, a_s, a_d, out, lse = ctx.saved_tensors
        half = f2.dtype in HALF_DTYPES
        g = _f32_2d(g.to(f2.dtype) if g.dtype != f2.dtype else g, allow16=half)
        E = int(fwd["cols"].shape[0])
        n_src, n_dst = int(f2.shape[0]), int(out.shape[0])
        alpha = torch.empty((E, H), dtype=torch.float32, device=g.device)
        dz = torch.empty((E, H), dtype=torch.float32, device=g.device)
        with torch.cuda.device(g.device):
            if drop is not None and half:
                check(lib.pglb_gat_bwd_edge_drop_x16(_ptr(fwd["rows"]), _ptr(fwd["cols"]), _ptr(fwd["eid"]), _ptr(f2),
                                                     f2.stride(0), _ptr(g), g.stride(0), _ptr(out), out.stride(0),
                                                     _ptr(a_s), _ptr(a_d), _ptr(lse), slope, E, H, Dh,
                                                     _DTYPE16[f2.dtype], *drop, _ptr(alpha), _ptr(dz), _stream()))
            elif drop is not None:
                check(lib.pglb_gat_bwd_edge_drop_f32(_ptr(fwd["rows"]), _ptr(fwd["cols"]), _ptr(fwd["eid"]), _ptr(f2),
                                                     f2.stride(0), _ptr(g), g.stride(0), _ptr(out), out.stride(0),
                                                     _ptr(a_s), _ptr(a_d), _ptr(lse), slope, E, H, Dh, *drop,
                                                     _ptr(alpha), _ptr(dz), _stream()))
            elif half:
                check(lib.pglb_gat_bwd_edge_x16(_ptr(fwd["rows"]), _ptr(fwd["cols"]), _ptr(fwd["eid"]), _ptr(f2),
                                                f2.stride(0), _ptr(g), g.stride(0), _ptr(out), out.stride(0),
                                                _ptr(a_s), _ptr(a_d), _ptr(lse), slope, E, H, Dh, _DTYPE16[f2.dtype],
                                                _ptr(alpha), _ptr(dz), _stream()))
            else:
                check(lib.pglb_gat_bwd_edge_f32(_ptr(fwd["rows"]), _ptr(fwd["cols"]), _ptr(fwd["eid"]), _ptr(f2),
                                                f2.stride(0), _ptr(g), g.stride(0), _ptr(out), out.stride(0),
                                                _ptr(a_s), _ptr(a_d), _ptr(lse), slope, E, H, Dh, _ptr(alpha),
                                                _ptr(dz), _stream()))
        gf = gs = gd = None
        # grad f[s] = sum over the out-edges of s of alpha[e] * g[dst[e]] (with dropout: the dropped attention)
        if ctx.needs_input_grad[0]:
            gf = _spmm_raw(bwd["indptr"], bwd["cols"], g, n_src, "sum", eid=bwd["eid"], y2=alpha, y_bcast=BCAST_HEAD,
                           head_dim=Dh, msg_op="mul", max_degree=bwd.get("max_degree", -1))
        if ctx.needs_input_grad[1]:   # z = as[src] + ad[dst]: send_uv(add)'s backward
            gs = _spmm_raw(bwd["indptr"], bwd["eid"], dz, n_src, "sum", max_degree=bwd.get("max_degree", -1))
        if ctx.needs_input_grad[2]:
            gd = _spmm_raw(fwd["indptr"], fwd["eid"], dz, n_dst, "sum", max_degree=fwd.get("max_degree", -1))
        return gf, gs, gd, None, None, None, None, None, None


GAT_FUSED_TRAIN = os.environ.get("PGLB_GAT_FUSED_TRAIN", "1") != "0"


def _attn_drop_stream(device):
    """(seed, offset) of one attention-dropout call from the default CUDA generator of ``device``: its seed and its
    current offset, which then advances by 4, so every call draws a fresh mask and torch.manual_seed replays a
    sequence of calls bit for bit."""
    gen = torch.cuda.default_generators[device.index if device.index is not None else torch.cuda.current_device()]
    seed, offset = int(gen.initial_seed()), int(gen.get_offset())
    gen.set_offset(offset + 4)
    return seed, offset


def gat_fused_train(fwd, bwd, f, attn_src, attn_dst, negative_slope=0.2, out_dtype=None, attn_drop=0.0, seed=None):
    """gat_fused with a backward.  f [N, H, Dh], 64 < H*Dh <= 128, H % 4 == 0, Dh a power of two >= 4,
    0 <= slope <= 1; returns [N, H, Dh], or None when the shape is outside the fused kernels (the caller keeps the
    op-by-op path).  ``bwd`` is the reverse CSR dict or a callable returning it.
    The result dtype is ``out_dtype``, or by default torch's promotion of f's and the attention's dtypes.  float32 f
    runs the float32 kernels (the result cast to the result dtype).  bfloat16 / float16 f runs the 16-bit kernels when
    the result dtype is f's (attention widened to float32; grad f in f's dtype, grad attention formed in float32 and
    returned in the attention's dtype); other 16-bit calls return None.
    ``attn_drop`` in (0, 1): dropout on the normalised attention, per edge and head, inside the same kernels (the
    *_drop_* entries of include/pglb.h).  The mask comes from ``seed`` = (seed, offset), offset a multiple of 4, or by
    default from the default CUDA generator of f's device (whose offset then advances by 4).  attn_drop >= 1 and calls
    during a CUDA graph capture return None (the caller keeps the op-by-op path with its own dropout)."""
    require_cuda(f, attn_src, attn_dst)
    n, H, Dh = int(f.shape[0]), int(f.shape[1]), int(f.shape[2])
    half = f.dtype in HALF_DTYPES
    res = _result_dtype(out_dtype, f, attn_src, attn_dst)
    if not GAT_FUSED_TRAIN or H * Dh > 128 or H * Dh <= 64 or H % 4 or H > 32:
        return None
    attn_drop = float(attn_drop)
    if not 0.0 <= attn_drop < 1.0:
        return None
    if attn_drop > 0.0 and torch.cuda.is_current_stream_capturing():
        return None     # the generator's offset advances on the host: not replayable by a graph
    if not (f.dtype == torch.float32 or (half and res == f.dtype and torch.float64 not in (attn_src.dtype,
                                                                                          attn_dst.dtype))):
        return None
    if Dh < 4 or (Dh & (Dh - 1)) or not (0.0 <= float(negative_slope) <= 1.0):
        return None
    n_dst = int(fwd["indptr"].shape[0]) - 1
    if n_dst != n or int(fwd["cols"].shape[0]) == 0 or fwd.get("rows") is None:
        return None
    f2 = _f32_2d(f, allow16=half)
    a_s, a_d = (_att32(attn_src), _att32(attn_dst)) if half else (_f32_2d(attn_src), _f32_2d(attn_dst))
    if f2.data_ptr() % 16 or (f2.stride(0) * f2.element_size()) % 16 or a_s.data_ptr() % 16:
        return None
    drop = None
    if attn_drop > 0.0:
        drop = (attn_drop,) + (tuple(int(v) for v in seed) if seed is not None else _attn_drop_stream(f2.device))
    try:
        out = _GatFused.apply(f2, a_s, a_d, fwd, bwd, float(negative_slope), H, Dh, drop)
    except _lib.PglbError as ex:
        if ex.code == -4:   # PGLB_EUNSUPPORTED: e.g. 32 heads, whose attention rows do not fit the kernel's rings
            return None
        raise
    out = out.reshape(n_dst, H, Dh)
    return out if out.dtype == res else out.to(res)


def _dot_attn_fwd_raw(fwd, q2, k2, v2, H, Dh, drop, want_lse, e2=None):
    """pglb_dot_attn_* on [N, H*Dh] rows of one dtype: (out, lse or None).  e2: edge features [E, H*Dh] in edge-id
    order (pglb_dot_attn_e_*)."""
    n = int(q2.shape[0])
    E = int(fwd["cols"].shape[0])
    out = torch.empty((n, H * Dh), dtype=q2.dtype, device=q2.device)
    lse = torch.zeros((n, H), dtype=torch.float32, device=q2.device) if want_lse else None
    need = ctypes.c_size_t(0)
    check(lib.pglb_spmm_csr_ws(n, E, H * Dh, ctypes.byref(need)))
    ws = workspace(q2.device, need.value)
    ef = () if e2 is None else (_ptr(fwd["eid"]),)
    rows = (_ptr(q2), q2.stride(0), _ptr(k2), k2.stride(0), _ptr(v2), v2.stride(0))
    if e2 is not None:
        rows += (_ptr(e2), e2.stride(0))
    args = (_ptr(fwd["indptr"]), _ptr(fwd["cols"]), *ef, *rows, _ptr(out), out.stride(0), _ptr(lse), n, n, E, H, Dh)
    dt = (_DTYPE16[q2.dtype],) if q2.dtype in HALF_DTYPES else ()
    fn = {(False, False): lib.pglb_dot_attn_csr_f32, (False, True): lib.pglb_dot_attn_csr_x16,
          (True, False): lib.pglb_dot_attn_drop_csr_f32, (True, True): lib.pglb_dot_attn_drop_csr_x16}
    if e2 is not None:
        fn = {(False, False): lib.pglb_dot_attn_e_csr_f32, (False, True): lib.pglb_dot_attn_e_csr_x16,
              (True, False): lib.pglb_dot_attn_e_drop_csr_f32, (True, True): lib.pglb_dot_attn_e_drop_csr_x16}
    with torch.cuda.device(q2.device):
        check(fn[(drop is not None, bool(dt))](*args, *dt, *(drop or ()), _ptr(ws), ws.numel(), _stream()))
    return out, lse


class _DotAttn(torch.autograd.Function):
    """TransformerConv's dot-product attention under autograd (reference pgl/nn/conv.py:808-847 differentiated by Paddle
    over send_uv(mul), sum, edge_softmax, dropout and send_ue_recv).  Forward = pglb_dot_attn_* (one pass; keeps only
    lse[N, H]).  Backward = one edge kernel (pglb_dot_attn_bwd_edge_*: scores and weights rebuilt, two head dots per
    edge) + three aggregations on the existing send_ue_recv kernels.  16-bit rows take the *_x16 entries; lse, beta and
    ds are float32 and the gradients are in the rows' dtype.  drop = (p, seed, offset): attention dropout recomputed from
    (seed, offset) in the forward and the backward.  e2 (None or edge features [E, H*Dh] in edge-id order): the
    pglb_dot_attn_e_* entries, k + e and v + e in place of k and v; the edge kernel also writes grad e, and grad q
    takes one more aggregation, of e by edge id."""

    @staticmethod
    def forward(ctx, q2, k2, v2, e2, fwd, bwd, H, Dh, drop):
        out, lse = _dot_attn_fwd_raw(fwd, q2, k2, v2, H, Dh, drop, True, e2)
        ctx.meta = (fwd, bwd, H, Dh, drop)
        ctx.save_for_backward(q2, k2, v2, e2, out, lse)
        return out

    @staticmethod
    def backward(ctx, g):
        fwd, bwd, H, Dh, drop = ctx.meta
        bwd = bwd() if callable(bwd) else bwd
        q2, k2, v2, e2, out, lse = ctx.saved_tensors
        half = q2.dtype in HALF_DTYPES
        g = _f32_2d(g.to(q2.dtype) if g.dtype != q2.dtype else g, allow16=half)
        E = int(fwd["cols"].shape[0])
        n = int(q2.shape[0])
        beta = torch.empty((E, H), dtype=torch.float32, device=g.device)
        ds = torch.empty((E, H), dtype=torch.float32, device=g.device)
        dt = (_DTYPE16[q2.dtype],) if half else ()
        rows = (_ptr(q2), q2.stride(0), _ptr(k2), k2.stride(0), _ptr(v2), v2.stride(0))
        ge, ef = None, ()
        if e2 is None:
            fn = {(False, False): lib.pglb_dot_attn_bwd_edge_f32, (False, True): lib.pglb_dot_attn_bwd_edge_x16,
                  (True, False): lib.pglb_dot_attn_bwd_edge_drop_f32, (True, True): lib.pglb_dot_attn_bwd_edge_drop_x16}
        else:
            fn = {(False, False): lib.pglb_dot_attn_e_bwd_edge_f32, (False, True): lib.pglb_dot_attn_e_bwd_edge_x16,
                  (True, False): lib.pglb_dot_attn_e_bwd_edge_drop_f32,
                  (True, True): lib.pglb_dot_attn_e_bwd_edge_drop_x16}
            rows += (_ptr(e2), e2.stride(0))
            ge = torch.empty_like(e2) if ctx.needs_input_grad[3] else None
            ef = (_ptr(ge), H * Dh)
        with torch.cuda.device(g.device):
            check(fn[(drop is not None, half)](
                _ptr(fwd["rows"]), _ptr(fwd["cols"]), _ptr(fwd["eid"]), *rows, _ptr(g), g.stride(0), _ptr(out),
                out.stride(0), _ptr(lse), E, H, Dh, *dt, *(drop or ()), _ptr(beta), _ptr(ds), *ef, _stream()))
        gq = gk = gv = None

        def agg(csr, x2, w):   # sum over the CSR's slots of w[eid, head] * x2[col]
            return _spmm_raw(csr["indptr"], csr["cols"], x2, n, "sum", eid=csr["eid"], y2=w, y_bcast=BCAST_HEAD,
                             head_dim=Dh, msg_op="mul", max_degree=csr.get("max_degree", -1))
        if ctx.needs_input_grad[0]:   # grad q[d] = sum over the in-edges of d of ds k[src] (+ ds e[eid])
            gq = agg(fwd, k2, ds)
            if e2 is not None:        # the e rows are addressed by edge id: the CSR's eid is their column array
                gq += agg({"indptr": fwd["indptr"], "cols": fwd["eid"], "eid": fwd["eid"],
                           "max_degree": fwd.get("max_degree", -1)}, e2, ds)
        if ctx.needs_input_grad[1]:   # grad k[u] = sum over the out-edges of u of ds q[dst]
            gk = agg(bwd, q2, ds)
        if ctx.needs_input_grad[2]:   # grad v[u] = sum over the out-edges of u of beta G[dst]
            gv = agg(bwd, g, beta)
        return gq, gk, gv, ge, None, None, None, None, None


def dot_attention(fwd, bwd, q, k, v, attn_drop=0.0, seed=None, edge_feat=None):
    """TransformerConv's attention in one pass:
    out[d,h,:] = sum over the in-edges j of d of softmax_j(<q[d,h,:], k[src_j,h,:]>) v[src_j,h,:]
    (q already scaled by 1 / sqrt(Dh)), with a fused backward when autograd needs one.  ``edge_feat`` [E, H, Dh] in
    edge-id order, q's dtype: k + e and v + e in place of k[src_j] and v[src_j] (the add first, then the dot), and the
    backward also returns grad edge_feat; None when it has another shape or dtype, or rows that are not 16-byte
    aligned.  q, k, v [N, H, Dh] of one dtype (float32, bfloat16 or float16) on one graph (n_dst == N); ``fwd`` is
    the dst-keyed CSR dict (with ``rows``), ``bwd`` the src-keyed one or a callable returning it.  Returns [N, H, Dh] in that dtype, or None when the call is
    outside the kernels (H*Dh > 128, Dh not a power of two >= 4, rows the kernels cannot read, mixed dtypes, float64, no
    edges, attn_drop >= 1, dropout during CUDA-graph capture); the caller then keeps the op-by-op path.
    ``attn_drop`` in (0, 1): dropout on the normalised attention per edge and head inside the kernels, the mask drawn
    from ``seed`` = (seed, offset), offset a multiple of 4, or by default from the default CUDA generator of q's device
    (whose offset then advances by 4), as GATConv's fused path does.  16-bit rows: the output is the float32 kernel's on
    the widened rows, rounded once."""
    require_cuda(q, k, v)
    if q.dim() != 3 or q.shape != k.shape or q.shape != v.shape:
        return None
    if not (q.dtype == k.dtype == v.dtype and (q.dtype == torch.float32 or q.dtype in HALF_DTYPES)):
        return None
    n, H, Dh = (int(s) for s in q.shape)
    if H * Dh > 128 or Dh < 4 or Dh & (Dh - 1) or (H * Dh * q.element_size()) % 16:
        return None
    attn_drop = float(attn_drop)
    if not 0.0 <= attn_drop < 1.0 or (attn_drop > 0.0 and H % 4):
        return None
    if attn_drop > 0.0 and torch.cuda.is_current_stream_capturing():
        return None     # the generator's offset advances on the host: not replayable by a graph
    if int(fwd["indptr"].shape[0]) - 1 != n or int(fwd["cols"].shape[0]) == 0 or fwd.get("rows") is None:
        return None
    e2 = None
    if edge_feat is not None:
        require_cuda(edge_feat)
        if edge_feat.dtype != q.dtype or tuple(edge_feat.shape) != (int(fwd["cols"].shape[0]), H, Dh):
            return None
        e2 = _f32_2d(edge_feat, allow16=True)
        if e2.data_ptr() % 16:
            return None
    q2, k2, v2 = (_f32_2d(t, allow16=True) for t in (q, k, v))
    if any(t.data_ptr() % 16 for t in (q2, k2, v2)):
        return None
    drop = None
    if attn_drop > 0.0:
        drop = (attn_drop,) + (tuple(int(s) for s in seed) if seed is not None else _attn_drop_stream(q2.device))
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (q, k, v, edge_feat)):
        out = _DotAttn.apply(q2, k2, v2, e2, fwd, bwd, H, Dh, drop)
    else:
        out = _dot_attn_fwd_raw(fwd, q2, k2, v2, H, Dh, drop, False, e2)[0]
    return out.reshape(n, H, Dh)


def _gatv2_fwd_raw(fwd, f2, a32, slope, H, Dh, drop, want_lse):
    """pglb_gatv2_attn_* on [N, H*Dh] rows: (out in f2's dtype, lse or None)."""
    n = int(f2.shape[0])
    E = int(fwd["cols"].shape[0])
    out = torch.empty((n, H * Dh), dtype=f2.dtype, device=f2.device)
    lse = torch.zeros((n, H), dtype=torch.float32, device=f2.device) if want_lse else None
    need = ctypes.c_size_t(0)
    check(lib.pglb_spmm_csr_ws(n, E, H * Dh, ctypes.byref(need)))
    ws = workspace(f2.device, need.value)
    args = (_ptr(fwd["indptr"]), _ptr(fwd["cols"]), _ptr(f2), f2.stride(0), _ptr(a32), float(slope), _ptr(out),
            out.stride(0), _ptr(lse), n, E, H, Dh)
    dt = (_DTYPE16[f2.dtype],) if f2.dtype in HALF_DTYPES else ()
    fn = {(False, False): lib.pglb_gatv2_attn_csr_f32, (False, True): lib.pglb_gatv2_attn_csr_x16,
          (True, False): lib.pglb_gatv2_attn_drop_csr_f32, (True, True): lib.pglb_gatv2_attn_drop_csr_x16}
    with torch.cuda.device(f2.device):
        check(fn[(drop is not None, bool(dt))](*args, *dt, *(drop or ()), _ptr(ws), ws.numel(), _stream()))
    return out, lse


class _GatV2(torch.autograd.Function):
    """GATv2Conv's attention under autograd (reference pgl/nn/conv.py:420-427 differentiated by Paddle over send_uv(add),
    LeakyReLU, the product with attn, a sum, edge_softmax, dropout and send_ue_recv).  Forward = pglb_gatv2_attn_* (one
    pass; keeps only lse[N, H]).  Backward = one edge kernel (pglb_gatv2_bwd_edge_*: scores and weights rebuilt, beta,
    ds and grad attn) + the score-gradient aggregation on the dst-keyed and the src-keyed CSR (pglb_gatv2_score_grad_*:
    the [E, H*Dh] dz is recomputed, never stored) + send_ue_recv(G, beta) on the src-keyed CSR.  16-bit f2 takes the
    *_x16 entries: lse, beta, ds, the score terms and a32 are float32, grad f comes back in f2's dtype.
    drop = (p, seed, offset): attention dropout recomputed from (seed, offset) in the forward and the backward."""

    @staticmethod
    def forward(ctx, f2, a32, fwd, bwd, slope, H, Dh, drop):
        out, lse = _gatv2_fwd_raw(fwd, f2, a32, slope, H, Dh, drop, True)
        ctx.meta = (fwd, bwd, slope, H, Dh, drop)
        ctx.save_for_backward(f2, a32, out, lse)
        return out

    @staticmethod
    def backward(ctx, g):
        fwd, bwd, slope, H, Dh, drop = ctx.meta
        bwd = bwd() if callable(bwd) else bwd
        f2, a32, out, lse = ctx.saved_tensors
        half = f2.dtype in HALF_DTYPES
        g = _f32_2d(g.to(f2.dtype) if g.dtype != f2.dtype else g, allow16=half)
        E = int(fwd["cols"].shape[0])
        n, D = int(f2.shape[0]), H * Dh
        dev = g.device
        beta = torch.empty((E, H), dtype=torch.float32, device=dev)
        ds = torch.empty((E, H), dtype=torch.float32, device=dev)
        ga = torch.empty((D,), dtype=torch.float32, device=dev) if ctx.needs_input_grad[1] else None
        need_e, need_a = ctypes.c_size_t(0), ctypes.c_size_t(0)
        check(lib.pglb_gatv2_bwd_edge_ws(E, ctypes.byref(need_e)))
        check(lib.pglb_spmm_csr_ws(n, E, D, ctypes.byref(need_a)))
        ws = workspace(dev, max(need_e.value, need_a.value))
        dt = (_DTYPE16[f2.dtype],) if half else ()
        fn = {(False, False): lib.pglb_gatv2_bwd_edge_f32, (False, True): lib.pglb_gatv2_bwd_edge_x16,
              (True, False): lib.pglb_gatv2_bwd_edge_drop_f32, (True, True): lib.pglb_gatv2_bwd_edge_drop_x16}
        gf = None
        with torch.cuda.device(dev):
            check(fn[(drop is not None, half)](
                _ptr(fwd["rows"]), _ptr(fwd["cols"]), _ptr(fwd["eid"]), _ptr(f2), f2.stride(0), _ptr(a32), float(slope),
                _ptr(g), g.stride(0), _ptr(out), out.stride(0), _ptr(lse), E, H, Dh, *dt, *(drop or ()), _ptr(beta),
                _ptr(ds), _ptr(ga), _ptr(ws), ws.numel(), _stream()))
            if ctx.needs_input_grad[0]:
                # grad f = the dst term (dst-keyed CSR) + the src term (src-keyed CSR) + sum over out-edges of beta G[dst]
                gr = torch.empty((n, D), dtype=torch.float32, device=dev)
                score = lib.pglb_gatv2_score_grad_x16 if half else lib.pglb_gatv2_score_grad_f32
                for csr, acc in ((fwd, 0), (bwd, 1)):
                    check(score(_ptr(csr["indptr"]), _ptr(csr["cols"]), _ptr(csr["eid"]), _ptr(f2), f2.stride(0),
                                _ptr(a32), float(slope), _ptr(ds), _ptr(gr), gr.stride(0), n, E, H, Dh, *dt, acc,
                                _ptr(ws), ws.numel(), _stream()))
                gv = _spmm_raw(bwd["indptr"], bwd["cols"], g, n, "sum", eid=bwd["eid"], y2=beta, y_bcast=BCAST_HEAD,
                               head_dim=Dh, msg_op="mul", max_degree=bwd.get("max_degree", -1))
                gf = gr.add_(gv.float() if half else gv)
                gf = gf.to(f2.dtype) if half else gf
        return gf, ga, None, None, None, None, None, None


def gatv2_attention(fwd, bwd, f, attn, negative_slope, out_dtype=None, attn_drop=0.0, seed=None):
    """GATv2Conv's attention in one pass:
    out[d,h,:] = sum over the in-edges j of d of softmax_j(sum_c attn[h,c] lrelu(f[src_j,h,c] + f[d,h,c])) f[src_j,h,:]
    with a fused backward when autograd needs one.  f [N, H, Dh] on one graph (n_dst == N), attn [H, Dh] or
    [1, H, Dh]; ``fwd`` is the dst-keyed CSR dict (with ``rows``), ``bwd`` the src-keyed one or a callable returning
    it.  The result dtype is ``out_dtype``, or by default torch's promotion of f's and attn's dtypes.  float32 f runs the
    float32 kernels (attn widened to float32); bfloat16 / float16 f runs the 16-bit kernels when the result dtype is f's
    (attn widened to float32, grad f in f's dtype, grad attn in attn's dtype).  Returns [N, H, Dh], or None when the
    call is outside the kernels (float64, another dtype mix, H*Dh > 128, Dh not a power of two >= 4, slope outside
    [0, 1], rows the kernels cannot read, n_dst != N, no edges, attn_drop >= 1, dropout with H % 4 != 0 or during
    CUDA-graph capture); the caller then keeps the op-by-op path.
    ``attn_drop`` in (0, 1): dropout on the normalised attention per edge and head inside the kernels, the mask drawn
    from ``seed`` = (seed, offset), offset a multiple of 4, or by default from the default CUDA generator of f's device
    (whose offset then advances by 4), as GATConv's fused path does."""
    require_cuda(f, attn)
    if f.dim() != 3:
        return None
    n, H, Dh = (int(s) for s in f.shape)
    if attn.numel() != H * Dh or attn.shape[-2:] != (H, Dh):
        return None
    half = f.dtype in HALF_DTYPES
    res = _result_dtype(out_dtype, f, attn)
    if torch.float64 in (f.dtype, attn.dtype) or not (f.dtype == torch.float32 or (half and res == f.dtype)):
        return None
    if H * Dh > 128 or Dh < 4 or Dh & (Dh - 1) or (H * Dh * f.element_size()) % 16:
        return None
    slope = float(negative_slope)
    if not 0.0 <= slope <= 1.0:
        return None
    attn_drop = float(attn_drop)
    if not 0.0 <= attn_drop < 1.0 or (attn_drop > 0.0 and H % 4):
        return None
    if attn_drop > 0.0 and torch.cuda.is_current_stream_capturing():
        return None     # the generator's offset advances on the host: not replayable by a graph
    if int(fwd["indptr"].shape[0]) - 1 != n or int(fwd["cols"].shape[0]) == 0 or fwd.get("rows") is None:
        return None
    f2 = _f32_2d(f, allow16=half)
    a32 = attn.reshape(H * Dh)
    a32 = (a32.float() if a32.dtype != torch.float32 else a32).contiguous()
    if f2.data_ptr() % 16 or (f2.stride(0) * f2.element_size()) % 16 or a32.data_ptr() % 16:
        return None
    drop = None
    if attn_drop > 0.0:
        drop = (attn_drop,) + (tuple(int(s) for s in seed) if seed is not None else _attn_drop_stream(f2.device))
    if torch.is_grad_enabled() and (f.requires_grad or attn.requires_grad):
        out = _GatV2.apply(f2, a32, fwd, bwd, slope, H, Dh, drop)
    else:
        out = _gatv2_fwd_raw(fwd, f2, a32, slope, H, Dh, drop, False)[0]
    out = out.reshape(n, H, Dh)
    return out if out.dtype == res else out.to(res)


def _fa_records(g_src, norm, g_dst):
    """The [N, 4] float32 node records (g_src, norm, g_dst, 0) of pglb_fa_attn_*: one 16-byte bulk copy per slot."""
    return torch.stack((g_src.float(), norm.float(), g_dst.float(), torch.zeros_like(g_src, dtype=torch.float32)), 1)


def _fa_fwd_raw(fwd, f2, rec, drop):
    """pglb_fa_attn_* on [N, D] rows: out in f2's dtype."""
    n, D = int(f2.shape[0]), int(f2.shape[1])
    E = int(fwd["cols"].shape[0])
    out = torch.empty((n, D), dtype=f2.dtype, device=f2.device)
    need = ctypes.c_size_t(0)
    check(lib.pglb_spmm_csr_ws(n, E, D, ctypes.byref(need)))
    ws = workspace(f2.device, need.value)
    args = (_ptr(fwd["indptr"]), _ptr(fwd["cols"]), _ptr(f2), f2.stride(0), _ptr(rec), _ptr(out), out.stride(0), n, E,
            D)
    dt = (_DTYPE16[f2.dtype],) if f2.dtype in HALF_DTYPES else ()
    fn = {(False, False): lib.pglb_fa_attn_csr_f32, (False, True): lib.pglb_fa_attn_csr_x16,
          (True, False): lib.pglb_fa_attn_drop_csr_f32, (True, True): lib.pglb_fa_attn_drop_csr_x16}
    with torch.cuda.device(f2.device):
        check(fn[(drop is not None, bool(dt))](*args, *dt, *(drop or ()), _ptr(ws), ws.numel(), _stream()))
    return out


class _FaFused(torch.autograd.Function):
    """FAConv's self-gated aggregation under autograd (reference pgl/nn/conv.py:1306-1339 differentiated by Paddle over
    send_uv(add), tanh, send_uv(mul), the product, dropout and send_ue_recv).  Forward = pglb_fa_attn_* (one pass;
    keeps only N-sized tensors: f2 and the [N, 4] node records, plus (seed, offset)).  Backward = one edge kernel
    (pglb_fa_bwd_edge_*: weights rebuilt bit for bit, beta and dz per edge, 8 bytes per edge alive only inside the
    backward) + three aggregations on the existing kernels: grad f = send_ue_recv(G, beta) and grad g_src = segment sum
    of dz over the src-keyed CSR, grad g_dst = segment sum of dz over the dst-keyed CSR.  16-bit f2 takes the *_x16
    entries; beta and dz are float32, grad f is aggregated in float32 on the widened G and comes back in f2's dtype,
    grad g_src / g_dst in their own dtypes.
    norm is a constant (no gradient)."""

    @staticmethod
    def forward(ctx, f2, g_src, g_dst, norm, fwd, bwd, drop):
        rec = _fa_records(g_src, norm, g_dst)
        out = _fa_fwd_raw(fwd, f2, rec, drop)
        ctx.meta = (fwd, bwd, drop, g_src.dtype, g_dst.dtype)
        ctx.save_for_backward(f2, rec)
        return out

    @staticmethod
    def backward(ctx, g):
        fwd, bwd, drop, gs_dtype, gd_dtype = ctx.meta
        bwd = bwd() if callable(bwd) else bwd
        f2, rec = ctx.saved_tensors
        half = f2.dtype in HALF_DTYPES
        g = _f32_2d(g.to(f2.dtype) if g.dtype != f2.dtype else g, allow16=half)
        E = int(fwd["cols"].shape[0])
        n, D = int(f2.shape[0]), int(f2.shape[1])
        beta = torch.empty((E, 1), dtype=torch.float32, device=g.device)
        dz = torch.empty((E, 1), dtype=torch.float32, device=g.device)
        dt = (_DTYPE16[f2.dtype],) if half else ()
        fn = {(False, False): lib.pglb_fa_bwd_edge_f32, (False, True): lib.pglb_fa_bwd_edge_x16,
              (True, False): lib.pglb_fa_bwd_edge_drop_f32, (True, True): lib.pglb_fa_bwd_edge_drop_x16}
        with torch.cuda.device(g.device):
            check(fn[(drop is not None, half)](
                _ptr(fwd["rows"]), _ptr(fwd["cols"]), _ptr(fwd["eid"]), _ptr(f2), f2.stride(0), _ptr(rec), _ptr(g),
                g.stride(0), E, D, *dt, *(drop or ()), _ptr(beta), _ptr(dz), _stream()))
        gf = gs = gd = None
        if ctx.needs_input_grad[0]:   # grad f[u] = sum over the out-edges of u of beta[e] G[dst]
            # 16-bit G is widened and aggregated on the float32 route, then rounded once: on cfg3's graph the 16-bit
            # edge-operand kernel made the bfloat16 D = 128 training step slower than the op-by-op route (DESIGN 4.18)
            gf = _spmm_raw(bwd["indptr"], bwd["cols"], g.float() if half else g, n, "sum", eid=bwd["eid"], y2=beta,
                           y_bcast=BCAST_SCALAR, head_dim=1, msg_op="mul", max_degree=bwd.get("max_degree", -1))
            gf = gf.to(f2.dtype) if half else gf
        if ctx.needs_input_grad[1]:   # z = g_src[src] + g_dst[dst]: send_uv(add)'s backward
            gs = _spmm_raw(bwd["indptr"], bwd["eid"], dz, n, "sum", max_degree=bwd.get("max_degree", -1))
            gs = gs.reshape(n).to(gs_dtype)
        if ctx.needs_input_grad[2]:
            gd = _spmm_raw(fwd["indptr"], fwd["eid"], dz, n, "sum", max_degree=fwd.get("max_degree", -1))
            gd = gd.reshape(n).to(gd_dtype)
        return gf, gs, gd, None, None, None, None


def fa_attention(fwd, bwd, f, g_src, g_dst, norm, attn_drop=0.0, seed=None, out_dtype=None):
    """FAConv's self-gated aggregation in one pass:
    out[d,:] = sum over the in-edges e = (u -> d) of d of keep_e s ((tanh(g_src[u] + g_dst[d]) norm[u]) norm[d]) f[u,:]
    with a fused backward when autograd needs one (grad f, g_src and g_dst; norm is a constant).  f [N, D]; g_src, g_dst
    and norm [N] or [N, 1] on one graph (n_dst == N); ``fwd`` is the dst-keyed CSR dict (with ``rows``), ``bwd`` the
    src-keyed one or a callable returning it.  The result dtype is ``out_dtype``, or by default torch's promotion of
    f's, g_src's and g_dst's dtypes.  float32 f runs the float32 kernels (g_src, g_dst and norm widened to float32);
    bfloat16 / float16 f runs the 16-bit kernels when the result dtype is f's (the output is the float32 kernel's on the
    widened f, rounded once; grad f in f's dtype, grad g_src / g_dst in theirs).  Returns [N, D], or None when the call
    is outside the kernels (float64, another dtype mix, D > 128 or rows not a multiple of 16 bytes, norm requiring
    grad, n_dst != N, no edges, attn_drop >= 1, misaligned f, dropout during CUDA-graph capture); the caller then keeps
    the op-by-op path.
    ``attn_drop`` in (0, 1): dropout on the edge weights inside the kernels, the keep bit of dst-CSR slot j being head 0
    of GAT's 4-head keep word, drawn from ``seed`` = (seed, offset), offset a multiple of 4, or by default from the
    default CUDA generator of f's device (whose offset then advances by 4); kept weights are scaled by 1 / (1 - p).
    The mask is not nn.Dropout's: only its distribution and its replay from (seed, offset) are promised."""
    require_cuda(f, g_src, g_dst, norm)
    if f.dim() != 2:
        return None
    n, D = int(f.shape[0]), int(f.shape[1])
    for t in (g_src, g_dst, norm):
        if not t.dtype.is_floating_point or t.numel() != n or not (t.dim() == 1 or (t.dim() == 2 and t.shape[1] == 1)):
            return None
    if norm.requires_grad:
        return None
    half = f.dtype in HALF_DTYPES
    if torch.float64 in (f.dtype, g_src.dtype, g_dst.dtype, norm.dtype):
        return None
    res = _result_dtype(out_dtype, f, g_src, g_dst)
    if not (f.dtype == torch.float32 or (half and res == f.dtype and
                                         torch.promote_types(f.dtype, torch.promote_types(g_src.dtype, g_dst.dtype))
                                         == f.dtype)):
        return None
    if D <= 0 or D > 128 or (D * f.element_size()) % 16:
        return None
    attn_drop = float(attn_drop)
    if not 0.0 <= attn_drop < 1.0:
        return None
    if attn_drop > 0.0 and torch.cuda.is_current_stream_capturing():
        return None     # the generator's offset advances on the host: not replayable by a graph
    if int(fwd["indptr"].shape[0]) - 1 != n or int(fwd["cols"].shape[0]) == 0 or fwd.get("rows") is None:
        return None
    f2 = _f32_2d(f, allow16=half)
    if f2.data_ptr() % 16 or (f2.stride(0) * f2.element_size()) % 16:
        return None
    gs, gd, nm = (t.reshape(n) for t in (g_src, g_dst, norm))
    drop = None
    if attn_drop > 0.0:
        drop = (attn_drop,) + (tuple(int(s) for s in seed) if seed is not None else _attn_drop_stream(f2.device))
    if torch.is_grad_enabled() and (f.requires_grad or g_src.requires_grad or g_dst.requires_grad):
        out = _FaFused.apply(f2, gs, gd, nm, fwd, bwd, drop)
    else:
        out = _fa_fwd_raw(fwd, f2, _fa_records(gs, nm, gd), drop)
    return out if out.dtype == res else out.to(res)


def _aligned16(t):
    """t contiguous with a 16-byte aligned base (rows are then 16-byte aligned for widths % 4 == 0)."""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _rgcn_agg_raw(csr, x2, w3, slot_w=None):
    """pglb_rgcn_agg_f32: out[d] = sum_r A_r[d] w3[r] on a typed CSR (heter_graph.typed_csr)."""
    n, K, N = csr["n_rows"], int(w3.shape[1]), int(w3.shape[2])
    if int(csr["cols"].shape[0]) == 0:
        # no edges (a sampled block whose targets have no in-edges): every run is empty, so every row is 0 -- what the
        # kernel would write; its empty slot arrays have no address to pass
        return torch.zeros((n, N), dtype=torch.float32, device=x2.device)
    out = torch.empty((n, N), dtype=torch.float32, device=x2.device)
    with torch.cuda.device(x2.device):
        check(lib.pglb_rgcn_agg_f32(_ptr(csr["indptr"]), _ptr(csr["cols"]), _ptr(csr["rel"]), _ptr(slot_w), _ptr(x2),
                                    x2.stride(0), _ptr(w3), int(w3.shape[0]), K, N, _ptr(out), out.stride(0), n,
                                    _stream()))
    return out


def _rgcn_wgrad_raw(fwd, x2, g, D, O):
    R = fwd["num_rels"]
    gw = torch.empty((R, D, O), dtype=torch.float32, device=x2.device)
    need = ctypes.c_size_t(0)
    check(lib.pglb_rgcn_wgrad_ws(fwd["n_items"], D, O, ctypes.byref(need)))
    ws = workspace(x2.device, need.value)
    with torch.cuda.device(x2.device):
        check(lib.pglb_rgcn_wgrad_f32(_ptr(fwd["run_row"]), _ptr(fwd["run_beg"]), _ptr(fwd["run_end"]),
                                      _ptr(fwd["run_off"]), _ptr(fwd["item_off"]), R, fwd["n_items"], fwd["chunk"],
                                      _ptr(fwd["cols"]), _ptr(x2), x2.stride(0), _ptr(g), g.stride(0), D, O, _ptr(gw),
                                      _ptr(ws), ws.numel(), _stream()))
    return gw


class _RGCNAgg(torch.autograd.Function):
    """RGCNConv's aggregation under autograd (reference pgl/nn/conv.py:1018-1024 differentiated by Paddle over the
    per-relation matmul, send_recv(mean) and sum).  Forward = one pglb_rgcn_agg_f32 on the typed dst-CSR.  Backward:
    grad x = pglb_rgcn_agg_f32 on the typed src-CSR with the per-slot weights 1 / cnt_r(dst) and W^T; grad weight =
    pglb_rgcn_wgrad_f32 over the run list (the A rows are gathered again, not stored)."""

    @staticmethod
    def forward(ctx, x2, w3, fwd, bwd):
        ctx.meta = (fwd, bwd)
        ctx.save_for_backward(x2, w3)
        return _rgcn_agg_raw(fwd, x2, w3)

    @staticmethod
    def backward(ctx, g):
        fwd, bwd = ctx.meta
        x2, w3 = ctx.saved_tensors
        g = _aligned16(g)
        gx = gw = None
        if ctx.needs_input_grad[0]:
            gx = _rgcn_agg_raw(bwd, g, w3.transpose(1, 2).contiguous(), slot_w=bwd["w"])
        if ctx.needs_input_grad[1]:
            gw = _rgcn_wgrad_raw(fwd, x2, g, int(w3.shape[1]), int(w3.shape[2]))
        return gx, gw, None, None


def rgcn_fused_pays(fwd, D, O):
    """The routing rule of rgcn_aggregate.  The fused kernel stages W_r (D x O) once per (64-row tile, relation) pair;
    the per-relation route runs R dense transforms over all N rows (D + O elements per row) and R launches per
    aggregation.  On a graph of >= 2^20 edges, where launches no longer dominate, the fused path is declined when
    the staged weights exceed half the dense transforms' row traffic (DESIGN 4.13: cfg3's RMAT graph split into 8
    relations at D = O = 128 sits at 1.7 and ran 2.1x slower fused; the example-shaped graph sits at 0.9 with
    2e5 edges and ran 7.8x faster)."""
    E = int(fwd["cols"].shape[0])
    return E < (1 << 20) or 2 * fwd["tile_rels"] * D * O <= fwd["num_rels"] * fwd["n_rows"] * (D + O)


def rgcn_aggregate(fwd, bwd, x, weight):
    """RGCNConv's relation-typed aggregation in one pass:
    out[d] = sum_r (mean over the in-edges of d in relation r of x[src]) @ weight[r]
    (the reference's sum_r send_recv(x @ weight[r], mean), reassociated) with a fused backward when autograd needs
    one.  ``fwd`` / ``bwd`` are the typed CSRs of heter_graph.typed_csr; weight [R, D, O].  Returns [N, O], or None
    when the call is outside the kernels (not CUDA, not float32, D or O not a multiple of 4 in [4, 128], x's rows not
    the graph's nodes, more than 32767 relations) or where the per-relation route is faster (rgcn_fused_pays); the
    caller then keeps the per-relation path."""
    if not (x.is_cuda and weight.is_cuda) or x.dtype != torch.float32 or weight.dtype != torch.float32:
        return None
    if x.dim() != 2 or weight.dim() != 3 or int(weight.shape[0]) != fwd["num_rels"] or fwd["num_rels"] > 32767:
        return None
    D, O = int(weight.shape[1]), int(weight.shape[2])
    if int(x.shape[1]) != D or int(x.shape[0]) != fwd["n_rows"]:
        return None
    if not all(4 <= v <= 128 and v % 4 == 0 for v in (D, O)):
        return None
    if not rgcn_fused_pays(fwd, D, O):
        return None
    x2 = _aligned16(x)
    w3 = weight.contiguous()
    if torch.is_grad_enabled() and (x.requires_grad or weight.requires_grad):
        return _RGCNAgg.apply(x2, w3, fwd, bwd)
    return _rgcn_agg_raw(fwd, x2, w3)


@f64_through
def aggregate_ue_slots(x, y_slots, fwd, n_dst, message_op="mul", reduce_op="sum"):
    """send_ue_recv whose edge operand is already in CSR slot order (read sequentially)."""
    require_cuda(x, y_slots)
    out_feat = tuple(x.shape[1:])
    cls = classify_bcast(x.shape, y_slots.shape)
    if cls is None:
        raise ValueError("pgl_b200: unsupported broadcast for slot-ordered edge operand")
    mode, hd = cls
    out = _spmm_raw(fwd["indptr"], fwd["cols"], _f32_2d(x), n_dst, reduce_op, eid=None,
                    y2=_f32_2d(y_slots), y_bcast=mode, head_dim=hd, msg_op=message_op,
                    max_degree=fwd.get("max_degree", -1))
    return out.reshape((n_dst,) + out_feat)


TC_GEMM = os.environ.get("PGLB_TC_GEMM", "1") != "0"
TC_GEMM_MIN_ROWS = int(os.environ.get("PGLB_TC_GEMM_MIN_ROWS", "4096"))


def linear_tc_ok(x, weight):
    """True when x @ weight can run on pglb_linear_tf32x3_f32 (tall-skinny fp32, K <= 128 and
    N in {64, 128}); small or odd shapes stay on torch.matmul (cuBLAS), which is plumbing here."""
    if not TC_GEMM or not x.is_cuda or x.dim() != 2 or x.dtype != torch.float32 \
            or weight.dtype != torch.float32:
        return False
    M, K = int(x.shape[0]), int(x.shape[1])
    N = int(weight.shape[1])
    return M >= TC_GEMM_MIN_ROWS and K % 4 == 0 and 4 <= K <= 128 and N in (64, 128) \
        and int(weight.shape[0]) == K


def _linear_tc_raw(x, weight, bias, act):
    x2 = x if (x.stride(1) == 1 and x.stride(0) % 4 == 0 and x.data_ptr() % 16 == 0) \
        else x.contiguous()
    w = weight.contiguous()
    M, K = int(x2.shape[0]), int(x2.shape[1])
    N = int(w.shape[1])
    out = torch.empty((M, N), dtype=torch.float32, device=x2.device)
    b = bias.contiguous() if bias is not None else None
    with torch.cuda.device(x2.device):
        check(lib.pglb_linear_tf32x3_f32(_ptr(x2), x2.stride(0), _ptr(w), _ptr(b) if b is not None else None,
                                         _ptr(out), N, M, K, N, 1 if act == "relu" else 0, _stream()))
    return out


class _LinearTC(torch.autograd.Function):
    """Forward on the 3xTF32 tensor-core kernel (bias + ReLU fused); backward is two plain fp32
    matmuls (training plumbing: the reference gets them from Paddle autograd)."""

    @staticmethod
    def forward(ctx, x, weight, bias, act):
        out = _linear_tc_raw(x, weight, bias, act)
        ctx.act = act
        ctx.has_bias = bias is not None
        ctx.save_for_backward(x, weight, out if act == "relu" else None)
        return out

    @staticmethod
    def backward(ctx, g):
        x, weight, out = ctx.saved_tensors
        if ctx.act == "relu":
            g = g * (out > 0)
        gx = g @ weight.t() if ctx.needs_input_grad[0] else None
        gw = x.t() @ g if ctx.needs_input_grad[1] else None
        gb = g.sum(0) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return gx, gw, gb, None


@f64_through
def linear_tc(x, weight, bias=None, act=None):
    """act(x @ weight + bias) with weight [in, out]; act in (None, "relu")."""
    require_cuda(x, weight)
    assert act in (None, "relu")
    if torch.is_grad_enabled() and (x.requires_grad or weight.requires_grad
                                    or (bias is not None and bias.requires_grad)):
        return _LinearTC.apply(x, weight, bias, act)
    return _linear_tc_raw(x, weight, bias, act)


def degree_norm(degree):
    require_cuda(degree)
    degree = _i64(degree).contiguous()
    n = int(degree.shape[0])
    out = torch.empty(n, dtype=torch.float32, device=degree.device)
    with torch.cuda.device(degree.device):
        check(lib.pglb_degree_norm_f32(_ptr(degree), n, _ptr(out), _stream()))
    return out.reshape(-1, 1)


def launch_count():
    return _lib.launch_count()


def stream_kernel_name(num_edges=None, num_rows=None):
    """Which wide-row streaming kernel pglb_spmm_csr_f32 routes copy-sum aggregations to (mirrors csrc/spmm_v5.inl
    v5_geo(): graphs of >= 12 slots per row take the groups-of-8 geometry)."""
    wide = num_edges is not None and num_rows and num_edges >= 12 * num_rows
    geo = "GRP=8,NG=3,W=9" if wide else "GRP=4,NG=4,W=13"
    return ("spmm_v5_kernel<bulk copy per row (cp.async.bulk), %s, device-side task queue> (+ task_plan, empty_rows, "
            "fix-up kernels)" % geo)
