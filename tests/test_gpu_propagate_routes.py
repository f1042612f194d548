"""Every route of the fused propagation step (pglb_propagate_f32 / pglb_propagate_narrow_f32, ops.propagate), forward
and backward, bit for bit against an exact float64 reference.

The step (include/pglb.h): t = s_dst * sum_{j -> d} s_src[j] x[j], y = a t (+ b h), acc_out = acc_in + c y, every
product and sum rounded on its own.  The reference restates it in float64 from the raw edge list (a scipy product,
never the library's CSR), in the contract's operation order, so the signs of zeros match too: a row without an edge
has t = +0, and with a < 0 and no h its y is -0.0.  `assert_bits` compares bit patterns, so -0.0 != +0.0.

The regime.  Features are small nonzero integers, norms powers of two, and a, b, c have few significant bits.  Every
term s_src[j] x[j] is then a multiple of a quantum q, and while the sum of |terms| of every row stays below 2^24 q,
every partial sum is exact whatever the order: sequential, 32-slot ranges, hub chunks, task partials plus fix-up.  If
every float64 intermediate (t, a t, b h, y, c y, acc_out) also survives a round trip through float32, each kernel
must return the reference exactly.  `prop_regime` asserts all of this for every case, so no case can quietly become a
tolerance test.  A dropped, doubled or misattributed slot, a skipped or misordered epilogue, a wrong operand row or
stride changes the exact value.

Routes.  The node-parallel kernel (one element per lane, or vec4 for D <= 64 without a narrow plan; hub passes for
rows past HUB_T = 1024), the narrow kernel (L = 4 / 8 / 16 lanes per row; SC = 0 / 1 / 2: no source norm, gathered,
or streamed per slot; HOT: L2 hints), and the wide-row v5 kernel (D in 68..128; geometry 0 or 2, chosen by
E >= 12 n; D128; HOT; SCALED) with its cut-row fix-up and empty-row fill.  `test_route_coverage` records which kernel
instantiations each call launches (torch.profiler).

The task size (PGLB_STREAM_TASK, read once per process, which also turns snapping off) runs the v5 and narrow forward
tests and the backward again in child processes, on a ladder graph whose boundary block is laid out for that task size
(`test_cut_coverage` checks the cuts it makes with `task_plan`)."""
import ctypes
import itertools
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import oracle as O
from test_gpu_exact_routes import LADDER, _int_features, _kernels_of, _packings, assert_bits, ladder_edges
from test_task_model import task_plan

CHILD = os.environ.get("PGLB_PROP_CHILD") == "1"
EXACT_LIMIT = float(1 << 24)
NORMS = np.array([0.5, 1.0, 2.0])
# (a, b, c): negative a and c, b = 0 with h given, few significant bits
COEFS = ((-0.75, 0.5, -1.5), (1.5, 0.0, 0.25), (-2.0, -1.0, 0.5))
H_KINDS = ("none", "h", "x")
ACC_KINDS = ("none", "out", "inplace", "c_dev")
HUB_T = 1024
PGLB_SPMM_L2_HINTS = 2


# ----------------------------------------------------------------------------------------------------------------
# float64 reference and the exact regime
# ----------------------------------------------------------------------------------------------------------------

def ref_prop(x, src, dst, n_dst, ss=None, sd=None, a=1.0, b=0.0, h=None, acc=None, c=1.0):
    """The step in float64 from the edge list: dict of t, at, bh, y, cy, acc_out (None where not formed)."""
    x = np.asarray(x, np.float64)
    src, dst = np.asarray(src, np.int64), np.asarray(dst, np.int64)
    w = np.ones(src.shape[0]) if ss is None else np.asarray(ss, np.float64)[src]
    A = sp.coo_matrix((w, (dst, src)), shape=(n_dst, x.shape[0])).tocsr()
    t = A @ x if src.size else np.zeros((n_dst, x.shape[1]))
    t = t + 0.0                                   # an empty row is +0
    if sd is not None:
        t = t * np.asarray(sd, np.float64)[:, None]
    at = a * t
    bh = None if h is None else b * np.asarray(h, np.float64)
    y = at if h is None else at + bh
    cy = None if acc is None else c * y
    acc_out = None if acc is None else np.asarray(acc, np.float64) + cy
    return {"t": t, "at": at, "bh": bh, "y": y, "cy": cy, "acc_out": acc_out}


def lowbit(v):
    """The largest power of two that divides each entry of v (0 for zeros)."""
    v = np.asarray(v, np.float64)
    m, e = np.frexp(v)
    M = (m * 2.0 ** 53).astype(np.int64)
    return np.where(v != 0, np.ldexp((M & -M).astype(np.float64), e - 53), 0.0)


def prop_regime(x, src, dst, n_dst, ss, ref, scalars=(), others=()):
    """Assert the preconditions of a bit-exact comparison for the step `ref` (ref_prop's result): float32 inputs;
    every term s_src[j] x[j] a multiple of q; the sum of |terms| of each row below 2^24 q; every intermediate finite
    and unchanged by a round trip through float32."""
    x = np.asarray(x, np.float64)
    for v in (x, ss, np.asarray(scalars, np.float64)) + tuple(others):
        if v is None:
            continue
        v = np.asarray(v, np.float64)
        assert np.array_equal(v, v.astype(np.float32).astype(np.float64)), "input not exactly representable in fp32"
    nz = x[x != 0]
    q = lowbit(nz).min() if nz.size else 1.0
    if ss is not None:
        q *= lowbit(np.asarray(ss, np.float64)[np.asarray(ss) != 0]).min(initial=1.0)
    w = np.ones(len(src)) if ss is None else np.abs(np.asarray(ss, np.float64))[src]
    A = sp.coo_matrix((w, (dst, src)), shape=(n_dst, x.shape[0])).tocsr()
    abs_sum = A @ np.abs(x)
    assert abs_sum.max(initial=0.0) < EXACT_LIMIT * q, \
        "case leaves the exact regime: a row's sum of |terms| reaches %g >= 2^24 q (q = %g)" % (abs_sum.max(), q)
    for name in ("t", "at", "bh", "y", "cy", "acc_out"):
        v = ref.get(name)
        if v is None:
            continue
        assert np.isfinite(v).all(), "case leaves the exact regime: %s is not finite" % name
        assert np.array_equal(v, v.astype(np.float32).astype(np.float64)), \
            "case leaves the exact regime: %s does not round-trip through float32" % name
    return q


def sum_regime(terms):
    """A float32 sum of `terms` (float64) in any order is exact: multiples of q whose |sum| stays below 2^24 q."""
    terms = np.asarray(terms, np.float64).ravel()
    nz = terms[terms != 0]
    q = lowbit(nz).min() if nz.size else 1.0
    assert np.array_equal(terms, terms.astype(np.float32).astype(np.float64)), "term not exactly representable"
    assert np.abs(terms).sum() < EXACT_LIMIT * q, "case leaves the exact regime: sum of |terms| >= 2^24 q"


def prop_case(x, src, dst, n_dst, ss=None, sd=None, a=1.0, b=0.0, h=None, acc=None, c=1.0):
    """(expected y, expected acc_out or None) as float32 arrays, after asserting the exact regime."""
    ref = ref_prop(x, src, dst, n_dst, ss, sd, a, b, h, acc, c)
    prop_regime(x, src, dst, n_dst, ss, ref, (a, b, c), (sd, h, acc))
    return ref["y"].astype(np.float32), (None if acc is None else ref["acc_out"].astype(np.float32))


# ----------------------------------------------------------------------------------------------------------------
# graphs and their task plans
# ----------------------------------------------------------------------------------------------------------------

def stream_task_size(E, sm_count, env_T=0):
    """(T, snap) of the copy-sum family: stream_task_size / stream_snap in pgl_b200/csrc/spmm_stream.cu."""
    if env_T:
        return env_T, env_T
    t = min(max((E // (sm_count * 28 * 4) + 31) // 32 * 32, 32), 2048)
    return t, max(t, 1024)


def narrow_task_sizes(T):
    """The narrow kernel's task size for L = 4, 8, 16 lanes per row: T rounded up to whole chunks of (32 / L) * 32
    slots (narrow2_task_size).  Narrow tasks start at multiples of it and never snap."""
    return {L: (T + (32 // L) * 32 - 1) // ((32 // L) * 32) * ((32 // L) * 32) for L in (4, 8, 16)}


def boundary_block(pos, T, snap):
    """In-degrees to append at slot `pos` (each row followed by 1 or 2 empty rows) so that tasks of T slots with the
    given snap cut: a row starting on a boundary, a cut row ending on one, a short row ending on one followed by
    empty rows, and, when rows of T + 1 slots are cut (snap <= T), a row cut into exactly a head and a tail."""
    degs = []

    def add(k, gap=1):
        nonlocal pos
        degs.extend([k] + [0] * gap)
        pos += k

    def pad_to(off):
        m = (off - pos) % T
        if m:
            add(m)
    long_ = max(snap, T)
    pad_to(0)
    add(long_ + 7)
    pad_to(-(long_ + 9) % T)
    add(long_ + 9)
    pad_to(T - 5)
    add(5, gap=2)
    if snap <= T:
        pad_to(T - 3)
        add(T + 1)
    return degs, pos


def ladder_degrees(T, snap, seed=5):
    """The LADDER in-degrees (shuffled) with runs of 1-3 empty rows between them, then a boundary block for the v5
    task size (T, snap) and one for each narrow task size."""
    rng = np.random.default_rng(seed)
    degs = []
    for k in rng.permutation(LADDER):
        degs.extend([int(k)] + [0] * int(rng.integers(1, 4)))
    pos = sum(degs)
    sizes = {T: snap}
    for tn in narrow_task_sizes(T).values():
        sizes.setdefault(tn, 0)
    for tt in sorted(sizes):
        block, pos = boundary_block(pos, tt, sizes[tt])
        degs.extend(block)
    return np.array(degs, np.int64)


def cut_cases(indptr, T, snap):
    """Which boundary cases the plan of tasks of T slots (snap as in task_plan) makes: dict name -> row ids."""
    n = indptr.shape[0] - 1
    E = int(indptr[-1])
    ntasks, _, start = task_plan(indptr, n, E, T, snap)
    inner = start[1:ntasks]
    s, e = indptr[:-1], indptr[1:]
    pieces = 1 + np.searchsorted(inner, e, side="left") - np.searchsorted(inner, s, side="right")
    deg = e - s
    on_boundary = np.isin(e, inner)
    empty_inside = (deg == 0) & (s > 0) & (s < E) & ~np.isin(s, start)
    return {"head_and_tail": np.flatnonzero((deg > 0) & (pieces == 2)),
            "three_or_more_tasks": np.flatnonzero((deg > 0) & (pieces >= 3)),
            "cut_row_ending_on_boundary": np.flatnonzero((deg > 0) & (pieces >= 2) & on_boundary),
            "short_row_ending_on_boundary": np.flatnonzero((deg > 0) & (pieces == 1) & on_boundary),
            "empty_run_inside_task": np.flatnonzero(empty_inside)}


def check_cut_cases(indptr, T, snap):
    """Assert every case the tests rely on exists under the plan (a head-and-tail cut only where snap allows it)."""
    cases = cut_cases(indptr, T, snap)
    need = [k for k in cases if k != "head_and_tail" or snap <= T]
    missing = [k for k in need if cases[k].size == 0]
    assert not missing, "tasks of %d slots (snap %d) make no %s" % (T, snap, ", ".join(missing))
    return cases


def v5_geometry(E, n_rows):
    """v5_geo in pgl_b200/csrc/spmm_v5.inl: groups of 8 at 12 or more slots per row, else groups of 4."""
    return 2 if (n_rows > 0 and E >= 12 * n_rows) else 0


def _env_T():
    try:
        v = int(os.environ.get("PGLB_STREAM_TASK", ""))
    except ValueError:
        return 0
    return v if v >= 32 and v % 32 == 0 else 0


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


class PGraph(object):
    """A graph of the suite: raw edges (the reference's input), a dst-CSR on the device (the C entries' input) and,
    for square graphs, a pgl Graph (ops.propagate's input)."""

    def __init__(self, name, edges, n_src, n_dst, with_graph=True):
        import pgl_b200 as pgl
        self.name, self.n_src, self.n_dst = name, n_src, n_dst
        self.src, self.dst = edges[:, 0].copy(), edges[:, 1].copy()
        self.E = int(edges.shape[0])
        order = np.argsort(self.dst, kind="stable")
        self.indptr = np.r_[0, np.cumsum(np.bincount(self.dst, minlength=n_dst))].astype(np.int64)
        self.deg = np.diff(self.indptr)
        self.ip_d = torch.from_numpy(self.indptr).cuda()
        self.cols_d = torch.from_numpy(self.src[order]).cuda()
        self.g = None
        if with_graph and n_src == n_dst:
            self.g = pgl.Graph(edges=edges, num_nodes=n_src)
            self.g.tensor()


_G = {}


def ladder_graph():
    """In-degree ladder with empty runs and this process's boundary block; E < 12 n (v5 geometry 0)."""
    if "ladder" not in _G:
        env = _env_T()
        T, snap = (env, env) if env else (32, 1024)
        degs = ladder_degrees(T, snap)
        E = int(degs.sum())
        n = max(degs.shape[0] + 64, E // 11 + 1)
        degs = np.r_[degs, np.zeros(n - degs.shape[0], np.int64)]
        assert stream_task_size(E, _sm_count(), env) == (T, snap), "the boundary block is laid out for another T"
        rng = np.random.default_rng(17)
        dst = np.repeat(np.arange(n), degs)
        src = rng.integers(0, n, E)
        perm = rng.permutation(E)
        G = PGraph("ladder", np.stack([src[perm], dst[perm]], 1).astype(np.int64), n, n)
        check_cut_cases(G.indptr, T, snap)
        for tn in narrow_task_sizes(T).values():
            check_cut_cases(G.indptr, tn, 0)
        assert v5_geometry(G.E, n) == 0
        _G["ladder"] = G
    return _G["ladder"]


def two_sided_graph():
    """In-degree ladder and out-degree ladder (different shuffles): the backward's reverse CSR has the same long rows
    and empty runs.  E < 12 n."""
    if "two" not in _G:
        rng = np.random.default_rng(23)

        def side():
            d = []
            for k in rng.permutation(LADDER):
                d.extend([int(k)] + [0] * int(rng.integers(1, 4)))
            return np.array(d, np.int64)
        din, dout = side(), side()
        E = int(din.sum())
        n = max(din.shape[0], dout.shape[0], E // 11 + 1)
        din = np.r_[din, np.zeros(n - din.shape[0], np.int64)]
        dout = np.r_[dout, np.zeros(n - dout.shape[0], np.int64)]
        dst = np.repeat(np.arange(n), din)
        src = rng.permutation(np.repeat(np.arange(n), dout))
        G = PGraph("two_sided", np.stack([src, dst], 1).astype(np.int64), n, n)
        assert np.array_equal(np.bincount(G.src, minlength=n), dout) and v5_geometry(G.E, n) == 0
        _G["two"] = G
    return _G["two"]


def dense_graph():
    """Chung-Lu graph with E >= 12 n: v5 geometry 2."""
    if "dense" not in _G:
        n = 3000
        G = PGraph("dense", O.chung_lu_edges(n, 48000, exponent=0.8, seed=41).astype(np.int64), n, n)
        assert v5_geometry(G.E, n) == 2
        _G["dense"] = G
    return _G["dense"]


def rect_graph():
    """n_dst = 900 != n_src = 3000, one 6000-slot row, rows past 700 empty: the C entries only."""
    if "rect" not in _G:
        rng = np.random.default_rng(31)
        e = np.stack([rng.integers(0, 3000, 20000), rng.integers(0, 700, 20000)], 1)
        e[:6000, 1] = 311
        _G["rect"] = PGraph("rect", e.astype(np.int64), 3000, 900)
    return _G["rect"]


def _graph(name):
    return {"ladder": ladder_graph, "dense": dense_graph, "rect": rect_graph, "two_sided": two_sided_graph}[name]()


# ----------------------------------------------------------------------------------------------------------------
# calls
# ----------------------------------------------------------------------------------------------------------------

def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float64), dtype=np.float32)).cuda()


def _check_rc(rc, what):
    from pgl_b200._lib import lib
    assert rc == 0, "%s refused: rc %d, %s" % (what, rc, lib.pglb_last_error())


def _ws(nbytes):
    from pgl_b200 import ops
    return ops.workspace(torch.device("cuda", torch.cuda.current_device()), nbytes)


def c_propagate(G, x, n_dst, ss=None, sslot=None, sd=None, a=1.0, b=0.0, h=None, acc_in=None, acc_out=None, c=1.0,
                c_dev=None, packed=None, hints=False, max_degree=-1, cols=None, indptr=None):
    """One pglb_propagate_f32 call; returns out."""
    from pgl_b200 import ops
    from pgl_b200._lib import lib
    ip = G.ip_d if indptr is None else indptr
    cols = G.cols_d if cols is None else cols
    n_src, D = int(x.shape[0]), int(x.shape[1])
    E = int(cols.shape[0])
    out = torch.empty((n_dst, D), dtype=torch.float32, device="cuda")
    need = ctypes.c_size_t(0)
    _check_rc(lib.pglb_spmm_csr_ws(n_dst, E, D, ctypes.byref(need)), "pglb_spmm_csr_ws")
    ws = _ws(need.value)
    p = ops._ptr
    rc = lib.pglb_propagate_f32(p(ip), p(cols) if E else None, p(x), x.stride(0), p(out), out.stride(0), n_dst, n_src,
                                E, D, p(ss), p(sslot), p(sd), a, b, p(h), h.stride(0) if h is not None else 0,
                                p(acc_in), acc_in.stride(0) if acc_in is not None else 0, p(acc_out),
                                acc_out.stride(0) if acc_out is not None else 0, c, p(c_dev), p(packed), max_degree,
                                PGLB_SPMM_L2_HINTS if hints else 0, p(ws), ws.numel(), ops._stream())
    _check_rc(rc, "pglb_propagate_f32")
    return out


def narrow_plan(G, packed=None):
    """(plan, nz_row, blk_k) of G's CSR, carrying bit 31 of `packed` (pglb_pack_cols ids) when given."""
    from pgl_b200 import ops
    from pgl_b200._lib import lib
    E = G.E
    plan = torch.empty(E, dtype=torch.int32, device="cuda")
    nz_row = torch.empty(G.n_dst + 2, dtype=torch.int32, device="cuda")
    blk_k = torch.empty((E + 31) // 32, dtype=torch.int32, device="cuda")
    need = ctypes.c_size_t(0)
    _check_rc(lib.pglb_narrow_plan_ws(G.n_dst, ctypes.byref(need)), "pglb_narrow_plan_ws")
    ws = _ws(need.value)
    _check_rc(lib.pglb_narrow_plan(ops._ptr(G.ip_d), ops._ptr(G.cols_d), ops._ptr(packed), G.n_dst, G.n_src, E,
                                   ops._ptr(plan), ops._ptr(nz_row), ops._ptr(blk_k), ops._ptr(ws), ws.numel(),
                                   ops._stream()), "pglb_narrow_plan")
    return plan, nz_row, blk_k


def c_propagate_narrow(G, x, n_dst, plan, ss=None, sslot=None, sd=None, a=1.0, b=0.0, h=None, acc_in=None,
                       acc_out=None, c=1.0, c_dev=None, hints=False):
    """One pglb_propagate_narrow_f32 call; returns out."""
    from pgl_b200 import ops
    from pgl_b200._lib import lib
    n_src, D = int(x.shape[0]), int(x.shape[1])
    out = torch.empty((n_dst, D), dtype=torch.float32, device="cuda")
    need = ctypes.c_size_t(0)
    _check_rc(lib.pglb_spmm_narrow_ws(G.E, D, ctypes.byref(need)), "pglb_spmm_narrow_ws")
    ws = _ws(need.value)
    p = ops._ptr
    rc = lib.pglb_propagate_narrow_f32(p(plan[0]), p(plan[1]), p(plan[2]), p(G.ip_d), p(x), x.stride(0), p(out),
                                       out.stride(0), n_dst, n_src, G.E, D, p(ss), p(sslot), p(sd), a, b, p(h),
                                       h.stride(0) if h is not None else 0, p(acc_in),
                                       acc_in.stride(0) if acc_in is not None else 0, p(acc_out),
                                       acc_out.stride(0) if acc_out is not None else 0, c, p(c_dev),
                                       PGLB_SPMM_L2_HINTS if hints else 0, p(ws), ws.numel(), ops._stream())
    _check_rc(rc, "pglb_propagate_narrow_f32")
    return out


# ----------------------------------------------------------------------------------------------------------------
# the epilogue matrix of one route
# ----------------------------------------------------------------------------------------------------------------

_CANARY = 0x7FA5A5A5


def _window(n, D, ld, off, fill=None):
    """A [n, D] window at column `off` of an [n, ld] buffer (canary-filled) and the buffer."""
    buf = torch.full((n, ld), _CANARY, dtype=torch.int32, device="cuda").view(torch.float32)
    w = buf[:, off:off + D]
    if fill is not None:
        w.copy_(fill)
    return w, buf


def _outside_untouched(buf, off, D, what):
    bits = buf.view(torch.int32).cpu().numpy()
    keep = np.ones(bits.shape, bool)
    keep[:, off:off + D] = False
    assert (bits[keep] == _CANARY).all(), "%s: wrote outside its window" % what


def epilogue_cases(kinds="all", square=True):
    """[(h kind, acc kind, layout, (a, b, c))]: every h kind with every acc kind (each with every coefficient set
    over the matrix), then the strided layouts; `kinds` = "few" keeps two cases and one strided layout."""
    cases = []
    for i, (hk, ak) in enumerate(itertools.product(H_KINDS, ACC_KINDS)):
        if hk == "x" and not square:
            continue
        cases.append((hk, ak, "contig", COEFS[i % 3]))
    strided = [("h", "out", "strided", COEFS[0]), ("h", "inplace", "strided", COEFS[2]),
               ("none", "c_dev", "strided", COEFS[1])]
    if kinds == "few":
        return [("h", "out", "contig", COEFS[0]), ("none", "inplace", "contig", COEFS[2])]
    return cases + strided


def run_epilogues(G, D, call, tag, scales="separate", kinds="all", strided=True, seed=0):
    """Run `call` over the epilogue cases on G at width D and compare every output bit for bit.
    call(x, ss, sd, a, b, h, acc_in, acc_out, c, c_dev) -> y; for an ops-level call, call.ops is True and the call
    returns (y, acc_out) itself from (x, norm, a, b, h, acc, c or c_dev, inplace).  scales: "separate" (s_src and
    s_dst differ), "shared" (one norm, as ops.propagate takes it) or None (unscaled).  Returns the comparisons made."""
    rng = np.random.default_rng(seed * 7919 + D)
    n_src, n_dst = G.n_src, G.n_dst
    x = _int_features(rng, n_src, D, torch.float32)
    hv = _int_features(rng, n_dst, D, torch.float32)
    av = _int_features(rng, n_dst, D, torch.float32)
    ss = sd = None
    if scales == "separate":
        ss, sd = rng.choice(NORMS, n_src), rng.choice(NORMS, n_dst)
    elif scales == "shared":
        ss = sd = rng.choice(NORMS, n_src)
    xd, hd0, ad0 = _dev(x), _dev(hv), _dev(av)
    ss_d = None if ss is None else _dev(ss)
    sd_d = None if sd is None else (ss_d if scales == "shared" else _dev(sd))
    is_ops = getattr(call, "ops", False)
    n_cmp = 0
    for hk, ak, layout, (a, b, c) in epilogue_cases(kinds, n_src == n_dst):
        if layout == "strided" and (is_ops or not strided):
            continue
        label = "%s %s D=%d h=%s acc=%s %s a=%g b=%g c=%g scales=%s" % (tag, G.name, D, hk, ak, layout, a, b, c,
                                                                        scales)
        h_np = {"none": None, "h": hv, "x": x}[hk]
        acc_np = None if ak == "none" else av
        want_y, want_acc = prop_case(x, G.src, G.dst, n_dst, ss, sd, a, b, h_np, acc_np, c)
        c_dev = torch.tensor([c], dtype=torch.float32, device="cuda") if ak == "c_dev" else None
        bufs = []
        if layout == "contig":
            h = {"none": None, "h": hd0, "x": xd}[hk]
            acc_in = None if ak == "none" else ad0.clone()
            acc_out = None if ak == "none" else (acc_in if ak == "inplace" else torch.empty_like(ad0))
        else:
            # h and acc windows of wider buffers; acc_in and acc_out at different strides unless in place
            h = None if hk == "none" else _window(n_dst, D, D + 8, 4, hd0)[0]
            acc_in, ib = _window(n_dst, D, D + 4, 0, ad0)
            if ak == "inplace":
                acc_out, ob, ooff = acc_in, ib, 0
            else:
                acc_out, ob = _window(n_dst, D, D + 12, 4)
                ooff = 4
            bufs.append((ob, ooff))
        if is_ops:
            r = call(xd, ss_d, a, b, h, acc_in, c_dev if c_dev is not None else c, ak == "inplace")
            y, ao = (r, None) if acc_in is None else r
            if ak == "inplace":
                assert ao is acc_in, label + ": in-place acc was not written in place"
        else:
            # with c on the device the host c is a decoy: an epilogue that read it would be off
            y = call(xd, ss_d, sd_d, a, b, h, acc_in, acc_out, c if c_dev is None else 3.0, c_dev)
            ao = acc_out
        assert_bits(y.cpu(), torch.from_numpy(want_y), label + " (y)", G.dst)
        n_cmp += 1
        if want_acc is not None:
            assert_bits(ao.cpu(), torch.from_numpy(want_acc), label + " (acc_out)", G.dst)
            n_cmp += 1
        for ob, ooff in bufs:
            _outside_untouched(ob, ooff, D, label)
    return n_cmp


def ops_call(G):
    """ops.propagate on G's library CSR (the route the library picks; one shared norm)."""
    from pgl_b200 import ops
    fwd = G.g._fwd_csr()

    def call(x, norm, a, b, h, acc, c, inplace):
        with torch.no_grad():
            r = ops.propagate(x, fwd, None, norm, a=a, b=b, h=h, acc=acc, c=c, inplace_acc=inplace)
        assert r is not None, "ops.propagate declined"
        return r
    call.ops = True
    return call


def csr_call(G, n_dst=None, **kw):
    def call(x, ss, sd, a, b, h, acc_in, acc_out, c, c_dev):
        return c_propagate(G, x, G.n_dst if n_dst is None else n_dst, ss=ss, sd=sd, a=a, b=b, h=h, acc_in=acc_in,
                           acc_out=acc_out, c=c, c_dev=c_dev, **kw)
    return call


def narrow_call(G, plan, hints=False, slot=False):
    """pglb_propagate_narrow_f32; slot: stream the source norm per slot (SC 2) instead of gathering it (SC 1)."""
    sl = torch.from_numpy(G.src[np.argsort(G.dst, kind="stable")]).cuda()

    def call(x, ss, sd, a, b, h, acc_in, acc_out, c, c_dev):
        sslot = ss[sl].contiguous() if (slot and ss is not None) else None
        return c_propagate_narrow(G, x, G.n_dst, plan, ss=ss, sslot=sslot, sd=sd, a=a, b=b, h=h, acc_in=acc_in,
                                  acc_out=acc_out, c=c, c_dev=c_dev, hints=hints)
    return call


def slot_scale_csr_call(G, packed=None, hints=False):
    """pglb_propagate_f32 with the source norm streamed per slot (scale_slot)."""
    sl = torch.from_numpy(G.src[np.argsort(G.dst, kind="stable")]).cuda()

    def call(x, ss, sd, a, b, h, acc_in, acc_out, c, c_dev):
        return c_propagate(G, x, G.n_dst, ss=ss, sslot=None if ss is None else ss[sl].contiguous(), sd=sd, a=a, b=b,
                           h=h, acc_in=acc_in, acc_out=acc_out, c=c, c_dev=c_dev, packed=packed, hints=hints)
    return call


# ----------------------------------------------------------------------------------------------------------------
# CPU: the reference, the regime helper and the task plans
# ----------------------------------------------------------------------------------------------------------------

def test_reference_matches_hand_computed_graph():
    """4 destination rows, row 2 without an edge: t by hand; -0.0 where a < 0 meets an empty row."""
    src = np.array([0, 1, 1, 3, 2])
    dst = np.array([0, 0, 1, 3, 3])
    x = np.array([[1.0, -2.0], [3.0, 4.0], [-5.0, 6.0], [7.0, 0.5]])
    ss = np.array([1.0, 0.5, 2.0, 4.0])
    sd = np.array([2.0, 1.0, 0.5, 0.25])
    r = ref_prop(x, src, dst, 4, ss, sd, a=-0.5)
    want_t = np.array([[2 * (1 + 1.5), 2 * (-2 + 2)], [3 * 0.5, 4 * 0.5], [0.0, 0.0],
                       [0.25 * (-10 + 28), 0.25 * (12 + 2)]])
    assert np.array_equal(r["t"], want_t)
    assert np.array_equal(r["y"], -0.5 * want_t)
    assert not np.signbit(r["t"][2]).any() and np.signbit(r["y"][2]).all()      # -0.0 on the empty row
    assert not np.signbit(r["t"][0, 1]) and np.signbit(r["y"][0, 1])             # -2 + 2 = +0, then -0.5 * +0
    # h, acc: y = a t + b h (b = 0 with h: -0 + +0 = +0), acc_out = acc + c y
    h = np.full((4, 2), 3.0)
    r = ref_prop(x, src, dst, 4, ss, sd, a=-0.5, b=0.0, h=h, acc=np.ones((4, 2)), c=-2.0)
    assert not np.signbit(r["y"][2]).any() and np.array_equal(r["acc_out"], 1.0 - 2.0 * r["y"])
    y32, a32 = prop_case(x, src, dst, 4, ss, sd, -0.5)
    assert a32 is None and np.signbit(y32[2]).all()


def test_reference_matches_ladder_by_edge_loop():
    edges, n, degs = ladder_edges()
    src, dst = edges[:, 0], edges[:, 1]
    rng = np.random.default_rng(2)
    x = _int_features(rng, n, 3, torch.float32)
    ss, sd = rng.choice(NORMS, n), rng.choice(NORMS, n)
    t = np.zeros((n, 3))
    for s, d in zip(src.tolist(), dst.tolist()):
        t[d] += ss[s] * x[s]
    t *= sd[:, None]
    h = _int_features(rng, n, 3, torch.float32)
    acc = _int_features(rng, n, 3, torch.float32)
    r = ref_prop(x, src, dst, n, ss, sd, -0.75, 0.5, h, acc, -1.5)
    assert np.array_equal(r["t"], t)
    assert np.array_equal(r["acc_out"], acc + -1.5 * (-0.75 * t + 0.5 * h))
    assert (degs == 0).any() and np.signbit(r["at"][degs == 0]).all()


def test_prop_regime_refuses_cases_outside_it():
    edges, n, _ = ladder_edges()
    src, dst = edges[:, 0], edges[:, 1]
    rng = np.random.default_rng(3)
    x = _int_features(rng, n, 4, torch.float32)
    ss = rng.choice(NORMS, n)
    prop_case(x, src, dst, n, ss, ss, -0.75, 0.5, x, x, -1.5)
    with pytest.raises(AssertionError, match="2\\^24"):          # 30k slots of 2^10 at quantum 1
        prop_case(np.full((n, 4), 1024.0) + 1, src, dst, n)
    with pytest.raises(AssertionError, match="round-trip"):      # a t with too many significant bits
        prop_case(x, src, dst, n, a=1.0 + 2.0 ** -20)
    with pytest.raises(AssertionError, match="round-trip"):      # acc_out: a large acc plus a fractional c y
        prop_case(x, src, dst, n, ss, ss, 0.75, acc=np.full((n, 4), 2.0 ** 24), c=1.0)
    with pytest.raises(AssertionError, match="representable"):
        prop_case(np.full((n, 4), 0.1), src, dst, n)
    with pytest.raises(AssertionError, match="representable"):
        prop_case(x, src, dst, n, a=0.1)
    with pytest.raises(AssertionError, match="2\\^24"):
        sum_regime(np.full(1 << 20, 17.0))
    sum_regime(np.full(1 << 10, 17.0))


CUT_TS = [32, 64, 160, 1024, 2048]


@pytest.mark.parametrize("T", CUT_TS + [0])
def test_cut_coverage(T):
    """The ladder laid out for task size T (0: the library's default on an H100, T = 32 with snapping at 1024) has,
    under the v5 plan and under each narrow plan, a row cut into exactly a head and a tail (where the snap allows
    one), a row spanning three or more tasks, a cut row and a short row ending on a task boundary, and an empty-row
    run inside a task."""
    Tv, snap = (T, T) if T else (32, 1024)
    degs = ladder_degrees(Tv, snap)
    E = int(degs.sum())
    for sms in (114, 132):
        assert stream_task_size(E, sms, T) == (Tv, snap)
    ip = np.r_[0, np.cumsum(degs)].astype(np.int64)
    cases = check_cut_cases(ip, Tv, snap)
    assert (degs[cases["three_or_more_tasks"]] == 30011).any()
    for tn in narrow_task_sizes(Tv).values():
        check_cut_cases(ip, tn, 0)
    # rows of at most snap slots are never cut by the v5 plan
    cut = np.zeros(degs.shape[0], bool)
    for k in ("head_and_tail", "three_or_more_tasks", "cut_row_ending_on_boundary"):
        cut[cases[k]] = True
    assert not cut[degs <= snap].any()


def test_v5_geometry_formula():
    assert v5_geometry(12 * 1000, 1000) == 2 and v5_geometry(12 * 1000 - 1, 1000) == 0 and v5_geometry(5, 0) == 0


# ----------------------------------------------------------------------------------------------------------------
# GPU: forward, every family
# ----------------------------------------------------------------------------------------------------------------

SCALAR_WIDTHS = [1, 3, 5, 7, 9, 33, 129, 1433]
VEC4_WIDTHS = [4, 8, 12, 16, 20, 32, 36, 64]
NARROW_WIDTHS = [4, 8, 12, 16, 20, 32, 36, 64]
V5_WIDTHS = [68, 100, 124, 128]
if CHILD:
    NARROW_WIDTHS = [16, 32, 64]


@pytest.mark.gpu
@pytest.mark.parametrize("D", SCALAR_WIDTHS)
def test_node_parallel_scalar_exact(D):
    """One element per lane (D % 4 != 0): ops.propagate's route, then the C entry with separate norms, strided
    operands, no norms, forced hub passes and a rectangular call."""
    for gname in ("ladder", "dense") if D < 1000 else ("ladder",):
        G = _graph(gname)
        n = run_epilogues(G, D, ops_call(G), "ops", scales="shared")
        n += run_epilogues(G, D, csr_call(G), "csr")
        n += run_epilogues(G, D, csr_call(G), "csr unscaled", scales=None, kinds="few")
        n += run_epilogues(G, D, csr_call(G, max_degree=-1), "csr hub forced", kinds="few")
        assert n > 0
    R = rect_graph()
    run_epilogues(R, D, csr_call(R), "csr rect", kinds="few")
    run_epilogues(R, D, csr_call(R), "csr rect unscaled", scales=None, kinds="few")


@pytest.mark.gpu
@pytest.mark.parametrize("D", [20, 36, 64])
def test_node_parallel_unaligned_x_exact(D):
    """x one element past a 16-byte boundary at row stride D + 3: the one-element-per-lane kernel at widths the
    vector kernels otherwise take."""
    for gname in ("ladder", "dense"):
        G = _graph(gname)
        base = torch.empty((G.n_src, D + 3), dtype=torch.float32, device="cuda")

        def call(x, ss, sd, a, b, h, acc_in, acc_out, c, c_dev):
            xs = base[:, 1:D + 1]
            xs.copy_(x)
            hh = xs if (h is not None and h.data_ptr() == x.data_ptr()) else h
            return c_propagate(G, xs, G.n_dst, ss=ss, sd=sd, a=a, b=b, h=hh, acc_in=acc_in, acc_out=acc_out, c=c,
                               c_dev=c_dev)
        assert run_epilogues(G, D, call, "csr unaligned x") > 0


@pytest.mark.gpu
@pytest.mark.parametrize("D", VEC4_WIDTHS)
def test_node_parallel_vec4_exact(D):
    """Four elements per lane: pglb_propagate_f32 without a narrow plan at D <= 64."""
    for gname in ("ladder", "dense"):
        G = _graph(gname)
        run_epilogues(G, D, csr_call(G), "csr vec4")
        run_epilogues(G, D, csr_call(G), "csr vec4 unscaled", scales=None, kinds="few")
        run_epilogues(G, D, csr_call(G, max_degree=-1), "csr vec4 hub forced", kinds="few")
    R = rect_graph()
    run_epilogues(R, D, csr_call(R), "csr vec4 rect", kinds="few")


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 16, 128, 256, 512])
def test_edgeless_exact(D):
    """A graph without edges through the C entry: every row empty, t = +0 (-0.0 outputs where a < 0); at D > 64 the
    only way to the four-element-per-lane kernel of 32-lane groups."""
    G = PGraph("edgeless", np.zeros((0, 2), np.int64), 300, 300, with_graph=False)
    run_epilogues(G, D, csr_call(G), "csr edgeless")


@pytest.mark.gpu
@pytest.mark.parametrize("D", NARROW_WIDTHS)
def test_narrow_exact(D):
    """The narrow kernel: ops.propagate (the norm on first sighting gathered, then streamed per slot), then the C
    entry with every packing, with and without L2 hints, gathered and streamed norms, no norms, and a rectangular
    call."""
    from pgl_b200 import ops
    graphs = ("ladder", "dense") if not CHILD else ("ladder",)
    for gname in graphs:
        G = _graph(gname)
        if not CHILD:
            run_epilogues(G, D, ops_call(G), "ops narrow", scales="shared")
        plans = {name: (narrow_plan(G, pk[0] if pk[1] else None), pk[1])
                 for name, pk in _packings(ops, G.cols_d, G.n_src).items()}
        plan0 = plans["none"][0]
        run_epilogues(G, D, narrow_call(G, plan0), "narrow SC=1")
        run_epilogues(G, D, narrow_call(G, plan0, slot=True), "narrow SC=2")
        run_epilogues(G, D, narrow_call(G, plan0), "narrow SC=0", scales=None, kinds="few")
        for name, (plan, has) in plans.items():
            for slot in (False, True):
                run_epilogues(G, D, narrow_call(G, plan, hints=True, slot=slot),
                              "narrow hints packing=%s (marked=%s) slot=%s" % (name, has, slot), kinds="few")
        run_epilogues(G, D, narrow_call(G, plans["all"][0], hints=True), "narrow SC=0 hot", scales=None,
                      kinds="few")
    R = rect_graph()
    run_epilogues(R, D, narrow_call(R, narrow_plan(R)), "narrow rect", kinds="few")


@pytest.mark.gpu
@pytest.mark.parametrize("D", V5_WIDTHS)
def test_v5_exact(D):
    """The wide-row kernel on both geometries (ladder: 0, dense: 2), with its cut-row fix-up and empty-row fill:
    ops.propagate, then the C entry with gathered and streamed norms, no norms, every packing (L2 hints at D = 128)
    and a rectangular call."""
    from pgl_b200 import ops
    for gname in ("ladder", "dense"):
        G = _graph(gname)
        if not CHILD:
            run_epilogues(G, D, ops_call(G), "ops v5", scales="shared")
        run_epilogues(G, D, csr_call(G), "v5 gathered norms")
        run_epilogues(G, D, slot_scale_csr_call(G), "v5 streamed norms", kinds="few")
        run_epilogues(G, D, csr_call(G), "v5 unscaled", scales=None, kinds="few")
        for name, (pk, has) in _packings(ops, G.cols_d, G.n_src).items():
            if D != 128 and name in ("few", "mixed"):
                continue
            run_epilogues(G, D, csr_call(G, packed=pk, hints=True), "v5 packing=%s (marked=%s)" % (name, has),
                          kinds="few")
            if D == 128:
                run_epilogues(G, D, csr_call(G, packed=pk, hints=True), "v5 packing=%s unscaled" % name,
                              scales=None, kinds="few")
                run_epilogues(G, D, slot_scale_csr_call(G, packed=pk, hints=True),
                              "v5 packing=%s streamed norms" % name, kinds="few")
    R = rect_graph()
    run_epilogues(R, D, csr_call(R), "v5 rect", kinds="few")
    run_epilogues(R, D, csr_call(R), "v5 rect unscaled", scales=None, kinds="few")


# ----------------------------------------------------------------------------------------------------------------
# GPU: op-by-op identity on random floats
# ----------------------------------------------------------------------------------------------------------------

def _eq(got, want, what, G):
    assert_bits(got.detach().cpu(), want.detach().cpu(), what, G.dst)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [7, 16, 36, 64, 100, 128, 129])
def test_op_by_op_identity(D):
    """On random floats the fused hop is bit for bit torch's op-by-op hop on the same aggregation route: one hop,
    10 hops of APPNP, SSGC's in-place running sum and GPR's device-side coefficient."""
    from pgl_b200 import ops
    from pgl_b200.nn.conv import _propagate
    for gname in ("ladder", "dense"):
        G = _graph(gname)
        g, fwd = G.g, G.g._fwd_csr()
        torch.manual_seed(D)
        x = torch.randn(G.n_src, D, device="cuda")
        h = torch.randn(G.n_src, D, device="cuda")
        acc = torch.randn(G.n_src, D, device="cuda")
        norm = torch.rand(G.n_src, device="cuda") + 0.25
        tag = "%s D=%d" % (gname, D)
        with torch.no_grad():
            for a, b, c in COEFS + ((0.9, 0.1, 0.3),):
                y, ao = ops.propagate(x, fwd, None, norm, a=a, b=b, h=h, acc=acc, c=c)
                wy = a * _propagate(g, x, norm) + b * h
                _eq(y, wy, "%s one hop a=%g b=%g" % (tag, a, b), G)
                _eq(ao, acc + c * wy, "%s one hop acc c=%g" % (tag, c), G)
                _eq(ops.propagate(x, fwd, None, norm, a=a), a * _propagate(g, x, norm), tag + " a only", G)
            alpha = 0.1
            f, r = x, x
            for _ in range(10):
                f = ops.propagate(f, fwd, None, norm, a=1 - alpha, b=alpha, h=x)
                r = alpha * x + (1 - alpha) * _propagate(g, r, norm)
            _eq(f, r, tag + " APPNP 10 hops", G)
            f, s = x, x.clone()
            rf, rs = x, x
            for _ in range(8):
                f, s2 = ops.propagate(f, fwd, None, norm, a=1 - alpha, acc=s, c=1.0, inplace_acc=True)
                assert s2 is s
                rf = (1 - alpha) * _propagate(g, rf, norm)
                rs = rs + rf
            _eq(f, rf, tag + " SSGC hops", G)
            _eq(s, rs, tag + " SSGC in-place running sum", G)
            temp = torch.randn(11, device="cuda")
            f, hid = x, x * temp[0]
            rf, rh = x, x * temp[0]
            for k in range(10):
                f, hid = ops.propagate(f, fwd, None, norm, acc=hid, c=temp[k + 1:k + 2])
                rf = _propagate(g, rf, norm)
                rh = rh + temp[k + 1] * rf
            _eq(hid, rh, tag + " GPR running sum, c on the device", G)


# ----------------------------------------------------------------------------------------------------------------
# GPU: backward
# ----------------------------------------------------------------------------------------------------------------

BWD_WIDTHS = [7, 12, 20, 36, 100, 128, 129]
if CHILD:
    BWD_WIDTHS = [12, 20, 36, 100, 128]


@pytest.mark.gpu
@pytest.mark.parametrize("D", BWD_WIDTHS)
def test_backward_exact(D):
    """ops.propagate's backward on dyadic inputs on the two-sided ladder (the reverse CSR has the long rows and empty
    runs too): g_x = a s * A^T (s * g_tot) with g_tot = g_y + c g_acc, g_h = b g_tot, g_acc passed through,
    g_c = sum(g_acc * y) -- all exact -- and the same bits from a second run."""
    from pgl_b200 import ops
    G = two_sided_graph()
    g = G.g
    n = G.n_src
    rng = np.random.default_rng(D + 5)
    x = _int_features(rng, n, D, torch.float32)
    hv = _int_features(rng, n, D, torch.float32)
    av = _int_features(rng, n, D, torch.float32)
    s = rng.choice(NORMS, n)
    gy = rng.integers(-3, 4, (n, D)).astype(np.float64)
    # g_acc sparse, so that sum(g_acc * y) stays in the exact regime
    gacc = rng.choice([-1.0, 1.0], (n, D)) * (rng.random((n, D)) < 2.0 / D)
    for a, b, c in ((-0.75, 0.5, -1.5), (1.5, -1.0, 0.25)):
        tag = "backward D=%d a=%g b=%g c=%g" % (D, a, b, c)
        fwd = ref_prop(x, G.src, G.dst, n, s, s, a, b, hv, av, c)
        gtot = gy + c * gacc
        bwd = ref_prop(gtot, G.dst, G.src, n, s, s, a)                 # the transpose: x's row j sums its out-edges
        prop_regime(gtot, G.dst, G.src, n, s, bwd, (a, b, c), (gy, gacc))
        prop_regime(x, G.src, G.dst, n, s, fwd, (a, b, c), (hv, av))
        gh = b * gtot
        assert np.array_equal(gtot, gtot.astype(np.float32)) and np.array_equal(gh, gh.astype(np.float32))
        sum_regime(gacc * fwd["y"])
        gc = float(np.sum(gacc * fwd["y"]))
        runs = []
        for _ in range(2):
            xd, hd, ad = (_dev(v).requires_grad_(True) for v in (x, hv, av))
            cd = torch.tensor([c], dtype=torch.float32, device="cuda", requires_grad=True)
            y, ao = ops.propagate(xd, g._fwd_csr(), g._bwd_csr, _dev(s), a=a, b=b, h=hd, acc=ad, c=cd)
            torch.autograd.backward([y, ao], [_dev(gy), _dev(gacc)])
            runs.append([t.grad.detach().clone() for t in (xd, hd, ad, cd)])
        assert_bits(runs[0][0].cpu(), torch.from_numpy(bwd["y"].astype(np.float32)), tag + " g_x", G.src)
        assert_bits(runs[0][1].cpu(), torch.from_numpy(gh.astype(np.float32)), tag + " g_h", G.dst)
        assert_bits(runs[0][2].cpu(), torch.from_numpy(gacc.astype(np.float32)), tag + " g_acc", G.dst)
        assert runs[0][3].item() == gc, (tag + " g_c", runs[0][3].item(), gc)
        for name, r0, r1 in zip(("g_x", "g_h", "g_acc", "g_c"), runs[0], runs[1]):
            assert_bits(r1.cpu().reshape(r1.shape[0], -1), r0.cpu().reshape(r0.shape[0], -1),
                        tag + " second run " + name)


# ----------------------------------------------------------------------------------------------------------------
# switches read once per process: child processes
# ----------------------------------------------------------------------------------------------------------------

CHILD_TS = [str(t) for t in CUT_TS]


@pytest.mark.gpu
@pytest.mark.parametrize("T", CHILD_TS)
def test_task_size_in_child(T):
    """PGLB_STREAM_TASK = T (snapping off, rows longer than T cut into partials and a fix-up): the v5 and narrow
    forward tests and the backward again, in a child process, on a ladder whose boundary block is laid out for T."""
    if CHILD:
        pytest.skip("already the child")
    sel = "v5_exact or narrow_exact or backward_exact"
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-m", "gpu", "-k", sel,
                        "-p", "no:cacheprovider"], env=dict(os.environ, PGLB_PROP_CHILD="1", PGLB_STREAM_TASK=T),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:]
    assert " passed" in r.stdout and " failed" not in r.stdout, r.stdout[-2000:]


# ----------------------------------------------------------------------------------------------------------------
# route coverage
# ----------------------------------------------------------------------------------------------------------------

_PSIG = re.compile(r"(spmm_csr_kernel|hub_plan_kernel|spmm_narrow2_kernel|spmm_v5_prop_kernel|"
                   r"spmm_stream_fixup_prop_kernel|empty_rows_prop_kernel)(?:<([^()]*)>)?")


def _prop_sigs(fn):
    names, _ = _kernels_of(fn)
    sigs = []
    for nm in names:
        m = _PSIG.search(nm)
        if m:
            sigs.append((m.group(1), [v.strip() for v in (m.group(2) or "").split(",") if v.strip()]))
    return names, sigs


def _csr_row(vec, g, iters):
    return "csr vec%d g%d x%d" % (vec, g, iters)


def _csr_shape(D, vec4):
    """pick_shape in pgl_b200/csrc/spmm.cu: (vec, group, iters)."""
    vec = 4 if vec4 else 1
    cv = D // vec
    if cv <= 16:
        return vec, (4 if cv <= 4 else 8 if cv <= 8 else 16), 1
    return vec, 32, (1 if cv <= 32 else 2 if cv <= 64 else 4)


# every PROP instantiation the C entries can reach
TABLE_ROWS = (
    {_csr_row(v, g, i) for v in (1, 4) for g, i in ((4, 1), (8, 1), (16, 1), (32, 1), (32, 2), (32, 4))}
    | {"hub passes"}
    | {"narrow L=%d SC=%d hot=%s" % (L, sc, hot) for L in (4, 8, 16) for sc in (0, 1, 2) for hot in ("false", "true")}
    | {"v5 geo=%d D128=%s hot=%s scaled=%s" % (geo, d128, hot, sc) for geo in (0, 2)
       for d128, hot in (("false", "false"), ("true", "false"), ("true", "true")) for sc in ("false", "true")}
    | {"fixup", "empty rows"})


def _route_calls():
    """[(label, fn, claim)]: claim(sigs) -> the table rows the call reached (a set), or fails."""
    from pgl_b200 import ops
    lad, den, rect = ladder_graph(), dense_graph(), rect_graph()
    rng = np.random.default_rng(0)
    calls = []

    def xs(G, D, n=None):
        return _dev(_int_features(rng, G.n_src if n is None else n, D, torch.float32))

    def csr_claim(D, vec4, hub=False, main_only=False):
        vec, g, it = _csr_shape(D, vec4)

        def claim(sigs):
            args = ["float", "float", str(vec), str(g), str(it), "0", "0", "true"]
            hit = [a for k, a in sigs if k == "spmm_csr_kernel" and a == args]
            assert hit, "expected spmm_csr_kernel<%s>" % ", ".join(args)
            rows = {_csr_row(vec, g, it)}
            if hub:
                assert any(k == "hub_plan_kernel" for k, _ in sigs), "expected the hub plan"
                assert len(hit) >= 2, "expected hub pass 2 on the PROP kernel"
                plain = [a for k, a in sigs if k == "spmm_csr_kernel" and a[:7] == args[:7] and a[7] == "false"]
                assert plain, "expected hub pass 1 on the plain kernel"
                rows.add("hub passes")
            if main_only:
                assert len(hit) == 1 and not any(k == "hub_plan_kernel" for k, _ in sigs), "expected no hub passes"
            return rows
        return claim

    def family_claim(fam, pred, what):
        def claim(sigs):
            assert any(k == fam and pred(a) for k, a in sigs), "expected %s (%s)" % (fam, what)
            return set()
        return claim

    def narrow_claim(L, sc, hot):
        def claim(sigs):
            hit = [a for k, a in sigs if k == "spmm_narrow2_kernel" and a == [str(L), str(sc), "false", hot, "true"]]
            assert hit, "expected spmm_narrow2_kernel<%d, %d, false, %s, true>" % (L, sc, hot)
            assert any(k == "spmm_stream_fixup_prop_kernel" for k, _ in sigs), "expected the fix-up"
            assert any(k == "empty_rows_prop_kernel" for k, _ in sigs), "expected the empty-row fill"
            return {"narrow L=%d SC=%d hot=%s" % (L, sc, hot), "fixup", "empty rows"}
        return claim

    def v5_claim(geo, d128, hot, scaled):
        grp = {0: ["4", "4", "13"], 2: ["8", "3", "9"]}[geo]

        def claim(sigs):
            hit = [a for k, a in sigs if k == "spmm_v5_prop_kernel" and a == [scaled, d128, hot] + grp]
            assert hit, "expected spmm_v5_prop_kernel<%s, %s, %s, %s>" % (scaled, d128, hot, ", ".join(grp))
            assert any(k == "spmm_stream_fixup_prop_kernel" for k, _ in sigs), "expected the fix-up"
            assert any(k == "empty_rows_prop_kernel" for k, _ in sigs), "expected the empty-row fill"
            return {"v5 geo=%d D128=%s hot=%s scaled=%s" % (geo, d128, hot, scaled), "fixup", "empty rows"}
        return claim

    ns_l, ns_d = _dev(rng.choice(NORMS, lad.n_src)), _dev(rng.choice(NORMS, den.n_src))
    # node-parallel, one element per lane, and vec4 without a plan, on a graph without a row past HUB_T
    flat = PGraph("flat", O.chung_lu_edges(3000, 48000, exponent=0.5, seed=41).astype(np.int64), 3000, 3000,
                  with_graph=False)
    assert flat.deg.max() <= HUB_T
    md = int(flat.deg.max())
    for D, vec4 in ((3, False), (7, False), (9, False), (17, False), (33, False), (129, False), (16, True),
                    (32, True), (64, True)):
        x = xs(flat, D)
        calls.append(("csr D=%d" % D, lambda x=x: c_propagate(flat, x, flat.n_dst, ss=ns_d, sd=ns_d, a=-0.75,
                                                               max_degree=md),
                      csr_claim(D, vec4, main_only=True)))
    E0 = PGraph("edgeless", np.zeros((0, 2), np.int64), 300, 300, with_graph=False)
    for D in (128, 256, 512):
        x = xs(E0, D)
        calls.append(("csr vec4 edgeless D=%d" % D, lambda x=x: c_propagate(E0, x, 300, a=-0.75),
                      csr_claim(D, True, main_only=True)))
    x7 = xs(lad, 7)
    calls.append(("csr hub D=7 ladder", lambda: c_propagate(lad, x7, lad.n_dst, ss=ns_l, sd=ns_l, a=-0.75,
                                                            max_degree=int(lad.deg.max())),
                  csr_claim(7, False, hub=True)))
    x20 = xs(lad, 20)
    calls.append(("csr vec4 hub D=20 ladder", lambda: c_propagate(lad, x20, lad.n_dst, ss=ns_l, sd=ns_l, a=-0.75),
                  csr_claim(20, True, hub=True)))
    # the routes ops.propagate takes
    fwd_l = lad.g._fwd_csr()
    x129, x64l, x128l = xs(lad, 129), xs(lad, 64), xs(lad, 128)
    calls.append(("ops D=129", lambda: ops.propagate(x129, fwd_l, None, ns_l, a=-0.75), csr_claim(129, False,
                                                                                                   hub=True)))
    calls.append(("ops D=64", lambda: ops.propagate(x64l, fwd_l, None, ns_l, a=-0.75),
                  family_claim("spmm_narrow2_kernel", lambda a: a[0] == "16" and a[4] == "true", "narrow L=16")))
    calls.append(("ops D=128", lambda: ops.propagate(x128l, fwd_l, None, ns_l, a=-0.75),
                  family_claim("spmm_v5_prop_kernel", lambda a: a[:2] == ["true", "true"] and a[3] == "4",
                               "v5 geometry 0, D = 128, scaled")))
    # narrow: every L, SC and HOT
    for D, L in ((16, 4), (32, 8), (64, 16)):
        x = xs(den, D)
        plan = narrow_plan(den, ops.pack_cols(den.cols_d, den.n_src, 512, budget_bytes=1 << 20)[0])
        sl = ns_d[torch.from_numpy(den.src[np.argsort(den.dst, kind="stable")]).cuda()].contiguous()
        for sc in (0, 1, 2):
            for hot in (False, True):
                kw = {} if sc == 0 else dict(ss=ns_d, sd=ns_d, sslot=sl if sc == 2 else None)
                calls.append(("narrow D=%d SC=%d hot=%s" % (D, sc, hot),
                              lambda x=x, plan=plan, kw=kw, hot=hot: c_propagate_narrow(den, x, den.n_dst, plan,
                                                                                        a=-0.75, hints=hot, **kw),
                              narrow_claim(L, sc, "true" if hot else "false")))
    # v5: both geometries, D128, HOT, SCALED
    for G, geo, ns in ((lad, 0, ns_l), (den, 2, ns_d)):
        pk = ops.pack_cols(G.cols_d, G.n_src, 512, budget_bytes=1 << 20)[0]
        for D in (100, 128):
            x = xs(G, D)
            for scaled in (False, True):
                kw = dict(ss=ns, sd=ns) if scaled else {}
                hots = (False, True) if D == 128 else (False,)
                for hot in hots:
                    calls.append(("v5 %s D=%d scaled=%s hot=%s" % (G.name, D, scaled, hot),
                                  lambda G=G, x=x, kw=kw, hot=hot, pk=pk: c_propagate(
                                      G, x, G.n_dst, a=-0.75, packed=pk if hot else None, hints=hot, **kw),
                                  v5_claim(geo, "true" if D == 128 else "false", "true" if hot else "false",
                                           "true" if scaled else "false")))
    xr = xs(rect, 128)
    calls.append(("v5 rect", lambda: c_propagate(rect, xr, rect.n_dst, a=-0.75),
                  v5_claim(2, "true", "false", "false")))
    return calls


@pytest.mark.gpu
def test_route_coverage():
    """Each representative call reaches the kernel instantiation it claims, and together they reach every PROP
    instantiation the C entries can reach."""
    if CHILD:
        pytest.skip("routing under the default task size only")
    a = torch.ones(1024, device="cuda")
    names, _ = _kernels_of(lambda: a.add_(1))
    if not names:
        pytest.skip("torch.profiler records no CUDA kernels here (probe: a plain torch kernel)")
    hit, failures, table = set(), [], []
    for label, fn, claim in _route_calls():
        names, sigs = _prop_sigs(fn)
        try:
            rows = claim(sigs)
            hit |= rows
            table.append("%-40s %s" % (label, ", ".join(sorted(rows))))
        except AssertionError as ex:
            failures.append("%s: %s; launched %s" % (label, ex, sorted(set(names))))
    assert not failures, "\n".join(failures)
    assert TABLE_ROWS <= hit, "instantiations not reached: %s" % sorted(TABLE_ROWS - hit)
    print("\n".join(table))
    print("reached: %s" % ", ".join(sorted(hit)))
