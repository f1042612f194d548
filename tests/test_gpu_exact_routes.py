"""Every route of the send/recv aggregation, bit for bit against an exact float64 reference.

The inputs are chosen so that the result does not depend on the summation order: features are small nonzero integers
(16-bit cases: +-1), scales and edge operands are powers of two, and the sum of |terms| of every output stays below
2^24.  Every product, partial sum and sum of partials is then exact in fp32, so every route -- sequential, 32-slot
ranges, task partials plus fix-up, hub chunks -- must return the exact sum; `mean` is one correctly rounded division
(the float64 quotient rounded to fp32 is __fdiv_rn's result, since 53 >= 2 * 24 + 2); `max` / `min` are exact anyway;
a 16-bit output is the round-to-nearest-even of that fp32 value.  A dropped, doubled or misattributed slot changes
the exact value of every column it touches, whatever the row length.  `exact_regime` asserts these preconditions for
every case, so a case cannot quietly become a tolerance test.

The reference is built from the raw edge list alone (scipy products, np.bincount, reduceat over edges stably sorted by
destination); it never uses the library's CSR.  Softmax-weighted routes (fused GAT, dot attention, edge softmax) are
not exact in this sense and are tested elsewhere.

Route coverage: `test_route_coverage` records the kernels each representative call launches (torch.profiler) and
asserts that every route of the wide/narrow/generic families was reached and that each call hit the family it claims.
The task size, which the library reads once per process, runs the numeric tests again in child processes."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
CHILD = os.environ.get("PGLB_EXACT_CHILD") == "1"
EXACT_LIMIT = float(1 << 24)
REDUCES = ("sum", "mean", "max", "min")
MSG_OPS = ("add", "sub", "mul", "div")
POW2 = np.array([0.25, 0.5, 1.0, 2.0, 4.0])
# in-degrees of the row-length ladder: every boundary of the 32-slot ranges, the generic kernel's hub threshold
# (HUB_T = 1024) and its chunks, plus one row of about 30k slots
LADDER = (0, 1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1023, 1024,
          1025, 2047, 2048, 2049, 4097, 30011)
_FINITE_MAX = {torch.float32: float(np.finfo(np.float32).max), torch.bfloat16: 3.3895313892515355e38,
               torch.float16: 65504.0}


# ----------------------------------------------------------------------------------------------------------------
# float64 reference (edge list only)
# ----------------------------------------------------------------------------------------------------------------

def _rows_sorted(dst):
    """(order, row starts, row ids): edges stably sorted by destination and where each non-empty row begins."""
    order = np.argsort(dst, kind="stable")
    ds = dst[order]
    starts = np.flatnonzero(np.r_[True, ds[1:] != ds[:-1]]) if ds.size else np.zeros(0, np.int64)
    return order, starts, ds[starts] if ds.size else np.zeros(0, np.int64)


def ref_messages(msg_fn, dst, n_dst, D, reduce_op, block=256):
    """out[d] = reduce over the edges e with dst[e] == d of msg_fn(edge ids, column slice) ([k, cols] float64).
    Rows without an edge are 0.  Sums are formed by a sparse product, max / min by reduceat, in column blocks."""
    E = dst.shape[0]
    out = np.zeros((n_dst, D), np.float64)
    if E == 0 or D == 0:
        return out
    cnt = np.bincount(dst, minlength=n_dst)[:n_dst]
    order, starts, rows = _rows_sorted(dst)
    S = sp.coo_matrix((np.ones(E), (dst, np.arange(E))), shape=(n_dst, E)).tocsr()
    for c0 in range(0, D, block):
        cs = slice(c0, min(D, c0 + block))
        if reduce_op in ("sum", "mean"):
            out[:, cs] = S @ msg_fn(np.arange(E), cs)
        else:
            red = np.maximum if reduce_op == "max" else np.minimum
            out[rows, cs] = red.reduceat(msg_fn(order, cs), starts, axis=0)
    if reduce_op == "mean":
        nz = cnt > 0
        out[nz] /= cnt[nz, None]
    return out


def ref_copy(x, src, dst, n_dst, reduce_op, scale_src=None, scale_dst=None, prev=None):
    """float64 send_u_recv: out[d] = reduce_{e: dst[e] = d} x[src[e]] * scale_src[src[e]], then (+ prev, when
    accumulating a sum) * scale_dst[d].  Rows without an edge: 0, or prev * scale_dst."""
    x = np.asarray(x, np.float64)
    src = np.asarray(src, np.int64)
    dst = np.asarray(dst, np.int64)
    D = x.shape[1]
    w = np.ones(src.shape[0]) if scale_src is None else np.asarray(scale_src, np.float64)[src]
    if reduce_op in ("sum", "mean"):
        A = sp.coo_matrix((w, (dst, src)), shape=(n_dst, x.shape[0])).tocsr()
        out = A @ x if src.size else np.zeros((n_dst, D))
        if prev is not None:
            assert reduce_op == "sum"
            out = out + np.asarray(prev, np.float64)
        if reduce_op == "mean":
            cnt = np.bincount(dst, minlength=n_dst)[:n_dst]
            nz = cnt > 0
            out[nz] /= cnt[nz, None]
    else:
        # the messages are exact in fp32 (the exact regime's inputs), and max / min need no wider type
        x32, w32 = x.astype(np.float32), w.astype(np.float32)
        assert np.array_equal(x32, x) and np.array_equal(w32, w), "max / min reference needs fp32 inputs"
        out = ref_messages(lambda e, cs: x32[src[e], cs] * w32[e, None], dst, n_dst, D, reduce_op)
    if scale_dst is not None:
        out = out * np.asarray(scale_dst, np.float64)[:, None]
    return out


def _apply_msg(op, a, b):
    return {"add": np.add, "sub": np.subtract, "mul": np.multiply, "div": np.divide}[op](a, b)


def ref_ue(x, y, src, dst, n_dst, msg_op, reduce_op, head_dim=None):
    """float64 send_ue_recv with x [N, D] and y in original edge order: [E, D] (full), [E, H] (per head: head_dim
    columns each) or [E] (scalar)."""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    D = x.shape[1]

    def msg(e, cs):
        cols = np.arange(D)[cs]
        if y.ndim == 1:
            ye = y[e][:, None]
        elif y.shape[1] == D:
            ye = y[e][:, cs]
        else:
            ye = y[e][:, cols // head_dim]
        return _apply_msg(msg_op, x[src[e]][:, cs], ye)
    return ref_messages(msg, np.asarray(dst, np.int64), n_dst, D, reduce_op)


def exact_regime(abs_sum, want, dtype):
    """Assert the preconditions of a bit-exact comparison: `abs_sum` (float64, the output's shape) bounds the sum of
    |terms| of every output (|prev| included, times |scale_dst|) and must stay below 2^24; the values must be finite
    in `dtype`."""
    abs_sum = np.asarray(abs_sum, np.float64)
    assert np.isfinite(abs_sum).all() and (abs_sum.max(initial=0.0) < EXACT_LIMIT), \
        "case leaves the exact regime: sum of |terms| reaches %g >= 2^24" % abs_sum.max(initial=0.0)
    big = np.abs(np.asarray(want, np.float64)).max(initial=0.0)
    assert big <= _FINITE_MAX[dtype], "case leaves the exact regime: |output| %g overflows %s" % (big, dtype)


def exact_inputs(*arrays):
    """Assert that the inputs are what the exact regime needs: fp32 values (integers, or powers of two for scales)."""
    for a in arrays:
        if a is None:
            continue
        a = np.asarray(a, np.float64)
        assert np.array_equal(a, a.astype(np.float32).astype(np.float64)), "input not exactly representable in fp32"


def copy_case(x, src, dst, n_dst, reduce_op, dtype, scale_src=None, scale_dst=None, prev=None):
    """(expected output as a torch tensor of `dtype`, after checking the exact regime) for one send_u_recv."""
    exact_inputs(x, scale_src, scale_dst, prev)
    want = ref_copy(x, src, dst, n_dst, reduce_op, scale_src, scale_dst, prev)
    ab = ref_copy(np.abs(np.asarray(x, np.float64)), src, dst, n_dst, "sum",
                  None if scale_src is None else np.abs(scale_src), None,
                  None if prev is None else np.abs(prev))
    if scale_dst is not None:
        ab = ab * np.abs(np.asarray(scale_dst, np.float64))[:, None]
    exact_regime(ab, want, dtype)
    return to_dtype(want, dtype)


def to_dtype(want64, dtype):
    """The fp32 rounding of a float64 value, then (16-bit) round to nearest even."""
    return torch.from_numpy(np.asarray(want64, np.float64).astype(np.float32)).to(dtype)


# ----------------------------------------------------------------------------------------------------------------
# graphs
# ----------------------------------------------------------------------------------------------------------------

def ladder_edges(seed=7, num_nodes=4096):
    """(edges [E, 2], num_nodes, row degrees): destination rows with the LADDER in-degrees (shuffled), runs of empty
    rows between them and after them; sources at random with duplicates and self-loops, source 0 and the last
    source in every row of 2+ slots; the edge list shuffled so edge ids differ from CSR slots."""
    rng = np.random.default_rng(seed)
    degs = []
    for k in rng.permutation(LADDER):
        degs.append(int(k))
        degs.extend([0] * int(rng.integers(0, 4)))
    assert len(degs) < num_nodes
    degs = np.array(degs + [0] * (num_nodes - len(degs)), np.int64)
    dst = np.repeat(np.arange(num_nodes), degs)
    src = rng.integers(0, num_nodes, dst.shape[0])
    first = np.r_[0, np.cumsum(degs)[:-1]]
    for d in np.flatnonzero(degs >= 2):
        b = first[d]
        src[b], src[b + 1] = 0, num_nodes - 1
        if degs[d] >= 4:
            src[b + 2] = d                    # self-loop
            src[b + 3] = src[b + 4] if degs[d] >= 5 else src[b + 2]   # duplicate
    perm = rng.permutation(dst.shape[0])
    return np.stack([src[perm], dst[perm]], 1).astype(np.int64), num_nodes, degs


def graph_specs():
    """name -> (edges, num_nodes, out_size or None)."""
    e, n, _ = ladder_edges()
    rng = np.random.default_rng(31)
    rect = np.stack([rng.integers(0, 3000, 20000), rng.integers(0, 700, 20000)], 1)
    rect[:6000, 1] = 311                      # one 6000-slot row
    return {
        "ladder": (e, n, None),
        "chunglu": (O.chung_lu_edges(3000, 60000, exponent=0.9, seed=32), 3000, None),
        "rect": (rect.astype(np.int64), 3000, 900),   # n_dst = 900 != n_src = 3000
        "noedges": (np.zeros((0, 2), np.int64), 40, None),
    }


# ----------------------------------------------------------------------------------------------------------------
# CPU tests of the reference and of the exactness helper
# ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("reduce_op", REDUCES)
def test_reference_matches_oracle_on_random_floats(reduce_op):
    rng = np.random.default_rng(5)
    for n, E, D, out_size in ((50, 300, 5, None), (30, 400, 3, 45), (20, 1, 2, None)):
        edges = rng.integers(0, n, (E, 2))
        x = rng.standard_normal((n, D)).astype(np.float32)
        n_out = out_size or n
        want = O.send_u_recv(x, edges[:, 0], edges[:, 1], reduce_op, out_size=out_size)
        got = ref_copy(x, edges[:, 0], edges[:, 1], n_out, reduce_op)
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5)
        for op in MSG_OPS:
            y = rng.uniform(0.5, 2.0, (E, D)).astype(np.float32)
            want = O.send_ue_recv(x, y, edges[:, 0], edges[:, 1], op, reduce_op)
            np.testing.assert_allclose(ref_ue(x, y, edges[:, 0], edges[:, 1], n, op, reduce_op), want,
                                       rtol=1e-5, atol=1e-5)
            yh = y[:, :1]
            want = O.send_ue_recv(x, yh, edges[:, 0], edges[:, 1], op, reduce_op)
            np.testing.assert_allclose(ref_ue(x, yh, edges[:, 0], edges[:, 1], n, op, reduce_op, head_dim=D),
                                       want, rtol=1e-5, atol=1e-5)


def test_reference_matches_hand_computed_ladder():
    edges, n, degs = ladder_edges()
    src, dst = edges[:, 0], edges[:, 1]
    assert sorted(int(k) for k in degs if k) == sorted(k for k in LADDER if k)
    assert np.array_equal(np.bincount(dst, minlength=n), degs)
    assert (src == 0).any() and (src == n - 1).any() and (src == dst).any()
    assert len(set(map(tuple, edges.tolist()))) < len(edges)          # duplicate edges
    x = (np.arange(n, dtype=np.float64) % 17 - 8)[:, None] * np.array([1.0, -2.0])
    sums, tops, lows = {}, {}, {}
    for s, d in zip(src.tolist(), dst.tolist()):
        sums[d] = sums.get(d, 0.0) + x[s, 0]
        tops[d] = max(tops.get(d, -np.inf), x[s, 0])
        lows[d] = min(lows.get(d, np.inf), x[s, 0])
    for reduce_op in REDUCES:
        got = ref_copy(x, src, dst, n, reduce_op)
        for d in range(n):
            if degs[d] == 0:
                assert (got[d] == 0).all()
                continue
            v = {"sum": sums[d], "mean": sums[d] / degs[d], "max": tops[d], "min": lows[d]}[reduce_op]
            assert got[d, 0] == v
            if reduce_op in ("sum", "mean"):
                assert got[d, 1] == -2.0 * v
    sd = np.full(n, 0.5)
    prev = np.full((n, 2), 3.0)
    got = ref_copy(x, src, dst, n, "sum", scale_dst=sd, prev=prev)
    assert got[np.flatnonzero(degs == 0)[0], 0] == 1.5          # empty row while accumulating: prev * scale_dst
    d = int(np.argmax(degs))
    assert got[d, 0] == (sums[d] + 3.0) * 0.5


def test_exact_regime_helper_refuses_cases_outside_it():
    edges, n, degs = ladder_edges()
    src, dst = edges[:, 0], edges[:, 1]
    rng = np.random.default_rng(3)
    x = _int_features(rng, n, 4, torch.float32)
    copy_case(x, src, dst, n, "sum", torch.float32, scale_src=np.full(n, 4.0), scale_dst=np.full(n, 4.0))
    with pytest.raises(AssertionError, match="exact regime"):      # 30k slots of 2^10: above 2^24
        copy_case(np.full((n, 4), 1024.0), src, dst, n, "sum", torch.float32)
    with pytest.raises(AssertionError, match="exact regime"):      # overflows float16
        copy_case(np.full((n, 4), 8.0), src, dst, n, "sum", torch.float16)
    with pytest.raises(AssertionError, match="representable"):
        copy_case(np.full((n, 4), 0.1), src, dst, n, "sum", torch.float32)
    with pytest.raises(AssertionError, match="representable"):
        copy_case(x, src, dst, n, "sum", torch.float32, scale_src=np.full(n, 1e-50))


# ----------------------------------------------------------------------------------------------------------------
# GPU helpers
# ----------------------------------------------------------------------------------------------------------------

def _int_features(rng, n, D, dtype):
    """fp32: uniform in [-8, 8] without 0; 16-bit: +-1 (keeps hub sums small enough to survive the 16-bit rounding)."""
    if dtype == torch.float32:
        v = rng.integers(1, 9, (n, D)) * rng.choice([-1, 1], (n, D))
    else:
        v = rng.choice([-1, 1], (n, D))
    return v.astype(np.float64)


def _pow2(rng, n, choices=POW2):
    return rng.choice(choices, n)


def _dev(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float64))).to(dtype).cuda()


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16).numpy()


def assert_bits(got, want, what, dst=None):
    """Bit equality; on failure name the first differing row, its in-degree and column."""
    assert tuple(got.shape) == tuple(want.shape), (what, tuple(got.shape), tuple(want.shape))
    assert got.dtype == want.dtype, (what, got.dtype, want.dtype)
    gb, wb = _bits(got).reshape(got.shape[0], -1), _bits(want).reshape(want.shape[0], -1)
    bad = np.argwhere(gb != wb)
    if bad.size:
        r, c = (int(v) for v in bad[0])
        deg = int(np.sum(np.asarray(dst) == r)) if dst is not None else -1
        g = got.reshape(got.shape[0], -1)[r, c].item()
        w = want.reshape(want.shape[0], -1)[r, c].item()
        rows = np.unique(bad[:, 0])
        pytest.fail("%s: %d elements differ in %d rows; first at row %d (in-degree %d) column %d: got %r, want %r"
                    % (what, bad.shape[0], rows.size, r, deg, c, g, w))


_GRAPHS = {}


def _graph(name):
    """(Graph on cuda, src, dst, num_nodes, n_out), built once per process."""
    if name not in _GRAPHS:
        import pgl_b200 as pgl
        edges, n, out_size = graph_specs()[name]
        g = pgl.Graph(edges=edges, num_nodes=n)
        g.tensor()
        _GRAPHS[name] = (g, edges[:, 0].copy(), edges[:, 1].copy(), n, out_size or n)
    return _GRAPHS[name]


def _csr(g, n_out):
    return g._csr_for_rows(n_out)


def _packings(ops, cols, n_src):
    """name -> (packed ids, has_hints): no, few, mixed and all rows marked hot."""
    packs = {name: tuple(ops.pack_cols(cols, n_src, 512, budget_bytes=b))
             for name, b in (("none", 0), ("few", 8 * 512), ("mixed", 1 << 20))}
    packs["all"] = (cols.to(torch.int32) | -(1 << 31), True)
    return packs


F32_WIDTHS = [1, 3, 4, 5, 8, 9, 16, 17, 20, 32, 33, 36, 64, 65, 68, 100, 124, 128, 129, 132, 256, 257, 260, 512, 513,
              516, 1024, 1433, 2052]
X16_WIDTHS = [(torch.bfloat16, d) for d in (1, 3, 4, 5, 8, 9, 16, 17, 32, 33, 64, 65, 68, 72, 120, 128, 129, 132,
                                            257, 513, 516, 1024, 1433)] + \
             [(torch.float16, d) for d in (17, 72, 128, 132, 516)]
if CHILD:                                         # the widths of the kernels that cut rows into tasks
    F32_WIDTHS = [36, 128, 260, 1024]
    X16_WIDTHS = [(torch.bfloat16, 128)]
V5_F32 = (68, 100, 124, 128)
V5_X16 = (72, 120, 128)
COPY_CASES = [(torch.float32, d) for d in F32_WIDTHS] + X16_WIDTHS
GRAPH_NAMES = ("ladder", "chunglu", "rect", "noedges")


def _run_copy_matrix(dtype, D, graph_names=None):
    """Every copy-message variant at one width on every graph (rows wider than 600 columns: the ladder, whose hub and
    cut rows are what they test, and the graph without edges); returns the number of comparisons."""
    from pgl_b200 import ops
    if graph_names is None:
        graph_names = GRAPH_NAMES if D <= 600 and not CHILD else ("ladder", "noedges") if D > 600 else \
            ("ladder", "chunglu")
    n_cmp = 0
    half = dtype != torch.float32
    for gname in graph_names:
        g, src, dst, n, n_out = _graph(gname)
        fwd = _csr(g, n_out)
        rng = np.random.default_rng(1000 * D + len(gname))
        x = _int_features(rng, n, D, dtype)
        xd = _dev(x, dtype)
        scale_choices = POW2 if dtype != torch.float16 else POW2[:4]
        ss, sd = _pow2(rng, n, scale_choices), _pow2(rng, n_out, scale_choices)
        ss_d, sd_d = _dev(ss), _dev(sd)
        for reduce_op in REDUCES:
            tag = "%s D=%d %s %s" % (dtype, D, gname, reduce_op)
            want = copy_case(x, src, dst, n_out, reduce_op, dtype)
            out_size = n_out if n_out != n else None
            assert_bits(g.send_recv(xd, reduce_op, out_size=out_size).cpu(), want, tag, dst)
            # the node-parallel kernel: no packed ids / narrow plan, no degree hint
            assert_bits(ops._spmm_raw(fwd["indptr"], fwd["cols"], xd, n_out, reduce_op, max_degree=-1).cpu(), want,
                        tag + " generic", dst)
            want = copy_case(x, src, dst, n_out, reduce_op, dtype, scale_src=ss, scale_dst=sd)
            # first sighting of the scale gathers it per edge, the second streams the per-slot copy
            for sighting in ("gathered", "streamed"):
                got = g._send_u_recv(xd, reduce_op, out_size, scale_src=ss_d, scale_dst=sd_d)
                assert_bits(got.cpu(), want, "%s scaled (%s norms)" % (tag, sighting), dst)
            n_cmp += 5
            if reduce_op == "sum" and not half:
                prev = _int_features(rng, n_out, D, torch.float32)
                want = copy_case(x, src, dst, n_out, "sum", dtype, scale_src=ss, scale_dst=sd, prev=prev)
                for packed in (ops._packed_of(fwd, xd), None):
                    out = _dev(prev)
                    ops._spmm_raw(fwd["indptr"], fwd["cols"], xd, n_out, "sum", scale_src=ss_d, scale_dst=sd_d,
                                  max_degree=fwd["max_degree"], out=out, packed=packed, accumulate=True)
                    assert_bits(out.cpu(), want, tag + " accumulate packed=%s" % (packed is not None), dst)
                    n_cmp += 1
            if reduce_op in ("sum", "mean") and fwd["cols"] is not None and int(fwd["cols"].shape[0]) > 0 and \
                    D in (V5_X16 if half else V5_F32):
                want_s = copy_case(x, src, dst, n_out, reduce_op, dtype, scale_src=ss, scale_dst=sd)
                want_p = copy_case(x, src, dst, n_out, reduce_op, dtype)
                for pname, pk in _packings(ops, fwd["cols"], n).items():
                    got = ops._spmm_raw(fwd["indptr"], fwd["cols"], xd, n_out, reduce_op, packed=pk,
                                        max_degree=fwd["max_degree"])
                    assert_bits(got.cpu(), want_p, "%s packing=%s" % (tag, pname), dst)
                    got = ops._spmm_raw(fwd["indptr"], fwd["cols"], xd, n_out, reduce_op, scale_src=ss_d,
                                        scale_dst=sd_d, packed=ops.PackedCols(pk, fwd["slot_scale"]),
                                        max_degree=fwd["max_degree"])
                    assert_bits(got.cpu(), want_s, "%s packing=%s scaled" % (tag, pname), dst)
                    n_cmp += 2
    return n_cmp


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,D", COPY_CASES, ids=["%s-%d" % (str(t).split(".")[-1], d) for t, d in COPY_CASES])
def test_copy_exact(dtype, D):
    assert _run_copy_matrix(dtype, D) > 0


UE_CASES = [(d, b) for d in (33, 64, 128, 256) for b in ("full", "head", "scalar")]


@pytest.mark.gpu
@pytest.mark.parametrize("D,bcast", UE_CASES, ids=["%d-%s" % c for c in UE_CASES])
def test_ue_exact(D, bcast):
    """send_ue_recv, fp32: every message op and reduction, y different on every edge (a wrong edge-id mapping
    shows)."""
    H = 4 if D % 4 == 0 else 3
    hd = D // H
    for gname in ("ladder", "chunglu", "rect") if D < 256 else ("ladder", "rect"):
        g, src, dst, n, n_out = _graph(gname)
        rng = np.random.default_rng(D + 7 * len(gname))
        E = src.shape[0]
        x = _int_features(rng, n, D, torch.float32)
        yshape = {"full": (E, D), "head": (E, H), "scalar": (E,)}[bcast]
        y = rng.choice([-4.0, -2.0, -1.0, -0.5, 0.5, 1.0, 2.0, 4.0], yshape)
        xd = _dev(x)
        if bcast == "head":
            xin, yin = xd.reshape(n, H, hd), _dev(y).reshape(E, H, 1)
        else:
            xin, yin = xd, _dev(y)
        out_size = n_out if n_out != n else None
        for op in MSG_OPS:
            ab = ref_ue(np.abs(x), np.abs(y), src, dst, n_out, op if op in ("mul", "div") else "add", "sum",
                        head_dim=hd)
            for reduce_op in REDUCES:
                want64 = ref_ue(x, y, src, dst, n_out, op, reduce_op, head_dim=hd)
                exact_regime(ab, want64, torch.float32)
                got = g.send_ue_recv(xin, yin, op, reduce_op, out_size=out_size).reshape(n_out, D)
                assert_bits(got.cpu(), to_dtype(want64, torch.float32),
                            "send_ue_recv D=%d %s %s %s %s" % (D, bcast, gname, op, reduce_op), dst)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_ue_x16_exact(dtype):
    """pglb_spmm_csr_ue_x16: 16-bit x, fp32 per-head or scalar y, mul / add messages, sum."""
    from pgl_b200 import ops
    for gname in ("ladder", "chunglu"):
        g, src, dst, n, n_out = _graph(gname)
        fwd = _csr(g, n_out)
        E = src.shape[0]
        rng = np.random.default_rng(77)
        for D, H in ((64, 8), (128, 4), (128, 1), (36, 3)):
            x = _int_features(rng, n, D, dtype)
            xd = _dev(x, dtype)
            for scalar in (False, True):
                y = rng.choice([-2.0, -1.0, -0.5, 0.5, 1.0, 2.0], (E,) if scalar else (E, H))
                y2 = _dev(y).reshape(E, -1)
                for op in ("mul", "add"):
                    want64 = ref_ue(x, y, src, dst, n_out, op, "sum", head_dim=D // H)
                    ab = ref_ue(np.abs(x), np.abs(y), src, dst, n_out, "mul" if op == "mul" else "add", "sum",
                                head_dim=D // H)
                    exact_regime(ab, want64, dtype)
                    got = ops._spmm_raw(fwd["indptr"], fwd["cols"], xd, n_out, "sum", eid=fwd["eid"], y2=y2,
                                        y_bcast=ops.BCAST_SCALAR if scalar else ops.BCAST_HEAD, head_dim=D // H,
                                        msg_op=op, max_degree=fwd["max_degree"])
                    assert_bits(got.cpu(), to_dtype(want64, dtype),
                                "ue_x16 %s D=%d H=%d scalar=%s %s %s" % (dtype, D, H, scalar, gname, op), dst)


SEG_CASES = [(torch.float32, d) for d in (17, 48, 68, 128, 256, 516)] + \
            [(torch.bfloat16, d) for d in (72, 128, 516)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,D", SEG_CASES, ids=["%s-%d" % (str(t).split(".")[-1], d) for t, d in SEG_CASES])
def test_segment_exact(dtype, D):
    """pgl.math.segment_*: identity columns (slot j reads row j), segments of ladder lengths with empty ones between."""
    import pgl_b200 as pgl
    rng = np.random.default_rng(D)
    lens = []
    for k in rng.permutation(LADDER):
        lens.append(int(k))
        lens.extend([0] * int(rng.integers(0, 3)))
    while lens[-1] == 0:
        lens.pop()
    ids = np.repeat(np.arange(len(lens)), lens)
    E = ids.shape[0]
    data = _int_features(rng, E, D, dtype)
    dd, idd = _dev(data, dtype), torch.from_numpy(ids).cuda()
    for reduce_op in REDUCES:
        want = copy_case(data, np.arange(E), ids, len(lens), reduce_op, dtype)
        got = getattr(pgl.math, "segment_" + reduce_op)(dd, idd)
        assert_bits(got.cpu(), want, "segment_%s %s D=%d" % (reduce_op, dtype, D), ids)


# ----------------------------------------------------------------------------------------------------------------
# layouts: column windows, poisoned rows and columns, misaligned bases, output windows with a canary
# ----------------------------------------------------------------------------------------------------------------

_POISON = {"sum": float("nan"), "mean": float("nan"), "max": float(1 << 20), "min": -float(1 << 20)}
_CANARY32 = 0x7FA5A5A5
_CANARY16 = 0x7FA5

LAYOUT_CASES = [(torch.float32, d) for d in (4, 16, 17, 36, 64, 68, 128, 132, 260, 1024)] + \
               [(torch.bfloat16, d) for d in (17, 72, 128, 132)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,D", LAYOUT_CASES, ids=["%s-%d" % (str(t).split(".")[-1], d) for t, d in LAYOUT_CASES])
def test_layouts_exact(dtype, D):
    """x as a column window of a wider buffer (ldx > D) whose other columns and extra rows past n_src are poisoned;
    out as a window of a canary-filled buffer (ldo > D) that must stay intact outside [n_dst, D]; both bases offset
    by one element (no vector loads)."""
    from pgl_b200 import ops
    for gname in ("ladder", "rect"):
        g, src, dst, n, n_out = _graph(gname)
        fwd = _csr(g, n_out)
        rng = np.random.default_rng(D + 3)
        x = _int_features(rng, n, D, dtype)
        ss, sd = _pow2(rng, n), _pow2(rng, n_out)
        ss_d, sd_d = _dev(ss), _dev(sd)
        extra, lpad, W = 5, 4, D + 12
        for reduce_op in REDUCES:
            tag = "%s D=%d %s %s" % (dtype, D, gname, reduce_op)
            want = copy_case(x, src, dst, n_out, reduce_op, dtype, scale_src=ss, scale_dst=sd)
            xb = torch.full((n + extra, W), _POISON[reduce_op], dtype=dtype, device="cuda")
            xb[:n, lpad:lpad + D] = _dev(x, dtype)
            xw = xb[:, lpad:lpad + D]
            canary = _CANARY32 if dtype == torch.float32 else _CANARY16
            ob = torch.full((n_out + 3, W), canary, dtype=torch.int32 if dtype == torch.float32 else torch.int16,
                            device="cuda").view(dtype)
            before = _bits(ob).copy()
            ow = ob[1:n_out + 1, lpad:lpad + D]
            ops._spmm_raw(fwd["indptr"], fwd["cols"], xw, n_out, reduce_op, scale_src=ss_d, scale_dst=sd_d,
                          max_degree=fwd["max_degree"], out=ow, packed=ops._packed_of(fwd, xw))
            assert_bits(ow.cpu(), want, tag + " windowed", dst)
            after = _bits(ob)
            keep = np.ones(after.shape, bool)
            keep[1:n_out + 1, lpad:lpad + D] = False
            assert np.array_equal(after[keep], before[keep]), tag + ": wrote outside the output window"
            # bases one element past a 16-byte boundary: the scalar paths
            xo = torch.empty(n * D + 1, dtype=dtype, device="cuda")[1:].view(n, D)
            xo.copy_(_dev(x, dtype))
            oo = torch.empty(n_out * D + 1, dtype=dtype, device="cuda")[1:].view(n_out, D)
            ops._spmm_raw(fwd["indptr"], fwd["cols"], xo, n_out, reduce_op, scale_src=ss_d, scale_dst=sd_d,
                          max_degree=fwd["max_degree"], out=oo, packed=ops._packed_of(fwd, xo))
            assert_bits(oo.cpu(), want, tag + " misaligned", dst)


@pytest.mark.gpu
@pytest.mark.parametrize("dim,chunks", [(200, 3), (130, 2)])
def test_host_aggregator_column_blocks_exact(dim, chunks):
    """HostAggregator's column blocks: dim 200 in 3 blocks of 68 / 68 / 64 columns read with ldx = 200 (wide and
    narrow kernels), dim 130 in 2 blocks (ldx % 4 != 0: the scalar node-parallel kernel)."""
    g, src, dst, n, _ = _graph("chunglu")
    rng = np.random.default_rng(dim)
    x = _int_features(rng, n, dim, torch.float32)
    ss, sd = _pow2(rng, n), _pow2(rng, n)
    xh = torch.from_numpy(x.astype(np.float32)).pin_memory()
    for reduce_op in ("sum", "mean", "max"):
        for scaled in (False, True):
            kw = dict(scale_src=_dev(ss), scale_dst=_dev(sd)) if scaled else {}
            want = copy_case(x, src, dst, n, reduce_op, torch.float32,
                             **(dict(scale_src=ss, scale_dst=sd) if scaled else {}))
            oh = torch.empty((n, dim), dtype=torch.float32).pin_memory()
            got = g.send_recv_host(xh, oh, reduce_op, chunks=chunks, **kw)
            assert_bits(got, want, "host aggregator dim=%d %s scaled=%s" % (dim, reduce_op, scaled), dst)


def _queue_order(run, ntasks):
    """'ascending' or 'descending': the order in which spmm_v5_kernel's device-side queue handed out the tasks of the
    one launch `run` makes, read from the per-task start times of pglb_debug_task_trace.  With several waves of tasks
    per resident warp the tasks handed out first start first."""
    from pgl_b200 import ops
    from pgl_b200._lib import check, lib
    buf = torch.zeros((ntasks, 4), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    check(lib.pglb_debug_task_trace(ops._ptr(buf), ntasks))
    try:
        run()
        torch.cuda.synchronize()
    finally:
        check(lib.pglb_debug_task_trace(None, 0))
    start = buf[:, 0].cpu().numpy()
    assert (start > 0).all(), "%d of %d tasks not traced" % (int((start <= 0).sum()), ntasks)
    k = ntasks // 8
    return "ascending" if np.median(start[:k]) < np.median(start[-k:]) else "descending"


@pytest.mark.gpu
def test_v5_queue_orders_exact():
    """At 64 slots per task: a graph of 3 tasks per resident warp takes spmm_v5_kernel's descending queue and one of
    more than 8 takes the ascending queue (dyn_mode in csrc/spmm_stream.cu).  Both orders, read from the task trace,
    give the exact sums, means and scaled sums of rows cut into many tasks."""
    if os.environ.get("PGLB_STREAM_TASK") != "64":
        pytest.skip("runs in the PGLB_STREAM_TASK=64 child")
    import pgl_b200 as pgl
    T, n = 64, 100_000
    resident_warps = torch.cuda.get_device_properties(0).multi_processor_count * 2 * 13
    for order, tasks in (("descending", 3 * resident_warps), ("ascending", 9 * resident_warps)):
        edges = O.chung_lu_edges(n, tasks * T, exponent=0.8, seed=tasks)
        src, dst = edges[:, 0], edges[:, 1]
        g = pgl.Graph(edges=edges, num_nodes=n)
        g.tensor()
        rng = np.random.default_rng(tasks)
        ss, sd = _pow2(rng, n), _pow2(rng, n)
        ss_d, sd_d = _dev(ss), _dev(sd)
        for dtype, D, reduce_op, scaled in ((torch.float32, 128, "sum", True), (torch.float32, 100, "mean", False),
                                            (torch.bfloat16, 128, "sum", False)):
            x = _int_features(rng, n, D, dtype)
            xd = _dev(x, dtype)
            kw = dict(scale_src=ss_d, scale_dst=sd_d) if scaled else {}
            want = copy_case(x, src, dst, n, reduce_op, dtype, **(dict(scale_src=ss, scale_dst=sd) if scaled else {}))
            tag = "%s queue, %d tasks: %s D=%d %s scaled=%s" % (order, tasks, dtype, D, reduce_op, scaled)
            got = {}
            seen = _queue_order(lambda: got.setdefault("out", g._send_u_recv(xd, reduce_op, None, **kw)), tasks)
            assert seen == order, "%s: the trace shows the %s order" % (tag, seen)
            assert_bits(got["out"].cpu(), want, tag, dst)


# ----------------------------------------------------------------------------------------------------------------
# backward
# ----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("D", [20, 128, 129])
def test_sum_backward_exact(D):
    g, src, dst, n, _ = _graph("ladder")
    rng = np.random.default_rng(D)
    x = _int_features(rng, n, D, torch.float32)
    go = rng.integers(-4, 5, (n, D)).astype(np.float64)
    xd = _dev(x).requires_grad_(True)
    g.send_recv(xd, "sum").backward(_dev(go))
    want = copy_case(go, dst, src, n, "sum", torch.float32)           # the transpose: x's row s sums its out-edges
    assert_bits(xd.grad.cpu(), want, "sum backward D=%d" % D, src)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [20, 128])
def test_mean_backward_bound(D):
    """grad x[s] = sum over out-edges of g[d] / deg(d): 1 / deg is not exact, so the bar is (k + 1) 2^-24 sum|terms|
    per element (k = out-degree of s)."""
    g, src, dst, n, _ = _graph("ladder")
    rng = np.random.default_rng(D + 1)
    x = _int_features(rng, n, D, torch.float32)
    go = rng.integers(-4, 5, (n, D)).astype(np.float64)
    xd = _dev(x).requires_grad_(True)
    g.send_recv(xd, "mean").backward(_dev(go))
    cnt = np.bincount(dst, minlength=n).astype(np.float64)
    inv = np.where(cnt > 0, 1.0 / np.maximum(cnt, 1), 0.0)
    want = ref_copy(go, dst, src, n, "sum", scale_src=inv)
    ab = ref_copy(np.abs(go), dst, src, n, "sum", scale_src=inv)
    k = np.bincount(src, minlength=n).astype(np.float64)[:, None]
    err = np.abs(xd.grad.cpu().numpy().astype(np.float64) - want)
    bound = (k + 1) * 2.0 ** -24 * ab
    bad = np.argwhere(err > bound)
    assert bad.size == 0, "mean backward: %d elements over the bound, first at %s" % (bad.shape[0], bad[0])


def _maxmin_grad_ref(x, out, go, src, dst, n_rows):
    """Every source entry equal to the reduced value receives the full gradient of that output (documented tie
    rule): grad[s, c] = sum over edges s -> d of go[d, c] * (x[s, c] == out[d, c])."""
    gx = np.zeros((n_rows, x.shape[1]), np.float64)
    np.add.at(gx, src, go[dst] * (x[src] == out[dst]))
    return gx


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("reduce_op", ["max", "min"])
@pytest.mark.parametrize("D", [24, 128])
def test_maxmin_backward_ties_exact(dtype, reduce_op, D):
    """Integer features make ties between distinct sources common, hub rows included."""
    for gname in ("ladder", "chunglu"):
        g, src, dst, n, _ = _graph(gname)
        rng = np.random.default_rng(D + 11)
        x = rng.choice([-2.0, -1.0, 1.0, 2.0], (n, D))
        go = rng.integers(-4, 5, (n, D)).astype(np.float64)
        xd = _dev(x, dtype).requires_grad_(True)
        out = g.send_recv(xd, reduce_op)
        out.backward(_dev(go, dtype))
        out64 = ref_copy(x, src, dst, n, reduce_op)
        assert_bits(out.detach().cpu(), to_dtype(out64, dtype), "%s forward %s" % (reduce_op, gname), dst)
        want = _maxmin_grad_ref(x, out64, go, src, dst, n)
        ties = np.zeros_like(out64)
        np.add.at(ties, dst, x[src] == out64[dst])
        deg = np.bincount(dst, minlength=n)
        assert (ties[deg >= 64] >= 2).all()                            # every output of a long row is a tie
        assert_bits(xd.grad.cpu(), to_dtype(want, dtype), "%s backward %s %s" % (reduce_op, dtype, gname), src)


@pytest.mark.gpu
@pytest.mark.parametrize("reduce_op", ["max", "min"])
def test_maxmin_backward_with_more_feature_rows_than_nodes(reduce_op):
    """Feature rows past the graph's nodes are never gathered: their gradient is zero."""
    g, src, dst, n, _ = _graph("chunglu")
    extra = 37
    rng = np.random.default_rng(9)
    x = rng.choice([-2.0, -1.0, 1.0, 2.0], (n + extra, 16))
    go = rng.integers(-4, 5, (n + extra, 16)).astype(np.float64)
    xd = _dev(x).requires_grad_(True)
    out = g.send_recv(xd, reduce_op)
    assert out.shape[0] == n + extra
    out.backward(_dev(go))
    out64 = ref_copy(x, src, dst, n + extra, reduce_op)
    want = _maxmin_grad_ref(x, out64, go, src, dst, n + extra)
    assert not want[n:].any()
    assert_bits(xd.grad.cpu(), to_dtype(want, torch.float32), "%s backward, extra rows" % reduce_op, src)


# ----------------------------------------------------------------------------------------------------------------
# feature matrices over 4 GiB
# ----------------------------------------------------------------------------------------------------------------

def _big_value(rows, cols):
    """x[i, c] of the over-4-GiB case: depends on the row id, and a row 2^23 below (where a 32-bit wrap of the byte
    offset of a 512-byte row lands) holds different values."""
    return (((rows[:, None] * 7 + cols[None, :]) % 127) - 63).astype(np.float64)


@pytest.mark.gpu
def test_feature_matrix_over_4gib_exact():
    """x of 9M x 128 fp32 (4.6 GB, under 2^31 elements) with sources mostly past the 4 GiB mark: v5 (sum, scaled),
    stream128 (max) and narrow (a D = 64 column window, ldx = 128).  A wrapped 32-bit offset stays inside the
    allocation, so a bug shows as wrong rows."""
    from pgl_b200 import ops
    N, D, n_dst, E = 9_000_000, 128, 1000, 300_000
    free = torch.cuda.mem_get_info()[0]
    if free < 12 * (1 << 30):
        pytest.skip("needs about 12 GB of free device memory, %.1f GB free (shared device)" % (free / 2 ** 30))
    rng = np.random.default_rng(4)
    wrap = (1 << 32) // (D * 4)
    src = np.where(rng.random(E) < 0.9, rng.integers(wrap, N, E), rng.integers(0, N, E))
    dst = np.sort(rng.integers(0, n_dst, E))
    src[:3] = [0, N - 1, wrap]
    order = np.argsort(dst, kind="stable")
    src, dst = src[order], dst[order]
    indptr = np.r_[0, np.cumsum(np.bincount(dst, minlength=n_dst))]
    x = torch.empty((N, D), dtype=torch.float32, device="cuda")
    step = 1 << 18
    cols_t = torch.arange(D, device="cuda", dtype=torch.int64)
    for r0 in range(0, N, step):
        r = torch.arange(r0, min(N, r0 + step), device="cuda", dtype=torch.int64)
        x[r0:r0 + r.shape[0]] = (((r[:, None] * 7 + cols_t[None, :]) % 127) - 63).to(torch.float32)
    uniq, inv = np.unique(src, return_inverse=True)
    xs = _big_value(uniq, np.arange(D))                               # only the gathered rows, on the host
    ss = rng.choice(POW2, N).astype(np.float32)
    ip_d, cols_d = torch.from_numpy(indptr).cuda(), torch.from_numpy(src).cuda()
    try:
        want = copy_case(xs, inv, dst, n_dst, "sum", torch.float32, scale_src=ss[uniq])
        got = ops._spmm_raw(ip_d, cols_d, x, n_dst, "sum", scale_src=_dev(ss))
        assert_bits(got.cpu(), want, "over 4 GiB: v5 sum scaled", dst)
        want = copy_case(xs, inv, dst, n_dst, "max", torch.float32)
        got = ops._spmm_raw(ip_d, cols_d, x, n_dst, "max")
        assert_bits(got.cpu(), want, "over 4 GiB: stream128 max", dst)
        xw = x[:, :64]
        plan = ops.NarrowPlan(*ops.narrow_plan(ip_d, cols_d, N, 256))
        want = copy_case(xs[:, :64], inv, dst, n_dst, "sum", torch.float32)
        got = ops._spmm_raw(ip_d, cols_d, xw, n_dst, "sum", packed=plan)
        assert_bits(got.cpu(), want, "over 4 GiB: narrow sum, ldx = 128", dst)
    finally:
        del x
        torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------------------------
# switches read once per process: child processes
# ----------------------------------------------------------------------------------------------------------------

# 32: one column batch per task; 64: every row longer than 64 slots cut; 160: 20 groups of 8 slots per full task, not
# a multiple of either ring's 3 or 4 groups; 1024: the snap limit, so the ladder's 1024-slot row stays whole and its
# 1025-slot row is cut; 2048: the default's largest task
CHILD_ENVS = [{"PGLB_STREAM_TASK": t} for t in ("64", "2048", "32", "160", "1024")]


@pytest.mark.gpu
@pytest.mark.parametrize("env", CHILD_ENVS, ids=["%s=%s" % next(iter(e.items())) for e in CHILD_ENVS])
def test_per_process_switches_in_child(env):
    """Pinned task sizes (rows longer than T cut, partials + fix-up; at T = 64 both queue orders of spmm_v5_kernel): the
    numeric tests again, in a child process with the switch set."""
    if CHILD:
        pytest.skip("already the child")
    sel = "copy_exact or (ue_exact and 128-head) or v5_queue_orders"
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-m", "gpu", "-k", sel,
                        "-p", "no:cacheprovider"], env=dict(os.environ, PGLB_EXACT_CHILD="1", **env),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:]


# ----------------------------------------------------------------------------------------------------------------
# route coverage
# ----------------------------------------------------------------------------------------------------------------

_SIG = re.compile(r"(spmm_csr_capped_kernel|spmm_csr_kernel|hub_plan_kernel|spmm_narrow2_kernel|spmm_v5_kernel|"
                  r"spmm_stream128_kernel|spmm_stream_kernel)(?:<([^()]*)>)?")


def _kernels_of(fn):
    """[(kernel family, [template arguments])] of the CUDA kernels fn launches."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    sigs = []
    for nm in names:
        m = _SIG.search(nm)
        if m:
            sigs.append((m.group(1), [a.strip() for a in (m.group(2) or "").split(",") if a.strip()]))
    return names, sigs


def _route_calls():
    """(label, call, claim): claim(sigs) -> the table rows the call must reach (a set), or fails."""
    import pgl_b200 as pgl
    from pgl_b200 import ops
    calls = []
    lad, _, _, n_l, _ = _graph("ladder")
    cl, _, _, n_c, _ = _graph("chunglu")
    f_l, f_c = lad._fwd_csr(), cl._fwd_csr()
    rng = np.random.default_rng(0)

    def x_of(n, D, dtype=torch.float32):
        return _dev(_int_features(rng, n, D, dtype), dtype)

    def generic(vec, g, iters, ti="float", capped=False, mode="0", hub=True):
        def claim(sigs):
            fam = "spmm_csr_capped_kernel" if capped else "spmm_csr_kernel"
            hit = [a for k, a in sigs if k == fam and a[:2] == [ti, ti] and a[2:5] == [str(vec), str(g), str(iters)]
                   and (capped or a[5] == mode)]
            assert hit, "expected %s<%s, %d, %d, %d>" % (fam, ti, vec, g, iters)
            assert not hub or any(k == "hub_plan_kernel" for k, _ in sigs), "expected the hub passes"
            rows = {"generic%s vec%d" % ("16" if ti != "float" else "32", vec)}
            if capped:
                rows.add("generic16 capped")
            if mode == "1" and ti != "float":
                rows.add("ue_x16")
            if hub:
                rows.add("generic hub passes")
            return rows
        return claim

    def family(fam, pred, row):
        def claim(sigs):
            hit = [a for k, a in sigs if k == fam and pred(a)]
            assert hit, "expected %s (%s)" % (fam, row)
            return {row}
        return claim

    xs = {D: x_of(n_l, D) for D in (17, 64, 1433, 256, 260, 1024)}
    calls.append(("f32 D=17 scalar", lambda: lad.send_recv(xs[17], "sum"), generic(1, 32, 1)))
    calls.append(("f32 D=1433 scalar, 12 tiles", lambda: lad.send_recv(xs[1433], "mean"), generic(1, 32, 4)))
    calls.append(("f32 D=64 vec4", lambda: ops._spmm_raw(f_l["indptr"], f_l["cols"], xs[64], n_l, "sum"),
                  generic(4, 16, 1)))
    calls.append(("f32 D=64 max", lambda: lad.send_recv(xs[64], "max"), generic(4, 16, 1)))
    xb = {D: x_of(n_l, D, torch.bfloat16) for D in (17, 132, 516, 1024, 128)}
    calls.append(("bf16 D=17", lambda: lad.send_recv(xb[17], "sum"), generic(1, 32, 1, ti="__nv_bfloat16")))
    calls.append(("bf16 D=132 capped", lambda: lad.send_recv(xb[132], "sum"),
                  generic(4, 32, 2, ti="__nv_bfloat16", capped=True)))
    calls.append(("bf16 D=516, 2 tiles", lambda: lad.send_recv(xb[516], "mean"), generic(4, 32, 4, ti="__nv_bfloat16")))
    calls.append(("bf16 D=1024, 2 tiles", lambda: lad.send_recv(xb[1024], "max"), generic(4, 32, 4, ti="__nv_bfloat16")))
    E_l = int(f_l["cols"].shape[0])
    yh = _dev(rng.choice([0.5, 2.0], (E_l, 4)))
    calls.append(("ue_x16 D=128", lambda: ops._spmm_raw(f_l["indptr"], f_l["cols"], xb[128], n_l, "sum",
                                                        eid=f_l["eid"], y2=yh, y_bcast=ops.BCAST_HEAD, head_dim=32,
                                                        msg_op="mul"),
                  generic(4, 32, 1, ti="__nv_bfloat16", mode="1")))
    for D, lanes in ((16, "4"), (20, "8"), (36, "16")):
        xn = x_of(n_c, D)
        calls.append(("narrow D=%d" % D, lambda xn=xn: cl.send_recv(xn, "sum"),
                      family("spmm_narrow2_kernel", lambda a, lanes=lanes: a[0] == lanes, "narrow lanes=" + lanes)))
    norm_c = _dev(_pow2(rng, n_c))

    def v5_claim(dtype, d128, hot, scaled, geo):
        grp = {0: ("4", "4", "13"), 2: ("8", "3", "9")}[geo]
        ti = "float" if dtype == torch.float32 else "__nv_bfloat16"

        def pred(a):
            return a[0] == ti and a[1:4] == [scaled, d128, hot] and tuple(a[4:7]) == grp
        return family("spmm_v5_kernel", pred, "v5 %s D128=%s hot=%s scaled=%s geo=%d" %
                      ("32" if ti == "float" else "16", d128, hot, scaled, geo))

    x128c, x100l = x_of(n_c, 128), x_of(n_l, 100)
    pk_mixed = tuple(ops.pack_cols(f_c["cols"], n_c, 512, budget_bytes=1 << 20))
    calls.append(("v5 D=128 hot", lambda: ops._spmm_raw(f_c["indptr"], f_c["cols"], x128c, n_c, "sum",
                                                        packed=pk_mixed),
                  v5_claim(torch.float32, "true", "true", "false", 2)))
    calls.append(("v5 D=128 scaled", lambda: cl._send_u_recv(x128c, "sum", None, scale_src=norm_c, scale_dst=norm_c),
                  v5_claim(torch.float32, "true", "false", "true", 2)))
    calls.append(("v5 D=100 ladder", lambda: lad.send_recv(x100l, "mean"),
                  v5_claim(torch.float32, "false", "false", "false", 0)))
    xb72 = x_of(n_c, 72, torch.bfloat16)
    calls.append(("v5 bf16 D=72", lambda: cl.send_recv(xb72, "sum"),
                  v5_claim(torch.bfloat16, "false", "false", "false", 2)))
    calls.append(("v5 bf16 D=128 ladder", lambda: lad.send_recv(xb[128], "sum"),
                  v5_claim(torch.bfloat16, "true", "false", "false", 0)))
    x128l = x_of(n_l, 128)
    calls.append(("stream128 max", lambda: lad.send_recv(x128l, "max"),
                  family("spmm_stream128_kernel", lambda a: a[0] == "1" and a[3] == "0", "stream128 max/min")))
    seg_ids = torch.from_numpy(np.repeat(np.arange(40), np.arange(40) * 3)).cuda()
    seg_x = x_of(int(seg_ids.shape[0]), 100)
    calls.append(("stream128 identity columns", lambda: pgl.math.segment_sum(seg_x, seg_ids),
                  family("spmm_stream128_kernel", lambda a: a[2] == "0" and a[3] == "0", "stream128 identity")))
    ye = _dev(rng.choice([0.5, 2.0], (E_l, 4))).reshape(E_l, 4, 1)
    calls.append(("stream128 edge operand", lambda: lad.send_ue_recv(x128l.reshape(n_l, 4, 32), ye, "mul", "sum"),
                  family("spmm_stream128_kernel", lambda a: a[3] == "1", "stream128 edge operand")))
    for D, iters, rk, red in ((256, "2", "0", "sum"), (260, "4", "1", "max"), (1024, "4", "0", "mean")):
        calls.append(("stream D=%d %s" % (D, red), lambda D=D, red=red: lad.send_recv(xs[D], red),
                      family("spmm_stream_kernel", lambda a, iters=iters, rk=rk: a == [iters, rk],
                             "stream<%s> rk=%s%s" % (iters, rk, ", >1 tiles" if D > 128 * int(iters) else ""))))
    return calls


TABLE_ROWS = {
    "generic32 vec1", "generic32 vec4", "generic16 vec1", "generic16 vec4", "generic16 capped", "generic hub passes",
    "ue_x16", "narrow lanes=4", "narrow lanes=8", "narrow lanes=16",
    "v5 32 D128=true hot=true scaled=false geo=2", "v5 32 D128=true hot=false scaled=true geo=2",
    "v5 32 D128=false hot=false scaled=false geo=0", "v5 16 D128=false hot=false scaled=false geo=2",
    "v5 16 D128=true hot=false scaled=false geo=0",
    "stream128 max/min", "stream128 identity", "stream128 edge operand",
    "stream<2> rk=0", "stream<4> rk=1", "stream<4> rk=0, >1 tiles",
}


@pytest.mark.gpu
def test_route_coverage():
    """Each representative call reaches the kernel family it claims, and together they reach every route."""
    if CHILD:
        pytest.skip("routing under the default switches only")
    a = torch.ones(1024, device="cuda")
    names, _ = _kernels_of(lambda: a.add_(1))
    if not names:
        pytest.skip("torch.profiler records no CUDA kernels here (probe: a plain torch kernel)")
    hit, failures = set(), []
    for label, fn, claim in _route_calls():
        names, sigs = _kernels_of(fn)
        try:
            hit |= claim(sigs)
        except AssertionError as ex:
            failures.append("%s: %s; launched %s" % (label, ex, sorted(set(names))))
    assert not failures, "\n".join(failures)
    assert TABLE_ROWS <= hit, "routes not reached: %s" % sorted(TABLE_ROWS - hit)
    print("routes reached: %s" % ", ".join(sorted(hit)))
