"""Every softmax-weighted route, bit for bit against an exact float64 reference on 0/1 attention weights.

The regime.  Scores are chosen so that, for every (row, head), they take two values: every selected slot scores
exactly sigma (the same bits), every masked slot scores the same value, at most sigma - 150.  Every route subtracts
the running maximum before it exponentiates (gat5's __expf(lg - m_run) and __expf(m_run - m_new), edge_ops'
expf(v - m), expf(m_i - M) in both fix-ups and in the readout merge), so every exponential is of 0 -- exactly 1 -- or of
at most -150 -- exactly 0 in fp32.  With small integer features (+-1 for 16-bit) whose selected sum stays below 2^24:
  - l = c and acc = A exactly, c the number of selected slots and A the sum of their feature rows, in any order and
    across any task cut;
  - out = fl(A / c) where the row is finished by a division (__fdiv_rn: both fix-ups, the per-slot kernel, the readout)
    and fl(A * fl(1 / c)) where gat5's row epilogue finishes it (__frcp_rn); with dropout A counts the kept selected
    slots and the quotient is multiplied by s once more; a 16-bit output is that fp32 value rounded to nearest even;
  - lse is within ulp(ln c) + ulp(lse) / 2 of sigma + ln c (logf is within 1 ulp), and equals sigma when c = 1;
  - stored-logit softmax (edge_softmax): alpha is fl(1 / c) on selected slots and 0 on masked ones.
A dropped, doubled or misattributed selected slot changes A or c, whatever the row length; a merge that gives a masked
partial weight 1, or a running max that forgets m_run, gives inf / NaN or counts masked slots.  `weights_regime`
asserts these preconditions on the scores of every case (computed in fp32 exactly as the kernels form them), so a
case cannot quietly become a tolerance test.

Which rows a task boundary cuts (and so which finish by the fix-up's division) follows from the library's task size and
`task_plan` (tests/test_task_model.py); the graphs carry rows cut exactly at task starts and ends, after a snapped
short row, and (when snapping is off) rows cut into exactly one head and one tail, and the tests assert that these
exist under the task size the library picks.

Backward: the edge-softmax backward, sddmm and the GATv2 score gradient are exact on power-of-two weights and integer
gradients.  The per-edge entries (GAT, dot attention, GATv2 with grad_attn; f32, x16, dropout) and the readout
backward run on a regime forward: masked edges must give exactly 0, selected ones must lie within a per-element bound
derived from the kernels' operations (`weight_bound`, `edge_grad_bound`), smaller than what one misattributed edge
changes.

The task size (PGLB_STREAM_TASK, read once per process, which also turns snapping off) runs the forward tests again in
child processes.  `test_route_coverage` records the
kernels each representative call launches (torch.profiler) and asserts that every softmax kernel, forward and
backward, was reached, and that every fused GAT case ran on the kernel family it claims."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import oracle as O
from oracle import oracle_pool as OP
from test_gpu_exact_routes import _kernels_of, assert_bits, to_dtype
from test_task_model import task_plan

CHILD = os.environ.get("PGLB_SOFTMAX_CHILD") == "1"
GAP = 150.0                     # masked scores sit at least this far below sigma: exp underflows to exactly 0
EXACT_LIMIT = float(1 << 24)
KINDS = ("prefix", "suffix", "alt", "first", "last", "middle", "all", "none", "odd")
# in-degrees of the row-length ladder: gat5's quads, 8-slot groups and ring of 3 groups, a warp's 32 slots, the edge
# softmax hub threshold (SM_HUB_T = 256), the snap (1024), the readout-sized rows and one row of about 30k slots
LADDER = tuple(range(0, 10)) + (15, 16, 17, 23, 24, 25, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025, 2047, 2048,
                                 2049, 4097, 30011)
HMAX, CMAX = 40, 4              # heads and score columns the mask patterns are drawn for
SEED = (1234, 8)                # attention-dropout stream: (seed, offset)
P_DROP = 0.375


# ----------------------------------------------------------------------------------------------------------------
# float64 references
# ----------------------------------------------------------------------------------------------------------------

def _row_of_slot(indptr):
    return np.repeat(np.arange(indptr.shape[0] - 1), np.diff(indptr))


def _reduceat(v, indptr, ufunc=np.add, empty=0.0):
    """ufunc over the slots of every row of v [E, ...]; rows without a slot get `empty`."""
    n = indptr.shape[0] - 1
    out = np.full((n,) + v.shape[1:], empty, np.float64)
    nz = np.flatnonzero(np.diff(indptr) > 0)
    if nz.size:
        out[nz] = ufunc.reduceat(v, indptr[nz], axis=0)
    return out


def ref_softmax(scores, indptr):
    """float64 softmax over the slots of every row: (alpha [E, H], lse [n, H], -inf on empty rows)."""
    s = np.asarray(scores, np.float64)
    row = _row_of_slot(indptr)
    m = _reduceat(s, indptr, np.maximum, -np.inf)
    e = np.exp(s - m[row])
    z = _reduceat(e, indptr)
    with np.errstate(divide="ignore"):
        lse = m + np.log(z)
    return e / z[row], lse


def ref_attend(alpha, feat_slots, indptr):
    """out[d, h, :] = sum over the slots j of row d of alpha[j, h] feat_slots[j, h, :] (float64)."""
    return _reduceat(np.asarray(alpha, np.float64)[:, :, None] * feat_slots, indptr)


def lrelu32(x, slope):
    """The kernels' LeakyReLU on fp32 values: x >= 0 ? x : fl(x * slope)."""
    x = np.asarray(x, np.float32)
    return np.where(x >= 0, x, x * np.float32(slope)).astype(np.float32)


def weights_regime(scores, indptr, allow_neg_inf=False):
    """Assert that fp32 `scores` [E, H] (CSR slot order) are in the 0/1-weight regime and return (sel [E, H] bool,
    sigma [n, H] float64 (NaN on empty rows), c [n, H] selected slots per row): for every (row, head) the selected
    slots score exactly sigma = the row's maximum, and the others one common value at most sigma - 150 (-inf allowed
    only with allow_neg_inf, and never for every slot of a row)."""
    s = np.asarray(scores, np.float32).astype(np.float64)
    assert not np.isnan(s).any(), "case leaves the 0/1-weight regime: a NaN score"
    assert not np.isposinf(s).any(), "case leaves the 0/1-weight regime: a +inf score"
    assert allow_neg_inf or np.isfinite(s).all(), "case leaves the 0/1-weight regime: a -inf score"
    row = _row_of_slot(indptr)
    sig = _reduceat(s, indptr, np.maximum, np.nan)
    deg = np.diff(indptr)
    assert np.isfinite(sig[deg > 0]).all(), "case leaves the 0/1-weight regime: a row whose every score is -inf"
    sel = s == sig[row]
    lo = _reduceat(np.where(sel, np.inf, s), indptr, np.minimum, np.inf)
    hi = _reduceat(np.where(sel, -np.inf, s), indptr, np.maximum, -np.inf)
    has = _reduceat((~sel).astype(np.float64), indptr) > 0
    assert (lo[has] == hi[has]).all(), "case leaves the 0/1-weight regime: masked slots of a row score differently"
    assert (hi[has] <= sig[has] - GAP).all(), \
        "case leaves the 0/1-weight regime: a masked score within %g of the row's maximum" % GAP
    c = _reduceat(sel.astype(np.float64), indptr)
    return sel, sig, c


def expected_attention(sel, feat_slots, indptr, rcp_rows=None, keep=None, drop_scale=None, dtype=torch.float32):
    """(out [n, H * Dh] in `dtype`, c [n, H]) of a softmax-weighted aggregation in the 0/1-weight regime:
    A = sum of the kept selected feature rows, c = number of selected slots, out = fl(A / c), or fl(A * fl(1 / c)) on
    the rows of rcp_rows (gat5's row epilogue), times fl32 drop_scale once more with dropout; 0 on empty rows."""
    f = np.asarray(feat_slots, np.float64)
    assert np.array_equal(f, np.round(f)), "case leaves the exact regime: features must be integers"
    w = sel if keep is None else (sel & keep)
    A = ref_attend(w, f, indptr)
    ab = ref_attend(sel, np.abs(f), indptr)
    assert ab.max(initial=0.0) < EXACT_LIMIT, "case leaves the exact regime: sum of |features| reaches 2^24"
    c = _reduceat(sel.astype(np.float64), indptr)
    cc = np.maximum(c, 1.0)[:, :, None]
    out = (A / cc).astype(np.float32)
    if rcp_rows is not None and np.any(rcp_rows):
        r = (1.0 / cc[rcp_rows]).astype(np.float32).astype(np.float64)
        out[rcp_rows] = (A[rcp_rows] * r).astype(np.float32)
    if drop_scale is not None:
        out = (out.astype(np.float64) * np.float64(np.float32(drop_scale))).astype(np.float32)
    out[np.diff(indptr) == 0] = 0.0
    return to_dtype(out.reshape(out.shape[0], -1), dtype), c


def check_lse(got, sig, c, what, empty_value=np.nan):
    """lse within ulp(ln c) + ulp(lse) / 2 of sigma + ln c (bitwise sigma where c = 1); empty rows hold
    `empty_value` (NaN: untouched prefill)."""
    got = np.asarray(got, np.float32).reshape(sig.shape)
    ne = c > 0
    if np.isnan(empty_value):
        assert np.isnan(got[~ne]).all(), "%s: lse written on a row without slots" % what
    else:
        assert (got[~ne] == empty_value).all(), "%s: lse of an empty row is not %r" % (what, empty_value)
    ln = np.log(np.where(ne, c, 1.0))
    want = sig + ln
    tol = np.spacing(np.abs(ln).astype(np.float32)).astype(np.float64) + \
        np.spacing(np.abs(want).astype(np.float32)).astype(np.float64) / 2
    err = np.abs(got.astype(np.float64) - want)
    bad = np.argwhere(ne & ~(err <= tol))
    assert bad.size == 0, "%s: lse of %d (row, head) off; first %s: got %r, want %r (c = %d)" % (
        what, bad.shape[0], tuple(bad[0]), float(got[tuple(bad[0])]), want[tuple(bad[0])], c[tuple(bad[0])])
    one = ne & (c == 1)
    assert (got[one] == sig[one].astype(np.float32)).all(), "%s: lse of a one-slot row is not sigma" % what


# ----------------------------------------------------------------------------------------------------------------
# task plan: which rows a task boundary cuts
# ----------------------------------------------------------------------------------------------------------------

def lib_task_size(E, sm_count, env_T=0):
    """(T, snap) of the fused-attention family: gat_task_size / stream_snap in pgl_b200/csrc/spmm_stream.cu."""
    if env_T:
        return env_T, env_T
    target = sm_count * 28 * 4
    t = min(max((E // target + 31) // 32 * 32, 32), 2048)
    t = max(32, (t // 2 + 31) // 32 * 32)
    return t, (t if t > 1024 else 1024)


def cut_rows(indptr, T, snap):
    """bool [n]: rows with a task start strictly inside them (finished by the fix-up), and the plan's starts."""
    n = indptr.shape[0] - 1
    E = int(indptr[-1])
    if E == 0:
        return np.zeros(n, bool), np.zeros(1, np.int64)
    ntasks, _, start = task_plan(indptr, n, E, T, snap)
    inner = start[1:ntasks]
    lo = np.searchsorted(inner, indptr[:-1], side="right")
    hi = np.searchsorted(inner, indptr[1:], side="left")
    return hi > lo, start


def boundary_degrees(pos, T, snap):
    """Degrees to append at slot `pos` (with the tags of the rows they make): a cut row starting exactly on a task
    boundary, one ending exactly on one, a short row straddling a boundary followed by a cut row, and -- when rows
    longer than T may be cut (snap == T) -- a row cut into exactly one head and one tail."""
    degs, tags = [], []

    def add(k, tag=None):
        nonlocal pos
        degs.append(k)
        tags.append(tag)
        pos += k
        degs.append(0)
        tags.append(None)

    def pad_to(mod):
        m = (mod - pos) % T
        if m:
            add(m)
    pad_to(0)
    add(max(snap, T) + 7, "starts_on_boundary")
    long2 = max(snap, T) + 9
    pad_to((-long2) % T)
    add(long2, "ends_on_boundary")
    pad_to(T - 3)
    add(6, "straddling_short")
    add(max(snap, T) + 11, "after_straddling")
    if snap < 2 * T - 1:
        pad_to(T - 1)
        add(T + 1, "one_head_one_tail")
    return degs, tags


def check_boundary_cases(indptr, tags, T, snap):
    """Assert that every tagged case exists under (T, snap)."""
    cut, start = cut_rows(indptr, T, snap)
    starts = set(int(v) for v in start)
    found = set()
    for r, tag in tags.items():
        b, e = int(indptr[r]), int(indptr[r + 1])
        inner = [s for s in starts if b < s < e]
        if tag == "starts_on_boundary":
            assert cut[r] and b in starts, (tag, b, T)
        elif tag == "ends_on_boundary":
            assert cut[r] and e in starts | {int(indptr[-1])} and e % T == 0, (tag, e, T)
        elif tag == "straddling_short":
            assert not cut[r] and b // T != (e - 1) // T and e <= snap + b, (tag, b, e, T)
        elif tag == "after_straddling":
            assert cut[r] and indptr[r - 2] + 6 == b, (tag, b)     # r - 2: the short row, then an empty one
        elif tag == "one_head_one_tail":
            assert cut[r] and len(inner) == 1, (tag, b, e, inner)
        found.add(tag)
    want = {"starts_on_boundary", "ends_on_boundary", "straddling_short", "after_straddling"}
    if snap < 2 * T - 1:
        want.add("one_head_one_tail")
    assert want <= found, sorted(want - found)
    return cut


# ----------------------------------------------------------------------------------------------------------------
# graphs: rows with mask patterns, sources carrying the score bits
# ----------------------------------------------------------------------------------------------------------------

def pattern(kind, deg, rng):
    """bool [deg]: which slots of one (row, head) are selected."""
    k = np.arange(deg)
    if deg == 0:
        return np.zeros(0, bool)
    cut = int(rng.integers(1, deg)) if deg >= 2 else 1
    return {
        "prefix": k >= cut if deg >= 2 else k >= 0,        # masked prefix, then selected
        "suffix": k < cut,                                  # selected, then masked
        "alt": (k % 2) == int(rng.integers(0, 2)) if deg >= 2 else k >= 0,
        "first": k == 0,
        "last": k == deg - 1,
        "middle": k == deg // 2,
        "all": k >= 0,
        "none": k >= 0,                                     # every slot at the low value: all selected, sigma lower
        "odd": np.isin(k, rng.choice(deg, min(deg, int(rng.choice([3, 5, 7]))), replace=False)),
    }[kind]


class RegimeGraph(object):
    """Rows 0..R-1 with the given in-degrees; every slot's source is a node >= R whose score bits (per head and score
    column) select it or not in that row, so the scores of the routes follow the per-(row, head) patterns.  Slots of
    one row with the same bits share a source at random (duplicate edges).  Edge ids are a random permutation, ascending
    inside every row, so the library's CSR has exactly these slots in this order while edge ids differ from slots.
      indptr [N + 1] (rows >= R empty), cols [E] (sources), eid [E] (slot -> edge id), edges [E, 2] (edge order),
      want [E, HMAX] selection intent, none [R, HMAX] whether the (row, head) uses the low score everywhere,
      col [R, HMAX] the score column of each (row, head), bits [N, HMAX, CMAX] the nodes' score bits."""

    def __init__(self, degs, seed):
        rng = np.random.default_rng(seed)
        degs = np.asarray(degs, np.int64)
        self.R = R = degs.shape[0]
        E = int(degs.sum())
        self.E = E
        self.col = rng.integers(0, CMAX, (R, HMAX))
        want = np.zeros((E, HMAX), bool)
        self.none = np.zeros((R, HMAX), bool)
        first = np.r_[0, np.cumsum(degs)]
        for d in range(R):
            k = int(degs[d])
            if not k:
                continue
            for h in range(HMAX):
                kind = KINDS[(3 * d + 5 * h + int(rng.integers(0, 2))) % len(KINDS)] if k < 1000 else \
                    KINDS[(d + h) % len(KINDS)]
                want[first[d]:first[d + 1], h] = pattern(kind, k, rng)
                self.none[d, h] = kind == "none"
        self.want = want
        # sources: one node per slot, or an earlier slot's node of the same row with the same requirement
        cols = np.empty(E, np.int64)
        node_req = []   # (owner row, first slot) of every source node
        for d in range(R):
            seen = {}
            for j in range(first[d], first[d + 1]):
                key = want[j].tobytes()
                if key in seen and rng.random() < 0.5:
                    cols[j] = seen[key]
                    continue
                node = R + len(node_req)
                node_req.append((d, j))
                seen[key] = node
                cols[j] = node
        self.N = N = R + len(node_req)
        bits = rng.random((N, HMAX, CMAX)) < 0.5
        bits[:R] = True
        self.node_row = np.r_[np.arange(R), [d for d, _ in node_req]].astype(np.int64)
        for i, (d, j) in enumerate(node_req):
            bits[R + i, np.arange(HMAX), self.col[d]] = want[j] ^ self.none[d]   # 'none': every source low
        self.bits = bits
        self.cols = cols
        self.indptr = np.r_[first, np.full(N - R, E)].astype(np.int64)
        perm = rng.permutation(E)
        eid = np.empty(E, np.int64)
        for d in range(R):
            eid[first[d]:first[d + 1]] = np.sort(perm[first[d]:first[d + 1]])
        self.eid = eid
        edges = np.empty((E, 2), np.int64)
        edges[eid, 0] = cols
        edges[eid, 1] = np.repeat(np.arange(R), degs)
        self.edges = edges

    def indptr_rows(self, n_rows):
        return self.indptr[:n_rows + 1]

    def eff(self, H):
        """bool [N, H]: each node's score bit in the column its owner row reads (rows themselves: high)."""
        return self.bits[np.arange(self.N)[:, None], np.arange(H)[None, :], self.col[self.node_row][:, :H]]


def ladder_degrees(seed, T, snap):
    """(degrees, tags): the LADDER shuffled with runs of empty rows between, then the task-boundary block."""
    rng = np.random.default_rng(seed)
    degs = []
    for k in rng.permutation(LADDER):
        degs.append(int(k))
        degs.extend([0] * int(rng.integers(0, 3)))
    bd, bt = boundary_degrees(int(sum(degs)), T, snap)
    tags = {len(degs) + i: t for i, t in enumerate(bt) if t}
    return degs + bd + [0, 0], tags


# ----------------------------------------------------------------------------------------------------------------
# scores of each route, in fp32 exactly as the kernels form them
# ----------------------------------------------------------------------------------------------------------------

GAT_B = 1000.0       # attn_src of a masked source sits this far below a selected one
DOT_B = 256.0        # k of a masked source in the score column
V2_HI, V2_LO = 96.0, -256.0


def gat_inputs(G, H, rng):
    """(attn_src [N, H], attn_dst [N, H]) float32: attn_src 0 (selected) or -GAT_B by the node's bit, attn_dst
    sigma in [150, 190) per (row, head) ('none' rows: every source at the low value)."""
    a_s = np.where(G.eff(H), 0.0, -GAT_B).astype(np.float32)
    a_d = np.zeros((G.N, H), np.float32)
    a_d[:G.R] = 150 + rng.integers(0, 40, (G.R, H))
    return a_s, a_d


def gat_scores(G, a_s, a_d, slope, n_rows):
    row = _row_of_slot(G.indptr_rows(n_rows))
    return lrelu32(a_s[G.cols] + a_d[row], slope)


def dot_inputs(G, H, Dh, rng):
    """(q, k) float64 [N, H * Dh]: q one-hot (1.0) at column col[d, h] of every head of row d; k at columns < CMAX
    4 c or 4 c - DOT_B by the node's bit, other columns small integers (multiplied by q's zeros)."""
    cm = min(CMAX, Dh)
    q = np.zeros((G.N, H, Dh))
    q[np.arange(G.R)[:, None], np.arange(H)[None, :], G.col[:, :H] % cm] = 1.0
    k = rng.integers(-3, 4, (G.N, H, Dh)).astype(np.float64)
    sig = 4.0 * np.arange(cm)
    k[:, :, :cm] = np.where(G.bits[:, :H, :cm], sig, sig - DOT_B)
    return q.reshape(G.N, -1), k.reshape(G.N, -1)


def dot_scores(G, q, k, H, n_rows):
    row = _row_of_slot(G.indptr_rows(n_rows))
    s = (q[row].reshape(-1, H, q.shape[1] // H) * k[G.cols].reshape(-1, H, k.shape[1] // H)).sum(-1)
    assert np.array_equal(s, s.astype(np.float32)), "dot score not exact in fp32"
    return s.astype(np.float32)


def v2_inputs(G, H, Dh, rng, half):
    """(f float64 [N, H * Dh], a float32 [H * Dh]): a = 1 at column 0 of every head, 0 elsewhere; f's column 0 of
    every head is the score column (V2_HI selected / V2_LO masked; rows: V2_HI), the others small integers."""
    f = _features(rng, G.N, H * Dh, half).reshape(G.N, H, Dh)
    f[:, :, 0] = np.where(G.eff(H), V2_HI, V2_LO)
    a = np.zeros((H, Dh), np.float32)
    a[:, 0] = 1.0
    return f.reshape(G.N, -1), a.reshape(-1)


def v2_scores(G, f, a, H, slope, n_rows):
    row = _row_of_slot(G.indptr_rows(n_rows))
    z = (f[G.cols].astype(np.float32) + f[row].astype(np.float32)).astype(np.float32)
    terms = a.astype(np.float64) * lrelu32(z, slope).astype(np.float64)
    s = terms.reshape(-1, H, terms.shape[1] // H).sum(-1)
    assert np.array_equal(s, s.astype(np.float32)), "GATv2 score not exact in fp32"
    return s.astype(np.float32)


def _features(rng, n, D, half):
    if half:
        return rng.choice([-1.0, 1.0], (n, D))
    return (rng.integers(1, 9, (n, D)) * rng.choice([-1, 1], (n, D))).astype(np.float64)


# ----------------------------------------------------------------------------------------------------------------
# CPU tests: the reference against the oracle, the regime helper, the task-boundary cases
# ----------------------------------------------------------------------------------------------------------------

def test_reference_matches_oracle_on_random_floats():
    rng = np.random.default_rng(3)
    for n, E, H, Dh in ((40, 300, 3, 4), (25, 500, 1, 2), (60, 80, 8, 3)):
        edges = rng.integers(0, n, (E, 2))
        edges[:7, 1] = 5
        lg = rng.standard_normal((E, H)).astype(np.float32) * 3
        deg, _, _, se, ip = O.adj_dst_index(edges, n)
        alpha, lse = ref_softmax(lg[se], ip)
        want = O.edge_softmax(edges, n, lg, "dst")
        np.testing.assert_allclose(alpha, want[se], rtol=1e-5, atol=1e-6)
        x = rng.standard_normal((n, H, Dh)).astype(np.float32)
        out = ref_attend(alpha, x[edges[se, 0]], ip)
        w3 = O.send_ue_recv(x, want.reshape(E, H, 1), edges[:, 0], edges[:, 1], "mul", "sum")
        np.testing.assert_allclose(out, w3, rtol=1e-5, atol=1e-5)
        for d in np.flatnonzero(deg)[:5]:
            s = lg[edges[:, 1] == d].astype(np.float64)
            np.testing.assert_allclose(lse[d], np.log(np.exp(s).sum(0)), rtol=1e-12)
        assert np.isneginf(lse[deg == 0]).all()
    # the readout: one segment's softmax over its rows, gate given
    x = rng.standard_normal((30, 5)).astype(np.float32)
    gate = rng.standard_normal(30).astype(np.float32)
    ip = np.array([0, 10, 10, 30])
    alpha, _ = ref_softmax(gate[:, None], ip)
    got = ref_attend(alpha, x[:, None, :], ip)[:, 0]
    want = OP.attn_readout(x, ip, gate=gate, indptr=True)
    want = want[0] if isinstance(want, tuple) else want
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-6)


def test_regime_matches_reference_and_rounding_choice():
    """In the regime the float64 softmax reference gives alpha in {0, 1 / c} and out = A / c; the two roundings of the
    quotient differ somewhere (so the route choice is observable)."""
    rng = np.random.default_rng(4)
    G = RegimeGraph([3, 0, 5, 7, 1, 40, 0], seed=5)
    a_s, a_d = gat_inputs(G, 4, rng)
    sc = gat_scores(G, a_s, a_d, 0.2, G.N)
    sel, sig, c = weights_regime(sc, G.indptr)
    alpha, lse = ref_softmax(sc, G.indptr)
    row = _row_of_slot(G.indptr)
    # e^-150 and below: under fp32's least denormal
    np.testing.assert_allclose(alpha, np.where(sel, 1.0 / np.maximum(c, 1)[row], 0.0), rtol=1e-15, atol=1e-60)
    ne = c > 0
    np.testing.assert_allclose(lse[ne], (sig + np.log(np.where(ne, c, 1)))[ne], rtol=1e-15)
    f = _features(rng, G.N, 4 * 8, False)
    fs = f[G.cols].reshape(-1, 4, 8)
    out, _ = expected_attention(sel, fs, G.indptr)
    np.testing.assert_allclose(out.numpy().reshape(G.N, 4, 8), ref_attend(alpha, fs, G.indptr), rtol=1e-7,
                               atol=1e-12)
    A = np.arange(1, 200, dtype=np.float64)
    assert any(np.float32(a / 3) != np.float32(a * np.float64(np.float32(1 / 3))) for a in A) or \
        any(np.float32(a / 7) != np.float32(a * np.float64(np.float32(1 / 7))) for a in A)


def test_weights_regime_refuses_cases_outside_it():
    ip = np.array([0, 3, 3, 5])
    ok = np.array([[5.0], [5.0], [-200.0], [1.0], [-300.0]], np.float32)
    sel, sig, c = weights_regime(ok, ip)
    assert sel[:, 0].tolist() == [True, True, False, True, False] and c[:, 0].tolist() == [2, 0, 1]
    assert np.isnan(sig[1, 0])
    for bad, msg in (([5.0, 5.0, -100.0, 1.0, -300.0], "within"),           # gap below 150
                     ([5.0, -200.0, -201.0, 1.0, -300.0], "differently"),    # two masked values in a row
                     ([5.0] + [np.nextafter(np.float32(5), np.float32(0))] * 2 + [1.0, -300.0], "within"),
                     ([5.0, 5.0, np.nan, 1.0, -300.0], "NaN"),
                     ([5.0, 5.0, np.inf, 1.0, -300.0], "inf"),
                     ([5.0, 5.0, -np.inf, 1.0, -300.0], "-inf")):
        with pytest.raises(AssertionError, match=msg):
            weights_regime(np.array(bad, np.float32)[:, None], ip)
    weights_regime(np.array([5.0, 5.0, -np.inf, 1.0, -np.inf], np.float32)[:, None], ip, allow_neg_inf=True)
    with pytest.raises(AssertionError, match="every score is -inf"):
        weights_regime(np.array([5.0, 5.0, -np.inf, -np.inf, -np.inf], np.float32)[:, None], ip, allow_neg_inf=True)
    # features: integers whose selected sum stays below 2^24
    sel = np.ones((5, 1), bool)
    expected_attention(sel, np.full((5, 1, 2), 3.0), ip)
    with pytest.raises(AssertionError, match="integers"):
        expected_attention(sel, np.full((5, 1, 2), 0.5), ip)
    with pytest.raises(AssertionError, match="2\\^24"):
        expected_attention(sel, np.full((5, 1, 2), 2.0 ** 23), ip)


@pytest.mark.parametrize("T,snap", [(32, 1024), (32, 32), (64, 64), (2048, 2048), (64, 1024)])
def test_task_boundary_cases_exist(T, snap):
    """The ladder's task-boundary block under fixed task sizes: every case is where it is meant to be, and the
    model's plan cuts exactly the rows longer than snap that a boundary crosses."""
    degs, tags = ladder_degrees(11, T, snap)
    ip = np.r_[0, np.cumsum(degs)].astype(np.int64)
    cut = check_boundary_cases(ip, tags, T, snap)
    deg = np.diff(ip)
    assert not cut[deg <= snap].any()
    crosses = (ip[:-1] // T) != ((ip[1:] - 1) // T)
    assert np.array_equal(cut, crosses & (deg > snap))
    if snap >= 1024:
        assert cut[deg == 30011].all() and not cut[deg == 1024].any()


def test_default_task_size_is_the_boundary_block_s():
    """The library's default fused task size on graphs of the ladder's size is 32 slots for any H100 SM count, which
    is what the default graph's block is laid out for."""
    degs, _ = ladder_degrees(11, 32, 1024)
    E = int(sum(degs))
    for sms in (114, 132):
        assert lib_task_size(E, sms) == (32, 1024)
    assert lib_task_size(10_000_000, 132) == (352, 1024)
    assert lib_task_size(1 << 30, 132) == (1024, 1024) and lib_task_size(50_000, 132, 2048) == (2048, 2048)


# ----------------------------------------------------------------------------------------------------------------
# GPU helpers
# ----------------------------------------------------------------------------------------------------------------

def _env_T():
    v = os.environ.get("PGLB_STREAM_TASK")
    try:
        v = int(v)
    except (TypeError, ValueError):
        return 0
    return v if v >= 32 and v % 32 == 0 else 0


_G = {}


def ladder():
    """(RegimeGraph, cut rows of the fused family, T, snap) for this process's task size."""
    if "ladder" not in _G:
        env = _env_T()
        T, snap = (env, env) if env else (32, 1024)
        degs, tags = ladder_degrees(11, T, snap)
        G = RegimeGraph(degs, seed=12)
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert lib_task_size(G.E, sms, env) == (T, snap), "the boundary block is laid out for another task size"
        cut = check_boundary_cases(G.indptr, tags, T, snap)
        _G["ladder"] = (G, cut, T, snap)
    return _G["ladder"]


def _dev(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float64))).to(dtype).cuda()


def _i64(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.int64)).cuda()


def _ws(n, E, D):
    from pgl_b200 import ops
    need = ctypes.c_size_t(0)
    ops.check(ops.lib.pglb_spmm_csr_ws(n, E, D, ctypes.byref(need)))
    return torch.empty(max(need.value, 16), dtype=torch.uint8, device="cuda")


def keep_mask(E, H, p=P_DROP, seed=SEED):
    """bool [E, H] keep bits of dst-CSR slot j from the library's host function."""
    from pgl_b200 import _lib
    w = np.zeros(max(E, 1), np.uint32)
    _lib.check(_lib.lib.pglb_attn_dropout_keep_host(seed[0], seed[1], p, 0, E, H, w.ctypes.data_as(ctypes.c_void_p)))
    return ((w[:E, None] >> np.arange(H, dtype=np.uint32)) & 1).astype(bool)


def drop_scale(p=P_DROP):
    return float(np.float32(1.0 / (1.0 - float(np.float32(p)))))


def _dt(dtype):
    from pgl_b200 import ops
    return () if dtype == torch.float32 else (ops._DTYPE16[dtype],)


def _nan(shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _call(name, *args):
    from pgl_b200 import ops
    with torch.cuda.device(0):
        ops.check(getattr(ops.lib, name)(*args))


def run_gat(G, n_dst, f, a_s, a_d, slope, H, Dh, dtype, mode, misalign=False):
    """One fused-GAT entry ('infer', 'train' or 'drop') on the ladder's first n_dst rows: (out, lse or None)."""
    from pgl_b200 import ops
    P = ops._ptr
    ip, cols = _i64(G.indptr_rows(n_dst)), _i64(G.cols)
    fd = _dev(f, dtype)
    a_sd = _dev(a_s)
    if misalign:
        buf = torch.empty(a_s.size + 1, device="cuda")
        a_sd = buf[1:].view(a_s.shape)
        a_sd.copy_(_dev(a_s))
    a_dd = _dev(a_d[:n_dst])
    D = H * Dh
    out = _nan((n_dst, D), dtype)
    lse = _nan((n_dst, H)) if mode != "infer" else None
    ws = _ws(n_dst, G.E, D)
    base = "pglb_gat_fused_%scsr_%s" % ("" if mode == "infer" else ("train_drop_" if mode == "drop" else "train_"),
                                       "f32" if dtype == torch.float32 else "x16")
    args = [P(ip), P(cols), P(fd), fd.stride(0), P(a_sd), P(a_dd), float(slope), P(out), out.stride(0)]
    if lse is not None:
        args.append(P(lse))
    args += [n_dst, G.N, G.E, H, Dh, *_dt(dtype)]
    if mode == "drop":
        args += [P_DROP, SEED[0], SEED[1]]
    args += [P(ws), ws.numel(), ops._stream()]
    _call(base, *args)
    return out, lse


def run_scored(kind, G, tensors, H, Dh, dtype, drop, slope=0.0, n_dst=None):
    """pglb_dot_attn_* (tensors = q, k, v; on the ladder's first n_dst rows, default all) or pglb_gatv2_attn_*
    (tensors = f, a; one node set, so square) on the ladder: (out, lse)."""
    from pgl_b200 import ops
    P = ops._ptr
    n_dst = G.N if n_dst is None else n_dst
    ip, cols = _i64(G.indptr_rows(n_dst)), _i64(G.cols)
    D = H * Dh
    out = _nan((n_dst, D), dtype)
    lse = _nan((n_dst, H))
    ws = _ws(n_dst, G.E, D)
    tail = [*_dt(dtype)] + ([P_DROP, SEED[0], SEED[1]] if drop else []) + [P(ws), ws.numel(), ops._stream()]
    sfx = ("drop_" if drop else "") + "csr_" + ("f32" if dtype == torch.float32 else "x16")
    if kind == "dot":
        q, k, v = _dev(tensors[0][:n_dst], dtype), _dev(tensors[1], dtype), _dev(tensors[2], dtype)
        _call("pglb_dot_attn_" + sfx, P(ip), P(cols), P(q), q.stride(0), P(k), k.stride(0), P(v), v.stride(0),
              P(out), out.stride(0), P(lse), n_dst, G.N, G.E, H, Dh, *tail)
    else:
        f, a = _dev(tensors[0], dtype), _dev(tensors[1])
        _call("pglb_gatv2_attn_" + sfx, P(ip), P(cols), P(f), f.stride(0), P(a), float(slope), P(out), out.stride(0),
              P(lse), G.N, G.E, H, Dh, *tail)
    return out, lse


def _check_fwd(what, out, lse, sel, sig, c, feat_slots, ip, rcp_rows, keep, dtype):
    want, _ = expected_attention(sel, feat_slots, ip, rcp_rows, keep, drop_scale() if keep is not None else None,
                                 dtype)
    # the sign of a zero is not part of the contract: a rescale of a negative partial by an underflowed weight leaves
    # -0 where the kept weights of a row are all 0 (x + 0 maps -0 to +0 and leaves every other value alone)
    assert_bits(out.cpu() + 0, want + 0, what, _row_of_slot(ip))
    if lse is not None:
        check_lse(lse.cpu().numpy(), sig, c, what)


def _gat5_rows(cut, n_rows, gat5):
    """Rows gat5's epilogue finishes (uncut); None for the per-slot kernel, which divides everywhere."""
    return (~cut[:n_rows]) if gat5 else None


# ----------------------------------------------------------------------------------------------------------------
# GPU: the canary, edge softmax, unfused GAT attention
# ----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_canary_one_slot_rows():
    """The premise on the hardware: a one-slot row gives out == f and lse == sigma bit for bit (gat5, train), and
    alpha == 1 (edge softmax)."""
    import pgl_b200 as pgl
    import pgl_b200.nn.functional as GF
    rng = np.random.default_rng(1)
    n, H, Dh = 64, 4, 32
    edges = np.stack([np.arange(n), (np.arange(n) * 7) % n], 1)
    f = _features(rng, n, H * Dh, False)
    a_s = rng.integers(-500, 500, (n, H)).astype(np.float32)
    a_d = rng.integers(-500, 500, (n, H)).astype(np.float32)
    G = RegimeGraph.__new__(RegimeGraph)
    deg, sv, su, se, ip = O.adj_dst_index(edges, n)
    G.indptr, G.cols, G.E, G.N, G.R = ip, sv, n, n, n
    out, lse = run_gat(G, n, f, a_s, a_d, 0.2, H, Dh, torch.float32, "train")
    want_f = np.zeros((n, H * Dh))
    want_f[edges[:, 1]] = f[edges[:, 0]]
    assert_bits(out.cpu(), to_dtype(want_f, torch.float32), "canary: one-slot rows, out")
    z = lrelu32(a_s[edges[:, 0]] + a_d[edges[:, 1]], 0.2)
    want_l = np.zeros((n, H), np.float32)
    want_l[edges[:, 1]] = z
    assert_bits(lse.cpu(), torch.from_numpy(want_l), "canary: one-slot rows, lse == sigma")
    g = pgl.Graph(edges=edges, num_nodes=n)
    g.tensor()
    al = GF.edge_softmax(g, _dev(rng.standard_normal((n, 3)) * 100))
    assert (al.cpu() == 1).all(), "canary: edge softmax of one-slot rows is not 1"


_PG = {}


def _pgl_graph(G):
    import pgl_b200 as pgl
    key = id(G)
    if key not in _PG:
        g = pgl.Graph(edges=G.edges, num_nodes=G.N)
        g.tensor()
        fwd = g._fwd_csr()
        assert np.array_equal(fwd["eid"].cpu().numpy(), G.eid), "library CSR slots differ from the graph's"
        assert np.array_equal(fwd["cols"].cpu().numpy(), G.cols)
        _PG[key] = g
    return _PG[key]


def _edge_logits(G, H, rng, neg_inf):
    """Stored logits in CSR slot order: sigma per (row, head) on selected slots, sigma - 200 (or -inf) on masked."""
    row = _row_of_slot(G.indptr)
    want = np.tile(G.want, (1, (H + HMAX - 1) // HMAX))[:, :H]
    sig = rng.integers(-60, 60, (G.N, H)).astype(np.float64)
    low = -np.inf if neg_inf else -200.0
    lg = np.where(want, sig[row], sig[row] + low)   # every row has a selected slot: never all -inf
    return lg.astype(np.float32)


EDGE_H = [1, 2, 3, 8, 32, 33, 40]


@pytest.mark.gpu
@pytest.mark.parametrize("H", EDGE_H)
def test_edge_softmax_exact(H):
    """pglb_edge_softmax_csr_f32 through F.edge_softmax (permuted eid; dst- and src-keyed) and through
    pgl.math.segment_softmax (eid NULL, segment ids with gaps): alpha = fl(1 / c) or 0, bit for bit; the warp and hub
    kernels and more than one head tile (H > 32)."""
    import pgl_b200 as pgl
    import pgl_b200.nn.functional as GF
    from pgl_b200 import ops
    G, _, _, _ = ladder()
    g = _pgl_graph(G)
    rng = np.random.default_rng(H)
    for neg_inf in (False, True):
        lg = _edge_logits(G, H, rng, neg_inf)
        sel, _, c = weights_regime(lg, G.indptr, allow_neg_inf=neg_inf)
        alpha = np.where(sel, (1.0 / np.maximum(c, 1)[_row_of_slot(G.indptr)]), 0.0).astype(np.float32)
        le = np.empty_like(lg)
        le[G.eid] = lg
        want = np.empty_like(alpha)
        want[G.eid] = alpha
        got = GF.edge_softmax(g, _dev(le), norm_by="dst")
        assert_bits(got.cpu(), torch.from_numpy(want), "edge_softmax dst H=%d -inf=%s" % (H, neg_inf))
        # the same edges on a CSR of R rows (fewer rows than nodes; no node past R has an in-edge)
        got = ops.edge_softmax_csr(_i64(G.indptr_rows(G.R)), _i64(G.eid), _dev(le), G.E)
        assert_bits(got.cpu(), torch.from_numpy(want), "edge_softmax CSR of %d rows H=%d" % (G.R, H))
        # segment_softmax: slots are rows, ids with gaps (empty segments)
        ids = _row_of_slot(G.indptr)
        got = pgl.math.segment_softmax(_dev(lg), _i64(ids))
        assert_bits(got.cpu(), torch.from_numpy(alpha), "segment_softmax H=%d -inf=%s" % (H, neg_inf))
    # src-keyed: the same scores seen from the sources (rows of the src CSR)
    src = G.edges[:, 0]
    order = np.argsort(src, kind="stable")
    sip = np.r_[0, np.cumsum(np.bincount(src, minlength=G.N))].astype(np.int64)
    sig = rng.integers(-60, 60, (G.N, H)).astype(np.float64)
    bit = rng.random((G.edges.shape[0], H)) < 0.5
    lg_e = np.where(bit, sig[src], sig[src] - 300.0).astype(np.float32)
    sel, _, c = weights_regime(lg_e[order], sip)
    a_slot = np.where(sel, 1.0 / np.maximum(c, 1)[_row_of_slot(sip)], 0.0).astype(np.float32)
    want = np.empty_like(a_slot)
    want[order] = a_slot
    got = GF.edge_softmax(g, _dev(lg_e), norm_by="src")
    assert_bits(got.cpu(), torch.from_numpy(want), "edge_softmax src H=%d" % H)


@pytest.mark.gpu
@pytest.mark.parametrize("slope", [0.0, 0.2, 1.0])
def test_gat_attention_unfused_exact(slope):
    """pglb_gat_attention_csr_f32 (GAT logits formed on the fly, alpha in slot order): fl(1 / c) or 0."""
    from pgl_b200 import ops
    G, _, _, _ = ladder()
    rng = np.random.default_rng(int(slope * 10) + 3)
    for H in (1, 4, 8, 33):
        a_s, a_d = gat_inputs(G, min(H, HMAX), rng)
        sc = gat_scores(G, a_s, a_d, slope, G.N)
        sel, _, c = weights_regime(sc, G.indptr)
        want = np.where(sel, 1.0 / np.maximum(c, 1)[_row_of_slot(G.indptr)], 0.0).astype(np.float32)
        csr = {"indptr": _i64(G.indptr), "cols": _i64(G.cols)}
        got = ops.gat_attention_csr(csr, _dev(a_s), _dev(a_d), slope)
        assert_bits(got.cpu(), torch.from_numpy(want), "gat_attention H=%d slope=%g" % (H, slope))


# ----------------------------------------------------------------------------------------------------------------
# GPU: fused GAT, dot attention, GATv2
# ----------------------------------------------------------------------------------------------------------------

# (dtype, H, Dh, slope, misaligned attn_src, gat5): gat5 runs inference, train and dropout; the per-slot kernel
# (spmm_stream128_kernel<..., 2>: H % 4 != 0, 32 heads of 4 in fp32, attn_src off 16 bytes, slope outside [0, 1])
# inference only
GAT_CASES = [
    (torch.float32, 4, 32, 0.2, False, True), (torch.float32, 8, 16, 0.0, False, True),
    (torch.float32, 4, 16, 1.0, False, True),
    (torch.float32, 2, 64, 0.2, False, False), (torch.float32, 3, 4, 0.2, False, False),
    (torch.float32, 32, 4, 0.2, False, False), (torch.float32, 8, 16, 0.2, True, False),
    (torch.float32, 4, 32, 2.0, False, False), (torch.float32, 4, 32, -0.5, False, False),
    (torch.bfloat16, 4, 32, 0.2, False, True), (torch.float16, 8, 16, 0.0, False, True),
    (torch.bfloat16, 32, 4, 0.2, False, True), (torch.float16, 32, 4, 1.0, False, True),
]
if CHILD:
    GAT_CASES = [GAT_CASES[i] for i in (0, 3, 9, 11)]
# launches of the same call before the checked one: every launch re-arms the persistent kernels' task queue head
WARM = ["0", "1", "2"] if not CHILD else ["2"]


def _gid(c):
    return "%s-%dx%d-s%g%s" % (str(c[0]).split(".")[-1], c[1], c[2], c[3], "-misaligned" if c[4] else "")


@pytest.mark.gpu
@pytest.mark.parametrize("warm", WARM)
@pytest.mark.parametrize("case", GAT_CASES, ids=[_gid(c) for c in GAT_CASES])
def test_gat_fused_exact(case, warm):
    dtype, H, Dh, slope, mis, gat5 = case
    G, cut, _, _ = ladder()
    rng = np.random.default_rng(H * 100 + Dh)
    f = _features(rng, G.N, H * Dh, dtype != torch.float32)
    a_s, a_d = gat_inputs(G, H, rng)
    for n_dst in (G.N, G.R):                                   # square, and fewer rows than sources
        ip = G.indptr_rows(n_dst)
        sel, sig, c = weights_regime(gat_scores(G, a_s, a_d, slope, n_dst), ip)
        fs = f[G.cols].reshape(-1, H, Dh)
        rcp = _gat5_rows(cut, n_dst, gat5)
        if gat5 and n_dst == G.N and dtype == torch.float32 and not CHILD:
            # a cut row finished by gat5's rounding instead of the fix-up's division would show
            fix, epi = (expected_attention(sel, fs, ip, r)[0].numpy()[cut[:n_dst]] for r in (None, cut[:n_dst]))
            assert (fix != epi).any(), "no cut row tells the fix-up's division from gat5's rounding"
        modes = ("infer", "train", "drop") if gat5 else ("infer",)
        for mode in modes:
            if mode != "infer" and n_dst != G.N:
                continue
            first = [run_gat(G, n_dst, f, a_s, a_d, slope, H, Dh, dtype, mode, misalign=mis)[0]
                     for _ in range(int(warm))]
            out, lse = run_gat(G, n_dst, f, a_s, a_d, slope, H, Dh, dtype, mode, misalign=mis)
            assert all(torch.equal(o, out) for o in first)
            keep = keep_mask(G.E, H) if mode == "drop" else None
            _check_fwd("gat %s %s n_dst=%d" % (_gid(case), mode, n_dst), out, lse, sel, sig, c, fs, ip, rcp, keep,
                       dtype)


DOT_CASES = [(torch.float32, 4, 32, False), (torch.float32, 2, 64, False), (torch.float32, 8, 16, False),
             (torch.float32, 32, 4, False), (torch.bfloat16, 4, 32, False), (torch.float16, 8, 16, False),
             (torch.float32, 4, 32, True), (torch.bfloat16, 8, 16, True)]
V2_CASES = [(torch.float32, 4, 32, 0.0, False), (torch.float32, 4, 32, 0.2, False), (torch.float32, 4, 32, 1.0, False),
            (torch.float32, 2, 64, 0.2, False), (torch.bfloat16, 4, 32, 0.2, False), (torch.float16, 8, 16, 0.0, False),
            (torch.float32, 4, 32, 0.2, True), (torch.bfloat16, 8, 16, 1.0, True)]
if CHILD:
    DOT_CASES = [DOT_CASES[i] for i in (0, 4, 6)]
    V2_CASES = [V2_CASES[i] for i in (1, 4, 6)]


@pytest.mark.gpu
@pytest.mark.parametrize("warm", WARM)
@pytest.mark.parametrize("case", DOT_CASES, ids=["%s-%dx%d%s" % (str(c[0]).split(".")[-1], c[1], c[2],
                                                                  "-drop" if c[3] else "") for c in DOT_CASES])
def test_dot_attn_exact(case, warm):
    dtype, H, Dh, drop = case
    G, cut, _, _ = ladder()
    rng = np.random.default_rng(H * 10 + Dh + 1)
    half = dtype != torch.float32
    q, k = dot_inputs(G, H, Dh, rng)
    v = _features(rng, G.N, H * Dh, half)
    for n_dst in (G.N, G.R):                                   # square, and fewer rows than sources
        ip = G.indptr_rows(n_dst)
        sel, sig, c = weights_regime(dot_scores(G, q, k, H, n_dst), ip)
        first = [run_scored("dot", G, (q, k, v), H, Dh, dtype, drop, n_dst=n_dst)[0] for _ in range(int(warm))]
        out, lse = run_scored("dot", G, (q, k, v), H, Dh, dtype, drop, n_dst=n_dst)
        assert all(torch.equal(o, out) for o in first)
        _check_fwd("dot %s H=%d Dh=%d drop=%s n_dst=%d" % (dtype, H, Dh, drop, n_dst), out, lse, sel, sig, c,
                   v[G.cols].reshape(-1, H, Dh), ip, ~cut[:n_dst], keep_mask(G.E, H) if drop else None, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("warm", WARM)
@pytest.mark.parametrize("case", V2_CASES, ids=["%s-%dx%d-s%g%s" % (str(c[0]).split(".")[-1], c[1], c[2], c[3],
                                                                     "-drop" if c[4] else "") for c in V2_CASES])
def test_gatv2_attn_exact(case, warm):
    dtype, H, Dh, slope, drop = case
    G, cut, _, _ = ladder()
    rng = np.random.default_rng(H * 10 + Dh + 2)
    f, a = v2_inputs(G, H, Dh, rng, dtype != torch.float32)
    sel, sig, c = weights_regime(v2_scores(G, f, a, H, slope, G.N), G.indptr)
    first = [run_scored("v2", G, (f, a), H, Dh, dtype, drop, slope)[0] for _ in range(int(warm))]
    out, lse = run_scored("v2", G, (f, a), H, Dh, dtype, drop, slope)
    assert all(torch.equal(o, out) for o in first)
    _check_fwd("gatv2 %s H=%d Dh=%d slope=%g drop=%s" % (dtype, H, Dh, slope, drop), out, lse, sel, sig, c,
               f[G.cols].reshape(-1, H, Dh), G.indptr, ~cut, keep_mask(G.E, H) if drop else None, dtype)


@pytest.mark.gpu
def test_edgeless_graph():
    """No edges: every row is empty: out 0, lse untouched."""
    G = RegimeGraph([0] * 40, seed=1)
    rng = np.random.default_rng(0)
    f = _features(rng, G.N, 128, False)
    a_s, a_d = gat_inputs(G, 4, rng)
    for mode in ("infer", "train"):
        out, lse = run_gat(G, G.N, f, a_s, a_d, 0.2, 4, 32, torch.float32, mode)
        assert (out.cpu() == 0).all()
        assert lse is None or torch.isnan(lse.cpu()).all()


# ----------------------------------------------------------------------------------------------------------------
# GPU: attention readout
# ----------------------------------------------------------------------------------------------------------------

READOUT_LENS = (2047, 0, 2048, 2049, 1, 4095, 0, 4096, 4097, 6, 3000)


@pytest.mark.gpu
@pytest.mark.parametrize("use_query", [False, True])
def test_attn_readout_exact(use_query):
    """pglb_attn_readout_f32, gate and query (one column), segments around one and two 2048-row chunks, every
    pattern; max_len exact and below the longest segment (one item per segment).  Empty segment: out 0, lse -inf."""
    from pgl_b200 import ops
    rng = np.random.default_rng(7 + use_query)
    lens = np.array(READOUT_LENS, np.int64)
    ip = np.r_[0, np.cumsum(lens)].astype(np.int64)
    N, B, D = int(ip[-1]), lens.shape[0], 40
    x = _features(rng, N, D, False)
    sel_i = np.zeros(N, bool)
    for g, k in enumerate(lens):
        kind = KINDS[g % len(KINDS)] if g % 3 else "prefix"
        p = pattern(kind, int(k), rng)
        if k > 2100 and g != 7:
            p = np.arange(k) >= 2100        # a whole masked chunk before the selected rows
        sel_i[ip[g]:ip[g + 1]] = p
    sig_g = rng.integers(-50, 50, B).astype(np.float64)
    row = _row_of_slot(ip)
    score = np.where(sel_i, sig_g[row], sig_g[row] - 400.0)
    gate = query = None
    if use_query:
        c0 = 7
        x[:, c0] = score
        query = np.zeros((B, D))
        query[:, c0] = 1.0
    else:
        gate = score
    sel, sig, c = weights_regime(score.astype(np.float32)[:, None], ip)
    want, _ = expected_attention(sel, x[:, None, :], ip)
    for max_len in (int(lens.max()), 100):
        out, lse = ops._attn_readout_raw(_dev(x), _i64(ip), None if gate is None else _dev(gate),
                                         None if query is None else _dev(query), max_len)
        tag = "readout query=%s max_len=%d" % (use_query, max_len)
        assert_bits(out.cpu(), want, tag, row)
        check_lse(lse.cpu().numpy()[:, None], sig, c, tag, empty_value=-np.inf)


# ----------------------------------------------------------------------------------------------------------------
# GPU: backward, bit-exact cases
# ----------------------------------------------------------------------------------------------------------------

def _exact_sum(terms, indptr, quantum):
    """float64 row sums of `terms` [E, ...], asserting that every term is a multiple of `quantum` and that the sum of
    |terms| over every row stays below 2^24 quanta: every partial sum is then exact in fp32."""
    t = np.asarray(terms, np.float64)
    assert np.array_equal(t / quantum, np.round(t / quantum)), "case leaves the exact regime: term off the quantum"
    ab = _reduceat(np.abs(t), indptr)
    assert ab.max(initial=0.0) / quantum < EXACT_LIMIT, "case leaves the exact regime: sum of |terms| too large"
    return _reduceat(t, indptr)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [1, 3, 8, 33])
def test_edge_softmax_bwd_exact(H):
    """pglb_edge_softmax_bwd_csr_f32: alpha = 2^-k (k <= 10), small integer gradients: alpha (g - sum alpha g) exact;
    eid permuted and NULL."""
    from pgl_b200 import ops
    G, _, _, _ = ladder()
    rng = np.random.default_rng(H + 40)
    E = G.E
    deg = np.diff(G.indptr)
    kmin = np.where(deg[_row_of_slot(G.indptr)] > 1024, 6, 0)[:, None]
    alpha = 2.0 ** -(kmin + rng.integers(0, 5, (E, H)))
    gr = rng.integers(-3, 4, (E, H)).astype(np.float64)
    s = _exact_sum(alpha * gr, G.indptr, 2.0 ** -10)
    want = alpha * (gr - s[_row_of_slot(G.indptr)])
    for eid in (G.eid, None):
        a_e, g_e, w_e = alpha, gr, want
        if eid is not None:
            a_e, g_e, w_e = (np.empty_like(t) for t in (alpha, gr, want))
            a_e[eid], g_e[eid], w_e[eid] = alpha, gr, want
        gl = torch.zeros((E, H), device="cuda")
        ipd, eidd, ad, gd = _i64(G.indptr), None if eid is None else _i64(eid), _dev(a_e), _dev(g_e)
        _call("pglb_edge_softmax_bwd_csr_f32", ops._ptr(ipd), ops._ptr(eidd), ops._ptr(ad), ops._ptr(gd),
              ops._ptr(gl), G.N, E, H, ops._stream())
        assert_bits(gl.cpu(), to_dtype(w_e, torch.float32), "edge_softmax_bwd H=%d eid=%s" % (H, eid is not None))


@pytest.mark.gpu
@pytest.mark.parametrize("H,Dh", [(4, 16), (8, 4), (3, 5), (1, 33)])
def test_sddmm_dot_exact(H, Dh):
    """pglb_sddmm_dot_f32 on integer rows (exact products and sums), Dh % 4 == 0 (float4 path) and not."""
    from pgl_b200 import ops
    G, _, _, _ = ladder()
    rng = np.random.default_rng(H * Dh)
    a = rng.integers(-8, 9, (G.N, H * Dh)).astype(np.float64)
    b = rng.integers(-8, 9, (G.N, H * Dh)).astype(np.float64)
    src, dst = G.edges[:, 0], G.edges[:, 1]
    want = (a[src].reshape(-1, H, Dh) * b[dst].reshape(-1, H, Dh)).sum(-1)
    got = ops.sddmm_dot(_dev(a), _dev(b), _i64(src), _i64(dst), H, Dh)
    assert_bits(got.cpu(), to_dtype(want, torch.float32), "sddmm_dot H=%d Dh=%d" % (H, Dh))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("slope", [0.25, 0.5, 1.0])
def test_gatv2_score_grad_exact(slope, dtype):
    """pglb_gatv2_score_grad_*: power-of-two ds and attn, integer f, on the dst- and the src-keyed CSR (rows over 1024
    slots take the chunked path), accumulate 0 and 1."""
    from pgl_b200 import ops
    P = ops._ptr
    G, _, _, _ = ladder()
    g = _pgl_graph(G)
    H, Dh = 4, 32
    D = H * Dh
    rng = np.random.default_rng(int(slope * 8))
    f = _features(rng, G.N, D, dtype != torch.float32)
    attn = rng.choice([-1.0, -0.5, -0.25, 0.25, 0.5, 1.0], D)
    ds = rng.choice([-1.0, 1.0], (G.E, H)) * 2.0 ** -rng.integers(0, 5, (G.E, H))   # edge order
    fd, ad, dsd = _dev(f, dtype), _dev(attn), _dev(ds)
    prev = rng.integers(-4, 5, (G.N, D)).astype(np.float64)
    for key in ("dst", "src"):
        csr = g._fwd_csr() if key == "dst" else g._bwd_csr()
        ip = csr["indptr"].cpu().numpy()
        cols, eid = csr["cols"].cpu().numpy(), csr["eid"].cpu().numpy()
        row = _row_of_slot(ip)
        z = f[row] + f[cols]
        der = np.where(z > 0, 1.0, slope)
        terms = ds[eid].repeat(Dh, axis=1) * attn[None, :] * der
        s = _exact_sum(terms, ip, 2.0 ** -8)
        ws = _ws(G.N, G.E, D)
        for acc in (0, 1):
            out = _dev(prev) if acc else _nan((G.N, D))
            _call("pglb_gatv2_score_grad_" + ("f32" if dtype == torch.float32 else "x16"), P(csr["indptr"]),
                  P(csr["cols"]), P(csr["eid"]), P(fd), fd.stride(0), P(ad), float(slope), P(dsd), P(out),
                  out.stride(0), G.N, G.E, H, Dh, *_dt(dtype), acc, P(ws), ws.numel(), ops._stream())
            want = s + prev if acc else s
            assert_bits(out.cpu(), to_dtype(want, torch.float32),
                        "gatv2_score_grad %s %s slope=%g accumulate=%d" % (dtype, key, slope, acc), row)


# ----------------------------------------------------------------------------------------------------------------
# GPU: backward, bounded cases on a regime forward
# ----------------------------------------------------------------------------------------------------------------

U = 2.0 ** -24       # unit roundoff of fp32


def _ulp_half(x):
    """ulp(x) / 2 in fp32 (half the spacing at |x|)."""
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64) / 2


def weight_bound(sig, lse, c):
    """Relative bound r_a with |a - 1/c| <= r_a / c for a selected slot's rebuilt weight a = expf(fl(sigma - lse)).
    lse is the forward's (within ulp(ln c) + ulp(lse) / 2 of sigma + ln c, see check_lse), so
      x = fl(sigma - lse) = -ln c - e,  |e| <= dx = |lse - sigma - ln c| + ulp(sigma - lse) / 2,
    and expf is within 2 ulp (relative 2^-22):  |a - 1/c| <= (1/c) (expm1(dx) + 2^-22 (1 + expm1(dx))).
    A masked slot's x is at most -150 - ln c: a is exactly 0."""
    dx = np.abs(lse - sig - np.log(c)) + _ulp_half(sig - lse)
    em = np.expm1(dx)
    return em + 2.0 ** -22 * (1.0 + em)


def edge_grad_bound(c, r_a, da, delta, s_go, Dh, scale=1.0, der=1.0):
    """(reference, bound) of a selected edge's score gradient d = der * a * (scale * da - delta) as the edge kernels
    form it: da = <G, f[src]> exact (integers), delta = <G, out> over Dh fma's and a head butterfly (error at most
    (Dh + 1) u sum|G out|), with dropout fl(scale * da) (u |scale da|), then the difference, the product with a and
    (GAT, negative side) the product with the slope, one rounding each:
      e_d = u |scale da| + (Dh + 1) u s_go,   |d_k| <= |dd| + e_d  (dd = scale da - delta, exact reals)
      bound = der ((1/c) r_a |dd| + (1/c)(1 + r_a) (e_d + 3 u (|dd| + e_d))).
    No global maximum enters: each element's bound comes from its own row."""
    dd = scale * da - delta
    e_d = U * np.abs(scale * da) + (Dh + 1) * U * s_go
    a1 = (1.0 + r_a) / c
    return der * dd / c, der * (r_a * np.abs(dd) / c + a1 * (e_d + 3 * U * (np.abs(dd) + e_d)))


def assert_within(got, want, bound, what):
    err = np.abs(np.asarray(got, np.float64) - want)
    bad = np.argwhere(~(err <= bound))
    assert bad.size == 0, "%s: %d elements off; first %s: got %r, want %r, bound %g" % (
        what, bad.shape[0], tuple(bad[0]), float(np.asarray(got)[tuple(bad[0])]), want[tuple(bad[0])],
        bound[tuple(bad[0])])


def run_edge_bwd(kind, G, ins, out, lse, g2, H, Dh, dtype, drop, slope=0.0):
    """The per-edge backward entry of kind 'gat' (ins = f, a_s, a_d), 'dot' (q, k, v) or 'v2' (f, a; with grad_attn):
    (weight [E, H], score gradient [E, H], grad attn or None), edge order."""
    from pgl_b200 import ops
    P = ops._ptr
    E = G.E
    rows, cols, eid = _i64(_row_of_slot(G.indptr)), _i64(G.cols), _i64(G.eid)
    w, d = torch.empty((E, H), device="cuda"), torch.empty((E, H), device="cuda")
    dt = [*_dt(dtype)] + ([P_DROP, SEED[0], SEED[1]] if drop else [])
    sfx = ("drop_" if drop else "") + ("f32" if dtype == torch.float32 else "x16")
    ga = None
    if kind == "gat":
        f, a_s, a_d = _dev(ins[0], dtype), _dev(ins[1]), _dev(ins[2])
        _call("pglb_gat_bwd_edge_" + sfx, P(rows), P(cols), P(eid), P(f), f.stride(0), P(g2), g2.stride(0), P(out),
              out.stride(0), P(a_s), P(a_d), P(lse), float(slope), E, H, Dh, *dt, P(w), P(d), ops._stream())
    elif kind == "dot":
        q, k, v = (_dev(t, dtype) for t in ins)
        _call("pglb_dot_attn_bwd_edge_" + sfx, P(rows), P(cols), P(eid), P(q), q.stride(0), P(k), k.stride(0), P(v),
              v.stride(0), P(g2), g2.stride(0), P(out), out.stride(0), P(lse), E, H, Dh, *dt, P(w), P(d),
              ops._stream())
    else:
        f, a = _dev(ins[0], dtype), _dev(ins[1])
        ga = torch.empty(H * Dh, device="cuda")
        need = ctypes.c_size_t(0)
        ops.check(ops.lib.pglb_gatv2_bwd_edge_ws(E, ctypes.byref(need)))
        ws = torch.empty(max(need.value, 16), dtype=torch.uint8, device="cuda")
        _call("pglb_gatv2_bwd_edge_" + sfx, P(rows), P(cols), P(eid), P(f), f.stride(0), P(a), float(slope), P(g2),
              g2.stride(0), P(out), out.stride(0), P(lse), E, H, Dh, *dt, P(w), P(d), P(ga), P(ws), ws.numel(),
              ops._stream())
    return w, d, ga


# (kind, dtype, H, Dh, slope, drop)
BWD_CASES = [("gat", torch.float32, 4, 32, 0.2, False), ("gat", torch.float32, 4, 16, 1.0, True),
             ("gat", torch.bfloat16, 8, 16, 0.0, True), ("gat", torch.float16, 32, 4, 0.2, False),
             ("dot", torch.float32, 4, 32, 0.0, False), ("dot", torch.float32, 2, 64, 0.0, False),
             ("dot", torch.bfloat16, 4, 32, 0.0, True), ("v2", torch.float32, 4, 32, 0.2, False),
             ("v2", torch.float32, 4, 32, 0.0, True), ("v2", torch.bfloat16, 8, 16, 1.0, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", BWD_CASES, ids=["%s-%s-%dx%d-s%g%s" % (c[0], str(c[1]).split(".")[-1], c[2], c[3],
                                                                          c[4], "-drop" if c[5] else "")
                                                   for c in BWD_CASES])
def test_edge_backward_bounded(case):
    """gat_bwd_edge / dot_attn_bwd_edge / gatv2_bwd_edge (with grad_attn), f32, x16 and drop, on the forward of a
    regime case: masked edges give weight and score gradient exactly 0; selected edges lie within edge_grad_bound of
    the float64 reference, a bound below what one misattributed edge changes (it changes c, and so the weight by
    1/(c(c+1)), or an integer da by at least 1)."""
    kind, dtype, H, Dh, slope, drop = case
    G, _, _, _ = ladder()
    half = dtype != torch.float32
    rng = np.random.default_rng(H * 31 + Dh)
    row = _row_of_slot(G.indptr)
    if kind == "gat":
        f = _features(rng, G.N, H * Dh, half)
        a_s, a_d = gat_inputs(G, H, rng)
        sc = gat_scores(G, a_s, a_d, slope, G.N)
        out, lse = run_gat(G, G.N, f, a_s, a_d, slope, H, Dh, dtype, "drop" if drop else "train")
        ins, feat = (f, a_s, a_d), f
        z = (a_s[G.cols] + a_d[row]).astype(np.float32)
        der = np.where(z > 0, 1.0, np.float64(np.float32(slope)))
    elif kind == "dot":
        q, k = dot_inputs(G, H, Dh, rng)
        v = _features(rng, G.N, H * Dh, half)
        sc = dot_scores(G, q, k, H, G.N)
        out, lse = run_scored("dot", G, (q, k, v), H, Dh, dtype, drop)
        ins, feat, der = (q, k, v), v, 1.0
    else:
        f, a = v2_inputs(G, H, Dh, rng, half)
        sc = v2_scores(G, f, a, H, slope, G.N)
        out, lse = run_scored("v2", G, (f, a), H, Dh, dtype, drop, slope)
        ins, feat, der = (f, a), f, 1.0
    sel, sig, c = weights_regime(sc, G.indptr)
    gr = rng.choice([-1.0, 1.0], (G.N, H * Dh)) if half else rng.integers(-3, 4, (G.N, H * Dh)).astype(np.float64)
    g2 = _dev(gr, dtype)
    w, d, ga = run_edge_bwd(kind, G, ins, out, lse, g2, H, Dh, dtype, drop, slope)
    w, d = w.cpu().numpy()[G.eid], d.cpu().numpy()[G.eid]           # slot order
    keep = keep_mask(G.E, H) if drop else np.ones((G.E, H), bool)
    s = drop_scale() if drop else 1.0
    tag = "%s backward %s H=%d Dh=%d slope=%g drop=%s" % (kind, dtype, H, Dh, slope, drop)
    assert (w[~sel] == 0).all() and (d[~sel] == 0).all(), tag + ": a masked edge has a nonzero weight or gradient"
    assert (w[sel & ~keep] == 0).all(), tag + ": a dropped edge has a nonzero weight"
    out64 = out.float().cpu().numpy().astype(np.float64)
    G3, F3, O3 = (t.reshape(-1, H, Dh) for t in (gr[row], feat[G.cols], out64[row]))
    da = (G3 * F3).sum(-1)
    assert (np.abs(G3 * F3).sum(-1) < EXACT_LIMIT).all()
    delta, s_go = (G3 * O3).sum(-1), np.abs(G3 * O3).sum(-1)
    lse64 = lse.cpu().numpy().astype(np.float64)[row]
    cc, sg = c[row], sig[row]
    r_a = weight_bound(sg, lse64, np.maximum(cc, 1))
    assert (r_a[sel] * (cc[sel] + 1) < 1).all(), tag + ": the weight bound does not resolve one edge more or less"
    a_want = np.where(keep, s / np.maximum(cc, 1), 0.0)
    a_bound = np.where(keep, s * (r_a + U * (1 + r_a)) / np.maximum(cc, 1), 0.0)
    assert_within(w[sel], a_want[sel], a_bound[sel], tag + " weight")
    d_want, d_bound = edge_grad_bound(np.maximum(cc, 1), r_a, np.where(keep, da, 0.0), delta, s_go, Dh, s,
                                      der if np.ndim(der) else np.full(da.shape, der))
    derv = der if np.ndim(der) else np.full(da.shape, der)
    assert (d_bound[sel] <= 0.5 * derv[sel] * s / cc[sel]).all(), tag + ": the bound does not resolve da by 1"
    assert_within(d[sel], d_want[sel], d_bound[sel], tag + " score gradient")
    if ga is not None:
        # grad a[h, c] = sum over edges of ds lrelu(z_c): a sum over every edge, so its bound is global: each edge's
        # share within |lrelu| d_bound, plus the fma chains and fixed trees of at most E + 300 additions
        z = (feat[G.cols].astype(np.float32) + feat[row].astype(np.float32)).astype(np.float32)
        lr = lrelu32(z, slope).astype(np.float64).reshape(-1, H, Dh)
        dw = np.where(sel, d_want, 0.0)[:, :, None] * lr
        want = dw.sum(0).reshape(-1)
        bound = (np.where(sel, d_bound, 0.0)[:, :, None] * np.abs(lr)).sum(0).reshape(-1) + \
            (G.E + 300) * U * np.abs(dw).sum(0).reshape(-1)
        assert_within(ga.cpu().numpy(), want, bound, tag + " grad attn")


@pytest.mark.gpu
@pytest.mark.parametrize("use_query", [False, True])
def test_attn_readout_backward_bounded(use_query):
    """pglb_attn_readout_bwd_f32 on the forward of a regime readout: masked rows give grad x (the gate part), grad
    gate exactly 0; selected rows lie within the bound of edge_grad_bound (the <r, G> block sum over D columns:
    (D + 16) u sum|r G|), and grad query within the sum of its rows' bounds plus (n + 16) u sum|ds x|."""
    from pgl_b200 import ops
    P = ops._ptr
    rng = np.random.default_rng(17 + use_query)
    lens = np.array(READOUT_LENS, np.int64)
    ip = np.r_[0, np.cumsum(lens)].astype(np.int64)
    N, B, D = int(ip[-1]), lens.shape[0], 40
    x = _features(rng, N, D, False)
    row = _row_of_slot(ip)
    sel_i = np.zeros(N, bool)
    for g, k in enumerate(lens):
        sel_i[ip[g]:ip[g + 1]] = pattern(KINDS[(g + 3) % len(KINDS)], int(k), rng)
    sig_g = rng.integers(-50, 50, B).astype(np.float64)
    score = np.where(sel_i, sig_g[row], sig_g[row] - 400.0)
    c0 = 7
    gate = query = None
    if use_query:
        x[:, c0] = score
        query = np.zeros((B, D))
        query[:, c0] = 1.0
    else:
        gate = score
    sel, sig, c = weights_regime(score.astype(np.float32)[:, None], ip)
    sel, sig, c = sel[:, 0], sig[:, 0], c[:, 0]
    xd, ipd = _dev(x), _i64(ip)
    gd, qd = (None if gate is None else _dev(gate)), (None if query is None else _dev(query))
    out, lse = ops._attn_readout_raw(xd, ipd, gd, qd, int(lens.max()))
    go = rng.integers(-3, 4, (B, D)).astype(np.float64)
    god = _dev(go)
    gx = _nan((N, D))
    gg = _nan((N,)) if gate is not None else None
    gq = _nan((B, D)) if query is not None else None
    ws = ops._readout_ws(B, N, D, int(lens.max()), xd.device)
    _call("pglb_attn_readout_bwd_f32", P(xd), N, D, P(ipd), B, int(lens.max()), P(gd), P(qd), P(out), P(lse),
          P(god), P(gx), P(gg), P(gq), P(ws), ws.numel() if ws is not None else 0, ops._stream())
    r64, l64 = out.cpu().numpy().astype(np.float64), lse.cpu().numpy().astype(np.float64)
    v = (x * go[row]).sum(1)
    delta, s_go = (r64 * go).sum(1)[row], np.abs(r64 * go).sum(1)[row]
    cc = np.maximum(c[row], 1)
    r_a = weight_bound(sig[row], l64[row], cc)
    ds_want, ds_bound = edge_grad_bound(cc, r_a, v, delta, s_go, D + 15)
    tag = "readout backward query=%s" % use_query
    gxn = gx.cpu().numpy()
    if gate is not None:
        ggn = gg.cpu().numpy()
        assert (ggn[~sel] == 0).all() and (gxn[~sel] == 0).all(), tag + ": a masked row has a nonzero gradient"
        assert_within(ggn[sel], ds_want[sel], ds_bound[sel], tag + " grad gate")
        gx_want = go[row] / cc[:, None]
        gx_bound = np.abs(go[row]) * ((r_a + U * (1 + r_a)) / cc)[:, None]
    else:
        gx_want = go[row] / cc[:, None] + ds_want[:, None] * query[row]
        gx_bound = np.abs(go[row]) * ((r_a + U * (1 + r_a)) / cc)[:, None] + \
            (ds_bound[:, None] + U * np.abs(gx_want)) * np.abs(query[row]) + U * np.abs(gx_want)
        dsx = np.where(sel, ds_want, 0.0)[:, None] * x
        gq_want = _reduceat(dsx, ip)
        gq_bound = _reduceat(np.where(sel, ds_bound, 0.0)[:, None] * np.abs(x), ip) + \
            (lens[:, None] + 16) * U * _reduceat(np.abs(dsx), ip)
        assert_within(gq.cpu().numpy(), gq_want, gq_bound, tag + " grad query")
    assert_within(gxn[sel], gx_want[sel], gx_bound[sel], tag + " grad x")


# ----------------------------------------------------------------------------------------------------------------
# switches read once per process: child processes
# ----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("T", ["32", "64", "2048"])
def test_task_size_in_child(T):
    """PGLB_STREAM_TASK = T (read once per process; snapping off, so rows longer than T are cut): the fused forward
    tests again in a child process, on a graph whose boundary block is laid out for T."""
    if CHILD:
        pytest.skip("already the child")
    sel = "gat_fused_exact or dot_attn_exact or gatv2_attn_exact"
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-m", "gpu", "-k", sel,
                        "-p", "no:cacheprovider"], env=dict(os.environ, PGLB_SOFTMAX_CHILD="1", PGLB_STREAM_TASK=T),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:]


# ----------------------------------------------------------------------------------------------------------------
# route coverage
# ----------------------------------------------------------------------------------------------------------------

_F, _BF, _FP = "float", "__nv_bfloat16", "__half"
ROUTES = {
    # edge softmax: stored logits (MODE 0) and GAT logits (MODE 1), warp and hub kernels
    "edge_softmax_warp<0>": r"edge_softmax_warp_kernel<0>", "edge_softmax_hub<0>": r"edge_softmax_hub_kernel<0>",
    "edge_softmax_warp<1>": r"edge_softmax_warp_kernel<1>", "edge_softmax_hub<1>": r"edge_softmax_hub_kernel<1>",
    "stream128 GAT per-slot": r"spmm_stream128_kernel<0, false, 0, 2>",
    "fixup_gat f32": r"spmm_stream_fixup_gat_kernel<float, false>",
    "fixup_gat f32 drop": r"spmm_stream_fixup_gat_kernel<float, true>",
    "fixup_gat bf16": r"spmm_stream_fixup_gat_kernel<__nv_bfloat16, false>",
    "fixup_gat fp16 drop": r"spmm_stream_fixup_gat_kernel<__half, true>",
    "edge_softmax_bwd": r"edge_softmax_bwd_kernel", "sddmm_dot<4>": r"sddmm_dot_kernel<4>",
    "sddmm_dot<1>": r"sddmm_dot_kernel<1>", "gatv2_score_grad": r"gatv2_score_grad_kernel",
    "readout gate": r"attn_readout_kernel<false>", "readout query": r"attn_readout_kernel<true>",
    "readout merge": r"ro_merge_kernel", "gat5 any": r"spmm_gat5_kernel<",
    "gat_bwd_edge f32": r"gat_bwd_edge_kernel<\d+, float, false>",
    "gat_bwd_edge bf16 drop": r"gat_bwd_edge_kernel<\d+, __nv_bfloat16, true>",
    "dot_bwd_edge f32": r"dot_attn_bwd_edge_kernel<\d+, float, false>",
    "dot_bwd_edge bf16 drop": r"dot_attn_bwd_edge_kernel<\d+, __nv_bfloat16, true>",
    "gatv2_bwd_edge f32": r"gatv2_bwd_edge_kernel<\d+, float, false>",
    "gatv2_bwd_edge bf16 drop": r"gatv2_bwd_edge_kernel<\d+, __nv_bfloat16, true>",
    "gatv2_ga_reduce": r"gatv2_ga_reduce_kernel",
    "readout bwd gate": r"attn_readout_bwd_kernel<false>", "readout bwd query": r"attn_readout_bwd_kernel<true>",
    "readout merge grad query": r"ro_merge_gq_kernel",
}
for _sk in (0, 1, 2):
    for _t in (_F, _BF, _FP):
        for _drop in ("false", "true"):
            ROUTES["gat5 sk=%d %s drop=%s" % (_sk, _t, _drop)] = \
                r"spmm_gat5_kernel<%s, \d+, \d+, \d+, %s(, %d)?>" % (re.escape(_t), _drop, _sk) \
                if _sk == 0 else r"spmm_gat5_kernel<%s, \d+, \d+, \d+, %s, %d>" % (re.escape(_t), _drop, _sk)


def _route_calls():
    """(label, call, [route names the call must reach])."""
    G, _, _, _ = ladder()
    g = _pgl_graph(G)
    rng = np.random.default_rng(0)
    calls = []
    import pgl_b200.nn.functional as GF
    from pgl_b200 import ops
    lg = _dev(_edge_logits(G, 8, rng, False))
    calls.append(("edge_softmax", lambda: GF.edge_softmax(g, lg), ["edge_softmax_warp<0>", "edge_softmax_hub<0>"]))
    a_s, a_d = gat_inputs(G, 8, rng)
    csr = {"indptr": _i64(G.indptr), "cols": _i64(G.cols)}
    calls.append(("gat_attention", lambda: ops.gat_attention_csr(csr, _dev(a_s), _dev(a_d), 0.2),
                  ["edge_softmax_warp<1>", "edge_softmax_hub<1>"]))
    for dtype, tn in ((torch.float32, _F), (torch.bfloat16, _BF), (torch.float16, _FP)):
        half = dtype != torch.float32
        H, Dh = 4, 32
        f = _features(rng, G.N, H * Dh, half)
        a_s4, a_d4 = gat_inputs(G, H, rng)
        q, k = dot_inputs(G, H, Dh, rng)
        fv, av = v2_inputs(G, H, Dh, rng, half)
        for drop in (False, True):
            dp = "true" if drop else "false"

            def gat_fn(drop=drop, dtype=dtype, f=f, a_s4=a_s4, a_d4=a_d4):
                run_gat(G, G.N, f, a_s4, a_d4, 0.2, 4, 32, dtype, "drop" if drop else "train")

            def dot_fn(drop=drop, dtype=dtype, q=q, k=k, f=f):
                run_scored("dot", G, (q, k, f), 4, 32, dtype, drop)

            def v2_fn(drop=drop, dtype=dtype, fv=fv, av=av):
                run_scored("v2", G, (fv, av), 4, 32, dtype, drop, 0.2)
            fix = {(_F, False): ["fixup_gat f32"], (_F, True): ["fixup_gat f32 drop"],
                   (_BF, False): ["fixup_gat bf16"], (_FP, True): ["fixup_gat fp16 drop"]}.get((tn, drop), [])
            for sk, fn in ((0, gat_fn), (1, dot_fn), (2, v2_fn)):
                calls.append(("%s sk=%d drop=%s" % (tn, sk, drop), fn, ["gat5 sk=%d %s drop=%s" % (sk, tn, dp)] + fix))
    for case in GAT_CASES:                                  # every fused GAT case runs on the family it claims
        dtype, H, Dh, slope, mis, gat5 = case
        fc = _features(rng, G.N, H * Dh, dtype != torch.float32)
        a_sc, a_dc = gat_inputs(G, H, rng)
        calls.append(("gat case " + _gid(case),
                      lambda fc=fc, a_sc=a_sc, a_dc=a_dc, dtype=dtype, H=H, Dh=Dh, slope=slope, mis=mis:
                      run_gat(G, G.N, fc, a_sc, a_dc, slope, H, Dh, dtype, "infer", misalign=mis),
                      ["gat5 any" if gat5 else "stream128 GAT per-slot"]))
    f1 = _features(rng, G.N, 128, False)
    a_s3, a_d3 = gat_inputs(G, 2, rng)
    calls.append(("gat per-slot", lambda: run_gat(G, G.N, f1, a_s3, a_d3, 0.2, 2, 64, torch.float32, "infer"),
                  ["stream128 GAT per-slot", "fixup_gat f32"]))
    al, gr = _dev(np.full((G.E, 3), 0.5)), _dev(np.ones((G.E, 3)))
    gl, ipd = torch.zeros((G.E, 3), device="cuda"), _i64(G.indptr)
    calls.append(("edge_softmax_bwd", lambda: _call("pglb_edge_softmax_bwd_csr_f32", ops._ptr(ipd), None,
                                                    ops._ptr(al), ops._ptr(gr), ops._ptr(gl), G.N, G.E, 3,
                                                    ops._stream()), ["edge_softmax_bwd"]))
    xa = _dev(np.ones((G.N, 20)))
    src, dst = _i64(G.edges[:, 0]), _i64(G.edges[:, 1])
    calls.append(("sddmm vec4", lambda: ops.sddmm_dot(xa, xa, src, dst, 5, 4), ["sddmm_dot<4>"]))
    calls.append(("sddmm vec1", lambda: ops.sddmm_dot(xa, xa, src, dst, 4, 5), ["sddmm_dot<1>"]))

    def sg():
        fwd = g._fwd_csr()
        fd, ad = _dev(np.ones((G.N, 128))), _dev(np.full(128, 0.5))
        dsd, out, ws = _dev(np.ones((G.E, 4))), torch.zeros((G.N, 128), device="cuda"), _ws(G.N, G.E, 128)
        P = ops._ptr
        _call("pglb_gatv2_score_grad_f32", P(fwd["indptr"]), P(fwd["cols"]), P(fwd["eid"]), P(fd), 128, P(ad), 0.5,
              P(dsd), P(out), 128, G.N, G.E, 4, 32, 0, P(ws), ws.numel(), ops._stream())
    calls.append(("gatv2 score grad", sg, ["gatv2_score_grad"]))
    ipr = _i64(np.r_[0, np.cumsum(READOUT_LENS)])
    xr = _dev(np.ones((int(sum(READOUT_LENS)), 16)))
    gate, qr = _dev(np.zeros(int(sum(READOUT_LENS)))), _dev(np.ones((len(READOUT_LENS), 16)))
    calls.append(("readout gate", lambda: ops._attn_readout_raw(xr, ipr, gate, None, max(READOUT_LENS)),
                  ["readout gate", "readout merge"]))
    calls.append(("readout query", lambda: ops._attn_readout_raw(xr, ipr, None, qr, max(READOUT_LENS)),
                  ["readout query", "readout merge"]))

    def readout_bwd(use_query):
        x = xr.clone().requires_grad_(True)
        if use_query:
            ops.attn_readout(x, ipr, query=qr.clone().requires_grad_(True)).sum().backward()
        else:
            ops.attn_readout(x, ipr, gate=gate.clone().requires_grad_(True)).sum().backward()
    calls.append(("readout backward gate", lambda: readout_bwd(False), ["readout bwd gate"]))
    calls.append(("readout backward query", lambda: readout_bwd(True), ["readout bwd query",
                                                                         "readout merge grad query"]))
    for kind in ("gat", "dot", "v2"):
        for dtype, drop in ((torch.float32, False), (torch.bfloat16, True)):
            half = dtype != torch.float32
            if kind == "gat":
                f = _features(rng, G.N, 128, half)
                a_s4, a_d4 = gat_inputs(G, 4, rng)
                ins = (f, a_s4, a_d4)
                out, lse = run_gat(G, G.N, f, a_s4, a_d4, 0.2, 4, 32, dtype, "drop" if drop else "train")
            elif kind == "dot":
                q, k = dot_inputs(G, 4, 32, rng)
                ins = (q, k, _features(rng, G.N, 128, half))
                out, lse = run_scored("dot", G, ins, 4, 32, dtype, drop)
            else:
                ins = v2_inputs(G, 4, 32, rng, half)
                out, lse = run_scored("v2", G, ins, 4, 32, dtype, drop, 0.2)
            g2 = _dev(np.ones((G.N, 128)), dtype)
            name = {"gat": "gat_bwd_edge", "dot": "dot_bwd_edge", "v2": "gatv2_bwd_edge"}[kind] + \
                (" bf16 drop" if drop else " f32")
            calls.append(("%s backward %s" % (kind, name),
                          lambda kind=kind, ins=ins, out=out, lse=lse, g2=g2, dtype=dtype, drop=drop:
                          run_edge_bwd(kind, G, ins, out, lse, g2, 4, 32, dtype, drop, 0.2),
                          [name] + (["gatv2_ga_reduce"] if kind == "v2" else [])))
    return calls


@pytest.mark.gpu
def test_route_coverage():
    """Each representative call reaches the kernels it claims, and together they reach every softmax route."""
    if CHILD:
        pytest.skip("routing under the default switches only")
    a = torch.ones(1024, device="cuda")
    names, _ = _kernels_of(lambda: a.add_(1))
    if not names:
        pytest.skip("torch.profiler records no CUDA kernels here (probe: a plain torch kernel)")
    hit, failures, seen = set(), [], set()
    for label, fn, claims in _route_calls():
        names, _ = _kernels_of(fn)
        seen |= set(names)
        for cl in claims:
            if any(re.search(ROUTES[cl], nm) for nm in names):
                hit.add(cl)
            else:
                failures.append("%s: expected %s; launched %s" % (label, cl, sorted(set(names))))
    assert not failures, "\n".join(failures)
    missing = sorted(set(ROUTES) - hit)
    assert not missing, "routes not reached: %s" % missing
    print("routes reached: %d; softmax kernels seen: %s" % (len(hit), sorted(
        nm for nm in seen if re.search(r"gat5|softmax|fixup_gat|readout|ro_merge|score_grad|sddmm", nm))))
