"""Every tensor-core GEMM route -- the dense transform (pglb_linear_tf32x3_f32: linear_wgmma_kernel and the two
linear_tf32x3_kernel<N>) and RGCNConv's forward, grad x and grad W (rgcn_agg_kernel<NP>,
rgcn_wgrad_kernel<DP, NP>, rgcn_wsum_kernel) -- bit for bit against an exact float64 reference.

What each kernel claims to compute.  Every operand v is split into tf32 halves and three products are accumulated in
fp32:  x_lo w_hi + x_hi w_lo + x_hi w_hi  (x_lo w_lo is dropped).
  - mma.sync kernels (linear_tc.cu, rgcn.cu), both operands:  hi = rna(v), lo = rna(v - hi)  (cvt.rna.tf32.f32: round
    to nearest, ties away from zero);
  - linear_wgmma_kernel, W: the same; x: the raw fp32 tile is the hi operand and .tf32 ignores its low 13 bits, so
    hi = trunc(x), lo = trunc(x - trunc(x))  (lo is stored as fp32 and truncated by the instruction in turn).
`rna_tf32` / `trunc_tf32` / `split_rna` / `split_trunc` restate this in numpy and `split_blocks` forms the three
operand pairs.  RGCN's A tile (the per-(row, relation) means) is reproduced bit for bit by `run_sums`: the kernel adds
a run's rows in slot order with fmaf(1, v, acc) = fl(acc + v) (fmaf(w, v, acc) with per-slot weights) and divides by
the run length with an IEEE division.

The regime.  `gemm_regime` takes, per output element, a common quantum q of every nonzero product term and of the bias
(the product of the smallest lowest set bit in the element's row of each left operand and in its column of the right
one, which every term of the pair is a multiple of) and asserts  sum |terms| + |bias| < 2^23 q.  Then every product is
exact, every partial sum in any order is a multiple of q below 2^23 q (so exact in fp32), and so is every alignment
inside an mma even for an adder that keeps only 24 bits aligned to its largest addend and truncates: the result is
the exact value whatever the accumulation order, tile cut, lap or work-item split, and the kernels must return it bit
for bit.  A case the helper refuses is a bug in the test, never a tolerance.  Two families are used:
  - D (dense, lo = 0): small integers, exact in tf32, times one power of two per operand -- pins the layout (TMA
    swizzle, W^T build, fragment indices, epilogue column mapping) for every (m, n, k);
  - L (sparse, lo != 0): at most two nonzero k terms per output, values s 2^a (h + l 2^-14) with odd h in [9, 15] and
    odd l in [1, 7] (l of either sign for mma.sync x and every W, positive for wgmma's x so truncation gives the
    short split).  Each lo term is then an odd multiple of 2^-14 2^a and a 2-term element needs 22.8 of the 23 bits.
    A missing or doubled term, or a wrong split, moves the element by at least q.
RGCN's exact cases use power-of-two run lengths (1 up to an 8192-slot hub, so A = S / 2^j is exact and carries a lo
once |S| > 2^11), integer x and g, and integer W or a lo-bearing W with at most one nonzero per row and column.

Random data (no regime) is checked per element: |got - ref| <= `gemm_bound` (derivation in its docstring), with rows
scaled by powers of two over +-30 so that small rows are checked at their own scale, and by two bit identities:
permuting x's rows permutes the output's rows, and scaling a row by 2^s scales its output row by 2^s.

The C entries are also called through ctypes with strided x (NaN in the padding) and an output view inside a wider,
sentinel-filled buffer (ldo > N, rows after M): every sentinel must survive.  `test_route_coverage` records the
kernels each case launches (torch.profiler) and asserts that every instantiation was reached and that each case ran
where it claims."""
import ctypes
import re

import numpy as np
import pytest
import torch

from oracle import oracle_conv as OC
from test_gpu_exact_routes import _kernels_of

NB = 1021                       # distinct x rows of a dense regime case; longer cases repeat them with period NB
M_LADDER = ("1", "2", "15", "16", "17", "63", "64", "65", "127", "128", "129", "193", "wg-1", "wg", "wg+1",
            "mma-1", "mma+1", "laps")

# ----------------------------------------------------------------------------------------------------------------
# tf32 split emulation and the exact reference
# ----------------------------------------------------------------------------------------------------------------

_MASK = np.uint32(0xffffe000)


def _bits(v):
    return np.ascontiguousarray(v, np.float32).view(np.uint32)


def rna_tf32(v):
    """cvt.rna.tf32.f32: add half a tf32 ulp to the magnitude bits, drop the low 13 (ties away from zero)."""
    return ((_bits(v) + np.uint32(0x1000)) & _MASK).view(np.float32)


def trunc_tf32(v):
    """What .tf32 reads from a raw fp32 value: the low 13 mantissa bits ignored."""
    return (_bits(v) & _MASK).view(np.float32)


def split_rna(v):
    v = np.asarray(v, np.float32)
    hi = rna_tf32(v)
    return hi, rna_tf32(v - hi)


def split_trunc(v):
    v = np.asarray(v, np.float32)
    hi = trunc_tf32(v)
    return hi, trunc_tf32(v - hi)


def split_blocks(x, w, x_trunc=False, rows=None):
    """The three operand pairs (x_lo, w_hi), (x_hi, w_lo), (x_hi, w_hi) in float64, as gemm_regime blocks."""
    xh, xl = (split_trunc if x_trunc else split_rna)(x)
    wh, wl = split_rna(w)
    f = lambda a: np.asarray(a, np.float64)
    return [(rows, f(xl), f(wh)), (rows, f(xh), f(wl)), (rows, f(xh), f(wh))]


def ref_exact(x, w, bias=None, act=None, x_trunc=False):
    """sum_k (x_hi w_hi + x_lo w_hi + x_hi w_lo) in float64, + bias, then ReLU (exact inside the regime)."""
    out = sum(X @ W for _, X, W in split_blocks(x, w, x_trunc))
    if bias is not None:
        out = out + np.asarray(bias, np.float64)
    return np.maximum(out, 0.0) if act == "relu" else out


def _lsb_log2(a):
    """log2 of the lowest set bit of each value (+inf for 0)."""
    a = np.abs(np.asarray(a, np.float64))
    m, e = np.frexp(a)
    mi = (m * 2.0 ** 53).astype(np.int64)
    _, el = np.frexp((mi & -mi).astype(np.float64))
    out = (e - 53 + el - 1).astype(np.float64)
    out[a == 0] = np.inf
    return out


def gemm_regime(blocks, shape, bias=None, what="case"):
    """Exact float64 value of sum over blocks of X @ W (+ bias per column), after asserting that it is exact in fp32
    in any order.  blocks: (rows, X [m, K], W [K, N]); rows (None = all) are the distinct output rows the block adds
    into.  Per element, q = min over blocks of lsb_row(X) * lsb_col(W) and lsb(bias): every term is a multiple of q
    (lowest set bits multiply), and q is no larger than the smallest lowest set bit of any term, so the test below
    is, if anything, stricter than one against the terms' own smallest bit."""
    S = np.zeros(shape)
    ref = np.zeros(shape)
    lq = np.full(shape, np.inf)
    for rows, X, W in blocks:
        X, W = np.asarray(X, np.float64), np.asarray(W, np.float64)
        assert np.isfinite(X).all() and np.isfinite(W).all(), what
        if X.shape[0] == 0:
            continue
        s, r = np.abs(X) @ np.abs(W), X @ W
        q = _lsb_log2(X).min(1)[:, None] + _lsb_log2(W).min(0)[None, :] if X.shape[1] else np.full(s.shape, np.inf)
        if rows is None:
            S += s
            ref += r
            lq = np.minimum(lq, q)
        else:
            assert np.unique(rows).size == len(rows), what
            S[rows] += s
            ref[rows] += r
            lq[rows] = np.minimum(lq[rows], q)
    if bias is not None:
        b = np.asarray(bias, np.float64)
        S += np.abs(b)[None, :]
        ref += b[None, :]
        lq = np.minimum(lq, _lsb_log2(b)[None, :])
    bad = np.argwhere(~(S < np.exp2(lq + 23)))
    if bad.size:
        i, j = (int(v) for v in bad[0])
        raise AssertionError("gemm_regime refuses %s: %d elements over the bit budget; first (%d, %d): sum|terms| = "
                             "%r, q = 2^%g (needs < 2^23 q)" % (what, bad.shape[0], i, j, S[i, j], lq[i, j]))
    return ref


def gemm_bound(absdot, kterms, x_trunc=False, absbias=0.0, adds=1.0):
    """Per-element bound on |got - ref| for a 3xTF32 dot product of kterms k-positions (padded to the mma's k8),
    ref = sum_k x_k w_k + b exactly, absdot = sum_k |x_k| |w_k|.
      split (x = x_hi + x_lo + dx, w likewise; the kernel forms x w - x_lo w_lo - x_hi dw - x_lo dw - dx w):
        rna / rna:   |x_lo| <= 2^-11 |x|, |dx| <= 2^-22 |x|          -> <= 6.01 2^-23 |x||w|, taken as 7
        trunc x:     |x_lo| <  2^-10 |x|, |dx| <  2^-20 |x|, w rna   -> <= 14.01 2^-23 |x||w|, taken as 15
      accumulation: 3 kterms / 8 mma instructions, each adding 8 products and the accumulator aligned to the
        largest addend and truncated (at most 9 addends each off by < 2^-23 of the sum of |terms|, which is
        <= (1 + 2^-8) absdot): 27 kterms / 8 (1 + 2^-8)
      epilogue and partial sums: `adds` round-to-nearest fp32 additions (bias, rgcn_wsum_kernel), each within
        2^-24 of |sum| <= absdot + |b|; +1 covers one.
    c = split + accumulation + adds, and |got - ref| <= c 2^-23 absdot + adds 2^-23 |b|."""
    c = (15.0 if x_trunc else 7.0) + 27.0 * kterms / 8.0 * (1 + 2.0 ** -8) + adds
    return c * 2.0 ** -23 * np.asarray(absdot, np.float64) + adds * 2.0 ** -23 * np.asarray(absbias, np.float64)


# ----------------------------------------------------------------------------------------------------------------
# dense regime cases
# ----------------------------------------------------------------------------------------------------------------

def lo_vals(rng, shape, neg_l=True):
    """s (h + l 2^-14): odd h in [9, 15], odd l in [1, 7] (of either sign when neg_l)."""
    h = rng.choice([9.0, 11.0, 13.0, 15.0], shape)
    l = rng.choice([1.0, 3.0, 5.0, 7.0], shape)
    if neg_l:
        l = l * rng.choice([-1.0, 1.0], shape)
    return rng.choice([-1.0, 1.0], shape) * (h + l * 2.0 ** -14)


def dense_case(regime, K, N, x_trunc, seed, B=NB):
    """(x [B, K], w [K, N], bias [N]) float32, exact in the regime.
    D: integers in [-3, 3] times 2^-5 (x) and 2^3 (w); rows of zeros, and one-hot rows x = 2^-5 e_0 whose
       pre-activation is exactly 0 in the even columns (bias = -x w there) and negative or positive elsewhere.
    L: per row two nonzero k (one on every 17th row, none on every 31st), positions sweeping all K columns over the
       rows; w dense lo-bearing times 2^-3; bias integers times 2^-3."""
    rng = np.random.default_rng(seed)
    if regime == "D":
        x = rng.integers(-3, 4, (B, K)).astype(np.float64)
        x[7::97] = 0.0
        x[11::97] = 0.0
        x[11::97, 0] = 1.0
        w = rng.integers(-3, 4, (K, N)).astype(np.float64)
        b = rng.integers(-3, 4, N).astype(np.float64)
        b[::2] = -w[0, ::2]
        x, w, b = x * 2.0 ** -5, w * 2.0 ** 3, b * 2.0 ** -2
    else:
        x = np.zeros((B, K))
        i = np.arange(B)
        k1 = i % K
        k2 = (k1 + 1 + (i // K) % (K - 1)) % K
        x[i, k1] = lo_vals(rng, B, neg_l=not x_trunc)
        two = (i % 17 != 5)
        x[i[two], k2[two]] = lo_vals(rng, int(two.sum()), neg_l=not x_trunc)
        x[i % 31 == 7] = 0.0
        w = lo_vals(rng, (K, N)) * 2.0 ** -3
        b = rng.integers(-3, 4, N) * 2.0 ** -3
    x32, w32, b32 = (np.asarray(a, np.float32) for a in (x, w, b))
    assert np.array_equal(x32, x) and np.array_equal(w32, w) and np.array_equal(b32, b)
    return x32, w32, b32


_DENSE = {}


def dense_ref(regime, K, N, x_trunc, with_bias, act):
    """(x_base, w, b or None, exact reference on x_base), through gemm_regime; cached."""
    key = (regime, K, N, x_trunc, with_bias, act)
    if key not in _DENSE:
        x, w, b = dense_case(regime, K, N, x_trunc, seed=K * 1000 + N + (regime == "L"))
        b = b if with_bias else None
        ref = gemm_regime(split_blocks(x, w, x_trunc), (x.shape[0], N), b, what="dense %s" % (key,))
        if regime == "L":
            xl, wl = (split_trunc if x_trunc else split_rna)(x)[1], split_rna(w)[1]
            assert (xl != 0).sum() > x.shape[0] and (wl != 0).all()     # the lo terms are really there
        _DENSE[key] = (x, w, b, np.maximum(ref, 0.0) if act == "relu" else ref)
    return _DENSE[key]


# ----------------------------------------------------------------------------------------------------------------
# RGCN: numpy model of the typed CSRs, the A tile and the regime graphs
# ----------------------------------------------------------------------------------------------------------------

def _runs(keys_row, keys_rel):
    """(beg, end) of the maximal (row, relation) groups of a slot sequence."""
    E = keys_row.shape[0]
    brk = np.ones(E, bool)
    brk[1:] = (keys_row[1:] != keys_row[:-1]) | (keys_rel[1:] != keys_rel[:-1])
    beg = np.flatnonzero(brk)
    return beg, np.r_[beg[1:], E].astype(np.int64)


class TypedModel(object):
    """heter_graph.typed_csr restated: dst CSR (slots grouped by relation ascending, eid ascending inside), its runs,
    the src CSR and its per-slot weights 1 / cnt_r(dst)."""

    def __init__(self, edge_lists, n):
        self.n, self.R = n, len(edge_lists)
        src = np.concatenate([e[:, 0] for e in edge_lists]).astype(np.int64)
        dst = np.concatenate([e[:, 1] for e in edge_lists]).astype(np.int64)
        rel = np.concatenate([np.full(e.shape[0], r, np.int64) for r, e in enumerate(edge_lists)])
        o = np.argsort(dst, kind="stable")
        self.indptr = np.r_[0, np.cumsum(np.bincount(dst, minlength=n))].astype(np.int64)
        self.cols, self.rel, rows = src[o], rel[o], dst[o]
        self.beg, self.end = _runs(rows, self.rel)
        self.run_row, self.run_rel = rows[self.beg], self.rel[self.beg]
        cnt_e = np.empty(src.shape[0], np.int64)
        cnt_e[o] = np.repeat(self.end - self.beg, self.end - self.beg)
        so = np.argsort(src, kind="stable")
        self.s_indptr = np.r_[0, np.cumsum(np.bincount(src, minlength=n))].astype(np.int64)
        self.s_cols, self.s_rel, s_rows = dst[so], rel[so], src[so]
        self.s_w = (1.0 / cnt_e[so].astype(np.float32)).astype(np.float32)
        self.s_beg, self.s_end = _runs(s_rows, self.s_rel)
        self.s_run_row, self.s_run_rel = s_rows[self.s_beg], self.s_rel[self.s_beg]


def run_sums(x32, cols, beg, end, w=None):
    """run_sum of csrc/rgcn.cu for every run: the rows x[cols[j]] added in slot order in fp32, acc = fmaf(w_j, v,
    acc) (= fl(acc + v) without weights).  fmaf is formed in float64 (w v is exact there) and rounded once, exact
    whenever the float64 sum is."""
    D = x32.shape[1]
    out = np.zeros((beg.shape[0], D), np.float32)
    L = end - beg
    for ln in np.unique(L):
        sel = np.flatnonzero(L == ln)
        b = beg[sel]
        acc = np.zeros((sel.shape[0], D), np.float32)
        for t in range(int(ln)):
            v = x32[cols[b + t]]
            if w is None:
                acc = acc + v
            else:
                acc = (w[b + t][:, None].astype(np.float64) * v + acc).astype(np.float32)
        out[sel] = acc
    return out


def a_tiles(m, x32):
    """A of every dst run, fl(run_sum / len) with an IEEE division, as the forward and grad W kernels form it."""
    return run_sums(x32, m.cols, m.beg, m.end) / (m.end - m.beg).astype(np.float32)[:, None]


def rgcn_refs(m, x, w3, g, regime=True):
    """Forward, grad x, grad W of the kernels' arithmetic: exact references through gemm_regime (regime=True) or
    float64 products of the emulated A tiles with per-element bounds (regime=False): (fwd, gx, gw, bounds)."""
    R, D, O = w3.shape
    A = a_tiles(m, x)
    Ag = run_sums(g, m.s_cols, m.s_beg, m.s_end, m.s_w)
    wT = np.ascontiguousarray(np.transpose(w3, (0, 2, 1)))
    outs, bounds = [], []
    for (rows_all, rel_all, AA, WW, n_out, K) in ((m.run_row, m.run_rel, A, w3, O, D),
                                                 (m.s_run_row, m.s_run_rel, Ag, wT, D, O)):
        blocks = []
        absdot = np.zeros((m.n, n_out))
        nrel = np.bincount(rows_all, minlength=m.n)
        for r in np.unique(rel_all):
            sel = rel_all == r
            if regime:
                blocks += split_blocks(AA[sel], WW[r], rows=rows_all[sel])
            else:
                blocks.append((rows_all[sel], AA[sel].astype(np.float64), WW[r].astype(np.float64)))
                absdot[rows_all[sel]] += np.abs(AA[sel].astype(np.float64)) @ np.abs(WW[r].astype(np.float64))
        if regime:
            outs.append(gemm_regime(blocks, (m.n, n_out), what="rgcn %dx%d" % (K, n_out)))
        else:
            outs.append(sum_blocks(blocks, (m.n, n_out)))
            bounds.append(gemm_bound(absdot, (nrel * ((K + 7) & ~7))[:, None], adds=0.0))
    gw = np.zeros((R, D, O))
    gb = np.zeros((R, D, O))
    for r in range(R):
        sel = m.run_rel == r
        if not sel.any():
            continue
        Ar, Gr = A[sel].T, g[m.run_row[sel]]
        if regime:
            gw[r] = gemm_regime(split_blocks(Ar, Gr), (D, O), what="rgcn gW[%d]" % r)
        else:
            gw[r] = Ar.astype(np.float64) @ Gr.astype(np.float64)
            gb[r] = (np.abs(Ar.astype(np.float64)) @ np.abs(Gr.astype(np.float64)))
    if not regime:
        bounds.append(gb)
    return outs[0], outs[1], gw, bounds


def sum_blocks(blocks, shape):
    out = np.zeros(shape)
    for rows, X, W in blocks:
        out[rows] += X @ W
    return out


def rgcn_graph(n, R, seed, lo_w=False):
    """Edge lists ([E_r, 2] (src, dst)) of R relations over n nodes with power-of-two run lengths:
      - about 15% of the rows receive nothing; the others take 0-3 relations (0-1 with lo_w) from a window that
        moves with the 64-row tile (6 more relations than an even share), so relations are absent from whole tiles;
        runs of 1-8 slots (1-4 with lo_w);
      - relation R // 2 (R >= 3) has no edges at all;
      - relation `many` gets a 1-slot run in every third live row: more runs than a weight-gradient work item;
      - without lo_w: hub rows 3, n / 4 + 10 and n / 2 + 7 each hold one run of 8192, 2048 and 512 slots (1024 and 256 for R = 1)
        in a hub relation no other row uses (R >= 3), from 48 dedicated source nodes with no other out-edges, whose x
        is positive in every 8th column so that A = S / 2^j carries a lo there;
      - with lo_w every node is the source of at most 3 edges."""
    rng = np.random.default_rng(seed)
    empty = R // 2 if R >= 3 else None
    hub_rel = None if lo_w else (R - 1 if R >= 3 else 0)
    hubs = [] if lo_w else list(zip([3, n // 4 + 10, n // 2 + 7], [8192, 2048, 512] if R >= 3 else [1024, 256]))
    pool = rng.choice(n, 48, replace=False)
    ordinary = np.setdiff1d(np.arange(n), pool)
    live = [r for r in range(R) if r != empty and (r != hub_rel or R == 1)]
    many = live[0]
    cap = np.full(n, 3) if lo_w else None
    edges = [[] for _ in range(R)]

    def pick(k):
        if not lo_w:
            return rng.choice(ordinary, k)
        avail = np.flatnonzero(cap > 0)
        if avail.size < k:
            return None
        s = rng.choice(avail, k, replace=False)
        cap[s] -= 1
        return s

    hub_rows = {h for h, _ in hubs}
    jmax = 2 if lo_w else 3
    tiles = -(-n // 64)
    width = min(len(live), 6 + -(-len(live) // tiles))
    for d in range(n):
        if d in hub_rows or rng.random() < 0.15:
            continue
        t = d // 64
        win = [live[(t * len(live) // tiles + i) % len(live)] for i in range(width)]
        rels = set(rng.choice(win, int(rng.integers(0, 2 if lo_w else 4)), replace=True).tolist())
        if d % 3 == 0:
            rels.add(many)
        for r in sorted(rels):
            ln = 1 if (r == many and d % 3 == 0) else 1 << int(rng.integers(0, jmax + 1))
            s = pick(ln)
            if s is not None:
                edges[r] += [(int(v), d) for v in s]
    for h, ln in hubs:
        edges[hub_rel] += [(int(v), h) for v in rng.choice(pool, ln)]
    lists = [np.asarray(e, np.int64).reshape(-1, 2) for e in edges]
    for r in range(R):      # shuffle each relation's edge ids: slot order inside a run is then not source order
        lists[r] = lists[r][rng.permutation(lists[r].shape[0])]
    return lists, pool


def rgcn_operands(n, R, D, O, pool, seed, lo_w=False):
    """x [n, D], w3 [R, D, O], g [n, O] float32 for the regime: integers (in [-3, 3]; [-2, 2] with lo_w), x of the
    hub sources in [1, 3] in every 8th column and in [-1, 1] elsewhere; W integer, or with lo_w a lo-bearing partial
    permutation (at most one nonzero per row and per column)."""
    rng = np.random.default_rng(seed)
    a = 2 if lo_w else 3
    x = rng.integers(-a, a + 1, (n, D)).astype(np.float32)
    g = rng.integers(-a, a + 1, (n, O)).astype(np.float32)
    if not lo_w:
        x[pool] = rng.integers(-1, 2, (pool.shape[0], D))
        x[np.ix_(pool, np.arange(0, D, 8))] = rng.integers(1, 4, (pool.shape[0], (D + 7) // 8))
        w3 = rng.integers(-3, 4, (R, D, O)).astype(np.float32)
    else:
        w3 = np.zeros((R, D, O), np.float32)
        k = min(D, O)
        for r in range(R):
            rows, cols = rng.permutation(D)[:k], rng.permutation(O)[:k]
            w3[r, rows, cols] = lo_vals(rng, k)
    return x, w3, g


# ----------------------------------------------------------------------------------------------------------------
# CPU tests: split, reference, regime helper, A tile
# ----------------------------------------------------------------------------------------------------------------

def test_tf32_split_hand_values():
    f = lambda bits: np.array([bits], np.uint32).view(np.float32)
    one = 1.0
    tie = f(0x3f801000)          # 1 + 2^-11: exactly half a tf32 ulp above 1
    assert rna_tf32(tie)[0] == one + 2.0 ** -10 and trunc_tf32(tie)[0] == one      # ties away from zero
    assert rna_tf32(-tie)[0] == -(one + 2.0 ** -10) and trunc_tf32(-tie)[0] == -one
    below = f(0x3f800fff)        # just under the tie: both keep 1
    assert rna_tf32(below)[0] == one and trunc_tf32(below)[0] == one
    v = f(0x3f801800)            # 1 + 2^-11 + 2^-12: rounding and truncation differ
    assert rna_tf32(v)[0] == one + 2.0 ** -10 and trunc_tf32(v)[0] == one
    h, l = split_rna(v)
    assert h[0] == one + 2.0 ** -10 and l[0] == -(2.0 ** -12)       # negative lo after rounding up
    h, l = split_trunc(v)
    assert h[0] == one and l[0] == 2.0 ** -11 + 2.0 ** -12
    x = np.float32(-(13 + 5 * 2.0 ** -14))                          # regime L value, negative
    h, l = split_rna(x)
    assert h == -13.0 and l == -5 * 2.0 ** -14
    h, l = split_rna(np.float32(13 - 5 * 2.0 ** -14))               # negative l: rna gives the short split
    assert h == 13.0 and l == -5 * 2.0 ** -14
    h, l = split_trunc(np.float32(13 - 5 * 2.0 ** -14))             # ... truncation the long one
    assert h == 13.0 - 2.0 ** -7 and l == 2.0 ** -7 - 5 * 2.0 ** -14
    for v in (3.0, -0.375, 2.0 ** -30, 1536.0):                     # tf32-exact: lo = 0 under both
        for s in (split_rna, split_trunc):
            h, l = s(np.float32(v))
            assert h == v and l == 0.0
    # a lo the instruction itself truncates: 1 + 2^-11 + 2^-23 -> lo = 2^-11 + 2^-23 keeps 2^-11 only
    h, l = split_trunc(f(0x3f801001))
    assert h == one and l == 2.0 ** -11


def test_reference_matches_fp64_within_split_error():
    rng = np.random.default_rng(3)
    for K, x_trunc in ((128, False), (128, True), (36, False)):
        x = (rng.standard_normal((300, K)) * np.exp2(rng.integers(-30, 31, (300, 1)))).astype(np.float32)
        w = rng.standard_normal((K, 64)).astype(np.float32)
        ref = ref_exact(x, w, x_trunc=x_trunc)
        exact = x.astype(np.float64) @ w.astype(np.float64)
        absdot = np.abs(x.astype(np.float64)) @ np.abs(w.astype(np.float64))
        err = np.abs(ref - exact)
        split_c = 15.0 if x_trunc else 7.0
        assert (err <= split_c * 2.0 ** -23 * absdot).all()
        assert err.max() > 0                                        # x_lo w_lo really is dropped
        # a missing x_lo w_hi term would be far outside the split's error
        xl = (split_trunc if x_trunc else split_rna)(x)[1]
        assert (np.abs(xl.astype(np.float64) @ w) > 4 * split_c * 2.0 ** -23 * absdot).mean() > 0.8


def test_gemm_regime_accepts_the_generators_and_refuses_outside():
    for regime in ("D", "L"):
        for K, N, tr in ((128, 128, True), (128, 64, False), (4, 64, False), (100, 128, False)):
            for wb in (False, True):
                dense_ref(regime, K, N, tr, wb, "relu" if wb else None)
    rng = np.random.default_rng(5)
    # dense lo-bearing operands: 128 lo terms per element are far over the budget
    x, w = lo_vals(rng, (64, 128)).astype(np.float32), lo_vals(rng, (128, 64)).astype(np.float32)
    with pytest.raises(AssertionError, match="gemm_regime refuses"):
        gemm_regime(split_blocks(x, w), (64, 64))
    # three lo-bearing k terms per element: just over the 23 bits two of them fit in
    x = np.zeros((64, 8), np.float32)
    x[:, :3] = 15 + 7 * 2.0 ** -14
    w = np.full((8, 64), 15 + 7 * 2.0 ** -14, np.float32)
    gemm_regime(split_blocks(x[:, :2].copy(), w[:2].copy()), (64, 64))
    with pytest.raises(AssertionError, match="gemm_regime refuses"):
        gemm_regime(split_blocks(x, w), (64, 64))
    # a bias off the quantum (2^-20 against q = 2^-14) and an integer bias too large for a lo-bearing element
    with pytest.raises(AssertionError, match="gemm_regime refuses"):
        gemm_regime(split_blocks(x[:, :2].copy(), w[:2].copy()), (64, 64), np.full(64, 2.0 ** -20))
    with pytest.raises(AssertionError, match="gemm_regime refuses"):
        gemm_regime(split_blocks(x[:, :2].copy(), w[:2].copy()), (64, 64), np.full(64, 64.0))
    # inside the regime the float64 reference is the exact sum
    x, w, b = dense_case("L", 64, 64, False, 9, B=200)
    got = gemm_regime(split_blocks(x, w), (200, 64), b)
    import fractions
    for i, j in ((0, 0), (17, 5), (199, 63)):
        xh, xl = split_rna(x[i])
        wh, wl = split_rna(w[:, j])
        F = fractions.Fraction
        want = sum(F(float(a)) * F(float(c)) for a, c in zip(np.r_[xl, xh, xh], np.r_[wh, wl, wh])) + F(float(b[j]))
        assert F(got[i, j]) == want


@pytest.mark.parametrize("R,lo_w", [(1, False), (3, False), (64, False), (300, False), (3, True), (64, True)])
def test_rgcn_regime_graphs(R, lo_w):
    """The generator's graphs have what the exact tests need, and every RGCN case is inside the regime."""
    n = 64 * 20 + 37
    el, pool = rgcn_graph(n, R, 40 + R, lo_w)
    m = TypedModel(el, n)
    ln = m.end - m.beg
    assert ((ln & (ln - 1)) == 0).all()                                  # power-of-two runs
    if not lo_w:
        assert ln.max() == (8192 if R >= 3 else 1024)
    assert (np.diff(m.indptr) == 0).sum() > n // 10                      # rows with no edges
    runs_per = np.bincount(m.run_rel, minlength=R)
    assert runs_per.max() > 64                                           # several work items for one relation
    if R >= 3:
        assert runs_per[R // 2] == 0
    if R == 300:
        assert (m.rel > 255).any()
    if R >= 64:
        tiles = m.run_row // 64
        assert all(np.unique(m.run_rel[tiles == t]).size < R for t in np.unique(tiles))
    cases = [c for c in RGCN_CASES if c[2] == R] or [(12, 36, R)]
    for D, O, _ in cases:
        x, w3, g = rgcn_operands(n, R, D, O, pool, 7, lo_w)
        fwd, gx, gw, _ = rgcn_refs(m, x, w3, g)
        A = a_tiles(m, x)
        if not lo_w:
            assert (split_rna(A)[1] != 0).any()                          # the hub's A carries a lo
        else:
            assert (split_rna(w3)[1] != 0).sum() >= R * min(D, O)


def test_rgcn_a_tile_matches_oracle_means():
    """A_r (the mean of x[src] over d's r-run) from the slot-order emulation equals the reference's
    send_u_recv(mean) of oracle_conv.rgcn_conv with W_r = I and the other relations zeroed: exactly on a regime
    graph, within the fp32 summation bound on random x."""
    n, R, D = 64 * 3 + 5, 3, 8
    el, pool = rgcn_graph(n, R, 2)
    m = TypedModel(el, n)
    rng = np.random.default_rng(1)
    for exact in (True, False):
        x = rgcn_operands(n, R, D, D, pool, 3)[0] if exact else rng.standard_normal((n, D)).astype(np.float32)
        A = a_tiles(m, x)
        for r in range(R):
            w = np.zeros((R, D, D))
            w[r] = np.eye(D)
            want = OC.rgcn_conv([("e%d" % i, e) for i, e in enumerate(el)], n, x.astype(np.float64), w)
            got = np.zeros((n, D))
            sel = m.run_rel == r
            got[m.run_row[sel]] = A[sel]
            if exact:
                assert np.array_equal(got, want), r
            else:       # slot-order fp32 sum of L rows, then a division: (L - 1) u mean|x| + u |mean|
                mabs = OC.rgcn_conv([("e%d" % i, e) for i, e in enumerate(el)], n, np.abs(x.astype(np.float64)), w)
                ln = np.zeros((n, 1))
                ln[m.run_row[sel], 0] = m.end[sel] - m.beg[sel]
                assert (np.abs(got - want) <= 2.0 ** -24 * (ln * mabs + np.abs(want))).all(), r


# ----------------------------------------------------------------------------------------------------------------
# GPU helpers
# ----------------------------------------------------------------------------------------------------------------

def _sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def m_of(label):
    sm = _sm()
    return {"wg-1": sm * 128 - 1, "wg": sm * 128, "wg+1": sm * 128 + 1, "mma-1": sm * 64 - 1, "mma+1": sm * 64 + 1,
            "laps": sm * 128 * 4 + 77}.get(label) or int(label)


def assert_exact(got, want, what, tile=64):
    """Value equality (a zero's sign is not compared); on failure name the first element, its tile and lap."""
    g = got.detach().double().cpu().numpy() if torch.is_tensor(got) else np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    assert g.shape == want.shape, (what, g.shape, want.shape)
    bad = np.argwhere(~(g == want))
    if bad.size:
        i, j = (int(v) for v in bad[0][:2])
        idx = tuple(bad[0])
        rows = np.unique(bad[:, 0])
        pytest.fail("%s: %d elements differ in %d rows; first %s (tile %d of %d rows, lap %d): got %r, want %r, "
                    "diff %r" % (what, bad.shape[0], rows.size, idx, i // tile, tile, i // tile // _sm(), g[idx],
                                 want[idx], g[idx] - want[idx]))


def assert_within(got, want, bound, what):
    g = got.detach().double().cpu().numpy()
    err = np.abs(g - want)
    bad = np.argwhere(~(err <= bound))
    assert bad.size == 0, "%s: %d elements off; first %s: got %r, want %r, bound %g" % (
        what, bad.shape[0], tuple(bad[0]), g[tuple(bad[0])], want[tuple(bad[0])], bound[tuple(bad[0])])


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def linear(x, w, b=None, act=None):
    from pgl_b200 import ops
    return ops._linear_tc_raw(x, w, b, act)


def _window(x, pad):
    """x on the device, read in place from a buffer with `pad` NaN columns after each row (ldx = K + pad)."""
    buf = torch.full((x.shape[0], x.shape[1] + pad), float("nan"), device="cuda")
    buf[:, :x.shape[1]] = _cuda(x)
    return buf[:, :x.shape[1]]


def check_dense(M, K, N, regime, x_trunc, with_bias, act, label, pad=0):
    x, w, b, ref = dense_ref(regime, K, N, x_trunc, with_bias, act)
    idx = np.arange(M) % x.shape[0]
    out = linear(_window(x[idx], pad), _cuda(w), _cuda(b) if b is not None else None, act)
    torch.cuda.synchronize()
    assert_exact(out, ref[idx], "%s M=%d K=%d N=%d regime %s bias=%s act=%s" % (label, M, K, N, regime, with_bias,
                                                                              act), tile=128 if x_trunc else 64)


VARIANTS = [("D", False, None), ("D", True, "relu"), ("L", False, None), ("L", True, "relu"), ("D", True, None)]


# ----------------------------------------------------------------------------------------------------------------
# GPU: dense transform, exact
# ----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("mlabel", M_LADDER)
def test_linear_exact_m_ladder(mlabel):
    """Every M of the ladder on wgmma (K = N = 128) and on the mma.sync kernel, both regimes."""
    M = m_of(mlabel)
    for K, N, tr, label in ((128, 128, True, "wgmma"), (128, 64, False, "mma.sync"), (60, 128, False, "mma.sync")):
        for regime, wb, act in VARIANTS:
            check_dense(M, K, N, regime, tr, wb, act, label)


@pytest.mark.gpu
@pytest.mark.parametrize("pad,N", [("8", 64), ("8", 128), ("16", 64), ("16", 128)])
def test_linear_exact_k_ladder(pad, N):
    """Every multiple of 4 in [4, 128] with x read in place at ldx = K + 8, a subset at ldx = K + 16 (NaN in the
    padding); K = N = 128 runs on wgmma (its TMA box strides over the padding), every other K on the mma.sync kernel."""
    ks = range(4, 129, 4) if pad == "8" else (4, 8, 12, 28, 36, 64, 68, 100, 124, 128)
    for K in ks:
        tr = K == 128 and N == 128
        for regime, wb, act in VARIANTS[:4]:
            check_dense(193, K, N, regime, tr, wb, act, "wgmma" if tr else "mma.sync", pad=int(pad))


SENT = np.array([0x7fc0beef], np.uint32).view(np.float32)[0]     # a NaN with a payload: only a write changes it


def _check_bounds_call(K, N, M, what, act=1, xpad=12):
    """The C entry with x strided (ldx = K + xpad, NaN in the padding and in the rows after M) and out a view at
    (1, 2) inside a sentinel-filled buffer with ldo = N + 6 and 70 rows after M: the sentinels survive and the
    in-bounds values equal the contiguous call's bit for bit."""
    from pgl_b200 import ops
    rng = np.random.default_rng(K + N + M)
    x = rng.standard_normal((M, K)).astype(np.float32)
    w = rng.standard_normal((K, N)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    ldx, ldo = K + xpad, N + 6
    xb = torch.full((M + 3, ldx), float("nan"), device="cuda")
    xb[:M, :K] = _cuda(x)
    ob = torch.empty((M + 71, ldo), device="cuda")
    ob.view(torch.int32).fill_(int(np.array([SENT]).view(np.int32)[0]))
    want = linear(_cuda(x), _cuda(w), _cuda(b), "relu" if act else None)
    wd, bd = _cuda(w), _cuda(b)
    P = ops._ptr
    out_ptr = ctypes.c_void_p(ob.data_ptr() + (ldo + 2) * 4)
    with torch.cuda.device(0):
        ops.check(ops.lib.pglb_linear_tf32x3_f32(P(xb), ldx, P(wd), P(bd), out_ptr, ldo, M, K, N, act, ops._stream()))
    torch.cuda.synchronize()
    bits = ob.view(torch.int32).cpu().numpy()
    inside = np.zeros(bits.shape, bool)
    inside[1:M + 1, 2:N + 2] = True
    sent = np.array([SENT]).view(np.int32)[0]
    assert (bits[~inside] == sent).all(), "%s: %d sentinels overwritten; first at %s" % (
        what, int((bits[~inside] != sent).sum()), tuple(np.argwhere((bits != sent) & ~inside)[0]))
    assert np.array_equal(bits[1:M + 1, 2:N + 2], want.view(torch.int32).cpu().numpy()), what
    # M = 0 launches nothing and writes nothing
    l0 = ops.launch_count()
    with torch.cuda.device(0):
        ops.check(ops.lib.pglb_linear_tf32x3_f32(P(xb), ldx, P(wd), P(bd), P(ob), ldo, 0, K, N, act, ops._stream()))
    torch.cuda.synchronize()
    assert ops.launch_count() == l0
    assert np.array_equal(ob.view(torch.int32).cpu().numpy(), bits)


@pytest.mark.gpu
@pytest.mark.parametrize("pad", ["8", "16"])
def test_linear_output_bounds(pad):
    sm = _sm()
    for K, N, M in ((128, 128, sm * 128 + 77), (128, 128, 100), (128, 64, sm * 64 + 3), (100, 128, 1000),
                    (36, 64, 77), (4, 128, 5)):
        _check_bounds_call(K, N, M, "K=%d N=%d M=%d ldx=K+%s" % (K, N, M, pad), act=M % 2, xpad=int(pad))


# ----------------------------------------------------------------------------------------------------------------
# GPU: dense transform, random data (bit identities and per-element bounds)
# ----------------------------------------------------------------------------------------------------------------

LIN_RANDOM = [(128, 128, "8"), (128, 64, "8"), (100, 128, "16"), (128, 64, "16"), (12, 64, "8")]


@pytest.mark.gpu
@pytest.mark.parametrize("K,N,pad", LIN_RANDOM)
def test_linear_random_identities_and_bounds(K, N, pad):
    """Rows permuted -> output rows permuted bit for bit; a row times 2^s -> its output row times 2^s bit for bit
    (no bias, s in [-30, 30]); and every element of a call on rows scaled by 2^[-30, 30], with bias and ReLU, read in
    place at ldx = K + pad, within gemm_bound of the float64 product."""
    x_trunc = K == 128 and N == 128
    M = _sm() * 128 * 2 + 77
    rng = np.random.default_rng(K * N)
    x = rng.standard_normal((M, K)).astype(np.float32)
    w = rng.standard_normal((K, N)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    xd, wd = _cuda(x), _cuda(w)
    base = linear(xd, wd)
    perm = rng.permutation(M)
    assert_exact(linear(_cuda(x[perm]), wd), base.cpu().numpy()[perm], "row permutation K=%d N=%d" % (K, N))
    s = rng.integers(-30, 31, (M, 1))
    xs = (x * np.exp2(s)).astype(np.float32)
    assert_exact(linear(_cuda(xs), wd), base.double().cpu().numpy() * np.exp2(s), "row scaling K=%d N=%d" % (K, N))
    got = linear(_window(xs, int(pad)), wd, _cuda(b), "relu")
    x64, w64 = xs.astype(np.float64), w.astype(np.float64)
    pre = x64 @ w64 + b
    bound = gemm_bound(np.abs(x64) @ np.abs(w64), (K + 7) & ~7, x_trunc, np.abs(b)[None, :])
    assert_within(got, np.maximum(pre, 0.0), bound, "per-element bound K=%d N=%d" % (K, N))


# ----------------------------------------------------------------------------------------------------------------
# GPU: RGCN
# ----------------------------------------------------------------------------------------------------------------

# (D, O, R): every agg<32|64|128> forward (by O) and grad x (by D), every wgrad<64|128, 32|64|128>, D and O not
# multiples of 8, R up to 300 (int16 relation ids above 255)
RGCN_CASES = [(4, 12, 1), (12, 4, 3), (20, 100, 64), (32, 128, 3), (36, 20, 300), (64, 64, 3), (100, 12, 3),
              (124, 36, 64), (128, 128, 300), (128, 32, 1), (64, 124, 3)]
RGCN_N = 64 * 20 + 37           # a last tile of 37 rows
_RG = {}


def rgcn_setup(R, lo_w):
    key = (R, lo_w)
    if key not in _RG:
        from pgl_b200.heter_graph import typed_csr
        el, pool = rgcn_graph(RGCN_N, R, 40 + R, lo_w)
        m = TypedModel(el, RGCN_N)
        fwd, bwd = typed_csr([_cuda(e) for e in el], RGCN_N)
        for k, v in (("indptr", m.indptr), ("cols", m.cols), ("rel", m.rel)):
            assert np.array_equal(fwd[k].cpu().numpy(), v), k
        for k, v in (("indptr", m.s_indptr), ("cols", m.s_cols), ("rel", m.s_rel), ("w", m.s_w)):
            assert np.array_equal(bwd[k].cpu().numpy(), v), k
        assert fwd["n_items"] > R, (fwd["n_items"], R)
        assert (np.diff(fwd["item_off"].cpu().numpy()) > 1).any()          # a relation split over several items
        _RG[key] = (el, pool, m, fwd, bwd)
    return _RG[key]


def rgcn_run(fwd, bwd, x, w3, g):
    from pgl_b200 import ops
    D, O = w3.shape[1], w3.shape[2]
    xd, wd, gd = _cuda(x), _cuda(w3), _cuda(g)
    out = ops._rgcn_agg_raw(fwd, xd, wd)
    gx = ops._rgcn_agg_raw(bwd, gd, wd.transpose(1, 2).contiguous(), slot_w=bwd["w"])
    gw = ops._rgcn_wgrad_raw(fwd, xd, gd, D, O)
    torch.cuda.synchronize()
    return out, gx, gw


def rgcn_bounds_call(fwd, x, w3, want, what):
    """pglb_rgcn_agg_f32 with x strided (NaN padding) into a view at (1, 2) of a sentinel buffer, ldo = O + 6."""
    from pgl_b200 import ops
    n, D = x.shape
    R, _, O = w3.shape
    ldx, ldo = D + 8, O + 6
    xb = torch.full((n, ldx), float("nan"), device="cuda")
    xb[:, :D] = _cuda(x)
    sent = np.array([SENT]).view(np.int32)[0]
    ob = torch.empty((n + 70, ldo), device="cuda")
    ob.view(torch.int32).fill_(int(sent))
    wd = _cuda(w3)
    P = ops._ptr
    with torch.cuda.device(0):
        ops.check(ops.lib.pglb_rgcn_agg_f32(P(fwd["indptr"]), P(fwd["cols"]), P(fwd["rel"]), None, P(xb), ldx, P(wd),
                                            R, D, O, ctypes.c_void_p(ob.data_ptr() + (ldo + 2) * 4), ldo, n,
                                            ops._stream()))
    torch.cuda.synchronize()
    bits = ob.view(torch.int32).cpu().numpy()
    inside = np.zeros(bits.shape, bool)
    inside[1:n + 1, 2:O + 2] = True
    assert (bits[~inside] == sent).all(), "%s: sentinel overwritten at %s" % (
        what, tuple(np.argwhere((bits != sent) & ~inside)[0]))
    assert_exact(ob[1:n + 1, 2:O + 2], want, what + " (ldo > N)")


@pytest.mark.gpu
@pytest.mark.parametrize("D,O,R", RGCN_CASES)
def test_rgcn_exact(D, O, R):
    """Forward, grad x and grad W bit for bit on the regime graph (integer W, hub runs up to 8192 slots), the forward
    once more through the C entry with ldo > N, and grad W of the relation without runs exactly 0."""
    el, pool, m, fwd, bwd = rgcn_setup(R, False)
    x, w3, g = rgcn_operands(RGCN_N, R, D, O, pool, D * 1000 + O)
    want_o, want_gx, want_gw, _ = rgcn_refs(m, x, w3, g)
    out, gx, gw = rgcn_run(fwd, bwd, x, w3, g)
    what = "D=%d O=%d R=%d" % (D, O, R)
    assert_exact(out, want_o, "rgcn forward " + what)
    assert_exact(gx, want_gx, "rgcn grad x " + what)
    assert_exact(gw, want_gw, "rgcn grad W " + what, tile=D)
    if R >= 3:
        assert not m.run_rel.tolist().count(R // 2) and (gw[R // 2] == 0).all()
    rgcn_bounds_call(fwd, x, w3, want_o, "rgcn forward " + what)


@pytest.mark.gpu
@pytest.mark.parametrize("D,O,R", [c for c in RGCN_CASES if c[2] in (3, 64)])
def test_rgcn_exact_lo_weights(D, O, R):
    """Forward and grad x bit for bit with a lo-bearing W (a partial permutation of s (h + l 2^-14) values) on a
    graph of short runs, few relations per row and at most 3 out-edges per node; grad W with it."""
    el, pool, m, fwd, bwd = rgcn_setup(R, True)
    x, w3, g = rgcn_operands(RGCN_N, R, D, O, pool, D * 1000 + O + 1, lo_w=True)
    want_o, want_gx, want_gw, _ = rgcn_refs(m, x, w3, g)
    out, gx, gw = rgcn_run(fwd, bwd, x, w3, g)
    what = "lo W D=%d O=%d R=%d" % (D, O, R)
    assert_exact(out, want_o, "rgcn forward " + what)
    assert_exact(gx, want_gx, "rgcn grad x " + what)
    assert_exact(gw, want_gw, "rgcn grad W " + what, tile=D)


@pytest.mark.gpu
@pytest.mark.parametrize("D,O,R", [(12, 4, 3), (36, 20, 300), (124, 36, 64), (128, 128, 300), (64, 124, 3)])
def test_rgcn_random_bounds_and_permutation(D, O, R):
    """Random x, W, g on the regime graph: every element of the forward, grad x and grad W within gemm_bound of the
    float64 product of the emulated A tiles; and relabelling the nodes (eid order inside runs kept) permutes the
    forward's rows bit for bit."""
    from pgl_b200 import ops
    from pgl_b200.heter_graph import typed_csr
    el, pool, m, fwd, bwd = rgcn_setup(R, False)
    rng = np.random.default_rng(D + O + R)
    n = RGCN_N
    x = (rng.standard_normal((n, D)) * np.exp2(rng.integers(-30, 31, (n, 1)))).astype(np.float32)
    w3 = (rng.standard_normal((R, D, O)) * 0.2).astype(np.float32)
    g = (rng.standard_normal((n, O)) * np.exp2(rng.integers(-30, 31, (n, 1)))).astype(np.float32)
    r_o, r_gx, r_gw, (b_o, b_gx, absgw) = rgcn_refs(m, x, w3, g, regime=False)
    out, gx, gw = rgcn_run(fwd, bwd, x, w3, g)
    what = "D=%d O=%d R=%d" % (D, O, R)
    assert_within(out, r_o, b_o, "rgcn forward " + what)
    assert_within(gx, r_gx, b_gx, "rgcn grad x " + what)
    chunk = int(fwd["chunk"])
    runs = np.bincount(m.run_rel, minlength=R)
    items = -(-runs // chunk)
    kterms = np.array([sum(-(-min(chunk, c - i * chunk) // 64) * 64 for i in range(it)) for c, it in zip(runs, items)])
    bgw = np.stack([gemm_bound(absgw[r], kterms[r], adds=float(items[r])) for r in range(R)])
    assert_within(gw, r_gw, bgw, "rgcn grad W " + what)
    # relabelled nodes: x'[pi[v]] = x[v], edges (pi[s], pi[d]) in the same order
    pi = rng.permutation(n)
    f2, _ = typed_csr([_cuda(pi[e]) for e in el], n)
    xp = np.empty_like(x)
    xp[pi] = x
    outp = ops._rgcn_agg_raw(f2, _cuda(xp), _cuda(w3))
    assert_exact(outp.cpu()[torch.from_numpy(pi)], out.double().cpu().numpy(), "rgcn relabelled rows " + what)


# ----------------------------------------------------------------------------------------------------------------
# route coverage
# ----------------------------------------------------------------------------------------------------------------

ROUTES = {"linear_wgmma": r"linear_wgmma_kernel"}
for _n in (64, 128):
    ROUTES["linear_tf32x3<%d>" % _n] = r"linear_tf32x3_kernel<%d>" % _n
for _np in (32, 64, 128):
    ROUTES["rgcn_agg<%d>" % _np] = r"rgcn_agg_kernel<%d>" % _np
    for _dp in (64, 128):
        ROUTES["rgcn_wgrad<%d, %d>" % (_dp, _np)] = r"rgcn_wgrad_kernel<%d, %d>" % (_dp, _np)
ROUTES["rgcn_wsum"] = r"rgcn_wsum_kernel"
_GEMM = re.compile(r"linear_wgmma_kernel|linear_tf32x3_kernel<[^>]*>|rgcn_\w+_kernel(<[^>]*>)?")


def _pad(v):
    return 32 if v <= 32 else 64 if v <= 64 else 128


def _route_calls():
    """(label, call, [routes the call must reach, and only these among the GEMM kernels])."""
    calls = []

    def lin(K, N):
        x, w, b, _ = dense_ref("D", K, N, K == 128 and N == 128, True, "relu")
        return lambda: linear(_cuda(x), _cuda(w), _cuda(b), "relu")
    calls.append(("K=N=128", lin(128, 128), ["linear_wgmma"]))
    for K, N in ((128, 64), (100, 128), (4, 64)):
        calls.append(("K=%d N=%d" % (K, N), lin(K, N), ["linear_tf32x3<%d>" % N]))
    for D, O, R in RGCN_CASES:
        def fn(D=D, O=O, R=R):
            _, pool, _, fwd, bwd = rgcn_setup(R, False)
            rgcn_run(fwd, bwd, *rgcn_operands(RGCN_N, R, D, O, pool, 1))
        calls.append(("rgcn D=%d O=%d R=%d" % (D, O, R), fn,
                      ["rgcn_agg<%d>" % _pad(O), "rgcn_agg<%d>" % _pad(D),
                       "rgcn_wgrad<%d, %d>" % (64 if D <= 64 else 128, _pad(O)), "rgcn_wsum"]))
    return calls


@pytest.mark.gpu
def test_route_coverage():
    """Each case reaches the kernels it claims and no other GEMM kernel; together they reach every instantiation."""
    a = torch.ones(1024, device="cuda")
    names, _ = _kernels_of(lambda: a.add_(1))
    if not names:
        pytest.skip("torch.profiler records no CUDA kernels here (probe: a plain torch kernel)")
    hit, failures = set(), []
    for label, fn, claims in _route_calls():
        names, _ = _kernels_of(fn)
        gemm = sorted({mt.group(0) for mt in (_GEMM.search(nm) for nm in names) if mt})
        reached = {r for r, pat in ROUTES.items() if any(re.search(pat + r"(?![\d])", nm) for nm in gemm)}
        if reached != set(claims):
            failures.append("%s: expected %s; launched %s" % (label, sorted(claims), gemm))
        hit |= reached
    assert not failures, "\n".join(failures)
    missing = sorted(set(ROUTES) - hit)
    assert not missing, "routes not reached: %s" % missing
    print("GEMM routes reached: %s" % sorted(hit))
