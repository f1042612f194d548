"""Every index-building kernel, bit for bit against a plain numpy int64 reference, at the sizes where its multi-block
paths engage.

These kernels build what every later layer reads and the EdgeIndex caches: the CSR (csrc/csr_build.cu: a three-kernel
int64 scan and a stable LSD radix sort), the segment ids and segment indptr, the narrow-row plan, the packed column
ids with their L2 hints (csrc/edge_ops.cu), the segment top-k order (csrc/readout.cu: one-CTA count, shared-memory
ranking or a 64-bit radix sort) and the halo plan (csrc/localgraph.cu).  A result that is wrong at one edge id is wrong
for every layer after it, so nothing here is a property or a tolerance check: every output is compared in full.

Which path a case reaches follows from a handful of constants, mirrored below (SCAN_TILE, the sort tiles, key_bits,
TOPK_T, TOPK_SMEM_MAX).  Every case names the boundaries it claims to cross (the scan's carry across rounds of 256 tile
sums, a radix pass count, the 64-bit sort's table-scan carry, the top-k count's carry, ...), and
`test_cases_cross_the_boundaries_they_name` checks those claims on the CPU, so a later change to the sizes cannot
quietly drop coverage.  The scan's carry is still 0 when the second round adds it, so a carry that forgot every round
but the last would only show from the third round on (more than 2 * 524,288 items): the row scans past the carry reach
a third round.  `test_route_coverage` records the kernels the entries launch (torch.profiler) and asserts that
every index kernel was reached.

Out of scope: csr_build's 64-bit-key route (2^32 edges or nodes, more memory than a shared device should be asked
for) and the aggregation task / hub plans, which are not exposed and are covered through the aggregations."""
import ctypes
import re

import numpy as np
import pytest
import torch

from oracle import oracle as O
from oracle import oracle_pool as OP

gpu = pytest.mark.gpu

# ---------------------------------------------------------------------------------------------------------------------
# the constants that pick the paths (csrc/csr_build.cu, csrc/readout.cu)
# ---------------------------------------------------------------------------------------------------------------------
SCAN_T = 256                    # threads of the scan kernels; scan_sums_kernel carries across rounds of SCAN_T sums
SCAN_TILE = 256 * 8             # items per scan tile
SCAN_CARRY = SCAN_T * SCAN_TILE  # the first carry happens above this many items
SORT_TILE32 = 4096              # pairs per radix-sort tile, 32-bit keys (csr_build)
SORT_TILE64 = 2048              # pairs per radix-sort tile, 64-bit keys (segment top-k)
TOPK_T = 1024                   # threads of topk_count_kernel; it carries across rounds of TOPK_T segments
TOPK_SMEM_MAX = 2048            # longest segment ranked by topk_smem_kernel


def key_bits(n):
    """Bits of a key below n (csr_build's key_bits, readout's key_bits_of)."""
    b = 1
    while b < 62 and (1 << b) < n:
        b += 1
    return b


def ceil_div(a, b):
    return -(-a // b)


def scan_rounds(n):
    """Rounds of scan_sums_kernel for a scan of n items; the carry is used from the second round on."""
    return ceil_div(ceil_div(n, SCAN_TILE), SCAN_T) if n > 0 else 0


def csr_passes(N):
    return ceil_div(key_bits(N), 8)


def csr_table(E):
    """Length of csr_build's digit-table scan."""
    return 256 * ceil_div(E, SORT_TILE32)


def u64_passes(B):
    return ceil_div(32 + key_bits(B), 8)


def u64_table(N):
    return 256 * ceil_div(N, SORT_TILE64)


# ---------------------------------------------------------------------------------------------------------------------
# numpy references
# ---------------------------------------------------------------------------------------------------------------------

def ref_csr(u, v, N):
    """(degree, sorted_v, sorted_u, sorted_eid, indptr): stable argsort + cumsum."""
    u = np.asarray(u, np.int64)
    v = np.asarray(v, np.int64)
    degree = np.bincount(u, minlength=N).astype(np.int64)
    indptr = np.zeros(N + 1, np.int64)
    np.cumsum(degree, out=indptr[1:])
    order = np.argsort(u, kind="stable").astype(np.int64)
    return degree, v[order], u[order], order, indptr


def ref_segment_ids(deg):
    """(uniq, segment ids) of the rows of a degree list: the non-empty rows and each slot's rank among them."""
    deg = np.asarray(deg, np.int64)
    nz = np.flatnonzero(deg).astype(np.int64)
    return nz, np.repeat(np.arange(nz.size, dtype=np.int64), deg[nz])


def ref_segment_indptr(ids, K):
    return np.searchsorted(np.asarray(ids, np.int64), np.arange(K + 1), side="left").astype(np.int64)


def ref_hot(count, k):
    """pack_cols' threshold: the k-th largest count, at least 2; None when it gives no hints."""
    if k <= 0 or k >= count.size:
        return None
    return max(int(np.sort(count)[::-1][k - 1]), 2)


def ref_packed(cols, count, min_count):
    hot = count[cols].astype(np.int64) >= min_count
    return cols.astype(np.uint32) | (hot.astype(np.uint32) << np.uint32(31))


def ref_narrow_plan(indptr, cols, packed):
    """(plan words, nz_row with its two padding copies, blk_k)."""
    N, E = indptr.size - 1, cols.size
    deg = np.diff(indptr)
    nz = np.flatnonzero(deg)
    plan = (packed & np.uint32(0xbfffffff)) if packed is not None else cols.astype(np.uint32)
    plan = plan.copy()
    plan[indptr[nz]] |= np.uint32(0x40000000)
    last = nz[-1] if nz.size else 0
    nz_row = np.concatenate([nz, [last, last]]).astype(np.int32)
    nblk = ceil_div(E, 32)
    owner = np.searchsorted(indptr, 32 * np.arange(1, nblk) - 1, side="right") - 1
    blk_k = np.concatenate([[-1], np.searchsorted(nz, owner)]).astype(np.int32)
    return plan, nz_row, blk_k


def topk_order(scores, indptr):
    """Nodes of [indptr[0], indptr[B]) in segment order, each segment in the documented order: score descending,
    -0.0 == +0.0, NaN after every number, ties by ascending node index; plus every sorted node's rank in its segment."""
    ip = np.asarray(indptr, np.int64)
    n = np.diff(ip)
    idx = np.arange(ip[0], ip[-1], dtype=np.int64)
    s = np.asarray(scores, np.float32)[idx].astype(np.float64)
    nan = np.isnan(s)
    key = np.where(nan, 0.0, -s) + 0.0
    seg = np.repeat(np.arange(n.size, dtype=np.int64), n)
    order = np.lexsort((idx, key, nan, seg))
    rank = np.arange(idx.size, dtype=np.int64) - (ip[seg] - ip[0])
    return idx[order], seg, rank


def ref_topk(order, indptr, ratio):
    """(offsets, perm) of segment_topk_perm from topk_order's result."""
    nodes, seg, rank = order
    k = OP.topk_k(np.diff(np.asarray(indptr, np.int64)), ratio)
    return np.concatenate([[0], np.cumsum(k)]).astype(np.int64), nodes[rank < k[seg]]


def ref_typed_csr(edge_lists, n):
    """heter_graph.typed_csr's integer layout and slot weights: relations concatenated, stably sorted by dst (fwd)
    and src (bwd); the (row, relation) runs sorted by relation (stable)."""
    src = np.concatenate([e[:, 0] for e in edge_lists])
    dst = np.concatenate([e[:, 1] for e in edge_lists])
    rel_e = np.concatenate([np.full(len(e), r, np.int16) for r, e in enumerate(edge_lists)])
    R, E = len(edge_lists), src.size
    o = np.argsort(dst, kind="stable")
    rows, rel = dst[o], rel_e[o]
    brk = np.ones(E, bool)
    brk[1:] = (rows[1:] != rows[:-1]) | (rel[1:] != rel[:-1])
    beg = np.flatnonzero(brk)
    end = np.append(beg[1:], E)
    ro = np.argsort(rel[beg], kind="stable")
    cnt_e = np.empty(E, np.int64)
    cnt_e[o] = np.repeat(end - beg, end - beg)
    ob = np.argsort(src, kind="stable")
    fwd = {"indptr": np.concatenate([[0], np.cumsum(np.bincount(dst, minlength=n))]), "cols": src[o], "rel": rel,
           "run_row": rows[beg][ro], "run_beg": beg[ro], "run_end": end[ro],
           "run_off": np.concatenate([[0], np.cumsum(np.bincount(rel[beg], minlength=R))])}
    bwd = {"indptr": np.concatenate([[0], np.cumsum(np.bincount(src, minlength=n))]), "cols": dst[ob],
           "rel": rel_e[ob], "w": np.float32(1) / cnt_e[ob].astype(np.float32)}
    return fwd, bwd


# ---------------------------------------------------------------------------------------------------------------------
# inputs and the boundaries each case claims
# ---------------------------------------------------------------------------------------------------------------------
# csr_build: (id, N, E, key kind, stride of the u / v views, claims)
CSR_CASES = [
    ("n1", 1, 5000, "uniform", 1, ["passes=1"]),
    ("e0", 7, 0, "uniform", 1, []),
    ("n256", 256, 60000, "uniform", 1, ["passes=1"]),
    ("n257", 257, 60000, "uniform", 1, ["passes=2"]),
    ("n65536", 65536, 300000, "uniform", 1, ["passes=2"]),
    ("n65537", 65537, 300000, "uniform", 2, ["passes=3"]),
    ("n2^24_top_digit", 1 << 24, 1000000, "top_digit", 1, ["passes=3", "deg_carry2"]),
    ("n2^24+1", (1 << 24) + 1, 1000000, "uniform", 1, ["passes=4", "deg_carry2"]),
    ("e4095", 300, 4095, "uniform", 1, ["tile_edge"]),
    ("e4096", 300, 4096, "uniform", 1, ["tile_edge"]),
    ("e4097", 300, 4097, "uniform", 3, ["tile_edge"]),
    ("e3tiles+1", 300, 3 * 4096 + 1, "uniform", 2, ["tile_edge"]),
    ("deg_below_carry", SCAN_CARRY, 2000000, "uniform", 2, ["deg_no_carry"]),
    ("deg_above_carry", SCAN_CARRY + 1, 2000000, "uniform", 2, ["deg_carry"]),
    ("deg_carried_twice", 1200000, 2000000, "uniform", 1, ["deg_carry2"]),
    ("table_carry", 1200000, 9000000, "uniform", 1, ["table_carry", "deg_carry2"]),
    ("table_carry_hub", 1200000, 17000000, "hub", 2, ["table_carry2", "deg_carry2"]),
    ("all_equal", 1000, 9000000, "equal", 1, ["table_carry"]),
    ("descending", 1200000, 1200000, "descending", 3, ["deg_carry2"]),
    ("stride3", 70000, 500000, "uniform", 3, ["passes=3"]),
]

# segment ids / segment indptr: (id, number of rows, degree pattern, claims)
SEG_CASES = [
    ("random", 1200000, "random", ["carry"]),
    ("empty_ends", 1200000, "empty_ends", ["carry"]),
    ("one_row", 1200000, "one_row", ["carry"]),
    ("all_empty", 1200000, "all_empty", ["carry"]),
    ("single", 1, "random", []),
]

# narrow plan: (id, number of rows, degree pattern, n_src, hot sources (0: no hints), claims)
NARROW_CASES = [
    ("random", 1200000, "random", 50000, 1000, ["carry", "hints"]),
    ("slot_boundaries", 20000, "boundaries", 5000, 0, ["starts_on_32", "crosses_32"]),
    ("one_row", 1200000, "one_row", 70, 0, ["carry"]),
    ("last_row_only", 1200000, "last_only", 70, 3, ["carry", "hints"]),
]

# segment top-k: (id, segment sizes, score kind, trailing nodes after indptr[B], paths, claims)
TOPK_CASES = [
    ("b1024", ("random", 1024, 40), "specials", 0, ("smem", "sort"), ["count_no_carry", "u64_passes=6"]),
    ("b1025", ("random", 1025, 40), "specials", 0, ("smem", "sort"), ["count_carry", "u64_passes=6"]),
    ("b256", ("random", 256, 60), "specials", 0, ("smem", "sort"), ["u64_passes=5"]),
    ("b257", ("random", 257, 60), "specials", 0, ("smem", "sort"), ["u64_passes=6"]),
    ("b65536", ("random", 65536, 9), "specials", 0, ("smem", "sort"), ["count_carry", "u64_passes=6"]),
    ("b65537", ("random", 65537, 9), "specials", 0, ("smem", "sort"), ["count_carry", "u64_passes=7"]),
    ("all_equal", ("random", 1500, 30), "equal", 0, ("smem", "sort"), ["count_carry"]),
    ("boundary_ties", ("random", 3000, 12), "segment_ties", 0, ("smem", "sort"), ["count_carry"]),
    ("trailing_nodes", ("random", 700, 30), "specials", 3000, ("smem", "sort"), []),
    ("n8.9M", ("hub", 4000, 100000), "specials", 0, ("natural",), ["u64_table_carry", "count_carry", "long"]),
]
TOPK_RATIOS = (0.01, 0.37, 1.0, 1, 3)


def claim_holds(claim, **kw):
    name, _, val = claim.partition("=")
    if name == "passes":
        return csr_passes(kw["N"]) == int(val)
    if name == "deg_carry":
        return scan_rounds(kw["N"]) >= 2
    if name == "deg_carry2":
        return scan_rounds(kw["N"]) >= 3
    if name == "deg_no_carry":
        return scan_rounds(kw["N"]) == 1 and kw["N"] == SCAN_CARRY
    if name == "table_carry":
        return scan_rounds(csr_table(kw["E"])) >= 2
    if name == "table_carry2":
        return scan_rounds(csr_table(kw["E"])) >= 3
    if name == "tile_edge":
        return kw["E"] % SORT_TILE32 in (0, 1, SORT_TILE32 - 1)
    if name == "carry":
        return scan_rounds(kw["N"]) >= 3
    if name == "count_carry":
        return ceil_div(kw["B"], TOPK_T) >= 2
    if name == "count_no_carry":
        return kw["B"] == TOPK_T
    if name == "u64_passes":
        return u64_passes(kw["B"]) == int(val)
    if name == "u64_table_carry":
        return scan_rounds(u64_table(kw["N"])) >= 3
    if name == "long":
        return kw["max_len"] > TOPK_SMEM_MAX
    if name == "hints":
        return kw["hot"] > 0
    if name == "starts_on_32":
        ip = kw["indptr"]
        return bool(np.any((ip[:-1] % 32 == 0) & (ip[:-1] > 0) & (np.diff(ip) > 0)))
    if name == "crosses_32":
        ip = kw["indptr"]
        d = np.diff(ip)
        return bool(np.any((d > 0) & (ip[:-1] // 32 != (ip[1:] - 1) // 32) & (ip[:-1] % 32 != 0)))
    raise KeyError(claim)


def csr_inputs(N, E, kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        u = rng.integers(0, N, E)
        if E:
            u[rng.integers(0, E, 8)] = N - 1        # the largest key, so the top digit is used
    elif kind == "top_digit":
        shift = 8 * (csr_passes(N) - 1)
        u = rng.integers(0, ceil_div(N, 1 << shift), E) << shift
    elif kind == "equal":
        u = np.full(E, N // 2)
    elif kind == "descending":
        u = np.arange(E)[::-1] * (N // E)
    elif kind == "hub":
        u = rng.integers(0, N, E)
        u[rng.random(E) < 0.6] = N // 3
    else:
        raise KeyError(kind)
    v = rng.integers(0, 1 << 40, E)
    return u.astype(np.int64), v.astype(np.int64)


def degrees(N, kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        d = rng.integers(0, 5, N)
        for s in rng.integers(0, N, 20):         # runs of empty rows
            d[s:s + int(rng.integers(1, 3000))] = 0
        d[-1] = 3                                # the last row counts in num_uniq
    elif kind == "empty_ends":
        d = rng.integers(0, 4, N)
        d[:777] = 0
        d[-555:] = 0
    elif kind == "one_row":
        d = np.zeros(N, np.int64)
        d[N // 3 + 17] = 100
    elif kind == "last_only":
        d = np.zeros(N, np.int64)
        d[-1] = 70
    elif kind == "all_empty":
        d = np.zeros(N, np.int64)
    elif kind == "boundaries":
        d = np.tile([32, 0, 16, 16, 5, 30, 29, 64, 1, 31, 0, 0, 33, 3], ceil_div(N, 14))[:N]
    else:
        raise KeyError(kind)
    return d.astype(np.int64)


def topk_sizes(spec, seed):
    kind, B, m = spec
    rng = np.random.default_rng(seed)
    if kind == "random":
        sizes = rng.integers(0, m + 1, B)
        sizes[[0, B // 2, B - 1]] = [0, 0, m]   # empty segments, the last one non-empty
        return sizes.astype(np.int64)
    sizes = rng.integers(1800, 2600, B)          # "hub": about 2200 B nodes plus one long segment
    sizes[B // 3] = m
    return sizes.astype(np.int64)


SPECIALS = np.array([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 1e-40, -1e-40, 1.1754942e-38, -1.1754942e-38,
                     3.4e38, -3.4e38], np.float32)
NANS = np.array([0x7fc00000, 0xffc00000, 0x7fc00001], np.uint32).view(np.float32)


def topk_scores(kind, sizes, extra, seed):
    rng = np.random.default_rng(seed)
    n = int(sizes.sum()) + extra
    if kind == "equal":
        return np.ones(n, np.float32)
    if kind == "segment_ties":                   # equal scores on both sides of every boundary
        s = np.repeat(rng.integers(-2, 3, sizes.size), sizes).astype(np.float32)
        s[rng.random(s.size) < 0.1] = 7.0
        return np.concatenate([s, np.full(extra, np.inf, np.float32)])
    s = rng.integers(-3, 4, n).astype(np.float32)
    pick = rng.random(n) < 0.25
    s[pick] = rng.choice(np.concatenate([SPECIALS, NANS]), int(pick.sum()))
    if extra:                                    # nodes after the last segment score above every member
        s[-extra:] = np.float32(np.inf)
    return s


def _claim_kwargs_topk(case):
    _, spec, _, extra, _, _ = case
    sizes = topk_sizes(spec, 7)
    return {"B": sizes.size, "N": int(sizes.sum()) + extra, "max_len": int(sizes.max())}


# ---------------------------------------------------------------------------------------------------------------------
# CPU tests: the references and the path engagement
# ---------------------------------------------------------------------------------------------------------------------

def test_references_match_the_oracle():
    rng = np.random.default_rng(3)
    for N, E in ((1, 9), (5, 0), (300, 5000), (70000, 100000)):
        edges = rng.integers(0, N, (E, 2)).astype(np.int64)
        for a, b in zip(ref_csr(edges[:, 1], edges[:, 0], N), O.adj_dst_index(edges, N)):
            assert np.array_equal(a, b)
    for kind in ("random", "empty_ends", "one_row", "boundaries"):
        d = degrees(5000, kind, 1)
        key = np.repeat(np.arange(d.size), d)
        uniq, seg = ref_segment_ids(d)
        ou, oseg = O.unique_segment(key)
        assert np.array_equal(uniq, ou) and np.array_equal(seg, oseg)
        ip = ref_segment_indptr(key, d.size)
        assert np.array_equal(ip, np.concatenate([[0], np.cumsum(d)]))
        assert np.array_equal(ip, OP.indptr_of(key, d.size))
        # segment_pool's sum over the ids is the degree list
        assert np.array_equal(O.segment_pool(np.ones((key.size, 1)), seg, "sum")[:, 0], d[uniq])
    for sizes in (np.array([0, 5, 1, 0, 9, 3]), topk_sizes(("random", 300, 40), 2)):
        ids = np.repeat(np.arange(sizes.size), sizes)
        s = topk_scores("specials", sizes, 0, 4)
        order = topk_order(s, np.concatenate([[0], np.cumsum(sizes)]))
        for ratio in TOPK_RATIOS:
            off, perm = ref_topk(order, np.concatenate([[0], np.cumsum(sizes)]), ratio)
            assert np.array_equal(perm, OP.segment_topk_perm(s, ids, ratio))
            assert off[-1] == perm.size


def test_typed_reference_matches_the_host_model():
    from test_hetergraph_host import typed_csr_model
    rng = np.random.default_rng(5)
    n = 300
    el = [rng.integers(0, n, (e, 2)).astype(np.int64) for e in (900, 0, 400)]
    el[2][:150, 1] = 7                           # a hub row shared by two relations
    fwd, bwd = ref_typed_csr(el, n)
    m = typed_csr_model(el, n)
    for k in ("indptr", "cols", "rel", "run_row", "run_beg", "run_end", "run_off"):
        assert np.array_equal(fwd[k], m["fwd"][k]), k
    for k in ("indptr", "cols", "rel", "w"):
        assert np.array_equal(bwd[k], m["bwd"][k]), k


def test_narrow_reference_by_hand():
    ip = np.array([0, 32, 32, 40, 70, 70])       # row 2 starts on slot 32, row 3 crosses slot 64
    cols = np.arange(70, dtype=np.int64)
    plan, nz, blk = ref_narrow_plan(ip, cols, None)
    assert nz.tolist() == [0, 2, 3, 3, 3]
    assert blk.tolist() == [-1, 0, 2]            # slot 31 -> row 0 (rank 0), slot 63 -> row 3 (rank 2)
    assert [j for j in range(70) if plan[j] & 0x40000000] == [0, 32, 40]
    packed = ref_packed(cols, np.bincount(cols, minlength=70) + np.arange(70) % 3, 3)
    plan2, _, _ = ref_narrow_plan(ip, cols, packed | np.uint32(0x40000000))
    assert np.array_equal(plan2 & np.uint32(0xbfffffff), packed & np.uint32(0xbfffffff))
    assert int((plan2 >> 31).sum()) == int((packed >> 31).sum()) > 0


def test_cases_cross_the_boundaries_they_name():
    assert SCAN_CARRY == 524288 and csr_table(8388608) == SCAN_CARRY and u64_table(4194304) == SCAN_CARRY
    assert [csr_passes(n) for n in (1, 256, 257, 65536, 65537, 1 << 24, (1 << 24) + 1)] == [1, 1, 2, 2, 3, 3, 4]
    for cid, N, E, _, _, claims in CSR_CASES:
        for c in claims:
            assert claim_holds(c, N=N, E=E), (cid, c)
    seen = {c for case in CSR_CASES for c in case[5]}
    assert {"passes=1", "passes=2", "passes=3", "passes=4", "deg_carry", "deg_carry2", "deg_no_carry",
            "table_carry", "table_carry2", "tile_edge"} <= seen
    assert {E for _, _, E, _, _, _ in CSR_CASES} >= {0, 4095, 4096, 4097}
    assert {c[4] for c in CSR_CASES} >= {1, 2, 3}
    for cid, N, kind, claims in SEG_CASES:
        for c in claims:
            assert claim_holds(c, N=N), (cid, c)
    for cid, N, kind, n_src, hot, claims in NARROW_CASES:
        d = degrees(N, kind, 11)
        ip = np.concatenate([[0], np.cumsum(d)])
        for c in claims:
            assert claim_holds(c, N=N, hot=hot, indptr=ip), (cid, c)
    for case in TOPK_CASES:
        kw = _claim_kwargs_topk(case)
        for c in case[5]:
            assert claim_holds(c, **kw), (case[0], c)
        if "natural" not in case[4]:
            assert kw["max_len"] <= TOPK_SMEM_MAX < kw["N"], case[0]   # both paths reachable by a max_len hint
    seen = {c for case in TOPK_CASES for c in case[5]}
    assert {"count_carry", "count_no_carry", "u64_passes=5", "u64_passes=6", "u64_passes=7", "u64_table_carry",
            "long"} <= seen
    # the carry sizes of the entries built on csr_build and of the halo plan
    assert scan_rounds(PART_K) >= 3 and scan_rounds(csr_table(PART_N)) >= 2
    assert scan_rounds(TYPED_N) >= 3 and scan_rounds(HALO_N) >= 3 and scan_rounds(HALO_E) >= 3


# ---------------------------------------------------------------------------------------------------------------------
# GPU tests
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    torch.cuda.set_device(0)
    return pgl_b200


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _call(name, *args):
    from pgl_b200 import _lib
    _lib.check(getattr(_lib.lib, name)(*args))


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def assert_same(got, want, what):
    g = got.cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    w = np.asarray(want)
    assert g.shape == w.shape, "%s: shape %s, want %s" % (what, g.shape, w.shape)
    bad = np.flatnonzero(g.reshape(-1) != w.reshape(-1))
    if bad.size:
        i = int(bad[0])
        pytest.fail("%s: %d of %d entries differ; first at %d: got %r, want %r"
                    % (what, bad.size, w.size, i, g.reshape(-1)[i], w.reshape(-1)[i]))


def _edge_views(u, v, stride):
    """u and v as device views of stride `stride` (read in place by csr_build)."""
    if stride == 1:
        return _dev(u), _dev(v)
    a = np.zeros((u.size, stride), np.int64)
    a[:, stride - 1], a[:, 0] = u, v
    t = _dev(a)
    return t[:, stride - 1], t[:, 0]


@gpu
@pytest.mark.parametrize("case", CSR_CASES, ids=[c[0] for c in CSR_CASES])
def test_csr_build(pgl, case):
    cid, N, E, kind, stride, _ = case
    u, v = csr_inputs(N, E, kind, seed=N + E)
    ud, vd = _edge_views(u, v, stride)
    assert stride == 1 or ud.stride(0) == stride
    got = pgl.ops.csr_build(ud, vd, N)
    want = ref_csr(u, v, N)
    for name, g, w in zip(("degree", "sorted_v", "sorted_u", "sorted_eid", "indptr"), got, want):
        assert_same(g, w, "%s %s" % (cid, name))


@gpu
def test_partition_relabel_above_the_carries(pgl):
    rng = np.random.default_rng(21)
    part = rng.integers(0, PART_K, PART_N).astype(np.int64)
    part[part == 5] = 0                          # an empty part
    new_id, offsets = pgl.ops.partition_relabel(_dev(part), PART_K)
    perm = np.argsort(part, kind="stable")
    want = np.empty(PART_N, np.int64)
    want[perm] = np.arange(PART_N)
    assert_same(new_id, want, "new_id")
    assert_same(offsets, np.concatenate([[0], np.cumsum(np.bincount(part, minlength=PART_K))]), "offsets")


PART_N, PART_K = 9000000, 1200000
TYPED_N = 1200000
HALO_N, HALO_E = 1200000, 2500000


@gpu
def test_typed_csr_above_the_carry(pgl):
    from pgl_b200.heter_graph import typed_csr
    rng = np.random.default_rng(22)
    el = [rng.integers(0, TYPED_N, (e, 2)).astype(np.int64) for e in (1500000, 400000, 900000)]
    el[2][: 300000, 1] = 12345                   # a hub row
    fwd, bwd = typed_csr([_dev(e) for e in el], TYPED_N)
    wf, wb = ref_typed_csr(el, TYPED_N)
    for k in ("indptr", "cols", "rel", "run_row", "run_beg", "run_end", "run_off"):
        assert_same(fwd[k], wf[k], "fwd " + k)
    for k in ("indptr", "cols", "rel", "w"):
        assert_same(bwd[k], wb[k], "bwd " + k)


def _segment_ids_case(case):
    cid, N, kind, _ = case
    d = degrees(N, kind, 31)
    return cid, d, np.concatenate([[0], np.cumsum(d)]).astype(np.int64)


@gpu
@pytest.mark.parametrize("case", SEG_CASES, ids=[c[0] for c in SEG_CASES])
def test_segment_ids_from_indptr(pgl, case):
    cid, d, ip = _segment_ids_case(case)
    uniq, seg = pgl.ops.segment_ids_from_indptr(_dev(ip), int(ip[-1]))
    wu, ws = ref_segment_ids(d)
    assert_same(uniq, wu, cid + " uniq")
    assert_same(seg, ws, cid + " segment_ids")


def _segment_indptr_raw(ids, K):
    out = torch.full((K + 1,), -7, dtype=torch.int64, device="cuda")   # every entry must be written
    _call("pglb_segment_indptr", _p(ids) if ids.numel() else None, int(ids.numel()), int(K), _p(out), _st())
    return out


@gpu
@pytest.mark.parametrize("case", SEG_CASES, ids=[c[0] for c in SEG_CASES])
def test_segment_indptr(pgl, case):
    cid, d, _ = _segment_ids_case(case)
    _, ids = ref_segment_ids(d)                  # sorted ids 0 .. K - 1 with gaps where rows were empty
    K = int(ids[-1]) + 1 if ids.size else 0
    idd = _dev(ids)
    for k in (K, K + 1, K + 1000):               # K larger than the largest id + 1 leaves trailing empty segments
        assert_same(_segment_indptr_raw(idd, k), ref_segment_indptr(ids, k), "%s K=%d" % (cid, k))
    assert_same(pgl.ops.segment_indptr(idd, K + 3), ref_segment_indptr(ids, K + 3), cid + " ops")


@gpu
def test_segment_indptr_no_ids(pgl):
    assert_same(_segment_indptr_raw(torch.zeros(0, dtype=torch.int64, device="cuda"), 5), np.zeros(6, np.int64),
                "E=0")
    ids = np.array([3, 3, 3, 9], np.int64)      # leading and inner empty segments
    assert_same(_segment_indptr_raw(_dev(ids), 12), ref_segment_indptr(ids, 12), "gaps")


@gpu
@pytest.mark.parametrize("case", NARROW_CASES, ids=[c[0] for c in NARROW_CASES])
def test_narrow_plan(pgl, case):
    from pgl_b200 import ops
    cid, N, kind, n_src, hot, _ = case
    d = degrees(N, kind, 11)
    ip = np.concatenate([[0], np.cumsum(d)]).astype(np.int64)
    E = int(ip[-1])
    rng = np.random.default_rng(41)
    cols = np.floor(n_src * rng.random(E) ** 3).astype(np.int64)     # skewed: a few sources gathered often
    row_bytes = ops.NARROW_HOT_BYTES // hot if hot else 64
    plan, nz_row, blk_k, hints = ops.narrow_plan(_dev(ip), _dev(cols), n_src, row_bytes)
    k = ops.NARROW_HOT_BYTES // row_bytes if ops.NARROW_HOT_BYTES > 0 else 0
    thr = ref_hot(np.bincount(cols, minlength=n_src), k)
    assert hints == (thr is not None), cid
    packed = ref_packed(cols, np.bincount(cols, minlength=n_src), thr) if hints else None
    if hot and ops.NARROW_HOT_BYTES > 0:
        assert hints and int((packed >> 31).sum()) > 0, cid
    wp, wn, wb = ref_narrow_plan(ip, cols, packed)
    assert_same(plan.cpu().numpy().view(np.uint32), wp, cid + " plan")
    K = wn.size - 2
    assert_same(nz_row[: K + 2], wn, cid + " nz_row")
    assert_same(blk_k, wb, cid + " blk_k")


def _pack_cols_raw(cols, n_src, min_count):
    count = torch.full((n_src,), -5, dtype=torch.int32, device="cuda")
    packed = torch.zeros(cols.numel(), dtype=torch.int32, device="cuda")
    _call("pglb_pack_cols", _p(cols), int(cols.numel()), int(n_src), _p(count), int(min_count), _p(packed), _st())
    return count, packed


@gpu
def test_pack_cols_threshold(pgl):
    rng = np.random.default_rng(51)
    n_src, E = 40000, 3000000
    cols = np.floor(n_src * rng.random(E) ** 2).astype(np.int64)
    cd = _dev(cols)
    count = np.bincount(cols, minlength=n_src)
    on_count = np.intersect1d(count, count + 1)  # thresholds c with sources of count c and of count c - 1
    assert on_count.size >= 3
    for c in (int(on_count[0]), int(on_count[on_count.size // 2]), int(on_count[-1])):
        assert (count == c).any() and (count == c - 1).any(), c
        got_count, packed = _pack_cols_raw(cd, n_src, c)
        assert_same(got_count, count.astype(np.int32), "count")
        assert_same(packed.cpu().numpy().view(np.uint32), ref_packed(cols, count, c), "packed min_count=%d" % c)


@gpu
@pytest.mark.parametrize("budget", ["zero", "few", "most", "all"])
def test_pack_cols_budgets(pgl, budget):
    rng = np.random.default_rng(52)
    n_src, E, row_bytes = 30000, 1000000, 256
    cols = np.floor(n_src * rng.random(E) ** 3).astype(np.int64)
    k = {"zero": 0, "few": 7, "most": n_src - 1, "all": n_src}[budget]
    packed, hints = pgl.ops.pack_cols(_dev(cols), n_src, row_bytes, budget_bytes=k * row_bytes)
    count = np.bincount(cols, minlength=n_src)
    thr = ref_hot(count, k)
    assert hints == (thr is not None)
    want = ref_packed(cols, count, thr) if hints else cols.astype(np.uint32)
    assert_same(packed.cpu().numpy().view(np.uint32), want, "packed")


def topk_raw(s, ip, ratio, max_len):
    """pglb_segment_topk_count + _fill with a max_len hint (a hint above TOPK_SMEM_MAX takes the sort path)."""
    B, N = int(ip.numel()) - 1, int(s.numel())
    k, r = (int(ratio), 0.0) if isinstance(ratio, int) else (0, float(ratio))
    offsets = torch.empty(B + 1, dtype=torch.int64, device="cuda")
    info = torch.empty(2, dtype=torch.int64, device="cuda")
    _call("pglb_segment_topk_count", _p(ip), B, r, k, _p(offsets), _p(info), _st())
    total, longest = (int(v) for v in info.tolist())
    perm = torch.full((total,), -1, dtype=torch.int64, device="cuda")   # every slot must be written
    need = ctypes.c_size_t(0)
    _call("pglb_segment_topk_ws", B, N, max_len, ctypes.byref(need))
    ws = torch.empty(max(need.value, 1), dtype=torch.uint8, device="cuda")
    _call("pglb_segment_topk_fill", _p(s), N, _p(ip), B, _p(offsets), max_len, _p(perm), _p(ws), ws.numel(), _st())
    return offsets, longest, perm


_TOPK = {}


def _topk_case(case):
    cid = case[0]
    if cid not in _TOPK:
        _, spec, kind, extra, _, _ = case
        sizes = topk_sizes(spec, 7)
        s = topk_scores(kind, sizes, extra, 8)
        ip = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        _TOPK.clear()
        _TOPK[cid] = (sizes, s, ip, topk_order(s, ip), _dev(s), _dev(ip))
    return _TOPK[cid]


TOPK_PARAMS = [(c, p) for c in TOPK_CASES for p in c[4]]


@gpu
@pytest.mark.parametrize("case,path", TOPK_PARAMS, ids=["%s-%s" % (c[0], p) for c, p in TOPK_PARAMS])
def test_segment_topk_perm(pgl, case, path):
    cid = case[0]
    sizes, s, ip, order, sd, ipd = _topk_case(case)
    N = s.size
    for ratio in TOPK_RATIOS:
        w_off, w_perm = ref_topk(order, ip, ratio)
        what = "%s %s ratio=%r" % (cid, path, ratio)
        if path == "sort":
            off, longest, perm = topk_raw(sd, ipd, ratio, N)
            assert_same(off, w_off, what + " offsets")
            assert longest == int(sizes.max()), what
        elif path == "smem":
            off, longest, perm = topk_raw(sd, ipd, ratio, int(sizes.max()))
            assert_same(off, w_off, what + " offsets")
            assert_same(pgl.ops.segment_topk_perm(sd, ipd, ratio), w_perm, what + " ops")
        else:
            perm = pgl.ops.segment_topk_perm(sd, ipd, ratio)
        assert_same(perm, w_perm, what + " perm")


@gpu
def test_halo_plan_above_the_carry(pgl):
    from pgl_b200.distributed.halo import block_offsets
    from test_gpu_localgraph import numpy_plan
    edges = O.chung_lu_edges(HALO_N, HALO_E, exponent=0.8, seed=61)
    ed = _dev(edges)
    offsets = block_offsets(HALO_N, 4)
    for r in (0, 2):
        lo, hi = offsets[r], offsets[r + 1]
        got = pgl.ops.halo_plan(ed, HALO_N, lo, hi, offsets)
        want = numpy_plan(edges, lo, hi, offsets)
        for name, g, w in zip(("eid", "dst_local", "col_local", "halo_ids", "recv_counts"), got, want):
            assert_same(g, np.asarray(w, np.int64), "rank %d %s" % (r, name))


# ---------------------------------------------------------------------------------------------------------------------
# route coverage
# ---------------------------------------------------------------------------------------------------------------------
ROUTES = {
    "scan tile sums": r"scan_tile_sums_kernel", "scan sums": r"scan_sums_kernel", "scan apply": r"scan_apply_kernel",
    "pack keys": r"pack_keys_kernel", "set first": r"set_first_kernel", "emit sorted": r"emit_sorted_kernel",
    "hist u32": r"rs_hist_kernel<unsigned int, 512>",
    "scatter u32": r"rs_scatter_kernel<unsigned int, unsigned int, 512>",
    "hist u64": r"rs_hist_kernel<unsigned long( long)?, 256>",
    "scatter u64": r"rs_scatter_kernel<unsigned long( long)?, unsigned long( long)?, 256>",
    "nonempty flag": r"nonempty_flag_kernel", "emit segments": r"emit_segments_kernel",
    "segment indptr": r"segment_indptr_kernel", "plan cols": r"plan_cols_kernel", "plan rows": r"plan_rows_kernel",
    "plan blocks": r"plan_blocks_kernel", "col count": r"col_count_kernel", "pack cols": r"pack_cols_kernel",
    "topk count": r"topk_count_kernel", "topk smem": r"topk_smem_kernel", "topk pack": r"topk_pack_kernel",
    "topk emit": r"topk_emit_kernel", "invert perm": r"invert_perm_kernel", "halo mark": r"halo_mark_kernel",
    "halo counts": r"halo_counts_kernel", "halo fill edges": r"halo_fill_edges_kernel",
    "halo fill nodes": r"halo_fill_nodes_kernel", "halo recv counts": r"halo_recv_counts_kernel",
}


def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@gpu
def test_route_coverage(pgl):
    """Small calls of every entry the file tests reach every index kernel."""
    a = torch.ones(1024, device="cuda")
    if not _kernel_names(lambda: a.add_(1)):
        pytest.skip("torch.profiler records no CUDA kernels here (probe: a plain torch kernel)")
    ops = pgl.ops
    rng = np.random.default_rng(71)
    edges = rng.integers(0, 500, (6000, 2)).astype(np.int64)
    ed = _dev(edges)
    sizes = np.array([3, 0, 2500, 7])
    ip = _dev(np.concatenate([[0], np.cumsum(sizes)]))
    s = _dev(rng.standard_normal(int(sizes.sum())).astype(np.float32))
    ip_short = _dev(np.array([0, 3, 3, 9]))

    def calls():
        deg, sv, su, se, indptr = ops.csr_build(ed[:, 1], ed[:, 0], 500)
        ops.segment_ids_from_indptr(indptr, 6000)
        ops.segment_indptr(su, 500)
        ops.narrow_plan(indptr, sv, 500, ops.NARROW_HOT_BYTES // 50 if ops.NARROW_HOT_BYTES else 64)
        ops.pack_cols(sv, 500, 64, budget_bytes=64 * 20)
        ops.segment_topk_perm(s, ip, 0.5)
        ops.segment_topk_perm(s[:9], ip_short, 2)
        ops.partition_relabel(ed[:, 0], 500)
        ops.halo_plan(ed, 500, 100, 300, [0, 100, 300, 500])
    names = _kernel_names(calls)
    missing = sorted(k for k, pat in ROUTES.items() if not any(re.search(pat, nm) for nm in names))
    assert not missing, "kernels not reached: %s (launched %s)" % (missing, sorted(set(names)))
