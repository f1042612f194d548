"""CPU model of the wide-row streaming kernels' control flow (csrc/spmm_stream.cu: task_plan_kernel, the row walk of
spmm_stream128_kernel, spmm_stream_fixup_kernel, empty_rows_kernel), statement by statement, checked against the oracle.
What it checks is the part most likely to be wrong -- rows ending at any slot of a commit group, empty-row runs, rows cut
by task boundaries, the partial / fix-up protocol -- over hub, gap and uniform graphs and several task sizes.  Memory
movement (cp.async rings) is not modelled: slot j simply reads x[cols[a + j]]; the issue / consume timeline IS modelled
as far as the per-batch source-scale registers (sc_cur / sc_prev) depend on it."""
import numpy as np
import pytest

from oracle import oracle as O

GRP = 4
LAG = 3
BIG = 1 << 30


def row_of_slot(indptr, n_rows, v):
    lo, hi = 0, n_rows
    while lo < hi:
        mid = (lo + hi) >> 1
        if indptr[mid] > v:
            hi = mid
        else:
            lo = mid + 1
    return lo - 1


def task_plan(indptr, n_rows, E, T, snap):
    ntasks = (E + T - 1) // T
    first_row = np.zeros(ntasks, np.int64)
    start = np.zeros(ntasks + 1, np.int64)
    start[ntasks] = E
    first_row[0] = row_of_slot(indptr, n_rows, 0)
    for t in range(1, ntasks):
        a = t * T
        r = row_of_slot(indptr, n_rows, a)
        s_r, e_r = indptr[r], indptr[r + 1]
        if s_r < a and e_r - s_r <= snap:
            a = e_r
            r = row_of_slot(indptr, n_rows, a) if a < E else n_rows - 1
        first_row[t] = r
        start[t] = a
    return ntasks, first_row, start


def stream_task(task, indptr, cols, x, scale, n_rows, E, start, first_row, out, partial, tail_row, mean):
    D = x.shape[1]
    a, b = int(start[task]), int(start[task + 1])
    cnt = b - a
    row = int(first_row[task])
    tail = -1
    if cnt > 0:
        def rel(v):
            d = int(v) - a
            return -BIG if d < -BIG else (BIG if d > BIG else d)

        st = {"row": row, "beg": rel(indptr[row]), "end": rel(indptr[row + 1]),
              "nxt": rel(indptr[row + 2]) if row + 2 <= n_rows else BIG,
              "head": rel(indptr[row]) < 0, "acc": np.zeros(D, np.float32)}

        def finish_row():
            acc = st["acc"]
            if st["head"]:
                partial[2 * task] = acc
                st["head"] = False
            else:
                deg = st["end"] - st["beg"]
                v = acc if deg != 0 else np.zeros(D, np.float32)
                if mean and deg != 0:
                    v = v / np.float32(deg)
                out[st["row"]] = v
            st["row"] += 1
            st["beg"] = st["end"]
            st["end"] = st["nxt"]
            st["nxt"] = rel(indptr[st["row"] + 2]) if st["row"] + 2 <= n_rows else BIG
            if st["end"] == st["beg"] and st["row"] < n_rows:
                pos_abs = a + st["beg"]
                if pos_abs >= E:
                    st["row"] = n_rows
                    st["end"] = BIG
                else:
                    st["row"] = row_of_slot(indptr, n_rows, pos_abs)
                    st["end"] = rel(indptr[st["row"] + 1])
                    st["nxt"] = rel(indptr[st["row"] + 2]) if st["row"] + 2 <= n_rows else BIG
            st["acc"] = np.zeros(D, np.float32)

        GPB = 32 // GRP
        ngroups = (cnt + GRP - 1) // GRP

        def batch_scales(batch):   # what a lane holds in sc_cur after loading column batch `batch`
            return [np.float32(scale[cols[a + batch * 32 + j]]) if batch * 32 + j < cnt else np.float32(1)
                    for j in range(32)]

        sc_cur, sc_prev = batch_scales(0), None
        for g in range(ngroups + LAG):
            if g < ngroups and g % GPB == 0 and g > 0:
                sc_prev, sc_cur = sc_cur, batch_scales(g // GPB)
            if g < LAG:
                continue
            gc = g - LAG
            if gc >= ngroups:
                continue
            csub = gc % GPB
            bcur = (g if g < ngroups else ngroups - 1) // GPB
            assert 0 <= bcur - gc // GPB <= 1, (bcur, gc)
            sc_reg = sc_cur if gc // GPB == bcur else sc_prev
            for k in range(GRP):
                s0 = gc * GRP + k
                if s0 >= cnt:
                    break
                while st["end"] <= s0:
                    finish_row()
                sval = sc_reg[csub * GRP + k]
                assert sval == np.float32(scale[cols[a + s0]])
                st["acc"] += x[cols[a + s0]] * sval
        while st["row"] < n_rows and st["end"] <= cnt:
            finish_row()
        if st["row"] < n_rows and st["beg"] < cnt:
            partial[2 * task if st["head"] else 2 * task + 1] = st["acc"]
            if not st["head"]:
                tail = st["row"]
    tail_row[task] = tail


def fixup(ntasks, T, indptr, partial, tail_row, out, mean):
    for t in range(ntasks):
        r = int(tail_row[t])
        if r < 0:
            continue
        s_r, e_r = int(indptr[r]), int(indptr[r + 1])
        acc = partial[2 * t + 1].copy()
        u_end = (e_r + T - 1) // T
        for u in range(t + 1, u_end):
            acc += partial[2 * u]
        if mean:
            acc = acc / np.float32(e_r - s_r)
        out[r] = acc


def model_spmm(edges, n, x, T, mean=False, snap=None, scale=None):
    deg, cols, _, _, indptr = O.build_index(edges[:, 1], edges[:, 0], n)
    E = len(edges)
    snap = T if snap is None else snap
    scale = np.ones(n, np.float32) if scale is None else scale
    ntasks, first_row, start = task_plan(indptr, n, E, T, snap)
    D = x.shape[1]
    out = np.full((n, D), np.nan, np.float32)           # every row must be written by someone
    partial = np.full((2 * ntasks, D), np.nan, np.float32)
    tail_row = np.full(ntasks, -7, np.int64)
    out[deg == 0] = 0.0                                  # empty_rows_kernel
    for t in range(ntasks):
        stream_task(t, indptr, cols, x, scale, n, E, start, first_row, out, partial, tail_row, mean)
    fixup(ntasks, T, indptr, partial, tail_row, out, mean)
    return out


def _graphs():
    rng = np.random.default_rng(901)
    yield "powerlaw", 300, O.chung_lu_edges(300, 2500, exponent=0.9, seed=902)
    yield "uniform", 200, rng.integers(0, 200, (1500, 2))
    e = O.chung_lu_edges(600, 1500, exponent=0.8, seed=903)
    e[:, 1] = e[:, 1] // 9 * 9
    yield "gaps", 600, e
    yield "tiny", 5, np.array([[0, 1], [1, 2], [3, 4], [4, 1], [1, 0]])
    hub = rng.integers(0, 60, (1800, 2))
    hub[:1300, 1] = 7
    yield "hub", 60, hub
    yield "last_rows_empty", 50, np.stack([rng.integers(0, 50, 300), rng.integers(0, 20, 300)], 1)
    yield "single_row", 4, np.stack([rng.integers(0, 4, 100), np.full(100, 2)], 1)


GRAPHS = dict((name, (n, edges)) for name, n, edges in _graphs())


@pytest.mark.parametrize("graph", sorted(GRAPHS))
@pytest.mark.parametrize("T", [32, 64, 2048])
def test_task_model_matches_oracle(graph, T):
    n, edges = GRAPHS[graph]
    edges = np.asarray(edges, np.int64)
    x = np.random.default_rng(910).standard_normal((n, 4)).astype(np.float32)
    for mean in (False, True):
        for snap in (T, max(T, 1024)):
            scale = (np.random.default_rng(911).random(n) + 0.5).astype(np.float32)
            got = model_spmm(edges, n, x, T, mean=mean, snap=snap, scale=scale)
            want = O.send_u_recv(x * scale[:, None], edges[:, 0], edges[:, 1], "mean" if mean else "sum")
            assert not np.isnan(got).any(), (graph, T, mean, snap, "a row was never written")
            err = np.abs(got - want).max() / max(np.abs(want).max(), 1e-12)
            assert err <= 1e-5, (graph, T, mean, snap, err)
