"""Per-slot source norms of the wide-row aggregation (spmm_v5_kernel): streaming scale_src[cols[j]] per CSR slot must
give bit for bit what gathering scale_src per edge gives, in both ring geometries, D = 128 (no hints, some rows hot,
every row hot) and D < 128, with hub rows cut into task partials and with empty rows.  Also the caching rule of EdgeIndex.slot_scale
and the argument check of the C entry point."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as O

EMPTY = 100  # trailing nodes without any edge: empty rows and never-gathered sources


def _graph(pgl, n, e, seed):
    """Chung-Lu graph (hubs of thousands of in-edges, far longer than a task) plus EMPTY isolated nodes."""
    edges = O.chung_lu_edges(n, e, exponent=0.8, seed=seed)
    g = pgl.Graph(edges=edges, num_nodes=n + EMPTY)
    g.tensor()
    return g, edges


def _mismatches(all_hot=False):
    """Every case the v5 kernel takes, streamed vs gathered norms; returns the cases that differ.  all_hot: at D = 128
    only, bit 31 on every id, so every row comes by per-lane cp.async (LDGSTS) and the gathered norms share its
    commit groups."""
    import pgl_b200 as pgl
    import pgl_b200.nn.functional as GF
    from pgl_b200 import ops
    bad = []
    for avg_deg in (5, 15):              # v5_geo: groups of 4 below 12 slots per row, groups of 8 above
        n = 20000
        g, _ = _graph(pgl, n, n * avg_deg, seed=avg_deg)
        N = n + EMPTY
        fwd = g._fwd_csr()
        norm = GF.degree_norm(g).reshape(-1)
        assert fwd["slot_scale"](norm) is None and fwd["slot_scale"](norm) is not None
        for D in ((128,) if all_hot else (128, 96)):
            x = torch.randn(N, D, device="cuda", generator=torch.Generator("cuda").manual_seed(D))
            for budget in ((None,) if all_hot else (0, 1 << 20)):  # no hints / the 2048 heaviest rows (D = 128 only)
                pk = (fwd["cols"].to(torch.int32) | -(1 << 31), True) if all_hot else \
                    tuple(ops.pack_cols(fwd["cols"], N, 4 * D, budget_bytes=budget))
                outs = [ops._spmm_raw(fwd["indptr"], fwd["cols"], x, N, "sum", scale_src=norm, scale_dst=norm,
                                      max_degree=fwd["max_degree"], packed=p)
                        for p in (pk, ops.PackedCols(pk, fwd["slot_scale"]))]
                if not torch.equal(outs[0], outs[1]):
                    bad.append((avg_deg, D, budget))
    return bad


@pytest.mark.gpu
def test_streamed_norms_bit_identical_to_gathered():
    assert _mismatches() == []


@pytest.mark.gpu
def test_streamed_norms_bit_identical_ldgsts_ring():
    assert _mismatches(all_hot=True) == []


@pytest.mark.gpu
def test_kernel_reads_the_slot_array():
    """The per-slot array is what the kernel multiplies by: twice the per-slot norms (exact in fp32) give exactly twice
    the output, although scale_src is unchanged."""
    import pgl_b200 as pgl
    import pgl_b200.nn.functional as GF
    from pgl_b200 import _lib, ops
    n = 20000
    g, _ = _graph(pgl, n, n * 15, seed=3)
    N = n + EMPTY
    fwd = g._fwd_csr()
    norm = GF.degree_norm(g).reshape(-1)
    x = torch.randn(N, 128, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    pk = ops.pack_cols(fwd["cols"], N, 512, budget_bytes=1 << 20)
    E = int(fwd["cols"].shape[0])
    need = ctypes.c_size_t(0)
    _lib.check(_lib.lib.pglb_spmm_csr_ws(N, E, 128, ctypes.byref(need)))
    ws = ops.workspace(x.device, need.value)
    outs = []
    for mult in (1.0, 2.0):
        slot = norm[fwd["cols"]] * mult
        out = torch.empty(N, 128, device="cuda")
        _lib.check(_lib.lib.pglb_spmm_csr_slot_scale_f32(
            ops._ptr(fwd["indptr"]), ops._ptr(fwd["cols"]), None, ops._ptr(x), 128, None, 0, 0, ops._ptr(out), 128, N,
            N, E, 128, 1, _lib.MSG["copy"], _lib.REDUCE["sum"], ops._ptr(norm), ops._ptr(slot), ops._ptr(norm),
            ops._ptr(pk[0]), -1, 2, ops._ptr(ws), ws.numel(), ops._stream()))
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(outs[1], outs[0] * 2)
    assert float(outs[0].abs().max()) > 0 and bool((outs[0][n:] == 0).all())   # isolated nodes: empty rows


@pytest.mark.gpu
def test_inplace_scale_change_is_picked_up():
    """Public path (Graph._send_u_recv with the GCN norms): an in-place change to the scale tensor must reach the
    kernel both before and after the per-slot copy is rebuilt."""
    import pgl_b200 as pgl
    import pgl_b200.nn.functional as GF
    n = 20000
    g, edges = _graph(pgl, n, n * 10, seed=4)
    N = n + EMPTY
    x = np.random.default_rng(5).standard_normal((N, 128)).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    norm = GF.degree_norm(g).reshape(-1)

    def run():
        return g._send_u_recv(xd, "sum", None, scale_src=norm, scale_dst=None)

    first, second = run(), run()          # gathered, then streamed from the per-slot copy
    assert torch.equal(first, second)
    cache = g.adj_dst_index._slot_scale_cache
    assert cache["ref"] is norm
    nrm = norm.cpu().numpy()
    want = O.send_u_recv(x * nrm[:, None], edges[:, 0], edges[:, 1], "sum", out_size=N)
    assert np.abs(second.cpu().numpy() - want).max() <= 1e-4 * np.abs(want).max()
    norm.mul_(2.0)                        # exact: every product and sum doubles
    third, fourth = run(), run()          # first sighting of the new version (gathered), then a rebuilt copy
    assert torch.equal(third, second * 2) and torch.equal(fourth, second * 2)


def test_slot_scale_materialised_on_second_sighting():
    """A scale tensor seen once (a one-off product, e.g. in the mean backward) is never laid out per slot; one seen
    twice in a row is, and stays cached while one-off tensors come and go."""
    from pgl_b200.utils.edge_index import EdgeIndex
    cols = torch.tensor([2, 0, 1, 2, 2], dtype=torch.int64)
    ei = EdgeIndex.from_index(cols, torch.zeros(5, dtype=torch.int64), torch.arange(5), torch.tensor([5, 0, 0]),
                              torch.tensor([0, 5, 5, 5]))
    s = torch.tensor([0.5, 0.25, 2.0])
    assert ei.slot_scale(s) is None
    v = ei.slot_scale(s)
    assert v is not None and v.tolist() == [2.0, 0.5, 0.25, 2.0, 2.0]
    assert ei.slot_scale(s) is v
    one_off = s * 3
    assert ei.slot_scale(one_off) is None
    assert ei.slot_scale(s) is v          # the one-off did not evict the cached copy
    s.mul_(2)                             # in place: a new version, seen once
    assert ei.slot_scale(s) is None
    assert ei.slot_scale(s).tolist() == [4.0, 1.0, 0.5, 4.0, 4.0]


def test_slot_scale_entry_needs_scale_src():
    """The kernels that do not stream the per-slot array gather scale_src, so it must come with it."""
    from pgl_b200 import _lib
    one = ctypes.c_void_p(16)   # non-NULL dummy, never dereferenced: the check comes before any device work
    rc = _lib.lib.pglb_spmm_csr_slot_scale_f32(one, one, None, one, 128, None, 0, 0, one, 128, 10, 10, 100, 128, 1,
                                               _lib.MSG["copy"], _lib.REDUCE["sum"], None, one, None, None, -1, 0,
                                               None, 0, None)
    assert rc < 0 and b"scale_slot needs scale_src" in _lib.lib.pglb_last_error()


def test_hot_budget_override(monkeypatch):
    from pgl_b200 import ops
    monkeypatch.setenv("PGLB_HOT_MB", "24")
    assert ops.hot_l2_bytes("cuda:0") == 24 << 20
    monkeypatch.setenv("PGLB_HOT_MB", "0")
    assert ops.hot_l2_bytes("cuda:0") == 0
