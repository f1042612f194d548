"""The fused skip-gram negative-sampling loss (csrc/sgns.cu forward, csr_build + aggregation backward; pgl.nn.functional
.skip_gram_loss, pgl.nn.SkipGramModel) on the GPU: the loss against the float64 oracle over D, K, P and strided tables;
both gradients, dense and sparse, separate and shared, with a hub row past 10^5 touches and repeated ids; saturated
logits; bit identity run to run and between the sparse and dense gradients; refusals before any launch; pinned launch
counts; peak memory at the DeepWalk config; one optimiser step against the torch route; DeepWalk on Cora."""
import math

import numpy as np
import pytest
import torch

import sgns_oracle as SO

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    torch.cuda.set_device(0)
    return pgl_b200


def _tables(seed, N, D, Nc=None, ld=None, scale=None, shared=False):
    """fp32 tables N(0, scale^2), scale 2 / sqrt(D) so |s| reaches a few units; ld > D gives strided views."""
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    scale = scale if scale is not None else 2.0 / math.sqrt(D)
    ld = ld or D
    emb = (torch.randn(N, ld, generator=gen, device="cuda") * scale)[:, :D]
    if shared:
        return emb, emb
    ctx = (torch.randn(Nc or N, ld, generator=gen, device="cuda") * scale)[:, :D]
    return emb, ctx


def _ids(seed, N, Nc, P, K):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed + 1)
    src = torch.randint(0, N, (P,), generator=gen, device="cuda")
    dsts = torch.randint(0, Nc, (P, 1 + K), generator=gen, device="cuda")
    if P >= 6 and N == Nc:
        dsts[0, 0] = src[0]          # src == pos
        dsts[1, 1:] = src[1]         # negatives equal to the centre
        dsts[2, :] = dsts[2, 0]      # repeated ids within a pair
        src[3:6] = src[2]
    return src, dsts


def _np(t):
    return t.detach().cpu().numpy()


def _loss_bound(emb, ctx, src, dsts, loss64):
    """Each logit is an fp32 dot of D products: |ds| <= (D + 2) u sum_d |e_d x_d|; softplus has slope <= 1, and the
    epilogue adds a few ulp per term.  So |d loss| <= mean over terms of that, plus 16 u loss."""
    e = _np(emb).astype(np.float64)[_np(src)]
    x = _np(ctx).astype(np.float64)[_np(dsts)]
    a = np.einsum("pd,pjd->pj", np.abs(e), np.abs(x))
    D = e.shape[1]
    return (D + 2) * U * a.mean() + 16 * U * loss64


def _grad_bound(abs_sum, n_max, D, smax):
    """Per element: the aggregation adds n terms in fp32 (bounded here at 8 sqrt(n) u of their absolute sum, the
    expected-case growth; the worst case n u is never approached by these random tables), each term carries its
    coefficient's error from its logit (relative <= (D + 2) u max sum |e x|) and two roundings."""
    return U * (8 * math.sqrt(n_max) + (D + 2) * max(1.0, smax) + 8) * abs_sum + 1e-30


LOSS_CASES = [(1, 1, 1000), (3, 5, 1_000_000), (16, 20, 5000), (64, 5, 20000), (100, 1, 3000), (128, 20, 8000),
              (200, 5, 4000), (256, 20, 2000), (300, 5, 500), (600, 3, 300), (257, 2, 300), (128, 5, 1)]


@pytest.mark.parametrize("D,K,P", LOSS_CASES)
@pytest.mark.parametrize("ld_extra", [0, 5])
def test_loss_matches_the_oracle(pgl, D, K, P, ld_extra):
    N = 5000
    emb, ctx = _tables(D * 7 + K, N, D, ld=D + ld_extra if ld_extra else None)
    src, dsts = _ids(D + K + P, N, N, P, K)
    with torch.no_grad():
        got = pgl.nn.functional.skip_gram_loss(emb, ctx, src, dsts)
    assert got.shape == () and got.dtype == torch.float32
    want = SO.sgns(_np(emb), _np(ctx), _np(src), _np(dsts))[0]
    assert abs(float(got) - want) <= _loss_bound(emb, ctx, src, dsts, want), (float(got), want)


def _check_grads(pgl, emb, ctx, src, dsts, shared, sparse, g=1.0):
    te = emb.detach().clone().requires_grad_(True)
    tc = te if shared else ctx.detach().clone().requires_grad_(True)
    loss = pgl.nn.functional.skip_gram_loss(te, tc, src, dsts, sparse=sparse)
    grads = torch.autograd.grad(loss * g, [te] if shared else [te, tc])
    e64, c64 = _np(te).astype(np.float64), (None if shared else _np(tc).astype(np.float64))
    s_np, d_np = _np(src), _np(dsts)
    loss64, _, de, dc, (ae, ac) = SO.sgns(e64, c64, s_np, d_np, g=g, shared=shared)
    x = e64 if shared else c64
    smax = np.einsum("pd,pjd->pj", np.abs(e64[s_np]), np.abs(x[d_np])).max()
    D = e64.shape[1]
    assert abs(float(loss) - loss64) <= _loss_bound(te, te if shared else tc, src, dsts, loss64)
    pairs = [(grads[0], de, ae, SO.touched(s_np, d_np) if shared else SO.touched(s_np),
              np.bincount(s_np).max() * (1 + d_np.shape[1]) + (np.bincount(d_np.reshape(-1)).max() if shared else 0))]
    if not shared:
        pairs.append((grads[1], dc, ac, SO.touched(d_np), np.bincount(d_np.reshape(-1)).max()))
    for grad, want, a, rows, n_max in pairs:
        if sparse:
            assert grad.is_sparse and grad.is_coalesced()
            assert np.array_equal(_np(grad.indices()[0]), rows)
            got = _np(grad.to_dense()).astype(np.float64)
        else:
            assert not grad.is_sparse
            got = _np(grad).astype(np.float64)
        assert np.isfinite(got).all()
        tol = _grad_bound(a, n_max, D, smax)
        bad = np.abs(got - want) > tol
        assert not bad.any(), (np.argwhere(bad)[:5], got[bad][:5], want[bad][:5], tol[bad][:5])


@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("D,K,P", [(3, 5, 2000), (64, 5, 20000), (128, 20, 5000), (100, 1, 3000), (600, 2, 300)])
def test_grads_match_autograd(pgl, shared, sparse, D, K, P):
    N = 3000 if P > 3000 else 50_000          # dense collisions, and a table mostly untouched
    emb, ctx = _tables(D + 11 * K, N, D, shared=shared)
    src, dsts = _ids(P + D, N, N, P, K)
    _check_grads(pgl, emb, ctx, src, dsts, shared, sparse, g=0.75)


# D (and leading dimension) reaching every training layout of the forward kernel, so c and w are checked on each:
# 16-byte rows G = 4, 8, 16, 32 with NV = 1, 2, 4 and the wide kernel; 4-byte rows G = 4, 8, 16, 32 with NV = 1, 2, 4,
# 8 (unaligned D, or D = 128 with an odd leading dimension) and the wide kernel.
LAYOUT_CASES = [(16, None), (32, None), (64, None), (128, None), (200, None), (300, None), (600, None), (3, None),
                (6, None), (13, None), (30, None), (50, None), (99, None), (130, None), (128, 129), (257, None)]


@pytest.mark.parametrize("D,ld", LAYOUT_CASES)
def test_every_training_layout(pgl, D, ld):
    P, K, N = 3000, 5, 2000
    emb, ctx = _tables(D + 5, N, D, ld=ld)
    src, dsts = _ids(D + 6, N, N, P, K)
    _check_grads(pgl, emb, ctx, src, dsts, False, False, g=1.25)


def test_inference_writes_the_loss_only(pgl):
    """Under torch.no_grad() the kernel takes its loss-only form even for tables that require grad (Parameters, as in a
    model's evaluation): the loss is the training forward's bit for bit, no [P, D] buffer is allocated, and nothing is
    saved for a backward."""
    P, K, D, N = 200_000, 5, 128, 50_000
    torch.manual_seed(2)
    m = pgl.nn.SkipGramModel(N, embed_size=D, neg_num=K).cuda()
    src, dsts = _ids(15, N, N, P, K)
    train_loss = m(src, dsts)
    assert train_loss.requires_grad
    want = train_loss.detach().clone()
    del train_loss
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        got = m(src, dsts)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert not got.requires_grad and torch.equal(got, want)
    assert peak < P * D * 4 // 8, peak
    # a table that needs no gradient in grad mode takes the same loss-only form
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    got2 = pgl.nn.functional.skip_gram_loss(m.emb.weight.detach(), m.v_emb.weight.detach(), src, dsts)
    torch.cuda.synchronize()
    assert torch.equal(got2, want) and torch.cuda.max_memory_allocated() - base < P * D * 4 // 8


def test_overlapping_row_views_are_copied(pgl):
    """An expanded row (stride(0) = 0) or a view whose rows overlap is read from a contiguous copy."""
    D, N = 8, 50
    row = torch.randn(1, D, device="cuda")
    emb = row.expand(N, D)
    base = torch.randn(N * 4 + D, device="cuda")
    ctx = base.as_strided((N, D), (4, 1))
    src, dsts = _ids(16, N, N, 40, 3)
    got = pgl.nn.functional.skip_gram_loss(emb, ctx, src, dsts)
    want = pgl.nn.functional.skip_gram_loss(emb.contiguous(), ctx.contiguous(), src, dsts)
    assert torch.equal(got, want)


@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("sparse", [False, True])
def test_hub_row(pgl, shared, sparse):
    """Node 0 is the centre of 60 % of 200 000 pairs and the positive of 60 %: > 10^5 touches in each role reach the
    aggregation's hub and cut-row paths."""
    P, K, D, N = 200_000, 3, 64, 10_000
    emb, ctx = _tables(77, N, D, shared=shared, scale=0.1)
    src, dsts = _ids(78, N, N, P, K)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(79)
    hub = torch.rand(P, generator=gen, device="cuda") < 0.6
    src = torch.where(hub, 0, src)
    dsts[:, 0] = torch.where(torch.rand(P, generator=gen, device="cuda") < 0.6, 0, dsts[:, 0])
    assert int((src == 0).sum()) > 100_000 and int((dsts == 0).sum()) > 100_000
    _check_grads(pgl, emb, ctx, src, dsts, shared, sparse)


def test_int32_ids_and_float64_tables(pgl):
    emb, ctx = _tables(5, 400, 16)
    src, dsts = _ids(6, 400, 400, 500, 4)
    want = pgl.nn.functional.skip_gram_loss(emb, ctx, src, dsts)
    assert torch.equal(pgl.nn.functional.skip_gram_loss(emb, ctx, src.int(), dsts.int()), want)
    e64 = emb.double().requires_grad_(True)
    got = pgl.nn.functional.skip_gram_loss(e64, ctx.double(), src.reshape(-1, 1), dsts)
    assert got.dtype == torch.float64 and float(got) == float(want)
    got.backward()
    assert e64.grad.dtype == torch.float64


def test_saturated_logits_are_finite(pgl):
    """|s| = 100 on every term, both signs: finite loss and gradients."""
    emb = torch.tensor([[10.0, 0, 0, 0], [-10.0, 0, 0, 0], [0, 10.0, 0, 0], [0, 0, 0, 0]], device="cuda")
    ctx = emb.clone()
    src = torch.tensor([0, 1, 0, 1, 2], device="cuda")
    dsts = torch.tensor([[0, 1, 0], [1, 0, 1], [1, 0, 0], [0, 1, 1], [2, 2, 3]], device="cuda")
    for sparse in (False, True):
        te = emb.clone().requires_grad_(True)
        tc = ctx.clone().requires_grad_(True)
        loss = pgl.nn.functional.skip_gram_loss(te, tc, src, dsts, sparse=sparse)
        loss.backward()
        want = SO.sgns(_np(emb), _np(ctx), _np(src), _np(dsts))
        assert math.isfinite(float(loss)) and abs(float(loss) - want[0]) <= 1e-5 * want[0]
        for grad in (te.grad, tc.grad):
            dense = grad.to_dense() if sparse else grad
            assert torch.isfinite(dense).all()


def test_bit_identity(pgl):
    """Two forward + backward runs are identical bit for bit; with separate tables the sparse gradients' values are
    the dense gradients' touched rows bit for bit."""
    P, K, D, N = 69_744, 20, 128, 1 << 16
    emb, ctx = _tables(3, N, D)
    src, dsts = _ids(4, N, N, P, K)
    runs = []
    for sparse in (False, False, True, True):
        te = emb.detach().clone().requires_grad_(True)
        tc = ctx.detach().clone().requires_grad_(True)
        loss = pgl.nn.functional.skip_gram_loss(te, tc, src, dsts, sparse=sparse)
        runs.append((loss.detach(),) + torch.autograd.grad(loss, [te, tc]))
    for a, b in ((runs[0], runs[1]), (runs[2], runs[3])):
        assert torch.equal(a[0], b[0])
        for ga, gb in ((a[1], b[1]), (a[2], b[2])):
            if ga.is_sparse:
                assert ga.is_coalesced() and gb.is_coalesced()
                assert torch.equal(ga.indices(), gb.indices()) and torch.equal(ga.values(), gb.values())
            else:
                assert torch.equal(ga, gb)
    assert torch.equal(runs[0][0], runs[2][0])
    for dense, sp in ((runs[0][1], runs[2][1]), (runs[0][2], runs[2][2])):
        rows = sp.indices()[0]
        assert torch.equal(dense[rows], sp.values())
        untouched = torch.ones(N, dtype=torch.bool, device="cuda")
        untouched[rows] = False
        assert not dense[untouched].any()


def test_refusals_before_any_launch(pgl):
    F = pgl.nn.functional
    emb, ctx = _tables(1, 100, 8)
    src, dsts = _ids(2, 100, 100, 50, 3)
    torch.cuda.synchronize()
    before = pgl.ops.launch_count()
    bad_src = src.clone()
    bad_src[7] = 100
    with pytest.raises(IndexError):
        F.skip_gram_loss(emb, ctx, bad_src, dsts)
    bad_dsts = dsts.clone()
    bad_dsts[3, 2] = -1
    with pytest.raises(IndexError):
        F.skip_gram_loss(emb, ctx, src, bad_dsts)
    with pytest.raises(IndexError):
        F.skip_gram_loss(emb, ctx[:50], src, dsts.clamp(max=99) * 0 + 60)
    with pytest.raises(TypeError):
        F.skip_gram_loss(emb.half(), ctx, src, dsts)
    with pytest.raises(TypeError):
        F.skip_gram_loss(emb, ctx.bfloat16(), src, dsts)
    with pytest.raises(ValueError):
        F.skip_gram_loss(emb, ctx, src.float(), dsts)
    with pytest.raises(ValueError):
        F.skip_gram_loss(emb, ctx, src, dsts[:, :1])
    with pytest.raises(ValueError):
        F.skip_gram_loss(emb, ctx, src, dsts.bool())
    with pytest.raises(ValueError):
        F.skip_gram_loss(emb, ctx, src.reshape(5, 10), dsts)
    torch.cuda.synchronize()
    assert pgl.ops.launch_count() == before


def test_launch_counts(pgl):
    """Forward: the fused kernel and the loss sum, with or without grad.  Backward: two csr_builds (the P centre keys,
    the P (1 + K) context keys) and one aggregation per table, nothing else from the library."""
    from pgl_b200 import ops
    P, K, D, N = 5000, 5, 64, 3000
    emb, ctx = _tables(9, N, D)
    src, dsts = _ids(10, N, N, P, K)
    with torch.no_grad():
        before = ops.launch_count()
        pgl.nn.functional.skip_gram_loss(emb, ctx, src, dsts)
        assert ops.launch_count() - before == 2
    te = emb.detach().clone().requires_grad_(True)
    tc = ctx.detach().clone().requires_grad_(True)
    before = ops.launch_count()
    loss = pgl.nn.functional.skip_gram_loss(te, tc, src, dsts)
    assert ops.launch_count() - before == 2
    before = ops.launch_count()
    loss.backward()
    bwd = ops.launch_count() - before
    # the same pieces, called one by one
    J = K + 1
    before = ops.launch_count()
    _, _, _, pair, ip_e = ops.csr_build(src, src, N)
    _, col_c, _, slot_c, ip_c = ops.csr_build(dsts.reshape(-1), src.repeat_interleave(J), N)
    w = torch.zeros(P, D, device="cuda")
    ops._spmm_raw(ip_e, pair, w, N, "sum", y2=torch.ones(P, 1, device="cuda"), y_bcast=ops.BCAST_SCALAR,
                  msg_op="mul", num_edges=P)
    ops._spmm_raw(ip_c, col_c, te.detach(), N, "sum", eid=slot_c, y2=torch.ones(P * J, 1, device="cuda"),
                  y_bcast=ops.BCAST_SCALAR, msg_op="mul", num_edges=P * J)
    assert bwd == ops.launch_count() - before
    print("skip_gram_loss launches: forward 2, backward %d" % bwd)


def test_peak_memory_at_the_deepwalk_config(pgl):
    """512 walks x 40, window 10, 20 negatives: 69 744 pairs, D = 128, 2^20-node tables.  Forward + backward needs
    below one [P, 1 + K, D] fp32 tensor beyond the tables and their two gradients (which the torch route needs too)."""
    P, K, D, N = 69_744, 20, 128, 1 << 20
    emb, ctx = _tables(11, N, D)
    emb.requires_grad_(True)
    ctx.requires_grad_(True)
    src, dsts = _ids(12, N, N, P, K)
    pgl.nn.functional.skip_gram_loss(emb, ctx, src, dsts).backward()     # warm the workspace caches
    emb.grad = ctx.grad = None
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    pgl.nn.functional.skip_gram_loss(emb, ctx, src, dsts).backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base - 2 * N * D * 4
    rows = P * (1 + K) * D * 4
    print("deepwalk config: transient peak %.1f MB, one [P, 1 + K, D] fp32 tensor %.1f MB" % (peak / 2 ** 20,
                                                                                             rows / 2 ** 20))
    assert peak < rows


def test_one_sgd_step_matches_the_torch_route(pgl):
    P, K, D, N = 20_000, 5, 64, 5000
    torch.manual_seed(0)
    m_fused = pgl.nn.SkipGramModel(N, embed_size=D, neg_num=K).cuda()
    with torch.no_grad():
        m_fused.v_emb.weight.uniform_(-0.1, 0.1)
    src, dsts = _ids(13, N, N, P, K)
    e0, c0 = m_fused.emb.weight.detach().clone(), m_fused.v_emb.weight.detach().clone()
    opt = torch.optim.SGD(m_fused.parameters(), lr=1000.0)
    m_fused(src, dsts).backward()
    opt.step()
    te, tc = e0.clone().requires_grad_(True), c0.clone().requires_grad_(True)
    from test_sgns_host import reference_model
    reference_model(te, tc, src, dsts).backward()
    with torch.no_grad():
        te -= 1000.0 * te.grad
        tc -= 1000.0 * tc.grad
    _, _, de, dc, (ae, ac) = SO.sgns(_np(e0), _np(c0), _np(src), _np(dsts))
    smax = 1.0 * D
    for got, ref, a, n in ((m_fused.emb.weight, te, ae, np.bincount(_np(src)).max() * (K + 1)),
                           (m_fused.v_emb.weight, tc, ac, np.bincount(_np(dsts).reshape(-1)).max())):
        # both routes' updates lie within the gradient bound of the exact step; the tables' own rounding adds 1 ulp
        tol = 1000.0 * 2 * _grad_bound(a, n, D, smax) + U * 2 * np.abs(_np(ref)).astype(np.float64)
        assert (np.abs(_np(got).astype(np.float64) - _np(ref).astype(np.float64)) <= tol).all()


@pytest.mark.parametrize("opt_name", ["SparseAdam", "SGD", "Adagrad"])
def test_sparse_optimisers_step(pgl, opt_name):
    P, K, D, N = 4000, 5, 32, 100_000
    torch.manual_seed(1)
    m = pgl.nn.SkipGramModel(N, embed_size=D, neg_num=K, sparse=True).cuda()
    with torch.no_grad():
        m.v_emb.weight.uniform_(-0.5, 0.5)
    src, dsts = _ids(14, 2000, 2000, P, K)
    before_e, before_c = m.emb.weight.detach().clone(), m.v_emb.weight.detach().clone()
    # SGD's step is lr g with g ~ 1 / P: a large lr moves it as far as the normalised optimisers' lr does
    opt = getattr(torch.optim, opt_name)(m.parameters(), lr=1000.0 if opt_name == "SGD" else 0.05)
    loss = m(src, dsts)
    loss.backward()
    assert m.emb.weight.grad.is_sparse and m.v_emb.weight.grad.is_sparse
    opt.step()
    changed = (m.emb.weight != before_e).any(1)
    assert changed[src].all() and not changed[2000:].any()
    assert (m.v_emb.weight != before_c).any(1)[dsts.reshape(-1)].all()
    assert float(m(src, dsts)) < float(loss)


# ---- DeepWalk on Cora: the fused and torch routes on identical batches, init and seeds ----------------------------

DW_STEPS, DW_BATCH, DW_WALK, DW_WIN, DW_NEG, DW_DIM, DW_LR = 200, 512, 40, 5, 5, 64, 0.05
# Probe accuracy of SkipGramModel (U(-1, 1) centre init) after DW_STEPS steps with Adam.  Measured on an H100 80GB HBM3
# (700 W): fused 0.7504, torch route 0.7504, fused sparse + SparseAdam 0.7526.  The floor sits below all three so it
# catches a broken model, and the gap allows the routes' different summation orders.
SG_FLOOR, SG_GAP = 0.72, 0.02


def _deepwalk_cora(pgl, fused, sparse):
    import os

    from oracle import oracle as O
    from test_gpu_skipgram import _probe
    cora = O.load_cora(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cora.npz"))
    n, edges = cora["num_nodes"], cora["edges"]
    edges = np.concatenate([edges, edges[:, ::-1]])
    g = pgl.Graph(edges=edges, num_nodes=n).tensor()
    y = torch.from_numpy(cora["y"]).cuda()
    deg = np.bincount(edges[:, 0], minlength=n).astype(np.float64)
    alias, events = pgl.sampling.alias_table(torch.from_numpy(deg ** 0.75).cuda())
    batches = np.random.default_rng(0).integers(0, n, (DW_STEPS, DW_BATCH))
    torch.manual_seed(0)
    m = pgl.nn.SkipGramModel(n, embed_size=DW_DIM, neg_num=DW_NEG, sparse=sparse).cuda()
    opt = (torch.optim.SparseAdam if sparse else torch.optim.Adam)(list(m.parameters()), lr=DW_LR)
    from test_sgns_host import reference_model
    for step in range(DW_STEPS):
        walks = pgl.sampling.random_walk(g, torch.from_numpy(batches[step]).cuda(), DW_WALK, seed=1000 + step)
        src, pos = pgl.sampling.skip_gram_pairs(walks, DW_WIN, seed=2000 + step)
        neg = pgl.sampling.alias_sample(alias, events, (src.numel(), DW_NEG), seed=3000 + step)
        dsts = torch.cat([pos[:, None], neg], 1)
        loss = m(src, dsts) if fused else reference_model(m.emb.weight, m.v_emb.weight, src, dsts)
        opt.zero_grad()
        loss.backward()
        opt.step()
    return _probe(m.emb.weight.detach(), y, 0)


def test_deepwalk_on_cora(pgl):
    acc_fused = _deepwalk_cora(pgl, True, False)
    acc_torch = _deepwalk_cora(pgl, False, False)
    acc_sparse = _deepwalk_cora(pgl, True, True)
    print("skip-gram deepwalk cora probe accuracy: fused %.4f torch %.4f fused sparse+SparseAdam %.4f"
          % (acc_fused, acc_torch, acc_sparse))
    assert acc_fused >= acc_torch - SG_GAP and acc_fused >= SG_FLOOR
    assert acc_sparse >= SG_FLOOR
