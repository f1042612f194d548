"""RGCNConv's relation-typed aggregation (ops.rgcn_aggregate, csrc/rgcn.cu) on a tensor-mode HeterGraph: the forward
against the reference's op order in float64 (oracle_conv.rgcn_conv), the gradients against float64 torch autograd of
that op order, run-to-run bit identity, the layer against the per-relation route on a dict of Graphs, launches, peak
memory, declined calls, and the reference R-GCN model trained on both routes."""
import numpy as np
import pytest
import torch

from oracle import oracle_conv as OC

pytestmark = pytest.mark.gpu
FWD_BOUND = 2e-5    # of the output's largest magnitude (test_gpu_linear_tc.py's 3xTF32 bound)
GRAD_BOUND = 1e-4


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    return pgl_b200


def rel_graph(n, R, seed, hub_slots=12000):
    """Edges of R relations over n nodes: empty rows (the last 10% of the nodes receive nothing), rows with only
    some relations, one-edge runs, multi-edges, self-loops, and a hub row (node 3) with hub_slots in-edges spread
    over the relations."""
    rng = np.random.default_rng(seed)
    live = int(n * 0.9)
    out = []
    for r in range(R):
        m = int(rng.integers(50, 400))
        src = rng.integers(0, n, m)
        dst = rng.integers(0, live, m)
        k = max(1, m // 10)
        loops = rng.integers(0, live, k)
        src = np.concatenate([src, loops, src[:k]])          # self-loops, then multi-edges
        dst = np.concatenate([dst, loops, dst[:k]])
        hub = hub_slots // R + (hub_slots % R if r == 0 else 0)
        src = np.concatenate([src, rng.integers(0, n, hub)])
        dst = np.concatenate([dst, np.full(hub, 3)])
        out.append(np.stack([src, dst], 1).astype(np.int64))
    return out


def make_heter(pgl, edge_lists, n, etypes):
    g = pgl.HeterGraph(edges={t: e for t, e in zip(etypes, edge_lists)}, num_nodes=n,
                       node_types=[(i, "v") for i in range(n)])
    return g.tensor()


def ref_torch(x, w, edge_lists, n):
    """The reference's op order: sum_r send_recv(x @ w[r], mean), in x's dtype with torch autograd."""
    out = None
    for r, e in enumerate(edge_lists):
        src = torch.as_tensor(e[:, 0], device=x.device)
        dst = torch.as_tensor(e[:, 1], device=x.device)
        h = x @ w[r]
        s = torch.zeros((n, h.shape[1]), dtype=x.dtype, device=x.device).index_add_(0, dst, h[src])
        cnt = torch.bincount(dst, minlength=n).clamp(min=1).to(x.dtype)
        h = s / cnt[:, None]
        out = h if out is None else out + h
    return out


def maxerr(a, b):
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-30))


@pytest.mark.parametrize("R,D,O", [(1, 64, 64), (3, 16, 12), (3, 128, 128), (64, 64, 64), (64, 32, 128)])
def test_forward_and_gradients_against_float64(pgl, R, D, O):
    n = 3000
    etypes = ["r%d" % i for i in range(R)]
    el = rel_graph(n, R, 10 + R)
    g = make_heter(pgl, el, n, etypes)
    fwd, bwd = g.typed_csr(etypes, torch.device("cuda"))
    gen = torch.Generator(device="cpu").manual_seed(R * 7 + D)
    x = torch.randn((n, D), generator=gen).cuda().requires_grad_()
    w = (torch.randn((R, D, O), generator=gen) * 0.2).cuda().requires_grad_()
    gout = torch.randn((n, O), generator=gen).cuda()
    out = pgl.ops.rgcn_aggregate(fwd, bwd, x, w)
    assert out is not None and out.shape == (n, O)
    want = OC.rgcn_conv([(t, e) for t, e in zip(etypes, el)], n, x.detach().cpu().double().numpy(),
                        w.detach().cpu().double().numpy())
    assert maxerr(out, torch.from_numpy(want)) <= FWD_BOUND
    gx, gw = torch.autograd.grad(out, (x, w), gout)

    x64 = x.detach().double().requires_grad_()
    w64 = w.detach().double().requires_grad_()
    ref = ref_torch(x64, w64, el, n)
    assert maxerr(out, ref) <= FWD_BOUND
    rgx, rgw = torch.autograd.grad(ref, (x64, w64), gout.double())
    assert maxerr(gx, rgx) <= GRAD_BOUND
    for r in range(R):     # per relation: small relations must not hide behind the hub's magnitude
        assert maxerr(gw[r], rgw[r]) <= GRAD_BOUND, r

    # bit-identical over two runs
    out2 = pgl.ops.rgcn_aggregate(fwd, bwd, x, w)
    gx2, gw2 = torch.autograd.grad(out2, (x, w), gout)
    assert torch.equal(out, out2) and torch.equal(gx, gx2) and torch.equal(gw, gw2)


def test_typed_csr_layout(pgl):
    """The device build matches the numpy model of test_hetergraph_host on a subset and a reordering of etypes."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location(
        "hetergraph_host_model", os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_hetergraph_host.py"))
    host = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(host)
    typed_csr_model = host.typed_csr_model
    n = 500
    el = rel_graph(n, 5, 3, hub_slots=3000)
    etypes = ["a", "b", "c", "d", "e"]
    g = make_heter(pgl, el, n, etypes)
    for sel in (["c", "a", "e"], ["e", "d", "c", "b", "a"]):
        fwd, bwd = g.typed_csr(sel, torch.device("cuda"))
        m = typed_csr_model([el[etypes.index(t)] for t in sel], n)
        for k in ("indptr", "cols", "rel", "run_row", "run_beg", "run_end", "run_off"):
            assert np.array_equal(fwd[k].cpu().numpy(), m["fwd"][k]), k
        for k in ("indptr", "cols", "rel"):
            assert np.array_equal(bwd[k].cpu().numpy(), m["bwd"][k]), k
        assert np.allclose(bwd["w"].cpu().numpy(), m["bwd"]["w"], rtol=1e-7, atol=0)
        assert int(fwd["item_off"][-1]) == fwd["n_items"]
        assert g.typed_csr(sel, torch.device("cuda"))[0] is fwd     # cached per etype tuple


@pytest.mark.parametrize("num_bases", [0, 2])
def test_layer_matches_dict_route(pgl, num_bases):
    n, d, od = 2500, 64, 64
    all_types = ["cites", "writes", "likes", "owns"]
    el = rel_graph(n, 4, 77)
    g = make_heter(pgl, el, n, all_types)
    graphs = {t: pgl.Graph(edges=e, num_nodes=n).tensor() for t, e in zip(all_types, el)}
    x0 = torch.randn((n, d), generator=torch.Generator().manual_seed(5)).cuda()
    for etypes in (all_types, ["likes", "cites", "owns"], ["owns", "likes", "writes", "cites"]):
        torch.manual_seed(11)
        conv = pgl.nn.RGCNConv(d, od, etypes, num_bases=num_bases).cuda()
        xa = x0.clone().requires_grad_()
        xb = x0.clone().requires_grad_()
        a = conv(g, xa)
        b = conv(graphs, xb)
        assert maxerr(a, b) <= 1e-4
        gout = torch.randn_like(a)
        ga = torch.autograd.grad(a, [xa] + list(conv.parameters()), gout)
        gb = torch.autograd.grad(b, [xb] + list(conv.parameters()), gout)
        for u, v in zip(ga, gb):
            assert maxerr(u, v) <= 1e-4


def test_launches_and_peak_memory(pgl):
    n, d, R = 20000, 64, 16
    etypes = ["r%d" % i for i in range(R)]
    el = rel_graph(n, R, 9, hub_slots=20000)
    g = make_heter(pgl, el, n, etypes)
    graphs = {t: pgl.Graph(edges=e, num_nodes=n).tensor() for t, e in zip(etypes, el)}
    conv = pgl.nn.RGCNConv(d, d, etypes, num_bases=8).cuda()
    x = torch.randn((n, d), device="cuda", requires_grad=True)

    def step(graph):
        out = conv(graph, x)
        out.sum().backward()

    step(g)     # typed CSR built and cached
    step(graphs)
    torch.cuda.synchronize()
    with torch.no_grad():
        l0 = pgl.ops.launch_count()
        conv(g, x)
        assert pgl.ops.launch_count() - l0 == 1
    counts, peaks = {}, {}
    for name, graph in (("fused", g), ("old", graphs)):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        l0 = pgl.ops.launch_count()
        step(graph)
        torch.cuda.synchronize()
        counts[name] = pgl.ops.launch_count() - l0
        peaks[name] = torch.cuda.max_memory_allocated() - base
    assert counts["fused"] < counts["old"], counts
    assert peaks["fused"] < peaks["old"], peaks
    assert peaks["fused"] < n * R * d * 4, peaks    # no [N, R, D] float tensor


def test_declined_calls_fall_back(pgl):
    n = 400
    etypes = ["a", "b"]
    el = rel_graph(n, 2, 21, hub_slots=100)
    g = make_heter(pgl, el, n, etypes)
    fwd, bwd = g.typed_csr(etypes, torch.device("cuda"))
    x = torch.randn((n, 8), device="cuda")
    for xx, ww in ((x.double(), torch.randn((2, 8, 8), device="cuda", dtype=torch.float64)),
                   (x.bfloat16(), torch.randn((2, 8, 8), device="cuda", dtype=torch.bfloat16)),
                   (torch.randn((n, 6), device="cuda"), torch.randn((2, 6, 8), device="cuda")),
                   (x, torch.randn((2, 8, 130), device="cuda")),
                   (x[:-1], torch.randn((2, 8, 8), device="cuda")),
                   (x.cpu(), torch.randn((2, 8, 8)))):
        assert pgl.ops.rgcn_aggregate(fwd, bwd, xx, ww) is None
    graphs = {t: g[t] for t in etypes}
    # a graph of 2^20 edges whose every 64-row tile holds both relations: W staging would outweigh the dense
    # transforms at D = O = 128 (ops.rgcn_fused_pays), so the layer keeps the per-relation route
    rng = np.random.default_rng(5)
    big = [rng.integers(0, 4096, (1 << 19, 2)) for _ in range(2)]
    gb = make_heter(pgl, big, 4096, etypes)
    f2, b2 = gb.typed_csr(etypes, torch.device("cuda"))
    assert not pgl.ops.rgcn_fused_pays(f2, 128, 128) and pgl.ops.rgcn_fused_pays(f2, 16, 16)
    assert pgl.ops.rgcn_aggregate(f2, b2, torch.randn((4096, 128), device="cuda"),
                                  torch.randn((2, 128, 128), device="cuda")) is None
    conv = pgl.nn.RGCNConv(128, 128, etypes).cuda()
    xb = torch.randn((4096, 128), device="cuda")
    with torch.no_grad():
        assert torch.equal(conv(gb, xb), conv({t: gb[t] for t in etypes}, xb))
    for dtype, d in ((torch.float64, 8), (torch.bfloat16, 8), (torch.float32, 6)):
        conv = pgl.nn.RGCNConv(d, 8, etypes).cuda().to(dtype)
        xx = torch.randn((n, d), device="cuda").to(dtype)
        with torch.no_grad():
            a = conv(g, xx)
            b = conv(graphs, xx)
        assert a.dtype == dtype and torch.equal(a, b)


def test_reference_rgcn_model_trains_alike(pgl):
    """examples/rgcn: two RGCNConv layers (64 -> 64, num_bases 8) over a learned nfeat and a linear head, on a seeded
    task whose label is the relation (of 4) through which a node receives edges from a marked half of the nodes."""
    n, R, C, hid = 3000, 8, 4, 64
    rng = np.random.default_rng(123)
    marked = rng.random(n) < 0.5
    label = rng.integers(0, C, n)
    mk, um = np.nonzero(marked)[0], np.nonzero(~marked)[0]
    el = [[] for _ in range(R)]
    for v in range(n):
        for r in range(R):
            k = int(rng.integers(1, 4))
            pool = mk if r == label[v] else um
            for s in rng.choice(pool, k):
                el[r].append((s, v))
    el = [np.asarray(e, np.int64) for e in el]
    etypes = ["rel%d" % r for r in range(R)]
    g = make_heter(pgl, el, n, etypes)
    graphs = {t: g[t] for t in etypes}
    perm = rng.permutation(n)
    train, test = torch.as_tensor(perm[:2000]).cuda(), torch.as_tensor(perm[2000:]).cuda()
    y = torch.as_tensor(label).cuda()

    def fit(graph):
        torch.manual_seed(0)
        nfeat = torch.nn.Parameter(torch.randn(n, hid, device="cuda") * 0.1)
        layers = torch.nn.ModuleList([pgl.nn.RGCNConv(hid, hid, etypes, num_bases=8) for _ in range(2)]).cuda()
        head = torch.nn.Linear(hid, C).cuda()
        opt = torch.optim.Adam([nfeat] + list(layers.parameters()) + list(head.parameters()), lr=0.01)
        for _ in range(60):
            h = nfeat
            for lay in layers:
                h = lay(graph, h)
            loss = torch.nn.functional.cross_entropy(head(h)[train], y[train])
            opt.zero_grad()
            loss.backward()
            opt.step()
        with torch.no_grad():
            h = nfeat
            for lay in layers:
                h = lay(graph, h)
            return float((head(h)[test].argmax(1) == y[test]).float().mean())

    acc_fused, acc_old = fit(g), fit(graphs)
    assert acc_fused >= 0.6 and acc_old >= 0.6, (acc_fused, acc_old)
    assert abs(acc_fused - acc_old) <= 0.05, (acc_fused, acc_old)
