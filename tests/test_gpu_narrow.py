"""GPU tests of the narrow-row kernel: rows of <= 64 floats, the shapes of a column-sharded feature matrix.
spmm_narrow2_kernel (csrc/spmm_narrow2.inl: sub-warp-major 32-slot ranges, plan with row-start flags).  The cut-row
variant (PGLB_STREAM_TASK=64: tasks of one chunk, every long row cut) runs the same tests in a child process -- the
library reads that switch once per process.

Sum order differs from the sequential oracle (ranges of a row are summed separately, then added), so the bar is the
fp32 tolerance, not bit equality."""
import os

import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu
RTOL = 1e-4


def rel_err(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-12) if a.size else 0.0


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    return pgl_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def graphs():
    yield "powerlaw", 3000, O.chung_lu_edges(3000, 60000, exponent=0.9, seed=801)
    yield "uniform", 2000, np.random.default_rng(802).integers(0, 2000, (30000, 2))
    e = O.chung_lu_edges(5000, 20000, exponent=0.8, seed=803)
    e[:, 1] = e[:, 1] // 7 * 7                       # runs of empty rows between the used ones
    yield "gaps", 5000, e
    yield "tiny", 5, np.array([[0, 1], [1, 2], [3, 4], [4, 1], [1, 0]])
    hub = np.random.default_rng(804).integers(0, 400, (40000, 2))
    hub[:30000, 1] = 7                               # one 30k-edge row (cut into tasks)
    yield "hub", 400, hub


@pytest.mark.parametrize("d", [4, 8, 12, 16, 24, 32, 48, 64])
def test_narrow_sum_mean_vs_oracle(pgl, d):
    for name, n, edges in graphs():
        edges = np.asarray(edges, np.int64)
        x = np.random.default_rng(810 + d).standard_normal((n, d)).astype(np.float32)
        g = pgl.Graph(edges=edges, num_nodes=n)
        g.tensor()
        l0 = pgl.ops.launch_count()
        for op in ("sum", "mean"):
            out = g.send_recv(dev(x), op).cpu().numpy()
            want = O.send_u_recv(x, edges[:, 0], edges[:, 1], op)
            assert out.shape == want.shape and rel_err(out, want) <= RTOL, (name, d, op)
        assert pgl.ops.launch_count() > l0


def test_narrow_scaled_and_accumulate(pgl):
    n, d = 3000, 16
    edges = O.chung_lu_edges(n, 50000, exponent=0.85, seed=821)
    rng = np.random.default_rng(822)
    x = rng.standard_normal((n, d)).astype(np.float32)
    g = pgl.Graph(edges=edges, num_nodes=n)
    g.tensor()
    norm = O.degree_norm(O.adj_dst_index(edges, n)[0], np.float32)
    out = g._send_u_recv(dev(x), "sum", None, scale_src=dev(norm.reshape(-1)), scale_dst=dev(norm.reshape(-1)))
    want = O.send_u_recv(x * norm, edges[:, 0], edges[:, 1], "sum") * norm
    assert rel_err(out.cpu().numpy(), want) <= RTOL
    # a column slice of a wider matrix is read in place (ldx > D), and equals the slice of the wide result
    xw = rng.standard_normal((n, 128)).astype(np.float32)
    wide = g.send_recv(dev(xw), "sum")
    xs = dev(xw)[:, 32:48]
    sl = g.send_recv(xs, "sum")
    assert rel_err(sl.cpu().numpy(), wide[:, 32:48].cpu().numpy()) <= RTOL
    # backward goes through the same kernel on the reverse CSR
    x1 = dev(x).requires_grad_(True)
    x2 = dev(x).requires_grad_(True)
    go = torch.randn(n, d, device="cuda")
    g.send_recv(x1, "sum").backward(go)
    ed = dev(edges)
    torch.zeros(n, d, device="cuda").index_add_(0, ed[:, 1], x2[ed[:, 0]]).backward(go)
    assert rel_err(x1.grad.cpu().numpy(), x2.grad.cpu().numpy()) <= RTOL


def _child(extra_env):
    import subprocess
    import sys
    if os.environ.get("PGLB_NARROW_CHILD") == "1":
        pytest.skip("already the child")
    env = dict(os.environ, PGLB_NARROW_CHILD="1", **extra_env)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-m", "gpu",
                        "-p", "no:cacheprovider"], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]


def test_cut_rows_in_child_process():
    """The same tests with 64-slot tasks (rounded up to one chunk: every long row is cut; partials + fix-up work)."""
    _child({"PGLB_STREAM_TASK": "64"})

