"""Argument checks of the GATv2 attention entries (pglb_gatv2_attn_csr_*, pglb_gatv2_attn_drop_csr_*,
pglb_gatv2_bwd_edge_*, pglb_gatv2_bwd_edge_drop_*, pglb_gatv2_score_grad_*): the new symbols are exported, and every
call below is refused (or has nothing to do) before any CUDA call, so they are checked without a GPU."""
import ctypes

import pytest

EINVAL, ESHAPE, EUNSUPPORTED, EWORKSPACE = -1, -2, -4, -3

NAMES = ["pglb_gatv2_attn_csr_f32", "pglb_gatv2_attn_csr_x16", "pglb_gatv2_attn_drop_csr_f32",
         "pglb_gatv2_attn_drop_csr_x16", "pglb_gatv2_bwd_edge_ws", "pglb_gatv2_bwd_edge_f32",
         "pglb_gatv2_bwd_edge_x16", "pglb_gatv2_bwd_edge_drop_f32", "pglb_gatv2_bwd_edge_drop_x16",
         "pglb_gatv2_score_grad_f32", "pglb_gatv2_score_grad_x16"]


@pytest.fixture(scope="module")
def lib():
    from pgl_b200 import _lib
    return _lib


P = ctypes.c_void_p(256)     # a non-NULL, 256-byte aligned dummy: must never be dereferenced here
P8 = ctypes.c_void_p(264)    # 8-byte but not 16-byte aligned


def _err(lib):
    return lib.lib.pglb_last_error()


def test_symbols_exported_and_declared(lib):
    import os
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "pglb.h")).read()
    for name in NAMES:
        assert hasattr(lib.lib, name), name
        assert name + "(" in hdr, name


def test_workspace_size(lib):
    need = ctypes.c_size_t(0)
    assert lib.lib.pglb_gatv2_bwd_edge_ws(1000, ctypes.byref(need)) == 0 and need.value >= 512
    assert lib.lib.pglb_gatv2_bwd_edge_ws(-1, ctypes.byref(need)) == EINVAL
    assert lib.lib.pglb_gatv2_bwd_edge_ws(10, None) == EINVAL


@pytest.mark.parametrize("kind", ["f32", "x16", "drop_f32", "drop_x16"])
def test_gatv2_forward_argument_checks(lib, kind):
    half = kind.endswith("x16")
    drop = kind.startswith("drop")
    el = 2 if half else 4

    def call(dtype=None, f=P, attn=P, ld=None, ldo=None, out=P, n=10, E=20, H=8, Dh=16, slope=0.2, p=0.5, offset=0,
             lse=P, cols=P):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        ld = H * Dh if ld is None else ld
        ldo = H * Dh if ldo is None else ldo
        # (indptr, cols, f, ldf, attn, slope, out, ldo, lse, n, E, H, head_dim, [dtype,] [attn_drop, seed, offset,]
        #  ws, ws_bytes, stream)
        args = [P, cols, f, ld, attn, slope, out, ldo, lse, n, E, H, Dh]
        if half:
            args.append(dtype)
        if drop:
            args += [p, 7, offset]
        fn = getattr(lib.lib, "pglb_gatv2_attn_%scsr_%s" % ("drop_" if drop else "", "x16" if half else "f32"))
        return fn(*args, P, 1 << 20, None)

    if half:
        assert call(dtype=0) == EINVAL and b"dtype" in _err(lib)
        assert call(dtype=3) == EINVAL
    assert call(H=0) == EINVAL and call(Dh=0) == EINVAL and call(n=-1) == EINVAL and call(E=-1) == EINVAL
    assert call(Dh=6) == EUNSUPPORTED            # head_dim % 4
    assert call(H=4, Dh=12) == EUNSUPPORTED      # head_dim not a power of two: the head sum is a xor butterfly
    assert call(H=16, Dh=16) == EUNSUPPORTED     # 256 elements per row
    assert call(H=1, Dh=7) == EUNSUPPORTED and b"head_dim" in _err(lib)   # the citation model's second layer
    if half:
        assert call(H=3, Dh=4) == EUNSUPPORTED   # 24-byte rows: not a multiple of 16 bytes
    assert call(slope=-0.1) == EUNSUPPORTED and call(slope=1.5) == EUNSUPPORTED
    assert call(slope=float("nan")) == EUNSUPPORTED and b"slope" in _err(lib)
    assert call(f=P8) == ESHAPE and call(attn=P8) == ESHAPE and call(out=P8) == ESHAPE
    assert call(ld=8 * 16 + 16 // el + 2) == ESHAPE      # a row stride that is not a multiple of 16 bytes
    assert call(ldo=64) == ESHAPE                        # ldo < D
    assert call(ld=64) == ESHAPE                         # ldf < D
    if drop:
        assert call(p=0.0) == EINVAL and call(p=1.0) == EINVAL and call(p=float("nan")) == EINVAL
        assert call(offset=2) == EINVAL and b"offset" in _err(lib)
        assert call(H=2, Dh=32) == EUNSUPPORTED and b"H % 4" in _err(lib)
        assert call(p=1.5, n=0) == EINVAL                # the dropout arguments are checked first
    else:
        assert call(H=2, Dh=32, n=0) == 0                # any head count without dropout
    assert call(slope=0.0, n=0) == 0 and call(slope=1.0, n=0) == 0
    assert call(n=0) == 0                                # nothing to do: no device work
    assert call(n=5, E=5, cols=None, lse=None) == EINVAL  # NULL cols with edges


@pytest.mark.parametrize("kind", ["f32", "x16", "drop_f32", "drop_x16"])
def test_gatv2_bwd_edge_argument_checks(lib, kind):
    half = kind.endswith("x16")
    drop = kind.startswith("drop")

    def call(dtype=None, f=P, g=P, attn=P, ld=128, ldg=128, E=20, H=8, Dh=16, slope=0.2, lse=P, beta=P, p=0.5,
             offset=0, ga=P, ws=P, ws_bytes=1 << 30):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        # (rows, cols, eid, f, ldf, attn, slope, grad_out, ldg, out, ldo, lse, E, H, head_dim, [dtype,]
        #  [attn_drop, seed, offset,] beta_e, ds_e, grad_attn, ws, ws_bytes, stream)
        args = [P, P, P, f, ld, attn, slope, g, ldg, P, ld, lse, E, H, Dh]
        if half:
            args.append(dtype)
        if drop:
            args += [p, 7, offset]
        fn = getattr(lib.lib, "pglb_gatv2_bwd_edge_%s%s" % ("drop_" if drop else "", "x16" if half else "f32"))
        return fn(*args, beta, P, ga, ws, ws_bytes, None)

    if half:
        assert call(dtype=0) == EINVAL and b"dtype" in _err(lib)
    assert call(H=0) == EINVAL and call(E=-1) == EINVAL
    assert call(Dh=6) == EUNSUPPORTED and call(H=4, Dh=12) == EUNSUPPORTED and call(H=16, Dh=16) == EUNSUPPORTED
    assert call(slope=2.0) == EUNSUPPORTED
    assert call(lse=None) == EINVAL and call(beta=None) == EINVAL
    assert call(f=P8) == ESHAPE and call(g=P8) == ESHAPE and call(attn=P8) == ESHAPE
    assert call(ldg=120) == ESHAPE                       # ldg < D
    assert call(ld=130) == ESHAPE                        # not a multiple of 16 bytes
    assert call(ws=None) == EWORKSPACE and call(ws_bytes=16) == EWORKSPACE   # grad attn needs the workspace
    assert call(E=0, ga=None) == 0
    if drop:
        assert call(p=0.0) == EINVAL and call(p=1.0) == EINVAL
        assert call(offset=6) == EINVAL
        assert call(H=2, Dh=32) == EUNSUPPORTED
    else:
        assert call(H=2, Dh=32, E=0, ga=None) == 0


@pytest.mark.parametrize("half", [False, True])
def test_gatv2_score_grad_argument_checks(lib, half):
    def call(dtype=None, f=P, attn=P, ds=P, out=P, ld=128, ldo=128, n=10, E=20, H=8, Dh=16, slope=0.2, cols=P):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        # (indptr, cols, eid, f, ldf, attn, slope, ds, out, ldo, n_rows, E, H, head_dim, [dtype,] accumulate,
        #  ws, ws_bytes, stream)
        args = [P, cols, P, f, ld, attn, slope, ds, out, ldo, n, E, H, Dh]
        if half:
            args.append(dtype)
        fn = lib.lib.pglb_gatv2_score_grad_x16 if half else lib.lib.pglb_gatv2_score_grad_f32
        return fn(*args, 0, P, 1 << 20, None)

    if half:
        assert call(dtype=0) == EINVAL and b"dtype" in _err(lib)
    assert call(H=0) == EINVAL and call(n=-1) == EINVAL and call(E=-1) == EINVAL
    assert call(Dh=6) == EUNSUPPORTED and call(H=16, Dh=16) == EUNSUPPORTED
    assert call(slope=-1.0) == EUNSUPPORTED
    assert call(cols=None) == EINVAL and call(ds=None) == EINVAL
    assert call(f=P8) == ESHAPE and call(out=P8) == ESHAPE and call(attn=P8) == ESHAPE
    assert call(ldo=64) == ESHAPE and call(ld=64) == ESHAPE
    assert call(n=0) == 0
