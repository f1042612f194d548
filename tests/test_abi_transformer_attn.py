"""Argument checks of the dot-product attention entries (pglb_dot_attn_csr_*, pglb_dot_attn_drop_csr_*,
pglb_dot_attn_bwd_edge_*, pglb_dot_attn_bwd_edge_drop_*): the new symbols are exported, and every call below is
refused (or has nothing to do) before any CUDA call, so they are checked without a GPU."""
import ctypes

import pytest

EINVAL, ESHAPE, EUNSUPPORTED = -1, -2, -4

NAMES = ["pglb_dot_attn_csr_f32", "pglb_dot_attn_csr_x16", "pglb_dot_attn_drop_csr_f32", "pglb_dot_attn_drop_csr_x16",
         "pglb_dot_attn_bwd_edge_f32", "pglb_dot_attn_bwd_edge_x16", "pglb_dot_attn_bwd_edge_drop_f32",
         "pglb_dot_attn_bwd_edge_drop_x16"]


@pytest.fixture(scope="module")
def lib():
    from pgl_b200 import _lib
    return _lib


P = ctypes.c_void_p(256)     # a non-NULL, 256-byte aligned dummy: must never be dereferenced here
P8 = ctypes.c_void_p(264)    # 8-byte but not 16-byte aligned


def _err(lib):
    return lib.lib.pglb_last_error()


def test_symbols_exported(lib):
    for name in NAMES:
        assert hasattr(lib.lib, name), name


@pytest.mark.parametrize("kind", ["f32", "x16", "drop_f32", "drop_x16"])
def test_dot_attn_forward_argument_checks(lib, kind):
    half = kind.endswith("x16")
    drop = kind.startswith("drop")
    el = 2 if half else 4

    def call(dtype=None, q=P, k=P, v=P, ld=None, ldo=None, out=P, n_dst=10, E=20, H=8, Dh=16, p=0.5, offset=0,
             lse=P, cols=P):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        ld = H * Dh if ld is None else ld
        ldo = H * Dh if ldo is None else ldo
        # (indptr, cols, q, ldq, k, ldk, v, ldv, out, ldo, lse, n_dst, n_src, E, H, head_dim, [dtype,]
        #  [attn_drop, seed, offset,] ws, ws_bytes, stream)
        args = [P, cols, q, ld, k, ld, v, ld, out, ldo, lse, n_dst, 10, E, H, Dh]
        if half:
            args.append(dtype)
        if drop:
            args += [p, 7, offset]
        fn = getattr(lib.lib, "pglb_dot_attn_%scsr_%s" % ("drop_" if drop else "", "x16" if half else "f32"))
        return fn(*args, P, 1 << 20, None)

    if half:
        assert call(dtype=0) == EINVAL and b"dtype" in _err(lib)
        assert call(dtype=3) == EINVAL
    assert call(H=0) == EINVAL and call(Dh=0) == EINVAL and call(n_dst=-1) == EINVAL and call(E=-1) == EINVAL
    assert call(Dh=6) == EUNSUPPORTED            # head_dim % 4
    assert call(H=4, Dh=12) == EUNSUPPORTED      # head_dim not a power of two: the head sum is a xor butterfly
    assert call(H=16, Dh=16) == EUNSUPPORTED     # 256 elements per row
    assert call(H=4, Dh=7) == EUNSUPPORTED and b"head_dim" in _err(lib)   # the citation model's concat=False layer
    if half:
        assert call(H=3, Dh=4) == EUNSUPPORTED   # 24-byte rows: not a multiple of 16 bytes
    assert call(q=P8) == ESHAPE and call(k=P8) == ESHAPE and call(v=P8) == ESHAPE and call(out=P8) == ESHAPE
    assert call(ld=8 * 16 + 16 // el + 2) == ESHAPE      # a row stride that is not a multiple of 16 bytes
    assert call(ldo=64) == ESHAPE                        # ldo < D
    assert call(ld=64) == ESHAPE                         # ldq / ldk / ldv < D
    if drop:
        assert call(p=0.0) == EINVAL and call(p=1.0) == EINVAL and call(p=float("nan")) == EINVAL
        assert call(offset=2) == EINVAL and b"offset" in _err(lib)
        assert call(H=2, Dh=32) == EUNSUPPORTED and b"H % 4" in _err(lib)
        assert call(p=1.5, n_dst=0) == EINVAL            # the dropout arguments are checked first
    else:
        assert call(H=2, Dh=32, n_dst=0) == 0            # any head count without dropout
    assert call(n_dst=0) == 0                            # nothing to do: no device work
    assert call(n_dst=5, E=5, cols=None, lse=None) == EINVAL      # NULL cols with edges


@pytest.mark.parametrize("kind", ["f32", "x16", "drop_f32", "drop_x16"])
def test_dot_attn_bwd_edge_argument_checks(lib, kind):
    half = kind.endswith("x16")
    drop = kind.startswith("drop")

    def call(dtype=None, q=P, g=P, ld=128, ldg=128, E=20, H=8, Dh=16, lse=P, beta=P, p=0.5, offset=0):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        # (rows, cols, eid, q, ldq, k, ldk, v, ldv, grad_out, ldg, out, ldo, lse, E, H, head_dim, [dtype,]
        #  [attn_drop, seed, offset,] beta_e, ds_e, stream)
        args = [P, P, P, q, ld, P, ld, P, ld, g, ldg, P, ld, lse, E, H, Dh]
        if half:
            args.append(dtype)
        if drop:
            args += [p, 7, offset]
        fn = getattr(lib.lib, "pglb_dot_attn_bwd_edge_%s%s" % ("drop_" if drop else "", "x16" if half else "f32"))
        return fn(*args, beta, P, None)

    if half:
        assert call(dtype=0) == EINVAL and b"dtype" in _err(lib)
    assert call(H=0) == EINVAL and call(E=-1) == EINVAL
    assert call(Dh=6) == EUNSUPPORTED and call(H=4, Dh=12) == EUNSUPPORTED and call(H=16, Dh=16) == EUNSUPPORTED
    assert call(lse=None) == EINVAL and call(beta=None) == EINVAL
    assert call(q=P8) == ESHAPE and call(g=P8) == ESHAPE
    assert call(ldg=120) == ESHAPE                       # ldg < D
    assert call(ld=130) == ESHAPE                        # not a multiple of 16 bytes
    assert call(E=0) == 0
    if drop:
        assert call(p=0.0) == EINVAL and call(p=1.0) == EINVAL
        assert call(offset=6) == EINVAL
        assert call(H=2, Dh=32) == EUNSUPPORTED
    else:
        assert call(H=2, Dh=32, E=0) == 0
