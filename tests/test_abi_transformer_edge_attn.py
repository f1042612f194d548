"""Argument checks of the dot-product attention entries with edge features (pglb_dot_attn_e_csr_*,
pglb_dot_attn_e_drop_csr_*, pglb_dot_attn_e_bwd_edge_*, pglb_dot_attn_e_bwd_edge_drop_*): the symbols are exported,
and every call below is refused (or has nothing to do) before any CUDA call, so they are checked without a GPU."""
import ctypes

import pytest

EINVAL, ESHAPE, EUNSUPPORTED = -1, -2, -4

NAMES = ["pglb_dot_attn_e_csr_f32", "pglb_dot_attn_e_csr_x16", "pglb_dot_attn_e_drop_csr_f32",
         "pglb_dot_attn_e_drop_csr_x16", "pglb_dot_attn_e_bwd_edge_f32", "pglb_dot_attn_e_bwd_edge_x16",
         "pglb_dot_attn_e_bwd_edge_drop_f32", "pglb_dot_attn_e_bwd_edge_drop_x16"]
KINDS = ["f32", "x16", "drop_f32", "drop_x16"]


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


@pytest.mark.parametrize("kind", KINDS)
def test_forward_argument_checks(lib, kind):
    half = kind.endswith("x16")
    drop = kind.startswith("drop")
    el = 2 if half else 4

    def call(dtype=None, q=P, k=P, v=P, e=P, eid=P, ld=None, lde=None, ldo=None, out=P, n_dst=10, E=20, H=8, Dh=16,
             p=0.5, offset=0, lse=P, cols=P):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        ld = H * Dh if ld is None else ld
        lde = H * Dh if lde is None else lde
        ldo = H * Dh if ldo is None else ldo
        # (indptr, cols, eid, q, ldq, k, ldk, v, ldv, e, lde, out, ldo, lse, n_dst, n_src, E, H, head_dim, [dtype,]
        #  [attn_drop, seed, offset,] ws, ws_bytes, stream)
        args = [P, cols, eid, q, ld, k, ld, v, ld, e, lde, out, ldo, lse, n_dst, 10, E, H, Dh]
        if half:
            args.append(dtype)
        if drop:
            args += [p, 7, offset]
        fn = getattr(lib.lib, "pglb_dot_attn_e_%scsr_%s" % ("drop_" if drop else "", "x16" if half else "f32"))
        return fn(*args, P, 1 << 20, None)

    if half:
        assert call(dtype=0) == EINVAL and b"dtype" in _err(lib)
        assert call(dtype=3) == EINVAL
    assert call(H=0) == EINVAL and call(Dh=0) == EINVAL and call(n_dst=-1) == EINVAL and call(E=-1) == EINVAL
    assert call(Dh=6) == EUNSUPPORTED            # head_dim % 4
    assert call(H=4, Dh=12) == EUNSUPPORTED      # head_dim not a power of two
    assert call(H=16, Dh=16) == EUNSUPPORTED     # 256 elements per row
    assert call(H=4, Dh=7) == EUNSUPPORTED and b"head_dim" in _err(lib)
    if half:
        assert call(H=3, Dh=4) == EUNSUPPORTED   # 24-byte rows
    assert call(q=P8) == ESHAPE and call(k=P8) == ESHAPE and call(v=P8) == ESHAPE and call(out=P8) == ESHAPE
    assert call(e=P8) == ESHAPE                              # e rows not 16-byte aligned
    assert call(lde=8 * 16 + 16 // el + 2) == ESHAPE         # an e row stride that is not a multiple of 16 bytes
    assert call(lde=64) == ESHAPE                            # lde < D
    assert call(ld=8 * 16 + 16 // el + 2) == ESHAPE
    assert call(ldo=64) == ESHAPE and call(ld=64) == ESHAPE
    if drop:
        assert call(p=0.0) == EINVAL and call(p=1.0) == EINVAL and call(p=float("nan")) == EINVAL
        assert call(offset=2) == EINVAL and b"offset" in _err(lib)
        assert call(H=2, Dh=32) == EUNSUPPORTED and b"H % 4" in _err(lib)
        assert call(p=1.5, n_dst=0) == EINVAL            # the dropout arguments are checked first
    else:
        assert call(H=2, Dh=32, n_dst=0) == 0            # any head count without dropout
    assert call(n_dst=0) == 0                            # nothing to do: no device work
    assert call(n_dst=0, e=None, eid=None) == 0
    assert call(n_dst=5, E=5, cols=None, lse=None) == EINVAL      # NULL cols with edges
    assert call(n_dst=5, E=5, eid=None, lse=None) == EINVAL       # NULL eid with edges
    assert call(n_dst=5, E=5, e=None, lse=None) == EINVAL         # NULL e with edges


@pytest.mark.parametrize("kind", KINDS)
def test_bwd_edge_argument_checks(lib, kind):
    half = kind.endswith("x16")
    drop = kind.startswith("drop")

    def call(dtype=None, q=P, g=P, e=P, ge=P, ld=128, ldg=128, lde=128, ldge=128, E=20, H=8, Dh=16, lse=P, beta=P,
             p=0.5, offset=0):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        # (rows, cols, eid, q, ldq, k, ldk, v, ldv, e, lde, grad_out, ldg, out, ldo, lse, E, H, head_dim, [dtype,]
        #  [attn_drop, seed, offset,] beta_e, ds_e, grad_e, ldge, stream)
        args = [P, P, P, q, ld, P, ld, P, ld, e, lde, g, ldg, P, ld, lse, E, H, Dh]
        if half:
            args.append(dtype)
        if drop:
            args += [p, 7, offset]
        fn = getattr(lib.lib, "pglb_dot_attn_e_bwd_edge_%s%s" % ("drop_" if drop else "", "x16" if half else "f32"))
        return fn(*args, beta, P, ge, ldge, None)

    if half:
        assert call(dtype=0) == EINVAL and b"dtype" in _err(lib)
    assert call(H=0) == EINVAL and call(E=-1) == EINVAL
    assert call(Dh=6) == EUNSUPPORTED and call(H=4, Dh=12) == EUNSUPPORTED and call(H=16, Dh=16) == EUNSUPPORTED
    assert call(lse=None) == EINVAL and call(beta=None) == EINVAL
    assert call(e=None) == EINVAL                        # e is required
    assert call(q=P8) == ESHAPE and call(g=P8) == ESHAPE
    assert call(e=P8) == ESHAPE and call(ge=P8) == ESHAPE
    assert call(ldg=120) == ESHAPE and call(lde=120) == ESHAPE and call(ldge=120) == ESHAPE   # below D
    assert call(ld=130) == ESHAPE and call(lde=130) == ESHAPE and call(ldge=130) == ESHAPE   # not 16-byte strides
    assert call(E=0) == 0
    assert call(E=0, e=None) == 0
    if drop:
        assert call(p=0.0) == EINVAL and call(p=1.0) == EINVAL
        assert call(offset=6) == EINVAL
        assert call(H=2, Dh=32) == EUNSUPPORTED
    else:
        assert call(H=2, Dh=32, E=0) == 0
