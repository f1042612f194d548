"""Argument checks of the FAConv aggregation entries (pglb_fa_attn_csr_*, pglb_fa_attn_drop_csr_*, pglb_fa_bwd_edge_*,
pglb_fa_bwd_edge_drop_*): the new symbols are exported, and every call below is refused (or has nothing to do) before
any CUDA call, so they are checked without a GPU."""
import ctypes
import os

import pytest

EINVAL, ESHAPE, EUNSUPPORTED = -1, -2, -4

NAMES = ["pglb_fa_attn_csr_f32", "pglb_fa_attn_csr_x16", "pglb_fa_attn_drop_csr_f32", "pglb_fa_attn_drop_csr_x16",
         "pglb_fa_bwd_edge_f32", "pglb_fa_bwd_edge_x16", "pglb_fa_bwd_edge_drop_f32", "pglb_fa_bwd_edge_drop_x16"]
KINDS = ["f32", "x16", "drop_f32", "drop_x16"]


@pytest.fixture(scope="module")
def lib():
    from pgl_b200 import _lib
    return _lib


P = ctypes.c_void_p(256)     # a non-NULL, 256-byte aligned dummy: must never be dereferenced here
P8 = ctypes.c_void_p(264)    # 8-byte but not 16-byte aligned


def _err(lib):
    return lib.lib.pglb_last_error()


def test_symbols_exported_and_declared(lib):
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "pglb.h")).read()
    for name in NAMES:
        assert hasattr(lib.lib, name), name
        assert name + "(" in hdr, name


@pytest.mark.parametrize("kind", KINDS)
def test_fa_forward_argument_checks(lib, kind):
    half = kind.endswith("x16")
    drop = kind.startswith("drop")
    el = 2 if half else 4

    def call(dtype=None, f=P, rec=P, ld=None, ldo=None, out=P, n=10, E=20, D=64, p=0.5, offset=0, cols=P,
             indptr=P):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        ld = D if ld is None else ld
        ldo = D if ldo is None else ldo
        # (indptr, cols, f, ldf, rec, out, ldo, n, E, D, [dtype,] [attn_drop, seed, offset,] ws, ws_bytes, stream)
        args = [indptr, cols, f, ld, rec, out, ldo, n, E, D]
        if half:
            args.append(dtype)
        if drop:
            args += [p, 7, offset]
        fn = getattr(lib.lib, "pglb_fa_attn_%scsr_%s" % ("drop_" if drop else "", "x16" if half else "f32"))
        return fn(*args, P, 1 << 20, None)

    if half:
        assert call(dtype=0) == EINVAL and b"dtype" in _err(lib)
        assert call(dtype=3) == EINVAL
    assert call(D=0) == EINVAL and call(n=-1) == EINVAL and call(E=-1) == EINVAL
    assert call(D=132) == EUNSUPPORTED and b"D <= 128" in _err(lib)
    assert call(D=256) == EUNSUPPORTED
    assert call(D=6) == EUNSUPPORTED            # rows not a multiple of 16 bytes
    if half:
        assert call(D=12) == EUNSUPPORTED       # 24-byte 16-bit rows
    else:
        assert call(D=12, n=0) == 0             # 48-byte float32 rows: D need not be a power of two
    assert call(indptr=None) == EINVAL and call(out=None) == EINVAL
    assert call(cols=None) == EINVAL and call(f=None) == EINVAL and call(rec=None) == EINVAL
    assert call(f=P8) == ESHAPE and call(rec=P8) == ESHAPE and call(out=P8) == ESHAPE
    assert call(ld=64 + 16 // el + 2) == ESHAPE         # a row stride that is not a multiple of 16 bytes
    assert call(ldo=32) == ESHAPE and call(ld=32) == ESHAPE   # strides below D
    if drop:
        assert call(p=0.0) == EINVAL and call(p=1.0) == EINVAL and call(p=-0.1) == EINVAL
        assert call(p=float("nan")) == EINVAL and b"attn_drop" in _err(lib)
        assert call(offset=2) == EINVAL and b"offset" in _err(lib)
        assert call(p=1.5, n=0) == EINVAL               # the dropout arguments are checked first
        assert call(p=1e-12, n=0) == 0
    assert call(n=0) == 0                               # nothing to do: no device work


@pytest.mark.parametrize("kind", KINDS)
def test_fa_bwd_edge_argument_checks(lib, kind):
    half = kind.endswith("x16")
    drop = kind.startswith("drop")

    def call(dtype=None, rows=P, cols=P, f=P, g=P, rec=P, ld=64, ldg=64, E=20, D=64, beta=P, dz=P, p=0.5, offset=0):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        # (rows, cols, eid, f, ldf, rec, grad_out, ldg, E, D, [dtype,] [attn_drop, seed, offset,] beta_e, dz_e,
        #  stream)
        args = [rows, cols, P, f, ld, rec, g, ldg, E, D]
        if half:
            args.append(dtype)
        if drop:
            args += [p, 7, offset]
        fn = getattr(lib.lib, "pglb_fa_bwd_edge_%s%s" % ("drop_" if drop else "", "x16" if half else "f32"))
        return fn(*args, beta, dz, None)

    if half:
        assert call(dtype=0) == EINVAL and b"dtype" in _err(lib)
    assert call(D=0) == EINVAL and call(E=-1) == EINVAL
    assert call(D=136) == EUNSUPPORTED and call(D=6) == EUNSUPPORTED
    if half:
        assert call(D=4) == EUNSUPPORTED        # 8-byte 16-bit rows
    assert call(rows=None) == EINVAL and call(cols=None) == EINVAL and call(rec=None) == EINVAL
    assert call(f=None) == EINVAL and call(g=None) == EINVAL and call(beta=None) == EINVAL and call(dz=None) == EINVAL
    assert call(f=P8) == ESHAPE and call(g=P8) == ESHAPE and call(rec=P8) == ESHAPE
    assert call(ldg=60) == ESHAPE and call(ld=66) == ESHAPE
    assert call(E=0) == 0
    if drop:
        assert call(p=0.0) == EINVAL and call(p=1.0) == EINVAL and call(p=2.0, E=0) == EINVAL
        assert call(offset=6) == EINVAL
