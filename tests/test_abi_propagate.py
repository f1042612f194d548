"""Argument checks of the propagation-step entries (pglb_propagate_f32, pglb_propagate_narrow_f32): the symbols are
exported and declared, and every call below is refused before any CUDA call, so they are checked without a GPU."""
import ctypes
import os

import pytest

EINVAL, ESHAPE, EUNSUPPORTED = -1, -2, -4
NAMES = ["pglb_propagate_f32", "pglb_propagate_narrow_f32"]


@pytest.fixture(scope="module")
def lib():
    from pgl_b200 import _lib
    return _lib


def _p(addr):
    return ctypes.c_void_p(addr)


N, E, D = 10, 20, 8
ROW = D * 4
X, OUT, H, ACC_IN, ACC_OUT = 1 << 20, 2 << 20, 3 << 20, 4 << 20, 5 << 20   # disjoint 256-byte aligned dummies


def _err(lib):
    return lib.lib.pglb_last_error()


def _call(lib, kind, x=X, out=OUT, h=H, ldh=D, acc_in=ACC_IN, ld_in=D, acc_out=ACC_OUT, ld_out=D, flags=0, n=N,
          D_=D, ldx=D, ldo=D):
    epi = [1.0, 0.0, _p(h) if h else None, ldh, _p(acc_in) if acc_in else None, ld_in,
           _p(acc_out) if acc_out else None, ld_out, 1.0, None]
    P = _p(256)
    if kind == "csr":
        return lib.lib.pglb_propagate_f32(P, P, _p(x), ldx, _p(out), ldo, n, n, E, D_, None, None, None, *epi, None,
                                          -1, flags, P, 1 << 20, None)
    return lib.lib.pglb_propagate_narrow_f32(P, P, P, P, _p(x), ldx, _p(out), ldo, n, n, E, D_, None, None, None,
                                             *epi, flags, P, 1 << 20, None)


def test_symbols_exported_and_declared(lib):
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "pglb.h")).read()
    for name in NAMES:
        assert hasattr(lib.lib, name), name
        assert name + "(" in hdr, name


@pytest.mark.parametrize("kind", ["csr", "narrow"])
def test_refusals(lib, kind):
    # acc_out without acc_in, and the reverse
    assert _call(lib, kind, acc_in=0) == EINVAL and b"acc_in and acc_out" in _err(lib)
    assert _call(lib, kind, acc_out=0) == EINVAL
    # out overlapping x, h, acc_in or acc_out
    for other in ("x", "h", "acc_in", "acc_out"):
        kw = {other: OUT + ROW}
        assert _call(lib, kind, **kw) == EINVAL, other
        assert b"out overlaps" in _err(lib)
    # acc_out overlapping acc_in other than exactly in place; acc_out overlapping x or h
    assert _call(lib, kind, acc_out=ACC_IN + ROW) == EINVAL and b"in place" in _err(lib)
    assert _call(lib, kind, acc_out=ACC_IN, ld_out=2 * D, ld_in=D) == EINVAL
    assert _call(lib, kind, acc_out=X) == EINVAL and b"acc_out overlaps x or h" in _err(lib)
    assert _call(lib, kind, acc_out=H) == EINVAL
    # leading dimensions of h / acc below D
    assert _call(lib, kind, ldh=D - 1) == ESHAPE
    assert _call(lib, kind, ld_in=D - 1, ld_out=D - 1, acc_out=ACC_IN) == ESHAPE
    assert _call(lib, kind, ld_out=D - 1) == ESHAPE
    # accumulate is not taken
    assert _call(lib, kind, flags=1) == EUNSUPPORTED
    # h / acc rows the vector kernels cannot read 16 bytes at a time
    assert _call(lib, kind, h=H + 4) == EUNSUPPORTED
    assert _call(lib, kind, acc_in=ACC_IN + 8, acc_out=ACC_IN + 8) == EUNSUPPORTED


def test_wide_rows_outside_the_v5_kernel_are_unsupported(lib):
    # 64 < D <= 128 with identity columns would take spmm_stream, which has no epilogue.  h == x and acc_out == acc_in
    # (in place) pass every argument check before that.
    D2 = 128
    P = _p(256)
    rc = lib.lib.pglb_propagate_f32(P, None, _p(X), D2, _p(OUT), D2, N, N, E, D2, None, None, None, 1.0, 0.5, _p(X),
                                    D2, _p(ACC_IN), D2, _p(ACC_IN), D2, 1.0, None, None, -1, 0, P, 1 << 20, None)
    assert rc == EUNSUPPORTED and b"spmm_stream" in _err(lib)
