"""Argument checks of RGCNConv's typed-aggregation entries (pglb_rgcn_agg_f32, pglb_rgcn_wgrad_ws,
pglb_rgcn_wgrad_f32): the symbols are exported and declared, and every call below is refused with PGLB_EINVAL (or has
nothing to do) before any CUDA call, so they are checked without a GPU."""
import ctypes
import os

import pytest

EINVAL = -1
NAMES = ["pglb_rgcn_agg_f32", "pglb_rgcn_wgrad_ws", "pglb_rgcn_wgrad_f32"]
P = ctypes.c_void_p(256)     # a non-NULL, 256-byte aligned dummy: must never be dereferenced here
P8 = ctypes.c_void_p(264)    # 8-byte but not 16-byte aligned


@pytest.fixture(scope="module")
def lib():
    from pgl_b200 import _lib
    return _lib.lib


def test_symbols_exported_and_declared(lib):
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "pglb.h")).read()
    for name in NAMES:
        assert hasattr(lib, name), name
        assert name + "(" in hdr, name


def agg(lib, indptr=P, cols=P, rel=P, slot_w=None, x=P, ldx=64, w=P, R=3, K=64, N=64, out=P, ldo=64, n=10):
    return lib.pglb_rgcn_agg_f32(indptr, cols, rel, slot_w, x, ldx, w, R, K, N, out, ldo, n, None)


def test_agg_argument_checks(lib):
    bad = [dict(n=-1), dict(R=0), dict(R=32768), dict(K=0), dict(K=6), dict(K=132), dict(N=2), dict(N=130),
           dict(ldx=60), dict(ldx=66), dict(ldo=60), dict(ldo=65), dict(indptr=None), dict(cols=None), dict(rel=None),
           dict(x=None), dict(w=None), dict(out=None), dict(x=P8), dict(out=ctypes.c_void_p(260)),
           dict(K=8, ldx=8, N=4, ldo=4, x=P8)]
    for kw in bad:
        assert agg(lib, **kw) == EINVAL, kw
        assert lib.pglb_last_error()
    # no rows: nothing to do, even with NULL pointers
    assert agg(lib, n=0, indptr=None, cols=None, rel=None, x=None, w=None, out=None) == 0


def test_wgrad_ws(lib):
    need = ctypes.c_size_t(0)
    assert lib.pglb_rgcn_wgrad_ws(10, 64, 32, ctypes.byref(need)) == 0 and need.value >= 10 * 64 * 32 * 4
    assert lib.pglb_rgcn_wgrad_ws(0, 64, 32, ctypes.byref(need)) == 0
    for args in ((-1, 64, 64), (1, 6, 64), (1, 64, 0), (1, 64, 256)):
        assert lib.pglb_rgcn_wgrad_ws(*args, ctypes.byref(need)) == EINVAL, args
    assert lib.pglb_rgcn_wgrad_ws(1, 64, 64, None) == EINVAL


def wgrad(lib, rows=P, beg=P, end=P, roff=P, ioff=P, R=3, items=4, chunk=64, cols=P, x=P, ldx=64, g=P, ldg=32,
          D=64, O=32, gw=P, ws=P, ws_bytes=1 << 20):
    return lib.pglb_rgcn_wgrad_f32(rows, beg, end, roff, ioff, R, items, chunk, cols, x, ldx, g, ldg, D, O, gw, ws,
                                   ws_bytes, None)


def test_wgrad_argument_checks(lib):
    bad = [dict(R=0), dict(R=40000), dict(items=-1), dict(chunk=0), dict(D=2), dict(D=130), dict(O=6), dict(O=132),
           dict(ldx=32), dict(ldx=66), dict(ldg=16), dict(ldg=34), dict(roff=None), dict(ioff=None), dict(gw=None),
           dict(rows=None), dict(beg=None), dict(end=None), dict(cols=None), dict(x=None), dict(g=None),
           dict(x=P8), dict(g=P8), dict(ws=None), dict(ws=P8), dict(ws_bytes=4 * 64 * 32 * 4 - 1)]
    for kw in bad:
        assert wgrad(lib, **kw) == EINVAL, kw
        assert lib.pglb_last_error()
