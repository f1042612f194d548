"""Argument checks of the relation-typed sampling entries (pglb_sample_typed_count, pglb_sample_typed_fill): the
symbols are exported and declared, and every call below is refused before any CUDA call (the fan-outs are a host
array, checked before they are copied to the device), so they are checked without a GPU."""
import ctypes
import os

import pytest

EINVAL, ESHAPE = -1, -2
NAMES = ["pglb_sample_typed_count", "pglb_sample_typed_fill"]
P = ctypes.c_void_p(256)     # a non-NULL dummy device pointer: must never be dereferenced here


@pytest.fixture(scope="module")
def lib():
    from pgl_b200 import _lib
    return _lib.lib


def sizes(*k):
    return ctypes.cast((ctypes.c_int64 * len(k))(*k), ctypes.c_void_p)


def test_symbols_exported_and_declared(lib):
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "pglb.h")).read()
    for name in NAMES:
        assert hasattr(lib, name), name
        assert name + "(" in hdr, name


def count(lib, indptr=P, rel=P, R=3, ss=None, sd=P, nodes=P, n=10, cnt=P, off=P):
    ss = sizes(5, 5, 5) if ss is None else ss
    return lib.pglb_sample_typed_count(indptr, rel, R, ss, sd, nodes, n, cnt, off, None)


def fill(lib, indptr=P, cols=P, rel=P, eid=None, R=3, ss=None, sd=P, nodes=P, n=10, off=P, nb=P, orel=P, oeid=None):
    ss = sizes(5, 5, 5) if ss is None else ss
    return lib.pglb_sample_typed_fill(indptr, cols, rel, eid, R, ss, sd, nodes, n, 7, off, nb, orel, oeid, None)


BAD = [dict(n=-1), dict(R=0), dict(R=-2), dict(R=32768), dict(ss=ctypes.c_void_p()), dict(sd=None),
       dict(ss=sizes(5, 4097, 5)), dict(ss=sizes(1 << 40, 0, 0)), dict(indptr=None), dict(rel=None), dict(nodes=None)]


def test_count_argument_checks(lib):
    for kw in BAD + [dict(cnt=None), dict(off=None)]:
        rc = count(lib, **kw)
        assert rc in (EINVAL, ESHAPE), kw
        assert lib.pglb_last_error()
    assert count(lib, ss=sizes(5, 4097, 5)) == ESHAPE


def test_fill_argument_checks(lib):
    for kw in BAD + [dict(cols=None), dict(off=None), dict(nb=None), dict(orel=None)]:
        rc = fill(lib, **kw)
        assert rc in (EINVAL, ESHAPE), kw
        assert lib.pglb_last_error()
    assert fill(lib, ss=sizes(4097, 0, 0)) == ESHAPE
