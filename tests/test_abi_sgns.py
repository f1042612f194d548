"""Argument checks of the fused skip-gram loss entry (pglb_sgns_fwd_f32, pglb_sgns_fwd_ws): the symbols are exported
and declared, and every call below is refused before any CUDA call, so they are checked without a GPU."""
import ctypes
import os

import pytest

EINVAL, ESHAPE, EWORKSPACE = -1, -2, -3
NAMES = ["pglb_sgns_fwd_ws", "pglb_sgns_fwd_f32"]


@pytest.fixture(scope="module")
def lib():
    from pgl_b200 import _lib
    return _lib


def _p(addr):
    return ctypes.c_void_p(addr) if addr else None


N, P, K, D = 100, 10, 3, 8
# disjoint 256-byte aligned dummies, each far larger than what it stands for
EMB, CTX, SRC, DSTS, LOSS, C, W, WS = [(i + 1) << 20 for i in range(8)]
WS_BYTES = 4096 * 8


def _call(lib, emb=EMB, n_emb=N, ld_emb=D, ctx=CTX, n_ctx=N, ld_ctx=D, src=SRC, dsts=DSTS, P_=P, K_=K, D_=D,
          loss=LOSS, c=C, w=W, ldw=D, ws=WS, ws_bytes=WS_BYTES):
    return lib.lib.pglb_sgns_fwd_f32(_p(emb), n_emb, ld_emb, _p(ctx), n_ctx, ld_ctx, _p(src), _p(dsts), P_, K_, D_,
                                     _p(loss), _p(c), _p(w), ldw, _p(ws), ws_bytes, None)


def _err(lib):
    return lib.lib.pglb_last_error()


def test_symbols_exported_and_declared(lib):
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "pglb.h")).read()
    for name in NAMES:
        assert hasattr(lib.lib, name), name
        assert name + "(" in hdr, name


def test_workspace_query(lib):
    need = ctypes.c_size_t(0)
    assert lib.lib.pglb_sgns_fwd_ws(P, ctypes.byref(need)) == 0 and 0 < need.value <= WS_BYTES
    assert lib.lib.pglb_sgns_fwd_ws(0, ctypes.byref(need)) == EINVAL
    assert lib.lib.pglb_sgns_fwd_ws(P, None) == EINVAL


def test_refusals(lib):
    # NULL tables, ids, loss
    for kw in ("emb", "ctx", "src", "dsts", "loss"):
        assert _call(lib, **{kw: 0}) == EINVAL and b"NULL" in _err(lib), kw
    # sizes below 1
    for kw in ("P_", "K_", "D_", "n_emb", "n_ctx"):
        assert _call(lib, **{kw: 0}) == EINVAL, kw
    assert _call(lib, K_=-1) == EINVAL
    # leading dimensions below D
    assert _call(lib, ld_emb=D - 1) == ESHAPE
    assert _call(lib, ld_ctx=D - 1) == ESHAPE
    assert _call(lib, ldw=D - 1) == ESHAPE
    # c and w together or not at all
    assert _call(lib, c=0) == EINVAL and b"together" in _err(lib)
    assert _call(lib, w=0) == EINVAL
    # outputs overlapping an input, or each other
    for out in ("loss", "c", "w"):
        for target in (EMB, CTX, SRC, DSTS):
            assert _call(lib, **{out: target + 64}) == EINVAL and b"overlaps an input" in _err(lib), (out, target)
    assert _call(lib, c=W + 16) == EINVAL and b"outputs overlap" in _err(lib)
    assert _call(lib, loss=C + 4) == EINVAL
    # the last row of a table reaches the next buffer: ((n - 1) ld + D) floats
    assert _call(lib, loss=EMB + ((N - 1) * D + D - 1) * 4) == EINVAL
    # workspace too small, NULL or misaligned
    assert _call(lib, ws_bytes=WS_BYTES - 1) == EWORKSPACE
    assert _call(lib, ws=0) == EWORKSPACE
    assert _call(lib, ws=WS + 4) == EWORKSPACE


def test_loss_only_takes_no_c_or_w(lib):
    # c = w = NULL is the loss-only form: ldw is not checked then.  A shared table (ctx == emb) is not an overlap.
    # With a too-small workspace these are refused at the last check, after every other argument passed.
    assert _call(lib, c=0, w=0, ldw=0, ws_bytes=1) == EWORKSPACE
    assert _call(lib, ctx=EMB, ws_bytes=1) == EWORKSPACE
