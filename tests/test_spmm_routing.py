"""Which index data ops._packed_of hands the aggregation for each dtype and row width, and the argument checks of the
two C aggregation entries.  Neither needs a GPU: _packed_of only reads shapes, and every call below fails a check (or
has no work) before any CUDA call."""
import ctypes

import pytest
import torch

from pgl_b200 import _lib, ops

DIMS = (4, 32, 60, 64, 68, 72, 96, 100, 128, 132, 200)


def _fake_csr(calls):
    def packed(n_src, row_bytes):
        calls.append(("packed", n_src, row_bytes))
        return ("ids", True)

    def plan(n_src, row_bytes):
        calls.append(("plan", n_src, row_bytes))
        return ("plan", "nz_row", "blk_k", True)

    return {"packed": packed, "plan": plan, "cols": torch.zeros(5, dtype=torch.int64), "slot_scale": "slot_scale"}


def _expected(dtype, D):
    """(kind, row bytes asked for) or None: packed ids for rows of 64 < D <= 128 that are a multiple of 16 bytes, the
    narrow plan for float32 rows of D <= 64 (D % 4 == 0), nothing otherwise."""
    row_bytes = D * (4 if dtype == torch.float32 else 2)
    if D > 128 or row_bytes % 16:
        return None
    if D <= 64:
        return ("plan", row_bytes) if dtype == torch.float32 else None
    return ("packed", row_bytes)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("D", DIMS)
def test_packed_of_by_dtype_and_width(dtype, D):
    calls = []
    x2 = torch.empty((10, D), dtype=dtype)
    got = ops._packed_of(_fake_csr(calls), x2)
    want = _expected(dtype, D)
    if want is None:
        assert got is None and calls == []
        return
    kind, row_bytes = want
    assert calls == [(kind, 10, row_bytes)]
    if kind == "plan":
        assert isinstance(got, ops.NarrowPlan)
        assert (got.plan, got.nz_row, got.blk_k, got.hints, got.slot_scale) == \
            ("plan", "nz_row", "blk_k", True, "slot_scale")
    else:
        assert isinstance(got, ops.PackedCols)
        assert tuple(got) == ("ids", True) and got.slot_scale == "slot_scale"


def test_packed_of_without_packed_ids():
    for dtype in (torch.float32, torch.bfloat16):
        assert ops._packed_of({"packed": None}, torch.empty((10, 128), dtype=dtype)) is None


ONE = ctypes.c_void_p(16)   # a non-NULL, 16-byte aligned dummy: never dereferenced, every call stops at a check
SUM, MEAN, MAX = _lib.REDUCE["sum"], _lib.REDUCE["mean"], _lib.REDUCE["max"]
COPY, MUL = _lib.MSG["copy"], _lib.MSG["mul"]
ACC = 1   # PGLB_SPMM_ACCUMULATE
BIG = 1 << 31


def _f32(indptr=ONE, x=ONE, ldx=128, y=None, y_bcast=_lib.BCAST_FULL, out=ONE, ldo=128, n_dst=10, n_src=10, E=20,
         D=128, head_dim=1, msg_op=COPY, reduce_op=SUM, scale_src=None, scale_slot=None, flags=0):
    return _lib.lib.pglb_spmm_csr_slot_scale_f32(indptr, ONE, None, x, ldx, y, 128, y_bcast, out, ldo, n_dst, n_src, E,
                                                 D, head_dim, msg_op, reduce_op, scale_src, scale_slot, None, None, -1,
                                                 flags, ONE, 1 << 20, None)


def _x16(indptr=ONE, x=ONE, ldx=128, out=ONE, ldo=128, n_dst=10, n_src=10, E=20, D=128, dtype=_lib.DTYPE_BF16,
         reduce_op=SUM, scale_src=None, scale_slot=None, flags=0):
    return _lib.lib.pglb_spmm_csr_x16(indptr, ONE, x, ldx, out, ldo, n_dst, n_src, E, D, dtype, reduce_op, scale_src,
                                      scale_slot, None, None, -1, flags, ONE, 1 << 20, None)


F32 = b"pglb_spmm_csr_f32: "
X16 = b"pglb_spmm_csr_x16: "

# (entry, arguments that differ from a valid call, return code, error text; None: no error expected)
CASES = [
    (_f32, dict(n_dst=-1), -1, F32 + b"negative size"),
    (_f32, dict(E=-1), -1, F32 + b"negative size"),
    (_f32, dict(reduce_op=7), -1, F32 + b"unknown reduce_op 7"),
    (_f32, dict(msg_op=9), -1, F32 + b"unknown msg_op 9"),
    (_f32, dict(msg_op=9, n_dst=0), -1, F32 + b"unknown msg_op 9"),
    (_f32, dict(scale_slot=ONE), -1, b"pglb_spmm_csr_slot_scale_f32: scale_slot needs scale_src"),
    (_f32, dict(n_dst=0), 0, None),
    (_f32, dict(D=0), 0, None),
    (_f32, dict(n_dst=0, indptr=None, out=None, x=None), 0, None),
    (_f32, dict(indptr=None), -1, F32 + b"indptr/out is NULL"),
    (_f32, dict(out=None), -1, F32 + b"indptr/out is NULL"),
    (_f32, dict(x=None), -1, F32 + b"x is NULL"),
    (_f32, dict(ldx=64), -2, F32 + b"leading dimension smaller than D"),
    (_f32, dict(ldo=64), -2, F32 + b"leading dimension smaller than D"),
    (_f32, dict(D=BIG, ldx=BIG, ldo=BIG), -2, F32 + b"D too large"),
    (_f32, dict(flags=ACC, reduce_op=MAX), -4, F32 + b"PGLB_SPMM_ACCUMULATE needs reduce_op SUM"),
    (_f32, dict(flags=ACC, reduce_op=MEAN), -4, F32 + b"PGLB_SPMM_ACCUMULATE needs reduce_op SUM"),
    (_f32, dict(flags=ACC, reduce_op=MAX, n_dst=0), 0, None),
    (_f32, dict(msg_op=MUL), -1, F32 + b"msg_op needs y"),
    (_f32, dict(msg_op=MUL, y=ONE, y_bcast=9), -1, F32 + b"unknown y_bcast 9"),
    (_f32, dict(msg_op=MUL, y=ONE, y_bcast=_lib.BCAST_HEAD, head_dim=3), -2, F32 + b"head_dim must divide D"),
    (_f32, dict(msg_op=MUL, y=ONE, y_bcast=_lib.BCAST_HEAD, head_dim=0), -2, F32 + b"head_dim must divide D"),
    (_x16, dict(dtype=3), -1, X16 + b"unknown dtype 3"),
    (_x16, dict(dtype=0), -1, X16 + b"unknown dtype 0"),
    (_x16, dict(n_dst=-1), -1, X16 + b"negative size"),
    (_x16, dict(D=-1), -1, X16 + b"negative size"),
    (_x16, dict(reduce_op=7), -1, X16 + b"unknown reduce_op 7"),
    (_x16, dict(scale_slot=ONE), -1, X16 + b"scale_slot needs scale_src"),
    (_x16, dict(flags=ACC), -4, X16 + b"PGLB_SPMM_ACCUMULATE would round the output twice"),
    (_x16, dict(flags=ACC, dtype=_lib.DTYPE_F16, n_dst=0), -4, X16 + b"PGLB_SPMM_ACCUMULATE would round the output twice"),
    (_x16, dict(n_dst=0), 0, None),
    (_x16, dict(D=0), 0, None),
    (_x16, dict(n_dst=0, indptr=None, out=None, x=None), 0, None),
    (_x16, dict(indptr=None), -1, X16 + b"indptr/out is NULL"),
    (_x16, dict(out=None), -1, X16 + b"indptr/out is NULL"),
    (_x16, dict(x=None), -1, X16 + b"x is NULL"),
    (_x16, dict(ldx=64), -2, X16 + b"leading dimension smaller than D"),
    (_x16, dict(ldo=64), -2, X16 + b"leading dimension smaller than D"),
    (_x16, dict(D=BIG, ldx=BIG, ldo=BIG), -2, X16 + b"D too large"),
]


@pytest.mark.parametrize("entry, kw, code, text", CASES,
                         ids=["%s-%s" % (c[0].__name__[1:], "-".join("%s=%s" % kv for kv in sorted(c[1].items())))
                              for c in CASES])
def test_single_failure_argument_checks(entry, kw, code, text):
    assert entry(**kw) == code
    if text is not None:
        assert _lib.lib.pglb_last_error() == text
