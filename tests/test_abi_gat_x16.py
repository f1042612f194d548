"""Argument checks of the 16-bit GAT entries (pglb_gat_fused_csr_x16, pglb_gat_fused_train_csr_x16,
pglb_gat_bwd_edge_x16, pglb_spmm_csr_ue_x16, pglb_head_dots_x16): every call below is refused (or has nothing to do)
before any CUDA call, so they are checked without a GPU."""
import ctypes

import pytest

EINVAL, ESHAPE, EUNSUPPORTED = -1, -2, -4


@pytest.fixture(scope="module")
def lib():
    from pgl_b200 import _lib
    return _lib


P = ctypes.c_void_p(256)     # a non-NULL, 256-byte aligned dummy: must never be dereferenced here
P8 = ctypes.c_void_p(264)    # 8-byte but not 16-byte aligned


def _err(lib):
    return lib.lib.pglb_last_error()


@pytest.mark.parametrize("train", [False, True])
def test_gat_fused_x16_argument_checks(lib, train):
    def call(dtype=None, f=P, ldf=128, out=P, ldo=128, n_dst=10, E=20, H=8, Dh=16, slope=0.2, attn=P, lse=P):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        # (indptr, cols, f, ldf, attn_src, attn_dst, slope, out, ldo, [lse,] n_dst, n_src, E, H, head_dim, dtype, ws,
        #  ws_bytes, stream)
        if train:
            return lib.lib.pglb_gat_fused_train_csr_x16(P, P, f, ldf, attn, P, slope, out, ldo, lse, n_dst, 10, E, H,
                                                        Dh, dtype, P, 1 << 20, None)
        return lib.lib.pglb_gat_fused_csr_x16(P, P, f, ldf, attn, P, slope, out, ldo, n_dst, 10, E, H, Dh, dtype, P,
                                              1 << 20, None)

    assert call(dtype=0) == EINVAL and b"dtype" in _err(lib)
    assert call(dtype=3) == EINVAL
    assert call(ldf=132) == ESHAPE          # 264-byte rows: not a multiple of 16 bytes
    assert call(dtype=lib.DTYPE_F16, ldo=124) == ESHAPE    # ldo < D
    assert call(f=P8) == ESHAPE
    assert call(out=P8) == ESHAPE
    assert call(H=3, Dh=32) == EUNSUPPORTED and b"16-bit kernel" in _err(lib)   # H % 4: no 16-bit fallback kernel
    assert call(H=36, Dh=4) == EUNSUPPORTED     # D = 144 > 128 (with head_dim % 4 == 0 this also bounds H by 32)
    assert call(slope=1.5) == EUNSUPPORTED and call(slope=-0.1) == EUNSUPPORTED
    assert call(attn=P8) == EUNSUPPORTED        # attention rows are bulk-copied: 16-byte aligned
    assert call(Dh=6) == EUNSUPPORTED           # head_dim % 4
    assert call(H=16, Dh=16) == EUNSUPPORTED    # 256 elements per row
    assert call(n_dst=0) == 0                   # nothing to do: no device work
    assert call(n_dst=0, dtype=lib.DTYPE_F16, E=0) == 0
    if train:
        assert call(lse=None) == EINVAL and b"lse" in _err(lib)
        assert call(lse=None, n_dst=0) == 0


def test_gat_bwd_edge_x16_argument_checks(lib):
    def call(dtype=None, ldf=128, ldg=128, ldo=128, f=P, E=20, H=8, Dh=16, lse=P):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        # (rows, cols, eid, f, ldf, grad_out, ldg, out, ldo, attn_src, attn_dst, lse, slope, E, H, head_dim, dtype,
        #  alpha_e, dz_e, stream)
        return lib.lib.pglb_gat_bwd_edge_x16(P, P, None, f, ldf, P, ldg, P, ldo, P, P, lse, 0.2, E, H, Dh, dtype, P, P,
                                             None)

    assert call(dtype=7) == EINVAL and b"dtype" in _err(lib)
    assert call(ldf=132) == ESHAPE
    assert call(ldg=140) == ESHAPE and call(dtype=lib.DTYPE_F16, ldo=120) == ESHAPE
    assert call(f=P8) == ESHAPE
    assert call(Dh=12) == EUNSUPPORTED and call(H=16, Dh=16) == EUNSUPPORTED
    assert call(lse=None) == EINVAL
    assert call(E=0) == 0


def test_spmm_csr_ue_x16_argument_checks(lib):
    from pgl_b200._lib import BCAST_FULL, BCAST_HEAD, BCAST_SCALAR, MSG, REDUCE

    def call(dtype=None, x=P, ldx=128, ldo=128, n_dst=10, D=128, hd=16, bcast=BCAST_HEAD, msg="mul", red="sum",
             flags=0, y=P):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        # (indptr, cols, eid, x, ldx, y, ldy, y_bcast, out, ldo, n_dst, n_src, E, D, head_dim, dtype, msg_op,
        #  reduce_op, scale_src, scale_dst, max_degree_hint, flags, ws, ws_bytes, stream)
        return lib.lib.pglb_spmm_csr_ue_x16(P, P, None, x, ldx, y, 8, bcast, P, ldo, n_dst, 10, 20, D, hd, dtype,
                                            MSG[msg], REDUCE[red], None, None, -1, flags, P, 1 << 20, None)

    assert call(dtype=0) == EINVAL and b"dtype" in _err(lib)
    assert call(msg="copy") == EUNSUPPORTED and call(msg="sub") == EUNSUPPORTED and call(msg="div") == EUNSUPPORTED
    assert call(red="max") == EUNSUPPORTED and call(red="mean") == EUNSUPPORTED
    assert call(bcast=BCAST_FULL) == EUNSUPPORTED
    assert call(flags=1) == EUNSUPPORTED        # PGLB_SPMM_ACCUMULATE would round twice
    assert call(D=6, ldx=8, ldo=8, bcast=BCAST_SCALAR) == EUNSUPPORTED   # D % 4
    assert call(ldx=130) == ESHAPE and call(ldo=126) == ESHAPE
    assert call(x=ctypes.c_void_p(260)) == ESHAPE
    assert call(hd=48) == ESHAPE                # head_dim must divide D
    assert call(y=None) == EINVAL
    assert call(bcast=5) == EINVAL and call(red="sum", msg="copy", bcast=3) == EINVAL
    assert lib.lib.pglb_spmm_csr_ue_x16(P, P, None, P, 128, P, 8, BCAST_HEAD, P, 128, 10, 10, 20, 128, 16,
                                        lib.DTYPE_BF16, MSG["mul"], 7, None, None, -1, 0, P, 1 << 20,
                                        None) == EINVAL   # unknown reduce_op
    assert call(n_dst=0) == 0


def test_head_dots_x16_argument_checks(lib):
    def call(dtype=None, f=P, ldf=128, n=10, H=8, Dh=16, w=P):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        # (f, ldf, n, H, head_dim, dtype, w_src, w_dst, attn_src, attn_dst, stream)
        return lib.lib.pglb_head_dots_x16(f, ldf, n, H, Dh, dtype, w, P, P, P, None)

    assert call(dtype=-1) == EINVAL and b"dtype" in _err(lib)
    assert call(ldf=132) == ESHAPE and call(f=P8) == ESHAPE and call(w=P8) == ESHAPE
    assert call(Dh=12) == EUNSUPPORTED and call(H=16, Dh=16) == EUNSUPPORTED
    assert call(w=None) == EINVAL
    assert call(n=0) == 0
