"""Argument checks of pglb_spmm_csr_x16 (16-bit copy aggregation): they all run before any CUDA call, so they are
checked without a GPU."""
import ctypes


def test_argument_validation_of_the_16bit_entry():
    from pgl_b200 import _lib
    lib = _lib.lib
    one = ctypes.c_void_p(16)   # a non-NULL, 16-byte aligned dummy: must never be dereferenced here

    def call(ldx=128, dtype=_lib.DTYPE_BF16, scale_src=None, scale_slot=None, flags=0, n_dst=10):
        # (indptr, cols, x, ldx, out, ldo, n_dst, n_src, E, D, dtype, reduce_op, scale_src, scale_slot, scale_dst,
        #  cols_packed, max_degree_hint, flags, ws, ws_bytes, stream)
        return lib.pglb_spmm_csr_x16(one, one, one, ldx, one, 128, n_dst, 10, 20, 128, dtype, 0, scale_src, scale_slot,
                                     None, None, -1, flags, one, 1 << 20, None)

    assert call(dtype=3) == -1 and b"dtype" in lib.pglb_last_error()
    assert call(dtype=0) == -1
    assert call(scale_slot=one) == -1 and b"scale_slot needs scale_src" in lib.pglb_last_error()
    assert call(ldx=64) == -2 and b"leading dimension" in lib.pglb_last_error()
    assert call(dtype=_lib.DTYPE_F16, flags=1) == -4      # PGLB_SPMM_ACCUMULATE would round twice
    assert call(n_dst=0) == 0                              # nothing to do: no device work
    assert lib.pglb_spmm_csr_x16(one, one, one, 128, one, 128, 10, 10, 20, 128, 1, 7, None, None, None, None, -1, 0,
                                 one, 1 << 20, None) == -1  # unknown reduce_op
