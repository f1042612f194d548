"""ctypes binding of libpglb.so (include/pglb.h).  The product path has no fallback: if the
shared library is missing this module raises at import time."""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_int, c_int64, c_size_t, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PGLB_LIB") or os.path.join(_HERE, "libpglb.so")
METIS_PATH = os.path.join(_HERE, "third_party", "libmetis_i64.so")

PGLB_OK = 0
PGLB_CUDA_ERR_BASE = 1000
REDUCE = {"sum": 0, "mean": 1, "max": 2, "min": 3}
MSG = {"copy": 0, "add": 1, "sub": 2, "mul": 3, "div": 4}
BCAST_FULL, BCAST_HEAD, BCAST_SCALAR = 0, 1, 2
DTYPE_BF16, DTYPE_F16 = 1, 2   # dtype of the *_x16 entries


class PglbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libpglb error %d: %s" % (code, msg))
        self.code = code


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "pgl_b200: %s not found. Build it first with `python pgl_b200/build.py` "
            "(or __graft_entry__.build()); there is no CPU / eager fallback." % LIB_PATH)
    return ctypes.CDLL(LIB_PATH)


lib = _load()

_p = c_void_p
_i64 = c_int64
_u64 = ctypes.c_uint64

_SIGS = {
    "pglb_version": (c_int, []),
    "pglb_last_error": (c_char_p, []),
    "pglb_launch_count": (c_int64, []),
    "pglb_csr_build_ws": (c_int, [_i64, _i64, POINTER(c_size_t)]),
    "pglb_csr_build": (c_int, [_p, _i64, _p, _i64, _i64, _i64, _p, _p, _p, _p, _p, _p, c_size_t, _p]),
    "pglb_build_index_host": (c_int, [_p, _i64, _p, _i64, _i64, _i64, _p, _p, _p, _p, _p]),
    "pglb_segment_ids_ws": (c_int, [_i64, POINTER(c_size_t)]),
    "pglb_segment_ids": (c_int, [_p, _i64, _i64, _p, _p, _p, _p, c_size_t, _p]),
    "pglb_segment_indptr": (c_int, [_p, _i64, _i64, _p, _p]),
    "pglb_spmm_csr_ws": (c_int, [_i64, _i64, _i64, POINTER(c_size_t)]),
    "pglb_spmm_csr_f32": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, c_int, _p, _i64, _i64, _i64, _i64,
                                  _i64, _i64, c_int, c_int, _p, _p, _p, _i64, c_int, _p, c_size_t, _p]),
    "pglb_spmm_csr_slot_scale_f32": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, c_int, _p, _i64, _i64, _i64, _i64,
                                             _i64, _i64, c_int, c_int, _p, _p, _p, _p, _i64, c_int, _p, c_size_t,
                                             _p]),
    "pglb_spmm_csr_x16": (c_int, [_p, _p, _p, _i64, _p, _i64, _i64, _i64, _i64, _i64, c_int, c_int, _p, _p, _p, _p,
                                  _i64, c_int, _p, c_size_t, _p]),
    "pglb_spmm_csr_ue_x16": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, c_int, _p, _i64, _i64, _i64, _i64, _i64, _i64,
                                     c_int, c_int, c_int, _p, _p, _i64, c_int, _p, c_size_t, _p]),
    "pglb_narrow_plan_ws": (c_int, [_i64, POINTER(c_size_t)]),
    "pglb_narrow_plan": (c_int, [_p, _p, _p, _i64, _i64, _i64, _p, _p, _p, _p, c_size_t, _p]),
    "pglb_spmm_narrow_ws": (c_int, [_i64, _i64, POINTER(c_size_t)]),
    "pglb_spmm_narrow_f32": (c_int, [_p, _p, _p, _p, _p, _i64, _p, _i64, _i64, _i64, _i64, _i64, c_int, _p, _p, _p,
                                     c_int, _p, c_size_t, _p]),
    "pglb_propagate_f32": (c_int, [_p, _p, _p, _i64, _p, _i64, _i64, _i64, _i64, _i64, _p, _p, _p, ctypes.c_float,
                                   ctypes.c_float, _p, _i64, _p, _i64, _p, _i64, ctypes.c_float, _p, _p, _i64, c_int,
                                   _p, c_size_t, _p]),
    "pglb_propagate_narrow_f32": (c_int, [_p, _p, _p, _p, _p, _i64, _p, _i64, _i64, _i64, _i64, _i64, _p, _p, _p,
                                          ctypes.c_float, ctypes.c_float, _p, _i64, _p, _i64, _p, _i64,
                                          ctypes.c_float, _p, c_int, _p, c_size_t, _p]),
    "pglb_memcpy2d_async": (c_int,[_p, c_size_t, _p, c_size_t, c_size_t, c_size_t, c_int, _p]),
    "pglb_ipc_alloc": (c_int, [c_size_t, POINTER(c_void_p), _p]),
    "pglb_ipc_free": (c_int, [_p]),
    "pglb_ipc_open": (c_int, [_p, POINTER(c_void_p)]),
    "pglb_ipc_close": (c_int, [_p]),
    "pglb_pack_cols": (c_int, [_p, _i64, _i64, _p, _i64, _p, _p]),
    "pglb_send_uv_f32": (c_int, [_p, _p, _p, _i64, _p, _i64, _i64, _i64, c_int, _p, _p]),
    "pglb_gather_rows_f32": (c_int, [_p, _i64, _p, _i64, _i64, _i64, _p, _i64, _p]),
    "pglb_scatter_rows_f32": (c_int, [_p, _i64, _p, _i64, _i64, _p, _i64, _p]),
    "pglb_edge_softmax_csr_ws": (c_int, [_i64, POINTER(c_size_t)]),
    "pglb_edge_softmax_csr_f32": (c_int, [_p, _p, _p, _p, _i64, _i64, _i64, _p, c_size_t, _p]),
    "pglb_degree_norm_f32": (c_int, [_p, _i64, _p, _p]),
    "pglb_sample_count": (c_int, [_p, _p, _i64, _i64, _p, _p, _p]),
    "pglb_sample_fill": (c_int, [_p, _p, _p, _p, _i64, _i64, ctypes.c_uint64, _p, _p, _p, _p]),
    "pglb_sample_typed_count": (c_int, [_p, _p, _i64, _p, _p, _p, _i64, _p, _p, _p]),
    "pglb_sample_typed_fill": (c_int, [_p, _p, _p, _p, _i64, _p, _p, _p, _i64, ctypes.c_uint64, _p, _p, _p, _p, _p]),
    "pglb_reindex_table_init": (c_int, [_p, _i64, _p]),
    "pglb_reindex_graph_ws": (c_int, [_i64, POINTER(c_size_t)]),
    "pglb_reindex_graph": (c_int, [_p, _i64, _p, _p, _i64, _p, _p, _p, _p, _p, _p, c_size_t, _p]),
    "pglb_random_walk": (c_int, [_p, _p, _i64, _p, _i64, _i64, _u64, _p, _p]),
    "pglb_node2vec_walk": (c_int, [_p, _p, _p, _i64, _p, _i64, _i64, ctypes.c_double, ctypes.c_double, c_int, _u64,
                                   _p, _p, _p]),
    "pglb_walk_host": (c_int, [_p, _p, _p, _i64, _p, _i64, _i64, ctypes.c_double, ctypes.c_double, c_int, _u64, _p,
                               _p]),
    "pglb_metapath_walk": (c_int, [_p, _p, c_int, _i64, _p, _i64, _i64, _u64, _p, _p]),
    "pglb_metapath_walk_host": (c_int, [_p, _p, c_int, _i64, _p, _i64, _i64, _u64, _p]),
    "pglb_skipgram_count_ws": (c_int, [_i64, POINTER(c_size_t)]),
    "pglb_skipgram_count": (c_int, [_p, _i64, _i64, _i64, _u64, _p, _p, c_size_t, _p]),
    "pglb_skipgram_fill": (c_int, [_p, _i64, _i64, _i64, _u64, _p, _p, _p, _p]),
    "pglb_skipgram_host": (c_int, [_p, _i64, _i64, _i64, _u64, _p, _p, _p]),
    "pglb_alias_build_host": (c_int, [_p, _i64, _p, _p]),
    "pglb_alias_sample": (c_int, [_p, _p, _i64, _i64, _u64, _p, _p]),
    "pglb_alias_sample_host": (c_int, [_p, _p, _i64, _i64, _u64, _p]),
    "pglb_sgns_fwd_ws": (c_int, [_i64, POINTER(c_size_t)]),
    "pglb_sgns_fwd_f32": (c_int, [_p, _i64, _i64, _p, _i64, _i64, _p, _p, _i64, _i64, _i64, _p, _p, _p, _i64, _p,
                                  c_size_t, _p]),
    "pglb_attn_readout_ws": (c_int, [_i64, _i64, _i64, _i64, POINTER(c_size_t)]),
    "pglb_attn_readout_f32": (c_int, [_p, _i64, _i64, _p, _i64, _i64, _p, _p, _p, _p, _p, c_size_t, _p]),
    "pglb_attn_readout_bwd_f32": (c_int, [_p, _i64, _i64, _p, _i64, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p,
                                          c_size_t, _p]),
    "pglb_segment_topk_count": (c_int, [_p, _i64, ctypes.c_float, _i64, _p, _p, _p]),
    "pglb_segment_topk_ws": (c_int, [_i64, _i64, _i64, POINTER(c_size_t)]),
    "pglb_segment_topk_fill": (c_int, [_p, _i64, _p, _i64, _p, _i64, _p, _p, c_size_t, _p]),
    "pglb_segment_pad": (c_int, [_p, _i64, _i64, c_int, _p, _i64, _i64, _u64, _p, _p]),
    "pglb_segment_unpad": (c_int, [_p, _i64, _i64, _i64, c_int, _p, _i64, _p, _p]),
    "pglb_linear_tf32x3_f32": (c_int, [_p, _i64, _p, _p, _p, _i64, _i64, _i64, _i64, c_int, _p]),
    "pglb_gat_fused_csr_f32": (c_int, [_p, _p, _p, _i64, _p, _p, ctypes.c_float, _p, _i64, _i64, _i64, _i64,
                                       _i64, _i64, _p, c_size_t, _p]),
    "pglb_head_dots_f32": (c_int, [_p, _i64, _i64, _i64, _i64, _p, _p, _p, _p, _p]),
    "pglb_gat_fused_train_csr_f32": (c_int, [_p, _p, _p, _i64, _p, _p, ctypes.c_float, _p, _i64, _p, _i64, _i64,
                                             _i64, _i64, _i64, _p, c_size_t, _p]),
    "pglb_gat_bwd_edge_f32": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _p, _p, ctypes.c_float,
                                      _i64, _i64, _i64, _p, _p, _p]),
    "pglb_gat_fused_csr_x16": (c_int, [_p, _p, _p, _i64, _p, _p, ctypes.c_float, _p, _i64, _i64, _i64, _i64,
                                       _i64, _i64, c_int, _p, c_size_t, _p]),
    "pglb_gat_fused_train_csr_x16": (c_int, [_p, _p, _p, _i64, _p, _p, ctypes.c_float, _p, _i64, _p, _i64, _i64,
                                             _i64, _i64, _i64, c_int, _p, c_size_t, _p]),
    "pglb_gat_bwd_edge_x16": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _p, _p, ctypes.c_float,
                                      _i64, _i64, _i64, c_int, _p, _p, _p]),
    "pglb_head_dots_x16": (c_int, [_p, _i64, _i64, _i64, _i64, c_int, _p, _p, _p, _p, _p]),
    "pglb_gat_fused_train_drop_csr_f32": (c_int, [_p, _p, _p, _i64, _p, _p, ctypes.c_float, _p, _i64, _p, _i64, _i64,
                                                  _i64, _i64, _i64, ctypes.c_float, _u64, _u64, _p, c_size_t, _p]),
    "pglb_gat_fused_train_drop_csr_x16": (c_int, [_p, _p, _p, _i64, _p, _p, ctypes.c_float, _p, _i64, _p, _i64, _i64,
                                                  _i64, _i64, _i64, c_int, ctypes.c_float, _u64, _u64, _p, c_size_t,
                                                  _p]),
    "pglb_gat_bwd_edge_drop_f32": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _p, _p, ctypes.c_float,
                                           _i64, _i64, _i64, ctypes.c_float, _u64, _u64, _p, _p, _p]),
    "pglb_gat_bwd_edge_drop_x16": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _p, _p, ctypes.c_float,
                                           _i64, _i64, _i64, c_int, ctypes.c_float, _u64, _u64, _p, _p, _p]),
    "pglb_attn_dropout_keep_host": (c_int, [_u64, _u64, ctypes.c_float, _i64, _i64, _i64, _p]),
    "pglb_dot_attn_csr_f32": (c_int, [_p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _i64, _i64, _i64, _i64,
                                      _p, c_size_t, _p]),
    "pglb_dot_attn_csr_x16": (c_int, [_p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _i64, _i64, _i64, _i64,
                                      c_int, _p, c_size_t, _p]),
    "pglb_dot_attn_drop_csr_f32": (c_int, [_p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _i64, _i64, _i64,
                                           _i64, ctypes.c_float, _u64, _u64, _p, c_size_t, _p]),
    "pglb_dot_attn_drop_csr_x16": (c_int, [_p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _i64, _i64, _i64,
                                           _i64, c_int, ctypes.c_float, _u64, _u64, _p, c_size_t, _p]),
    "pglb_dot_attn_bwd_edge_f32": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _i64,
                                           _i64, _p, _p, _p]),
    "pglb_dot_attn_bwd_edge_x16": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _i64,
                                           _i64, c_int, _p, _p, _p]),
    "pglb_dot_attn_bwd_edge_drop_f32": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64,
                                                _i64, _i64, ctypes.c_float, _u64, _u64, _p, _p, _p]),
    "pglb_dot_attn_bwd_edge_drop_x16": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64,
                                                _i64, _i64, c_int, ctypes.c_float, _u64, _u64, _p, _p, _p]),
    "pglb_dot_attn_e_csr_f32": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _i64,
                                        _i64, _i64, _i64, _p, c_size_t, _p]),
    "pglb_dot_attn_e_csr_x16": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _i64,
                                        _i64, _i64, _i64, c_int, _p, c_size_t, _p]),
    "pglb_dot_attn_e_drop_csr_f32": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64,
                                             _i64, _i64, _i64, _i64, ctypes.c_float, _u64, _u64, _p, c_size_t, _p]),
    "pglb_dot_attn_e_drop_csr_x16": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64,
                                             _i64, _i64, _i64, _i64, c_int, ctypes.c_float, _u64, _u64, _p, c_size_t,
                                             _p]),
    "pglb_dot_attn_e_bwd_edge_f32": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64,
                                             _p, _i64, _i64, _i64, _p, _p, _p, _i64, _p]),
    "pglb_dot_attn_e_bwd_edge_x16": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64,
                                             _p, _i64, _i64, _i64, c_int, _p, _p, _p, _i64, _p]),
    "pglb_dot_attn_e_bwd_edge_drop_f32": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p,
                                                  _i64, _p, _i64, _i64, _i64, ctypes.c_float, _u64, _u64, _p, _p, _p,
                                                  _i64, _p]),
    "pglb_dot_attn_e_bwd_edge_drop_x16": (c_int, [_p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p, _i64, _p,
                                                  _i64, _p, _i64, _i64, _i64, c_int, ctypes.c_float, _u64, _u64, _p,
                                                  _p, _p, _i64, _p]),
    "pglb_gatv2_attn_csr_f32": (c_int, [_p, _p, _p, _i64, _p, ctypes.c_float, _p, _i64, _p, _i64, _i64, _i64, _i64,
                                        _p, c_size_t, _p]),
    "pglb_gatv2_attn_csr_x16": (c_int, [_p, _p, _p, _i64, _p, ctypes.c_float, _p, _i64, _p, _i64, _i64, _i64, _i64,
                                        c_int, _p, c_size_t, _p]),
    "pglb_gatv2_attn_drop_csr_f32": (c_int, [_p, _p, _p, _i64, _p, ctypes.c_float, _p, _i64, _p, _i64, _i64, _i64,
                                             _i64, ctypes.c_float, _u64, _u64, _p, c_size_t, _p]),
    "pglb_gatv2_attn_drop_csr_x16": (c_int, [_p, _p, _p, _i64, _p, ctypes.c_float, _p, _i64, _p, _i64, _i64, _i64,
                                             _i64, c_int, ctypes.c_float, _u64, _u64, _p, c_size_t, _p]),
    "pglb_gatv2_bwd_edge_ws": (c_int, [_i64, _p]),
    "pglb_gatv2_bwd_edge_f32": (c_int, [_p, _p, _p, _p, _i64, _p, ctypes.c_float, _p, _i64, _p, _i64, _p, _i64, _i64,
                                        _i64, _p, _p, _p, _p, c_size_t, _p]),
    "pglb_gatv2_bwd_edge_x16": (c_int, [_p, _p, _p, _p, _i64, _p, ctypes.c_float, _p, _i64, _p, _i64, _p, _i64, _i64,
                                        _i64, c_int, _p, _p, _p, _p, c_size_t, _p]),
    "pglb_gatv2_bwd_edge_drop_f32": (c_int, [_p, _p, _p, _p, _i64, _p, ctypes.c_float, _p, _i64, _p, _i64, _p, _i64,
                                             _i64, _i64, ctypes.c_float, _u64, _u64, _p, _p, _p, _p, c_size_t, _p]),
    "pglb_gatv2_bwd_edge_drop_x16": (c_int, [_p, _p, _p, _p, _i64, _p, ctypes.c_float, _p, _i64, _p, _i64, _p, _i64,
                                             _i64, _i64, c_int, ctypes.c_float, _u64, _u64, _p, _p, _p, _p, c_size_t,
                                             _p]),
    "pglb_gatv2_score_grad_f32": (c_int, [_p, _p, _p, _p, _i64, _p, ctypes.c_float, _p, _p, _i64, _i64, _i64, _i64,
                                          _i64, c_int, _p, c_size_t, _p]),
    "pglb_gatv2_score_grad_x16": (c_int, [_p, _p, _p, _p, _i64, _p, ctypes.c_float, _p, _p, _i64, _i64, _i64, _i64,
                                          _i64, c_int, c_int, _p, c_size_t, _p]),
    "pglb_fa_attn_csr_f32": (c_int, [_p, _p, _p, _i64, _p, _p, _i64, _i64, _i64, _i64, _p, c_size_t, _p]),
    "pglb_fa_attn_csr_x16": (c_int, [_p, _p, _p, _i64, _p, _p, _i64, _i64, _i64, _i64, c_int, _p, c_size_t, _p]),
    "pglb_fa_attn_drop_csr_f32": (c_int, [_p, _p, _p, _i64, _p, _p, _i64, _i64, _i64, _i64, ctypes.c_float, _u64,
                                          _u64, _p, c_size_t, _p]),
    "pglb_fa_attn_drop_csr_x16": (c_int, [_p, _p, _p, _i64, _p, _p, _i64, _i64, _i64, _i64, c_int, ctypes.c_float,
                                          _u64, _u64, _p, c_size_t, _p]),
    "pglb_fa_bwd_edge_f32": (c_int, [_p, _p, _p, _p, _i64, _p, _p, _i64, _i64, _i64, _p, _p, _p]),
    "pglb_fa_bwd_edge_x16": (c_int, [_p, _p, _p, _p, _i64, _p, _p, _i64, _i64, _i64, c_int, _p, _p, _p]),
    "pglb_fa_bwd_edge_drop_f32": (c_int, [_p, _p, _p, _p, _i64, _p, _p, _i64, _i64, _i64, ctypes.c_float, _u64, _u64,
                                          _p, _p, _p]),
    "pglb_fa_bwd_edge_drop_x16": (c_int, [_p, _p, _p, _p, _i64, _p, _p, _i64, _i64, _i64, c_int, ctypes.c_float,
                                          _u64, _u64, _p, _p, _p]),
    "pglb_rgcn_agg_f32": (c_int, [_p, _p, _p, _p, _p, _i64, _p, _i64, _i64, _i64, _p, _i64, _i64, _p]),
    "pglb_rgcn_wgrad_ws": (c_int, [_i64, _i64, _i64, POINTER(c_size_t)]),
    "pglb_rgcn_wgrad_f32": (c_int, [_p, _p, _p, _p, _p, _i64, _i64, _i64, _p, _p, _i64, _p, _i64, _i64, _i64, _p, _p,
                                    c_size_t, _p]),
    "pglb_gat_attention_csr_f32":(c_int, [_p, _p, _p, _p, ctypes.c_float, _p, _i64, _i64, _i64, _p,
                                           c_size_t, _p]),
    "pglb_sddmm_dot_f32": (c_int, [_p, _p, _p, _i64, _p, _i64, _i64, _i64, _i64, _p, _p]),
    "pglb_edge_softmax_bwd_csr_f32": (c_int, [_p, _p, _p, _p, _p, _i64, _i64, _i64, _p]),
    "pglb_maxmin_bwd_f32": (c_int, [_p, _p, _p, _p, _p, _p, _i64, _i64, _p]),
    "pglb_debug_task_trace": (c_int, [_p, _i64]),
    "pglb_map_nodes": (c_int, [_p, _i64, _p, _i64, _p, _p, _p]),
    "pglb_map_edges": (c_int, [_p, _i64, _p, _i64, _p, _i64, _p, _p, _p]),
    "pglb_invert_perm": (c_int, [_p, _i64, _p, _p]),
    "pglb_halo_plan_ws": (c_int, [_i64, _i64, POINTER(c_size_t)]),
    "pglb_halo_plan_count": (c_int, [_p, _i64, _i64, _i64, _i64, _p, _p, _p, c_size_t, _p]),
    "pglb_halo_plan_fill": (c_int, [_p, _i64, _i64, _i64, _i64, _p, _i64, _p, _p, _p, _p, _p, _p, c_size_t, _p]),
    "pglb_metis_partition": (c_int, [c_char_p, _i64, _p, _p, _i64, _p, _p, c_int, _p]),
}

for _name, (_res, _args) in _SIGS.items():
    _f = getattr(lib, _name)
    _f.restype = _res
    _f.argtypes = _args


def check(rc):
    if rc != PGLB_OK:
        msg = lib.pglb_last_error()
        raise PglbError(rc, msg.decode("utf-8", "replace") if msg else "")


def launch_count():
    return int(lib.pglb_launch_count())
