"""Graph-level readouts without a GPU: the numpy oracle (oracle/oracle_pool.py) against the reference tests' known
answers (tests/golden/kat_readout.json), the fp32 top-k count, the total order of segment_topk, the Python layer's
argument checks and the C entries' PGLB_EINVAL before any device work."""
import ctypes
import json
import os

import numpy as np
import pytest

from oracle import oracle_pool as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def kat():
    with open(os.path.join(ROOT, "tests", "golden", "kat_readout.json")) as f:
        return json.load(f)


def test_segment_padding_kat(kat):
    k = kat["segment_padding"]
    out, seq_len, index = P.segment_padding(np.array(k["data"], np.float32), k["segment_ids"])
    assert out.tolist() == k["out"]
    assert seq_len.dtype == np.int32 and seq_len.tolist() == [2, 0, 1]
    assert index.tolist() == [[0, 0], [0, 1], [2, 0]]


def test_segment_topk_kat(kat):
    k = kat["segment_topk"]
    x = np.array(k["data"], np.float32)
    out, perm = P.segment_topk(x, k["scores"], k["segment_ids"], k["ratio"])
    assert perm.tolist() == k["index"] and out.tolist() == k["out"]
    out, perm = P.segment_topk(x, k["scores"], k["segment_ids"], k["ratio"], min_score=k["min_score"])
    assert perm.tolist() == k["index_min_score"]


def test_topk_count_is_fp32(kat):
    for ratio, n, want in kat["topk_k_fp32"]["cases"]:
        assert int(P.topk_k(n, ratio)) == want
    assert P.topk_k(np.array([5, 1, 0]), 3).tolist() == [3, 1, 0]


def test_topk_total_order():
    s = np.array([1.0, np.nan, -0.0, 0.0, np.inf, -np.inf, 1.0, -1e30, np.nan], np.float32)
    assert P.rank_order(s).tolist() == [4, 0, 6, 2, 3, 7, 5, 1, 8]
    # every score ranks: below -1e20 too, and other segments' nodes never enter
    perm = P.segment_topk_perm(np.array([-1e30, -1e25, 5.0], np.float32), [0, 0, 1], 1.0)
    assert perm.tolist() == [1, 0, 2]
    # gapped ids: the missing segment keeps nothing
    assert P.segment_topk_perm([3, 1, 2], [0, 2, 2], 2).tolist() == [0, 2, 1]


def test_to_dense_batch_kat(kat):
    k = kat["to_dense_batch"]
    ids = np.repeat(np.arange(3), k["graph_sizes"])
    out, mask = P.to_dense_batch(np.array(k["data"], np.float32), ids, fill_value=0)
    assert out.tolist() == k["out"] and mask.tolist() == k["mask"]
    assert out.dtype == np.float32


def test_filter_adj_kat(kat):
    k = kat["filter_adj"]
    assert P.filter_adj(k["edges"], k["perm"]).tolist() == k["out"]
    # num_nodes is honoured: a wider table changes nothing, kept order is the edge order
    assert P.filter_adj(k["edges"], k["perm"], num_nodes=20).tolist() == k["out"]


def test_graph_norm_kat(kat):
    k = kat["graph_norm"]
    ids = np.repeat(np.arange(2), [g["num_nodes"] for g in k["graphs"]])
    assert P.graph_norm(ids, np.array(k["feature"], np.float32)).tolist() == k["out"]


def test_attn_readout_oracle_overflow_and_empty(kat):
    k = kat["segment_softmax_overflow"]
    x = np.eye(2)
    out, lse = P.attn_readout(x, [0, 0], gate=k["scores"])
    assert out[0].tolist() == k["weights"]
    out, lse = P.attn_readout(np.ones((2, 3)), [0, 2, 2], gate=np.zeros(2), indptr=True)
    assert out.tolist() == [[1, 1, 1], [0, 0, 0]] and lse[1] == -np.inf and lse[0] == np.log(2.0)


def test_python_argument_checks():
    import torch
    import pgl_b200 as pgl
    x = torch.zeros(3, 2)
    ids = torch.zeros(3, dtype=torch.int64)
    for bad in (0.0, 1.5, -0.1, float("nan")):
        with pytest.raises(ValueError):
            pgl.math.segment_topk(x, x[:, 0], ids, bad)
    with pytest.raises(ValueError):
        pgl.math.segment_topk(x, x[:, 0], ids, 0)
    with pytest.raises(ValueError):
        pgl.ops.segment_topk_perm(x[:, 0], ids, 2.0)
    with pytest.raises(ValueError):
        pgl.ops.attn_readout(x, ids)
    with pytest.raises(ValueError):
        pgl.ops.attn_readout(x, ids, gate=x[:, 0], query=x)


def test_entries_reject_bad_arguments_without_a_device():
    from pgl_b200 import _lib
    lib = _lib.lib
    one = ctypes.c_void_p(256)   # non-NULL, aligned dummy: never dereferenced here
    need = ctypes.c_size_t(0)
    # attention readout: exactly one of gate / query, sizes, workspace
    assert lib.pglb_attn_readout_ws(4, 100, 8, 10, ctypes.byref(need)) == 0 and need.value == 0
    assert lib.pglb_attn_readout_ws(4, 10 ** 6, 8, 10 ** 6, ctypes.byref(need)) == 0 and need.value > 0
    assert lib.pglb_attn_readout_ws(-1, 100, 8, 10, ctypes.byref(need)) == -1
    assert lib.pglb_attn_readout_f32(one, 10, 8, one, 2, 5, None, None, one, one, None, 0, None) == -1
    assert b"exactly one" in lib.pglb_last_error()
    assert lib.pglb_attn_readout_f32(one, 10, 8, one, 2, 5, one, one, one, one, None, 0, None) == -1
    assert lib.pglb_attn_readout_f32(one, 10, 0, one, 2, 5, one, None, one, one, None, 0, None) == -1
    assert lib.pglb_attn_readout_f32(one, 10, 8, one, 2, -1, one, None, one, one, None, 0, None) == -1
    assert lib.pglb_attn_readout_f32(one, 10, 8, None, 2, 5, one, None, one, one, None, 0, None) == -1
    assert lib.pglb_attn_readout_f32(one, 10 ** 6, 8, one, 2, 10 ** 6, one, None, one, one, None, 0, None) == -3
    assert lib.pglb_attn_readout_f32(None, 0, 8, None, 0, 0, one, None, None, None, None, 0, None) == 0
    assert lib.pglb_attn_readout_bwd_f32(one, 10, 8, one, 2, 5, None, None, one, one, one, one, None, None, None, 0,
                                         None) == -1
    assert lib.pglb_attn_readout_bwd_f32(one, 10, 8, one, 2, 5, None, one, one, one, one, one, None, None, None, 0,
                                         None) == -1   # query given, grad_query NULL
    # top-k: float ratio in (0, 1], k >= 0, pointers
    assert lib.pglb_segment_topk_count(one, 2, 0.0, 0, one, one, None) == -1
    assert b"(0, 1]" in lib.pglb_last_error()
    assert lib.pglb_segment_topk_count(one, 2, 1.5, 0, one, one, None) == -1
    assert lib.pglb_segment_topk_count(one, 2, float("nan"), 0, one, one, None) == -1
    assert lib.pglb_segment_topk_count(one, 2, 0.5, -1, one, one, None) == -1
    assert lib.pglb_segment_topk_count(one, 2, 0.5, 0, None, one, None) == -1
    assert lib.pglb_segment_topk_ws(2, 100, 50, ctypes.byref(need)) == 0 and need.value == 0
    assert lib.pglb_segment_topk_ws(2, 10 ** 5, 10 ** 5, ctypes.byref(need)) == 0 and need.value >= 32 * 10 ** 5
    assert lib.pglb_segment_topk_fill(one, 10, one, 2, one, 11, one, None, 0, None) == -1   # max_len > N
    assert lib.pglb_segment_topk_fill(one, 10 ** 5, one, 2, one, 10 ** 5, one, None, 0, None) == -3
    # pad / unpad: element size 2, 4 or 8
    assert lib.pglb_segment_pad(one, 10, 4, 3, one, 2, 5, 0, one, None) == -1
    assert lib.pglb_segment_pad(one, 10, 4, 4, None, 2, 5, 0, one, None) == -1
    assert lib.pglb_segment_pad(one, -1, 4, 4, one, 2, 5, 0, one, None) == -1
    assert lib.pglb_segment_unpad(one, 2, 5, 4, 1, one, 10, one, None) == -1
    assert lib.pglb_segment_unpad(one, 0, 5, 4, 4, None, 10, one, None) == -1
    assert lib.pglb_segment_pad(None, 0, 4, 4, None, 0, 0, 0, None, None) == 0
