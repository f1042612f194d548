"""The attention-dropout stream of the fused GAT training path, without a GPU.

The keep bit of dst-CSR slot j and head h is word h % 4 of Philox4x32-10(counter = (j lo, j hi, h / 4, offset / 4),
key = (seed lo, seed hi)), kept iff the word >= thresh = min(floor(p 2^32), 2^32 - 1).  Here a numpy restatement of
Philox is pinned to Random123's published known-answer vectors, the library's host entry (the kernels' own function)
is pinned to the restatement, the keep fraction is checked against 1 - p, and the argument checks of the dropout
entries are shown to refuse before any CUDA call."""
import ctypes
import math

import numpy as np
import pytest

EINVAL, ESHAPE, EUNSUPPORTED = -1, -2, -4
MASK = np.uint64(0xFFFFFFFF)


@pytest.fixture(scope="module")
def lib():
    from pgl_b200 import _lib
    return _lib


def philox4x32_10(ctr, key):
    """ctr: four uint32 arrays (broadcastable), key: two uint32 values -> four uint32 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, np.uint64) for c in ctr)
    k0, k1 = (np.uint64(k) for k in key)
    m0, m1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(0x9E3779B9)) & MASK
            k1 = (k1 + np.uint64(0xBB67AE85)) & MASK
        p0, p1 = m0 * c0, m1 * c2     # exact: both factors < 2^32
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & MASK, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & MASK
    return [c.astype(np.uint32) for c in (c0, c1, c2, c3)]


def threshold(p):
    """thresh of the float32 p the entries receive, in double as the library derives it."""
    return min(math.floor(float(np.float32(p)) * 2.0 ** 32), 2 ** 32 - 1)


def keep_words(seed, offset, p, slot0, n, H):
    j = np.arange(n, dtype=np.uint64) + np.uint64(slot0)
    t = np.uint32(threshold(p))
    w = np.zeros(n, np.uint32)
    for q in range(H // 4):
        r = philox4x32_10((j & MASK, j >> np.uint64(32), np.full(n, q, np.uint64), np.full(n, (offset // 4) & 0xFFFFFFFF, np.uint64)),
                          (seed & 0xFFFFFFFF, seed >> 32))
        for i in range(4):
            w |= (r[i] >= t).astype(np.uint32) << np.uint32(4 * q + i)
    return w


def host_words(lib, seed, offset, p, slot0, n, H):
    out = np.zeros(n, np.uint32)
    rc = lib.lib.pglb_attn_dropout_keep_host(seed, offset, p, slot0, n, H, out.ctypes.data_as(ctypes.c_void_p))
    assert rc == 0, lib.lib.pglb_last_error()
    return out


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    got = philox4x32_10([np.array([c], np.uint64) for c in ctr], key)
    assert [int(g[0]) for g in got] == list(want)


@pytest.mark.parametrize("H", [4, 8, 12, 16, 32])
def test_host_entry_is_the_restated_stream(lib, H):
    """Bit for bit over slot ranges at 0 and across 2^32 (the counter's high word), with seeds of both halves set."""
    for seed, offset, p in ((0, 0, 0.6), (0x0123456789ABCDEF, 4 * 7919, 0.1), (2 ** 64 - 1, 2 ** 34 + 8, 0.9)):
        for slot0 in (0, 2 ** 32 - 3000):
            want = keep_words(seed, offset, p, slot0, 6000, H)
            got = host_words(lib, seed, offset, p, slot0, 6000, H)
            assert np.array_equal(got, want), (seed, offset, p, slot0)
            if H < 32:
                assert not (got >> np.uint32(H)).any()   # only the low H bits are set


def test_stream_depends_on_every_input(lib):
    base = host_words(lib, 11, 8, 0.5, 0, 4096, 8)
    assert not np.array_equal(base, host_words(lib, 12, 8, 0.5, 0, 4096, 8))         # seed
    assert not np.array_equal(base, host_words(lib, 11 + 2 ** 40, 8, 0.5, 0, 4096, 8))  # seed high word
    assert not np.array_equal(base, host_words(lib, 11, 12, 0.5, 0, 4096, 8))        # offset
    assert not np.array_equal(base, host_words(lib, 11, 8, 0.5, 2 ** 32, 4096, 8))   # slot high word
    assert np.array_equal(base, host_words(lib, 11, 8, 0.5, 0, 4096, 8))             # a pure function
    # the first four heads of an 8-head word are the 4-head word (one Philox call per four heads)
    assert np.array_equal(base & np.uint32(0xF), host_words(lib, 11, 8, 0.5, 0, 4096, 4))


def test_tiny_p_keeps_everything(lib):
    """p = 1e-12 gives thresh 0: every draw is kept (the bit anchor of the GPU tests)."""
    assert threshold(1e-12) == 0
    assert (host_words(lib, 5, 0, 1e-12, 0, 10000, 32) == np.uint32(0xFFFFFFFF)).all()


@pytest.mark.parametrize("p", [0.1, 0.5, 0.6, 0.9])
def test_keep_fraction(lib, p):
    """2^16 slots x 16 heads = 1,048,576 draws: the kept fraction is within 6 sigma of 1 - p."""
    n, H = 1 << 16, 16
    w = host_words(lib, 1234567, 40, p, 3, n, H)
    kept = int(np.unpackbits(w.view(np.uint8)).sum())
    draws = n * H
    q = 1.0 - threshold(p) / 2.0 ** 32
    sigma = math.sqrt(draws * q * (1 - q))
    assert abs(kept - draws * q) <= 6 * sigma, (kept, draws * q, sigma)
    assert abs(q - (1 - p)) < 1e-7
    # and per head: no head is starved
    per_head = np.array([int(((w >> np.uint32(h)) & np.uint32(1)).sum()) for h in range(H)])
    sig_h = math.sqrt(n * q * (1 - q))
    assert np.all(np.abs(per_head - n * q) <= 6 * sig_h), per_head


P = ctypes.c_void_p(256)     # a non-NULL, 256-byte aligned dummy: must never be dereferenced here
BAD_P = (0.0, 1.0, -0.5, 1.5, float("nan"), float("inf"))


def _err(lib):
    return lib.lib.pglb_last_error()


@pytest.mark.parametrize("x16", [False, True])
def test_forward_drop_argument_checks(lib, x16):
    def call(p=0.5, offset=0, lse=P, n_dst=10, H=8, Dh=16, dtype=None):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        # (indptr, cols, f, ldf, attn_src, attn_dst, slope, out, ldo, lse, n_dst, n_src, E, H, head_dim, [dtype,]
        #  attn_drop, seed, offset, ws, ws_bytes, stream)
        head = (P, P, P, 128, P, P, 0.2, P, 128, lse, n_dst, 10, 20, H, Dh)
        if x16:
            return lib.lib.pglb_gat_fused_train_drop_csr_x16(*head, dtype, p, 7, offset, P, 1 << 20, None)
        return lib.lib.pglb_gat_fused_train_drop_csr_f32(*head, p, 7, offset, P, 1 << 20, None)

    for p in BAD_P:
        assert call(p=p) == EINVAL and b"attn_drop" in _err(lib), p
        assert call(p=p, n_dst=0) == EINVAL, p        # refused before anything else
    assert call(offset=2) == EINVAL and b"offset" in _err(lib)
    assert call(offset=2 ** 63 + 1) == EINVAL
    assert call(lse=None) == EINVAL and b"lse" in _err(lib)
    assert call(H=2, Dh=64) == EUNSUPPORTED            # H % 4: outside the kernel
    assert call(H=16, Dh=16) == EUNSUPPORTED           # 256 elements per row
    assert call(n_dst=0) == 0                           # nothing to do: no device work
    if x16:
        assert call(dtype=0) == EINVAL and b"dtype" in _err(lib)


@pytest.mark.parametrize("x16", [False, True])
def test_backward_drop_argument_checks(lib, x16):
    def call(p=0.5, offset=0, lse=P, E=20, H=8, Dh=16, dtype=None):
        dtype = lib.DTYPE_BF16 if dtype is None else dtype
        # (rows, cols, eid, f, ldf, grad_out, ldg, out, ldo, attn_src, attn_dst, lse, slope, E, H, head_dim, [dtype,]
        #  attn_drop, seed, offset, alpha_e, dz_e, stream)
        head = (P, P, None, P, 128, P, 128, P, 128, P, P, lse, 0.2, E, H, Dh)
        if x16:
            return lib.lib.pglb_gat_bwd_edge_drop_x16(*head, dtype, p, 7, offset, P, P, None)
        return lib.lib.pglb_gat_bwd_edge_drop_f32(*head, p, 7, offset, P, P, None)

    for p in BAD_P:
        assert call(p=p) == EINVAL and b"attn_drop" in _err(lib), p
        assert call(p=p, E=0) == EINVAL, p
    assert call(offset=6) == EINVAL and b"offset" in _err(lib)
    assert call(lse=None) == EINVAL
    assert call(H=2, Dh=64) == EUNSUPPORTED and b"H % 4" in _err(lib)
    assert call(Dh=12) == EUNSUPPORTED
    assert call(E=0) == 0
    if x16:
        assert call(dtype=9) == EINVAL and b"dtype" in _err(lib)


def test_host_entry_argument_checks(lib):
    buf = np.zeros(4, np.uint32)
    ptr = buf.ctypes.data_as(ctypes.c_void_p)
    f = lib.lib.pglb_attn_dropout_keep_host
    for p in BAD_P:
        assert f(1, 0, p, 0, 4, 8, ptr) == EINVAL, p
    assert f(1, 3, 0.5, 0, 4, 8, ptr) == EINVAL
    assert f(1, 0, 0.5, -1, 4, 8, ptr) == EINVAL and f(1, 0, 0.5, 0, -4, 8, ptr) == EINVAL
    assert f(1, 0, 0.5, 0, 4, 8, None) == EINVAL
    for H in (0, 2, 6, 36):
        assert f(1, 0, 0.5, 0, 4, H, ptr) == EUNSUPPORTED, H
    assert f(1, 0, 0.5, 0, 0, 8, None) == 0
