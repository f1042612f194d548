"""The float64 oracle of the skip-gram loss (tests/sgns_oracle.py) against a float64 torch autograd restatement of the
reference's SkipGramModel.forward, and the Python-side refusals of pgl.nn.functional.skip_gram_loss that precede any
device work.  No GPU needed."""
import numpy as np
import pytest
import torch

import sgns_oracle as SO


def reference_model(emb, ctx, src, dsts):
    """examples/deepwalk/model.py SkipGramModel.forward in torch: embedding lookups, matmuls, BCEWithLogitsLoss."""
    src_embed = emb[src.reshape(-1, 1)]                       # [P, 1, D]
    dsts_embed = ctx[dsts]                                    # [P, 1 + K, D]
    pos = torch.matmul(src_embed, dsts_embed[:, 0:1].transpose(1, 2))
    neg = torch.matmul(src_embed, dsts_embed[:, 1:].transpose(1, 2))
    bce = torch.nn.BCEWithLogitsLoss()
    return (bce(pos, torch.ones_like(pos)) + bce(neg, torch.zeros_like(neg))) / 2


def _case(seed, N, P, K, D, scale, shared):
    rng = np.random.default_rng(seed)
    emb = rng.standard_normal((N, D)) * scale
    ctx = None if shared else rng.standard_normal((N + 3, D)) * scale
    src = rng.integers(0, N, P)
    dsts = rng.integers(0, N, (P, 1 + K))
    dsts[0, 0] = src[0]                  # src == pos
    dsts[1, 1:] = src[1]                 # every negative is the centre
    dsts[2, :] = dsts[2, 0]              # repeated ids within a pair
    src[3:6] = src[2]                    # a repeated centre
    return emb, ctx, src, dsts


@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("N,P,K,D,scale", [(7, 9, 1, 3, 1.0), (50, 40, 5, 16, 1.0), (20, 64, 20, 8, 0.3),
                                           (10, 12, 3, 4, 6.0)])
def test_oracle_is_the_reference_model(shared, N, P, K, D, scale):
    emb, ctx, src, dsts = _case(N * 100 + P, N, P, K, D, scale, shared)
    g = 1.7
    loss, c, d_emb, d_ctx, _ = SO.sgns(emb, ctx, src, dsts, g=g, shared=shared)
    te = torch.tensor(emb, requires_grad=True)
    tc = te if shared else torch.tensor(ctx, requires_grad=True)
    s = torch.from_numpy(src)
    d = torch.from_numpy(dsts)
    ref = reference_model(te, tc, s, d)
    (ref * g).backward()
    assert abs(loss - ref.item()) <= 1e-12 * max(1.0, abs(loss))
    np.testing.assert_allclose(d_emb, te.grad.numpy(), rtol=1e-10, atol=1e-14)
    if not shared:
        np.testing.assert_allclose(d_ctx, tc.grad.numpy(), rtol=1e-10, atol=1e-14)
    # c is d loss / d s
    sv = torch.einsum("pd,pjd->pj", torch.tensor(emb)[s], (te if shared else tc).detach()[d]).requires_grad_(True)
    lv = (torch.nn.functional.softplus(-sv[:, 0]).mean() + torch.nn.functional.softplus(sv[:, 1:]).mean()) / 2
    lv.backward()
    # torch forms sigmoid(-s) as 1 - sigmoid(s) in softplus's backward: absolute agreement near 1e-13 at |s| ~ 30
    np.testing.assert_allclose(c, sv.grad.numpy(), rtol=1e-9, atol=1e-12 / P)


def test_saturated_logits_are_finite():
    """|s| up to 100: the stable softplus / sigmoid forms give finite values equal to the reference model's."""
    emb = np.array([[5.0, 0, 0, 0], [-5.0, 0, 0, 0]])
    ctx = np.array([[20.0, 0, 0, 0], [-20.0, 0, 0, 0], [0.0, 0, 0, 0]])
    src = np.array([0, 1, 0, 1])
    dsts = np.array([[0, 1, 2], [1, 0, 2], [1, 0, 0], [0, 1, 1]])
    loss, c, d_emb, d_ctx, _ = SO.sgns(emb, ctx, src, dsts)
    assert np.isfinite(loss) and np.isfinite(c).all() and np.isfinite(d_emb).all() and np.isfinite(d_ctx).all()
    te = torch.tensor(emb, requires_grad=True)
    tc = torch.tensor(ctx, requires_grad=True)
    ref = reference_model(te, tc, torch.from_numpy(src), torch.from_numpy(dsts))
    ref.backward()
    assert abs(loss - ref.item()) <= 1e-12 * loss
    np.testing.assert_allclose(d_emb, te.grad.numpy(), rtol=1e-10, atol=1e-300)
    np.testing.assert_allclose(d_ctx, tc.grad.numpy(), rtol=1e-10, atol=1e-300)


def test_touched_rows():
    assert SO.touched([3, 1, 3], [[5, 1], [0, 0]]).tolist() == [0, 1, 3, 5]


def test_refusals_before_any_device_work():
    import pgl_b200 as pgl
    F = pgl.nn.functional
    emb = torch.zeros(10, 4)
    src = torch.zeros(3, dtype=torch.int64)
    dsts = torch.zeros(3, 6, dtype=torch.int64)
    for dt in (torch.float16, torch.bfloat16):
        with pytest.raises(TypeError):
            F.skip_gram_loss(emb.to(dt), emb, src, dsts)
        with pytest.raises(TypeError):
            F.skip_gram_loss(emb, emb.to(dt), src, dsts)
    for bad in (src.float(), src.bool()):
        with pytest.raises(ValueError):
            F.skip_gram_loss(emb, emb, bad, dsts)
    for bad in (dsts.double(), dsts.bool()):
        with pytest.raises(ValueError):
            F.skip_gram_loss(emb, emb, src, bad)
    with pytest.raises(ValueError):
        F.skip_gram_loss(emb, emb, src, dsts[:, :1])                  # K = 0
    with pytest.raises(ValueError):
        F.skip_gram_loss(emb, emb, src.reshape(3, 1, 1), dsts)        # rank
    with pytest.raises(ValueError):
        F.skip_gram_loss(emb, emb, src.reshape(1, 3), dsts)
    with pytest.raises(ValueError):
        F.skip_gram_loss(emb, emb, src, dsts.reshape(-1))
    with pytest.raises(ValueError):
        F.skip_gram_loss(emb, emb, src[:2], dsts)                     # P mismatch
    with pytest.raises(ValueError):
        F.skip_gram_loss(emb, torch.zeros(10, 5), src, dsts)          # widths
    with pytest.raises(RuntimeError):
        F.skip_gram_loss(emb, emb, src, dsts)                         # CPU tensors: no CPU fallback


def test_model_constructor():
    import pgl_b200 as pgl
    torch.manual_seed(0)
    m = pgl.nn.SkipGramModel(1000, embed_size=32, neg_num=5)
    assert m.emb.weight.shape == (1000, 32) and m.v_emb.weight.shape == (1000, 32)
    assert m.emb.weight.abs().max() <= 1.0 and m.emb.weight.abs().max() > 0.9
    assert m.v_emb.weight.abs().max() <= 1e-8
    ms = pgl.nn.SkipGramModel(10, shared_embedding=True, sparse=True)
    assert not hasattr(ms, "v_emb") and ms.emb.sparse
