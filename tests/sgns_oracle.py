"""A float64 numpy statement of the skip-gram negative-sampling loss (include/pglb.h, pglb_sgns_fwd_f32;
pgl_b200.ops.skip_gram_loss), written from the rule, with both gradients, dense and per touched row.

For centre ids src [P], targets dsts [P, 1 + K] (column 0 the positive), tables emb [N_e, D] and ctx [N_c, D]:
  s[p, j] = <emb[src[p]], ctx[dsts[p, j]]>
  loss    = ( mean_p softplus(-s[p, 0]) + mean_{p, k >= 1} softplus(s[p, k]) ) / 2
  c[p, 0] = -sigmoid(-s[p, 0]) / (2P),  c[p, k] = sigmoid(s[p, k]) / (2PK)
  d emb[n] = g sum_{p: src[p] = n} sum_j c[p, j] ctx[dsts[p, j]]
  d ctx[m] = g sum_{(p, j): dsts[p, j] = m} c[p, j] emb[src[p]]
A shared table (ctx is emb) receives the sum of both."""
import numpy as np


def softplus(x):
    return np.maximum(x, 0.0) + np.log1p(np.exp(-np.abs(x)))


def sigmoid(x):
    e = np.exp(-np.abs(x))
    return np.where(x >= 0, 1.0 / (1.0 + e), e / (1.0 + e))


def sgns(emb, ctx, src, dsts, g=1.0, shared=False):
    """(loss, c, d_emb, d_ctx) in float64; d_ctx is None and d_emb holds both roles when shared.  Also returns the
    per-element sums of |terms| of each gradient, for error bounds: (abs_emb, abs_ctx)."""
    emb = np.asarray(emb, np.float64)
    ctx = emb if shared else np.asarray(ctx, np.float64)
    src = np.asarray(src, np.int64).reshape(-1)
    dsts = np.asarray(dsts, np.int64)
    P, J = dsts.shape
    K = J - 1
    u = emb[src]                                   # [P, D]
    v = ctx[dsts]                                  # [P, J, D]
    s = np.einsum("pd,pjd->pj", u, v)
    loss = (softplus(-s[:, 0]).mean() + softplus(s[:, 1:]).mean()) / 2
    c = np.empty_like(s)
    c[:, 0] = -sigmoid(-s[:, 0]) / (2 * P)
    c[:, 1:] = sigmoid(s[:, 1:]) / (2 * P * K)
    w = np.einsum("pj,pjd->pd", c, v)
    wa = np.einsum("pj,pjd->pd", np.abs(c), np.abs(v))
    d_emb = np.zeros_like(emb)
    a_emb = np.zeros_like(emb)
    np.add.at(d_emb, src, g * w)
    np.add.at(a_emb, src, abs(g) * wa)
    cu = (g * c)[:, :, None] * u[:, None, :]      # [P, J, D]
    cua = np.abs(cu)
    if shared:
        np.add.at(d_emb, dsts.reshape(-1), cu.reshape(-1, u.shape[1]))
        np.add.at(a_emb, dsts.reshape(-1), cua.reshape(-1, u.shape[1]))
        return loss, c, d_emb, None, (a_emb, None)
    d_ctx = np.zeros_like(ctx)
    a_ctx = np.zeros_like(ctx)
    np.add.at(d_ctx, dsts.reshape(-1), cu.reshape(-1, u.shape[1]))
    np.add.at(a_ctx, dsts.reshape(-1), cua.reshape(-1, u.shape[1]))
    return loss, c, d_emb, d_ctx, (a_emb, a_ctx)


def touched(*ids):
    """The ascending rows any of the id arrays touch: the rows of a sparse gradient."""
    return np.unique(np.concatenate([np.asarray(i, np.int64).reshape(-1) for i in ids]))
