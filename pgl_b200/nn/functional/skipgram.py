"""The skip-gram negative-sampling loss of the reference's walk models (examples/deepwalk/model.py and
examples/metapath2vec/model.py, SkipGramModel.forward) on the fused kernel."""

from ... import ops

__all__ = ["skip_gram_loss"]


def skip_gram_loss(emb, ctx, src, dsts, sparse=False):
    """(BCEWithLogits(<emb[src], ctx[dsts[:, 0]]>, 1) + BCEWithLogits(<emb[src], ctx[dsts[:, 1:]]>, 0)) / 2.

    emb [N_e, D] / ctx [N_c, D]: the centre and context tables (``ctx is emb``: one shared table, as the reference's
    ``shared_embedding=True`` and its metapath2vec model).  src [P] or [P, 1] centre ids; dsts [P, 1 + K] with the
    positive in column 0 and K >= 1 negatives (metapath2vec's in-batch negatives are ``cat(pos, pos[idx])``).
    sparse=True gives coalesced sparse gradients over the touched rows, as ``nn.Embedding(sparse=True)``."""
    return ops.skip_gram_loss(emb, ctx, src, dsts, sparse=sparse)
