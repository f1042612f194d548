"""SkipGramModel: the reference's DeepWalk / node2vec model (examples/deepwalk/model.py) on the fused skip-gram loss."""
import torch

from . import functional as GF

__all__ = ["SkipGramModel"]


class SkipGramModel(torch.nn.Module):
    """The deepwalk example's constructor and initialisers: node embeddings U(-1, 1) and, unless shared_embedding,
    context embeddings U(-1e-8, 1e-8).  forward(src [P] or [P, 1], dsts [P, 1 + neg_num]) returns the scalar loss.
    sparse=True gives the tables sparse gradients (torch.optim.SparseAdam, SGD, Adagrad), as nn.Embedding(sparse=True).
    The reference's num_emb_part and sparse_embedding options are Paddle static-graph devices and are not taken."""

    def __init__(self, num_nodes, embed_size=16, neg_num=5, sparse=False, shared_embedding=False):
        super().__init__()
        self.num_nodes = num_nodes
        self.neg_num = neg_num
        self.sparse = sparse
        self.shared_embedding = shared_embedding
        self.emb = torch.nn.Embedding(num_nodes, embed_size, sparse=sparse)
        torch.nn.init.uniform_(self.emb.weight, -1.0, 1.0)
        if not shared_embedding:
            self.v_emb = torch.nn.Embedding(num_nodes, embed_size, sparse=sparse)
            torch.nn.init.uniform_(self.v_emb.weight, -1e-8, 1e-8)

    def forward(self, src, dsts):
        ctx = self.emb.weight if self.shared_embedding else self.v_emb.weight
        return GF.skip_gram_loss(self.emb.weight, ctx, src, dsts, sparse=self.sparse)
