"""GPU neighbour sampling (mirror of reference pgl/sampling/sage.py:130-155): csrc/sampling.cu, validated on
hardware in round 2 (tests/test_gpu_sampling.py, DESIGN.md section 4.6); relation-typed sampling on a HeterGraph
(HeteroNeighborSampler, DESIGN.md section 4.14); random walks (reference
pgl/sampling/walk.py): csrc/walk.cu (DESIGN.md section 4.9); metapath walks on a HeterGraph (the reference's
examples/metapath2vec metapath_randomwalk): csrc/walk.cu (DESIGN.md section 4.15); skip-gram pairs and alias-table
negative sampling of the walks: csrc/skipgram.cu (DESIGN.md section 4.17)."""
from .custom import subgraph  # noqa: F401
from .sage import (HeteroNeighborSampler, NeighborSampler, reindex_graph, sample_neighbors,  # noqa: F401
                   sample_typed_neighbors)
from .skipgram import alias_sample, alias_table, skip_gram_pairs  # noqa: F401
from .walk import metapath_randomwalk, node2vec_walk, node2vec_walk_plus, random_walk  # noqa: F401
