from . import helper, op, edge_index, relabel, transform  # noqa: F401
