"""Skip-gram training pairs and alias-table negative samples on the device (csrc/skipgram.cu), for the walk-based
models (DeepWalk, node2vec, metapath2vec): walks -> pairs -> negatives without a host round trip.

* ``skip_gram_pairs(walks, win_size=5, seed=None)``: the pairs of a whole batch of walks in one count -> scan -> fill
  sequence.  Centre i of walk b draws a window w uniform on [1, win_size] (Philox, a pure function of (seed, b, i)) and
  pairs with every position within w of it whose node differs from its own -- the reference's ``skip_gram_gen_pair``
  rule, walk after walk, with device-drawn windows.
* ``alias_table(weights)``: Vose's alias table of the normalised weights (the reference's ``alias_sample_build_table``,
  bit for bit), built once on the host.
* ``alias_sample(alias, events, size, seed=None)``: draws of that table on the device.

Mode rule: CUDA tensors in, CUDA tensors out (on their device); numpy arrays or lists in, numpy arrays out (the work
runs on the current CUDA device).  ``seed=None`` draws a 64-bit seed from ``np.random``, as the walks do."""
import math

import numpy as np
import torch

from .. import ops
from ..graph_kernel import alias_sample_build_table
from .walk import _seed

__all__ = ["skip_gram_pairs", "alias_table", "alias_sample"]


def _check_win(win_size):
    if isinstance(win_size, bool) or int(win_size) != win_size or not 1 <= int(win_size) < 2 ** 31:
        raise ValueError("win_size must be an integer in [1, 2^31), got %r" % (win_size,))
    return int(win_size)


def _pad(walks):
    """A list of walks (lists or 1-D arrays of non-negative ids) as one [B, L] int64 array padded with -1."""
    rows = []
    for w in walks:
        a = np.asarray(w)
        if a.ndim != 1:
            raise ValueError("walks must be 2-D: a list of 1-D walks")
        if a.size and (a.dtype.kind not in "iu"):
            raise ValueError("walks must hold integer node ids, got %s" % a.dtype)
        a = a.astype(np.int64)
        if a.size and a.min() < 0:
            raise ValueError("a listed walk holds a negative node id")
        rows.append(a)
    L = max((len(r) for r in rows), default=0)
    out = np.full((len(rows), L), -1, np.int64)
    for b, r in enumerate(rows):
        out[b, :len(r)] = r
    return out


def skip_gram_pairs(walks, win_size=5, seed=None):
    """Skip-gram (centre, context) pairs of a batch of walks.

    Args:
        walks: an int64 CUDA tensor ``[B, L]`` padded with -1 after each walk (the tensor-mode walk output), or a list
            of walks (the numpy-mode walk output), padded here and run on the current CUDA device.
        win_size: the largest window, in [1, 2^31).
        seed: 64-bit seed of the windows; None draws one from ``np.random``.

    Returns ``(src, pos)``, int64 of equal length, in walk, centre, context-position order: CUDA tensors for a tensor
    input, numpy arrays for a list.  Raises ValueError, before any launch, for float or bool walks, walks that are not
    2-D, or a bad win_size."""
    win_size = _check_win(win_size)
    if isinstance(walks, torch.Tensor):
        if walks.dtype.is_floating_point or walks.dtype.is_complex or walks.dtype == torch.bool:
            raise ValueError("walks must hold integer node ids, got %s" % walks.dtype)
        if walks.dim() != 2:
            raise ValueError("walks must be a 2-D [B, L] tensor, got %d-D" % walks.dim())
        ops.require_cuda(walks)
        return ops.skip_gram_pairs(walks, win_size, _seed(seed))
    if isinstance(walks, np.ndarray):
        if walks.ndim != 2:
            raise ValueError("walks must be 2-D, got %d-D" % walks.ndim)
        if walks.size and walks.dtype.kind not in "iu":
            raise ValueError("walks must hold integer node ids, got %s" % walks.dtype)
        padded = walks.astype(np.int64)
    else:
        padded = _pad(walks)
    seed = _seed(seed)
    dev = torch.device("cuda", torch.cuda.current_device())
    src, pos = ops.skip_gram_pairs(torch.from_numpy(padded).to(dev), win_size, seed)
    return src.cpu().numpy(), pos.cpu().numpy()


def alias_table(weights):
    """(alias, events) of the distribution proportional to ``weights`` (non-negative, finite, positive sum),
    normalised in float64 and built by the reference's construction.  CUDA input: float64 / int64 CUDA tensors on its
    device; CPU tensor: CPU tensors; numpy or list: numpy arrays."""
    if isinstance(weights, torch.Tensor):
        w = weights.detach().to("cpu", torch.float64).numpy()
    else:
        w = np.asarray(weights, dtype=np.float64)
    if w.ndim != 1:
        raise ValueError("weights must be 1-D, got shape %s" % (w.shape,))
    if w.size == 0:
        raise ValueError("weights is empty")
    if not np.isfinite(w).all():
        raise ValueError("weights must be finite")
    if (w < 0).any():
        raise ValueError("weights must be non-negative")
    total = w.sum()
    if not total > 0 or not math.isfinite(total):
        raise ValueError("weights must have a positive finite sum, got %r" % total)
    alias, events = alias_sample_build_table(w / total)
    if isinstance(weights, torch.Tensor):
        return torch.from_numpy(alias).to(weights.device), torch.from_numpy(events).to(weights.device)
    return alias, events


def alias_sample(alias, events, size, seed=None):
    """``size`` int64 draws (an int or a shape) of the table from ``alias_table``: draw k takes slot
    s = mulhi64(r64, n) and keeps it with probability alias[s], else takes events[s].  CUDA tensors in, a CUDA tensor
    out; numpy in, numpy out (drawn on the current CUDA device)."""
    shape = (int(size),) if np.isscalar(size) else tuple(int(s) for s in size)
    if any(s < 0 for s in shape):
        raise ValueError("size must be non-negative, got %r" % (size,))
    count = int(np.prod(shape, dtype=np.int64))
    n = alias.shape[0] if alias.ndim == 1 else -1
    if n < 1 or events.ndim != 1 or events.shape[0] != n:
        raise ValueError("alias and events must be 1-D of one length >= 1")
    if n >= 2 ** 32:
        raise ValueError("an alias table has fewer than 2^32 entries, got %d" % n)
    seed = _seed(seed)
    if isinstance(alias, torch.Tensor):
        return ops.alias_sample(alias, events, count, seed).reshape(shape)
    dev = torch.device("cuda", torch.cuda.current_device())
    out = ops.alias_sample(torch.from_numpy(np.ascontiguousarray(alias, np.float64)).to(dev),
                           torch.from_numpy(np.ascontiguousarray(events, np.int64)).to(dev), count, seed)
    return out.cpu().numpy().reshape(shape)
