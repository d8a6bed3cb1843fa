"""Read ranges of equal marker weight for the ranks of a read-sharded run (the sharded path itself is csrc/dist.cu)."""
from __future__ import annotations

import numpy as np


def balanced_read_ranges(weights, world):
    """Contiguous read ranges with roughly equal total weight (markers). Returns world+1 boundaries."""
    w = np.asarray(weights, dtype=np.float64)
    total = float(w.sum())
    csum = np.concatenate([[0.0], np.cumsum(w)])
    bounds = [0]
    for g in range(1, world):
        bounds.append(int(np.searchsorted(csum, total * g / world, side="left")))
    bounds.append(len(w))
    for g in range(1, world + 1):
        bounds[g] = max(bounds[g], bounds[g - 1])
    return bounds
