"""numpy restatement of centroid-linkage clustering as reverb_b200/csrc/diar_cluster.cu computes it.

tests/test_linkage_oracle.py pins this against `scipy.cluster.hierarchy.linkage(x, method="centroid")` (np.array_equal
on the whole Z), which pins the algorithm before anything runs on the GPU:

  * distances: sqrt of (x_ik - x_jk)^2 summed over k in index order (scipy's pdist; a split accumulator is not equal)
  * merges: the globally closest active pair (a, b), a < b, ties to the smallest (a, b); the merged cluster keeps slot
    b and slot a is retired
  * update: d(k,b) = sqrt(((sa*d_ak*d_ak) + (sb*d_bk*d_bk) - (sa*sb*d*d)/s) / s), s = sa + sb, in this order
  * rows in merge order (not sorted), relabelled by a union-find in merge order; column 3 is the size
"""
from __future__ import annotations

import numpy as np


def embeddings(kind: str, n: int, dim: int = 256, seed: int = 0) -> np.ndarray:
    """test inputs, unit-normalised float64: "random" normal vectors, or "clustered" around 5 speakers"""
    rng = np.random.default_rng(seed + n)
    if kind == "random":
        x = rng.normal(size=(n, dim))
    else:
        centres = rng.normal(size=(5, dim))
        x = centres[rng.integers(0, 5, n)] * 0.12 + 0.05 * rng.normal(size=(n, dim))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def pairwise(x: np.ndarray) -> np.ndarray:
    """(n, n) Euclidean distances, each sum accumulated over the dimensions in index order."""
    x = np.asarray(x, np.float64)
    n, dim = x.shape
    acc = np.zeros((n, n), np.float64)
    for k in range(dim):
        t = x[:, None, k] - x[None, :, k]
        acc += t * t
    return np.sqrt(acc)


def condensed(D: np.ndarray) -> np.ndarray:
    """upper triangle of a square matrix in scipy's pdist order"""
    iu = np.triu_indices(D.shape[0], k=1)
    return D[iu]


def centroid_linkage(x: np.ndarray) -> np.ndarray:
    """-> Z (n - 1, 4) float64, scipy's linkage layout."""
    x = np.asarray(x, np.float64)
    n = x.shape[0]
    D = pairwise(x)
    np.fill_diagonal(D, np.inf)
    size = np.ones(n)
    active = np.ones(n, bool)
    raw = np.zeros((n - 1, 4))
    for r in range(n - 1):
        M = np.where(active[:, None] & active[None, :], D, np.inf)
        i, j = np.unravel_index(np.argmin(M), M.shape)        # first minimum in row-major order = smallest (a, b)
        a, b = min(i, j), max(i, j)
        d = D[a, b]
        sa, sb = size[a], size[b]
        s = sa + sb
        raw[r] = (a, b, d, s)
        k = active.copy()
        k[a] = k[b] = False
        v = np.sqrt(((sa * D[a, k] * D[a, k]) + (sb * D[b, k] * D[b, k]) - (sa * sb * d * d) / s) / s)
        D[b, k] = v
        D[k, b] = v
        active[a] = False
        size[b] = s
    parent = np.arange(2 * n - 1)

    def find(u: int) -> int:
        while parent[u] != u:
            u = parent[u]
        return u

    Z = raw.copy()
    for r in range(n - 1):
        p, q = sorted((find(int(raw[r, 0])), find(int(raw[r, 1]))))
        Z[r, 0], Z[r, 1] = p, q
        parent[p] = parent[q] = n + r
    return Z
