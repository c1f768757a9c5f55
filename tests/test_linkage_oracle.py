"""The centroid-linkage specification that csrc/diar_cluster.cu implements (oracle/linkage_ref.py) gives exactly scipy's
`linkage(x, method="centroid")`: np.array_equal on the whole Z, inversions and merge order included."""
import numpy as np
import pytest
from scipy.cluster.hierarchy import linkage
from scipy.spatial.distance import pdist

from oracle.linkage_ref import embeddings


@pytest.mark.parametrize("kind", ["random", "clustered"])
@pytest.mark.parametrize("n", [2, 3, 5, 40, 200, 600])
def test_oracle_equals_scipy_centroid_linkage(n, kind):
    from oracle import linkage_ref
    x = embeddings(kind, n)
    want = linkage(x, method="centroid", metric="euclidean")
    got = linkage_ref.centroid_linkage(x)
    assert np.array_equal(got, want)


def test_sequential_distances_equal_pdist():
    from oracle import linkage_ref
    x = embeddings("clustered", 300)
    assert np.array_equal(linkage_ref.condensed(linkage_ref.pairwise(x)), pdist(x))
