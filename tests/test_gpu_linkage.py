"""Centroid linkage on the GPU (csrc/diar_cluster.cu through rvb_centroid_linkage) against scipy: the same Z bit for
bit, the same pairwise distances as pdist, a valid dendrogram on exact ties, and the same diarization turns as the
scipy clustering path."""
import numpy as np
import pytest
from scipy.cluster.hierarchy import fcluster, linkage
from scipy.spatial.distance import pdist

from oracle.linkage_ref import embeddings

pytestmark = pytest.mark.gpu

THRESHOLD = 0.7045654963945799


@pytest.mark.parametrize("kind", ["random", "clustered"])
@pytest.mark.parametrize("n", [2, 3, 17, 256, 1000, 4000, 8000])
def test_linkage_equals_scipy(n, kind):
    from reverb_b200.diarization.pipeline import centroid_linkage
    x = embeddings(kind, n, seed=1)
    want = linkage(x, method="centroid", metric="euclidean")
    got = centroid_linkage(x, "cuda")
    assert got.shape == (n - 1, 4)
    assert np.array_equal(got, want), f"first differing row {np.argmax(np.any(got != want, axis=1))}"


@pytest.mark.parametrize("n", [17, 1000])
def test_distance_phase_equals_pdist(n):
    from reverb_b200.diarization.pipeline import centroid_linkage
    x = embeddings("clustered", n, seed=2)
    _, dist = centroid_linkage(x, "cuda", return_distances=True)
    assert np.array_equal(dist, pdist(x))


def _partition(labels):
    """cluster labels -> set of frozensets of member indices"""
    return {frozenset(np.nonzero(labels == k)[0].tolist()) for k in np.unique(labels)}


def test_exact_ties_give_a_valid_dendrogram():
    """Duplicated embeddings tie at height 0 (and their clusters tie again later): the tie rule (smallest height, then
    smallest (a, b)) is the oracle's, so Z equals the oracle's row for row, every height is what the oracle's formula
    gives for the pair merged, and the cut at the pipeline's threshold is scipy's partition."""
    from oracle import linkage_ref
    from reverb_b200.diarization.pipeline import centroid_linkage
    base = embeddings("clustered", 60, seed=3)
    x = base[np.random.default_rng(4).integers(0, 60, 300)]
    got = centroid_linkage(x, "cuda")
    assert np.array_equal(got, linkage_ref.centroid_linkage(x))
    assert (got[:, 2] == 0.0).sum() >= 240                # 300 points, 60 distinct
    want = linkage(x, method="centroid", metric="euclidean")
    assert _partition(fcluster(got, THRESHOLD, criterion="distance")) == \
        _partition(fcluster(want, THRESHOLD, criterion="distance"))


def test_bad_input_fails_loudly():
    from reverb_b200 import _lib
    from reverb_b200.diarization.pipeline import centroid_linkage
    x = embeddings("random", 8)
    x[3, 5] = np.nan
    with pytest.raises(ValueError, match="finite"):
        centroid_linkage(x, "cuda")
    lib = _lib.load()
    assert lib.rvb_centroid_linkage_workspace_bytes(1) == -1
    need = lib.rvb_centroid_linkage_workspace_bytes(8)
    assert need >= 8 * 7 // 2 * 8
    assert lib.rvb_centroid_linkage(None, 8, 256, None, None, None, need, None) != 0
    assert "bad arguments" in _lib.last_error()


def _turns_both_ways(pipe, audio, monkeypatch):
    """turns with the GPU linkage, then with scipy's linkage swapped in; the embeddings must not differ between runs"""
    from reverb_b200.diarization import pipeline as P
    gpu_Z = []
    real = P.centroid_linkage

    def recording(emb, device, **kw):
        Z = real(emb, device, **kw)
        gpu_Z.append((emb.copy(), Z))
        return Z

    monkeypatch.setattr(P, "centroid_linkage", recording)
    turns_gpu = pipe(audio)
    emb_gpu = pipe.last["embeddings"]
    monkeypatch.setattr(P, "centroid_linkage", lambda emb, device: linkage(emb, method="centroid", metric="euclidean"))
    turns_cpu = pipe(audio)
    assert np.array_equal(pipe.last["embeddings"], emb_gpu, equal_nan=True)
    assert len(gpu_Z) == 1
    emb, Z = gpu_Z[0]
    assert np.array_equal(Z, linkage(emb, method="centroid", metric="euclidean"))
    return turns_gpu, turns_cpu, emb.shape[0]


def test_pipeline_turns_equal_the_scipy_clustering(monkeypatch):
    from reverb_b200.diarization import synth
    from reverb_b200.diarization.embedding import EmbeddingModel
    from reverb_b200.diarization.pipeline import SpeakerDiarization
    from reverb_b200.diarization.segmentation import SegmentationModel
    seg = SegmentationModel(synth.segmentation_state_dict(0))
    emb = EmbeddingModel(synth.embedding_state_dict(0))
    # the recording of test_gpu_diarization's end-to-end test
    pipe = SpeakerDiarization(seg, emb, min_cluster_size=3)
    a, b, n = _turns_both_ways(pipe, synth.synthetic_speech(40.0, seed=5, turns=2), monkeypatch)
    assert a == b
    # 20 minutes: thousands of (window, speaker) embeddings
    pipe = SpeakerDiarization(seg, emb, batch_size=64)
    a, b, n = _turns_both_ways(pipe, synth.synthetic_speech(1200.0, seed=11, turns=3), monkeypatch)
    print(f"20-minute recording: {n} embeddings clustered, {len(a)} turns")
    assert n >= 1000
    assert a == b
