"""Speaker-diarization pipeline around the two GPU networks (segmentation.py, embedding.py).

What the reference runs (reference: diarization/infer_pyannote3.0.py:33-42):

    pipeline = Pipeline.from_pretrained('Revai/reverb-diarization-v1'); annotation = pipeline(audio)
    annotation.write_rttm(f)

i.e. `pyannote.audio.pipelines.SpeakerDiarization.apply` (pyannote.audio==3.3.1, diarization/requirements.txt:1).
** parity unpinned **: pyannote's source is absent offline; this module restates the PUBLISHED algorithm of that
pipeline (3.1 defaults: 10 s windows every 1 s, powerset segmentation, overlap-excluded masked embeddings,
centroid-linkage agglomerative clustering at threshold 0.7046 with min_cluster_size 12, count-constrained
reconstruction) step by step, naming the upstream function each step follows.  The two networks and the centroid
linkage (thousands of 256-d vectors for a long call; csrc/diar_cluster.cu) run on the GPU; the rest of the glue
(aggregation over windows, cutting the dendrogram, run-length encoding) is host numpy/scipy, as it is upstream.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, List, Optional, Tuple

import numpy as np
import torch

from .rttm import Turn, write_rttm
from .segmentation import powerset_mapping


@dataclass(frozen=True)
class SlidingWindow:
    """pyannote.core.SlidingWindow: frame i covers [start + i*step, start + i*step + duration)."""
    start: float
    duration: float
    step: float

    def closest_frame(self, t: float) -> int:
        return int(np.rint((t - self.start - 0.5 * self.duration) / self.step))

    def middle(self, i: int) -> float:
        return self.start + i * self.step + 0.5 * self.duration

    def frame_start(self, i: int) -> float:
        return self.start + i * self.step


def receptive_field(sample_rate: int = 16000) -> SlidingWindow:
    """PyanNet's receptive field (`Model.receptive_field`): size 991 samples, step 270 samples for SincNet stride 10,
    k = 251 followed by three MaxPool(3) and two k = 5 convolutions; no padding, so frame 0 starts at 0."""
    size, step = 1, 1
    for kernel, stride in reversed([(251, 10), (3, 3), (5, 1), (3, 3), (5, 1), (3, 3)]):
        size = (size - 1) * stride + kernel
    for _, stride in [(251, 10), (3, 3), (5, 1), (3, 3), (5, 1), (3, 3)]:
        step *= stride
    return SlidingWindow(0.0, size / sample_rate, step / sample_rate)


def chunk_starts(num_samples: int, window: int, step: int) -> Tuple[int, bool]:
    """`Inference.slide`: number of full windows and whether a zero-padded last window follows."""
    num_chunks = (num_samples - window) // step + 1 if num_samples >= window else 0
    has_last = (num_samples < window) or ((num_samples - window) % step > 0)
    return num_chunks, has_last


def aggregate(scores: np.ndarray, chunks: SlidingWindow, frames: SlidingWindow, *, epsilon: float = 1e-12,
              missing: float = np.nan, skip_average: bool = False) -> np.ndarray:
    """`Inference.aggregate` (hamming=False, no warm-up): overlap-add the per-window scores (num_chunks, frames_per_chunk,
    classes) onto the global frame grid; NaN entries do not contribute.  -> (num_frames, classes)."""
    num_chunks, per_chunk, num_classes = scores.shape
    frames = SlidingWindow(chunks.start, frames.duration, frames.step)
    masks = 1.0 - np.isnan(scores)
    data = np.nan_to_num(scores, copy=True, nan=0.0)
    num_frames = frames.closest_frame(chunks.start + chunks.duration + (num_chunks - 1) * chunks.step + 0.5 * frames.duration) + 1
    out = np.zeros((num_frames, num_classes), np.float32)
    count = np.zeros((num_frames, num_classes), np.float32)
    seen = np.zeros((num_frames, num_classes), np.float32)
    for c in range(num_chunks):
        s = frames.closest_frame(chunks.start + c * chunks.step + 0.5 * frames.duration)
        e = min(s + per_chunk, num_frames)
        n = e - s
        out[s:e] += data[c, :n] * masks[c, :n]
        count[s:e] += masks[c, :n]
        seen[s:e] = np.maximum(seen[s:e], masks[c, :n])
    avg = out if skip_average else out / np.maximum(count, epsilon)
    avg[seen == 0.0] = missing
    return avg


def condensed_euclidean(emb: np.ndarray, device: Optional[str] = None) -> np.ndarray:
    """scipy `pdist(emb)` (float64, direct differences) computed with torch on `device`: for the ~8 000 embeddings of a
    45-minute recording the pairwise distances are a large share of the clustering time on the host (not re-timed on the
    H100).
    The linkage itself stays scipy's (same dendrogram: `linkage(y)` == `linkage(X)` for Euclidean input)."""
    x = torch.from_numpy(np.ascontiguousarray(emb, dtype=np.float64)).to(device or "cpu")
    n = x.shape[0]
    d = torch.cdist(x, x, p=2.0, compute_mode="donot_use_mm_for_euclid_dist")
    iu = torch.triu_indices(n, n, offset=1, device=d.device)
    return d[iu[0], iu[1]].cpu().numpy()


def centroid_linkage(emb: np.ndarray, device, return_distances: bool = False):
    """scipy `linkage(emb, method="centroid", metric="euclidean")` on a CUDA device (csrc/diar_cluster.cu): the same Z
    bit for bit unless two candidate merge heights tie (then the smallest pair (a, b) merges first).  The n (n - 1) / 2
    pairwise distances live in device memory for the call.  `return_distances` also returns them (scipy's pdist)."""
    from .. import _lib
    lib = _lib.load()
    x = np.ascontiguousarray(emb, dtype=np.float64)
    n, dim = x.shape
    if not np.isfinite(x).all():
        raise ValueError("The condensed distance matrix must contain only finite values.")   # scipy's check
    need = int(lib.rvb_centroid_linkage_workspace_bytes(n))
    if need < 0:
        raise ValueError(f"centroid linkage needs 2 or more embeddings and a workspace that fits a counter, got n = {n}")
    device = torch.device(device)
    try:
        ws = torch.empty(need, dtype=torch.uint8, device=device)
    except torch.OutOfMemoryError as e:
        raise RuntimeError(f"centroid linkage of {n} embeddings needs {need / 2**30:.2f} GiB of device memory for the "
                           f"pairwise distances, more than {device} has free") from e
    xd = torch.from_numpy(x).to(device)
    Z = torch.empty((n - 1, 4), dtype=torch.float64, device=device)
    dist = torch.empty(n * (n - 1) // 2, dtype=torch.float64, device=device) if return_distances else None
    with torch.cuda.device(device):
        _lib.check(lib.rvb_centroid_linkage(xd.data_ptr(), n, dim, Z.data_ptr(),
                                            dist.data_ptr() if dist is not None else None, ws.data_ptr(), need,
                                            torch.cuda.current_stream(device).cuda_stream), "rvb_centroid_linkage")
        Z = Z.cpu().numpy()
    return (Z, dist.cpu().numpy()) if return_distances else Z


def agglomerative_clustering(embeddings: np.ndarray, threshold: float, min_cluster_size: int,
                             device: Optional[str] = None) -> np.ndarray:
    """`AgglomerativeClustering.cluster` (method "centroid", metric "cosine"): unit-normalise, centroid linkage on
    Euclidean distances, cut at `threshold`, then merge every small cluster (< min_cluster_size members) into the large
    cluster with the nearest centroid (cosine) and renumber from 0.  On a CUDA `device` the linkage runs on it
    (centroid_linkage); the dendrogram is scipy's."""
    from scipy.cluster.hierarchy import fcluster, linkage
    from scipy.spatial.distance import cdist
    n = embeddings.shape[0]
    min_cluster_size = min(min_cluster_size, max(1, round(0.1 * n)))
    if n == 1:
        return np.zeros((1,), np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        emb = embeddings / np.linalg.norm(embeddings, axis=-1, keepdims=True)
    if device is not None and torch.device(device).type == "cuda":
        dendrogram = centroid_linkage(emb, device)
    elif device is not None and n > 256:
        dendrogram = linkage(condensed_euclidean(emb, device), method="centroid")
    else:
        dendrogram = linkage(emb, method="centroid", metric="euclidean")
    clusters = fcluster(dendrogram, threshold, criterion="distance") - 1
    unique, counts = np.unique(clusters, return_counts=True)
    large = unique[counts >= min_cluster_size]
    if len(large) == 0:
        clusters[:] = 0
        return clusters
    small = unique[counts < min_cluster_size]
    if len(small) == 0:
        return clusters
    large_c = np.vstack([emb[clusters == k].mean(axis=0) for k in large])
    small_c = np.vstack([emb[clusters == k].mean(axis=0) for k in small])
    dist = cdist(large_c, small_c, metric="cosine")
    for small_k, large_k in enumerate(np.argmin(dist, axis=0)):
        clusters[clusters == small[small_k]] = large[large_k]
    _, clusters = np.unique(clusters, return_inverse=True)
    return clusters


def assign_embeddings(embeddings: np.ndarray, train_idx: Tuple[np.ndarray, np.ndarray], train_clusters: np.ndarray):
    """`BaseClustering.assign_embeddings` (constrained=False): centroids of the training clusters, every (window,
    local speaker) embedding goes to its nearest centroid (cosine).  -> hard (C, S), soft (C, S, K), centroids."""
    from scipy.spatial.distance import cdist
    num_clusters = int(train_clusters.max()) + 1
    C, S, D = embeddings.shape
    train = embeddings[train_idx[0], train_idx[1]]
    centroids = np.vstack([train[train_clusters == k].mean(axis=0) for k in range(num_clusters)])
    with np.errstate(invalid="ignore"):
        e2k = cdist(embeddings.reshape(C * S, D), centroids, metric="cosine").reshape(C, S, num_clusters)
    soft = 2.0 - e2k
    soft = np.nan_to_num(soft, nan=-np.inf)        # zero-norm embeddings have no cosine: never preferred
    hard = np.argmax(soft, axis=2)
    return hard, soft, centroids


def binarize(activity: np.ndarray, frames: SlidingWindow, onset: float = 0.5, offset: float = 0.5,
             min_duration_off: float = 0.0) -> List[Tuple[float, float, int]]:
    """`pyannote.audio.utils.signal.Binarize` on a (num_frames, K) activity matrix: per column, hysteresis thresholding
    with region boundaries at frame MIDDLES; regions of the same label closer than min_duration_off are merged."""
    out: List[Tuple[float, float, int]] = []
    n, K = activity.shape
    if n == 0:
        return out
    ts = frames.start + np.arange(n) * frames.step + 0.5 * frames.duration
    for k in range(K):
        col = activity[:, k]
        if onset == offset and not np.any(col == onset):
            state = col > onset                                   # no hysteresis band: the state is the comparison
        else:
            state = np.zeros(n, bool)
            active = bool(col[0] > onset)
            state[0] = active
            for i in range(1, n):
                if active:
                    if col[i] < offset:
                        active = False
                elif col[i] > onset:
                    active = True
                state[i] = active
        # a region opens at the first active frame's middle and closes at the middle of the first inactive frame after
        # it (the last frame's middle when still active at the end)
        edge = np.diff(state.astype(np.int8))
        starts = list(ts[np.nonzero(edge == 1)[0] + 1])
        ends = list(ts[np.nonzero(edge == -1)[0] + 1])
        if state[0]:
            starts.insert(0, ts[0])
        if state[-1]:
            ends.append(ts[-1])
        merged: List[List[float]] = []
        for a0, b0 in zip(starts, ends):
            if merged and min_duration_off > 0.0 and a0 - merged[-1][1] <= min_duration_off:
                merged[-1][1] = float(b0)
            else:
                merged.append([float(a0), float(b0)])
        out.extend((a0, b0, k) for a0, b0 in merged if b0 > a0)
    return out


class SpeakerDiarization:
    """`pyannote.audio.pipelines.SpeakerDiarization` with the 3.1 hyper-parameters (the reverb-diarization-v1 pipeline
    config is not available offline; these are the published defaults of the pipeline it fine-tunes)."""

    def __init__(self, segmentation: Callable, embedding: Callable, *, sample_rate: int = 16000, duration: float = 10.0,
                 step_ratio: float = 0.1, clustering_threshold: float = 0.7045654963945799, min_cluster_size: int = 12,
                 min_duration_off: float = 0.0, embedding_exclude_overlap: bool = True, max_speakers_per_chunk: int = 3,
                 max_speakers_per_frame: int = 2, batch_size: int = 32, segmentation_batch_size: Optional[int] = None,
                 embedding_min_samples: int = 400,
                 device: str = "cuda"):
        # `device` exists for the host-logic tests, which drive the glue with stub networks; the real networks are CUDA-only
        self.device = device
        self.segmentation = segmentation
        self.embedding = embedding
        self.sample_rate = sample_rate
        self.duration = duration
        self.step = step_ratio * duration
        self.threshold = clustering_threshold
        self.min_cluster_size = min_cluster_size
        self.min_duration_off = min_duration_off
        self.exclude_overlap = embedding_exclude_overlap
        self.batch_size = batch_size
        # the LSTM recurrence runs 8 windows per 2-CTA cluster and direction: 264 windows fill the 132 SMs of an H100
        self.seg_batch_size = segmentation_batch_size or max(batch_size, 264)
        self.embedding_min_samples = embedding_min_samples
        self.mapping = powerset_mapping(max_speakers_per_chunk, max_speakers_per_frame)
        # the segmentation model's own frame grid when it declares one (WavLM: 400 / 320 samples), else PyanNet's
        rf = getattr(segmentation, "receptive_field", None)
        self.frames = (SlidingWindow(0.0, rf[0] / sample_rate, rf[1] / sample_rate) if rf is not None
                       else receptive_field(sample_rate))

    # -- stage 1: local segmentation of every window (`get_segmentations` + hard powerset conversion) -----------------
    def windows(self, wave: torch.Tensor) -> torch.Tensor:
        """(N,) CUDA waveform -> (num_chunks, window) windows every `step`; the last one zero-padded (Inference.slide)."""
        window, step = int(round(self.duration * self.sample_rate)), int(round(self.step * self.sample_rate))
        n, has_last = chunk_starts(wave.shape[0], window, step)
        total = n + (1 if has_last else 0)
        need = (total - 1) * step + window
        if need > wave.shape[0]:
            wave = torch.nn.functional.pad(wave, (0, need - wave.shape[0]))
        return wave.unfold(0, window, step)[:total]

    def get_segmentations(self, chunks: torch.Tensor) -> np.ndarray:
        mapping = torch.from_numpy(self.mapping).to(chunks.device)
        out = []
        for i in range(0, chunks.shape[0], self.seg_batch_size):
            logp = self.segmentation(chunks[i:i + self.seg_batch_size].contiguous())
            out.append(mapping[logp.argmax(dim=-1)])
        return torch.cat(out).cpu().numpy()                       # (num_chunks, frames, local speakers) in {0, 1}

    # -- stage 2: instantaneous speaker count (`speaker_count`) --------------------------------------------------------
    def speaker_count(self, binarized: np.ndarray, chunks: SlidingWindow) -> np.ndarray:
        count = aggregate(binarized.sum(axis=-1, keepdims=True), chunks, self.frames, missing=0.0)
        return np.rint(count).astype(np.uint8)                    # (num_frames, 1)

    # -- stage 3: one embedding per (window, local speaker) (`get_embeddings`) -----------------------------------------
    def get_embeddings(self, chunks: torch.Tensor, binarized: np.ndarray) -> np.ndarray:
        num_chunks, num_frames, S = binarized.shape
        masks = binarized.astype(np.float32)
        if self.exclude_overlap:
            window = chunks.shape[1]
            min_frames = math.ceil(num_frames * self.embedding_min_samples / window)
            clean = masks * (masks.sum(axis=2, keepdims=True) < 2)
            use_clean = clean.sum(axis=1) > min_frames            # (num_chunks, S)
            masks = np.where(use_clean[:, None, :], clean, masks)
        weights = torch.from_numpy(np.ascontiguousarray(masks.transpose(0, 2, 1))).to(chunks.device)   # (C, S, frames)
        out = []
        for i in range(0, num_chunks, self.batch_size):
            out.append(self.embedding(chunks[i:i + self.batch_size].contiguous(), weights[i:i + self.batch_size].contiguous()))
        return torch.cat(out).cpu().numpy()                       # (num_chunks, S, dim)

    # -- stage 4: global clustering (`AgglomerativeClustering.__call__`) ----------------------------------------------
    def cluster(self, embeddings: np.ndarray, binarized: np.ndarray, min_active_ratio: float = 0.2):
        num_chunks, num_frames, S = binarized.shape
        active = binarized.sum(axis=1) > min_active_ratio * num_frames
        valid = ~np.any(np.isnan(embeddings), axis=2)
        chunk_idx, speaker_idx = np.where(active & valid)
        if len(chunk_idx) < 2:
            hard = np.zeros((num_chunks, S), np.int64)
            return hard, None
        train = embeddings[chunk_idx, speaker_idx].astype(np.float64)
        train_clusters = agglomerative_clustering(train, self.threshold, self.min_cluster_size,
                                                  device=self.device if self.device != "cpu" else None)
        hard, soft, centroids = assign_embeddings(embeddings.astype(np.float64), (chunk_idx, speaker_idx), train_clusters)
        return hard, centroids

    # -- stage 5: reconstruction (`reconstruct` + `to_diarization`) -----------------------------------------------------
    def reconstruct(self, binarized: np.ndarray, hard: np.ndarray, count: np.ndarray, chunks: SlidingWindow) -> np.ndarray:
        num_chunks, num_frames, S = binarized.shape
        K = int(hard.max()) + 1
        clustered = np.full((num_chunks, num_frames, K), np.nan, np.float32)
        for c in range(num_chunks):
            for k in np.unique(hard[c]):
                if k < 0:
                    continue                                       # -2 marks an inactive local speaker
                clustered[c, :, k] = binarized[c][:, hard[c] == k].max(axis=1)
        activations = aggregate(clustered, chunks, self.frames, missing=0.0, skip_average=True)
        max_per_frame = int(count.max()) if count.size else 0
        if activations.shape[1] < max_per_frame:
            activations = np.pad(activations, ((0, 0), (0, max_per_frame - activations.shape[1])))
        n = min(activations.shape[0], count.shape[0])
        activations, count = activations[:n], count[:n]
        # per frame, the count[t] most active clusters speak (ties: lower index first, like a stable argsort)
        order = np.argsort(-activations, axis=-1, kind="stable")
        rank = np.empty_like(order)
        np.put_along_axis(rank, order, np.broadcast_to(np.arange(order.shape[1]), order.shape), axis=1)
        return (rank < count[:, :1].astype(np.int64)).astype(np.float32)

    # -- the call ------------------------------------------------------------------------------------------------------
    def apply(self, wave) -> List[Turn]:
        """wave: (N,) float waveform in [-1, 1] (numpy or torch) -> speaker turns (SPEAKER_00, SPEAKER_01, ...)."""
        if not torch.is_tensor(wave):
            wave = torch.from_numpy(np.asarray(wave, np.float32))
        wave = wave.to(device=self.device, dtype=torch.float32).flatten()
        import time
        sync = torch.cuda.synchronize if wave.is_cuda else (lambda: None)
        tm = {}
        t0 = time.perf_counter()
        chunks = self.windows(wave)
        window = SlidingWindow(0.0, self.duration, self.step)
        binarized = self.get_segmentations(chunks)
        sync()
        tm["segmentation"] = time.perf_counter() - t0
        count = self.speaker_count(binarized, window)
        if int(count.max()) == 0:
            self.last = dict(binarized=binarized, count=count, timing=tm)
            return []
        t1 = time.perf_counter()
        embeddings = self.get_embeddings(chunks, binarized)
        sync()
        tm["embedding"] = time.perf_counter() - t1
        t1 = time.perf_counter()
        hard, _ = self.cluster(embeddings, binarized)
        tm["clustering"] = time.perf_counter() - t1
        t1 = time.perf_counter()
        count = np.minimum(count, binarized.shape[2]).astype(np.int8)
        hard = hard.copy()
        hard[binarized.sum(axis=1) == 0] = -2
        discrete = self.reconstruct(binarized, hard, count, window)
        frames = SlidingWindow(0.0, self.frames.duration, self.frames.step)
        regions = binarize(discrete, frames, min_duration_off=self.min_duration_off)
        labels = sorted({k for _, _, k in regions})
        names = {k: f"SPEAKER_{i:02d}" for i, k in enumerate(labels)}
        turns = [Turn(a, b, names[k]) for a, b, k in regions]
        turns.sort(key=lambda t: (t.start, t.end))
        tm["reconstruction"] = time.perf_counter() - t1
        tm["total"] = time.perf_counter() - t0
        self.last = dict(binarized=binarized, count=count, embeddings=embeddings, hard=hard, discrete=discrete, timing=tm)
        return turns

    __call__ = apply

    def write_rttm(self, f, uri: str, turns: List[Turn]) -> None:
        write_rttm(f, uri, turns)
