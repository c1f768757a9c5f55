/* rvb_diar.h — C ABI of the diarization forward in librvb_b200.so (SURVEY.md §8f rank 1).
 *
 * The reference runs the two networks below through `pyannote.audio==3.3.1`
 * (reference: diarization/infer_pyannote3.0.py:14,33-40: `Pipeline.from_pretrained(...)`, `pipeline(audio)`;
 * requirements.txt:1).  There is no FFI in the reference for this path; these are the entry points a binding of
 * `pyannote.audio.Model.__call__` for the segmentation / embedding models would replace:
 *
 *   rvb_seg_*  PyanNet segmentation: waveform windows -> per-frame log-probabilities over the powerset classes
 *   rvb_emb_*  WeSpeaker ResNet34 speaker embedding: waveform windows (+ per-frame weights) -> 256-d vectors
 *
 * ** parity unpinned **: pyannote's source and the model weights are not available offline (SURVEY.md §8c-iii); the
 * architecture follows the upstream project's published description (oracle/diar_ref.py states what is assumed).
 *
 * Conventions as in rvb_b200.h: return 0 on success, negative on error (rvb_last_error()); d_* pointers are device
 * memory owned by the caller; work is enqueued on `stream`; models are owned by the library (create / destroy).
 */
#ifndef RVB_DIAR_H_
#define RVB_DIAR_H_

#include "rvb_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct rvb_seg_model rvb_seg_model;

typedef struct rvb_seg_config {
  int sample_rate;    /* 16000 */
  int sinc_filters;   /* 80 = 40 cosine + 40 sine band-pass filters (ParamSincFB) */
  int sinc_kernel;    /* 251 */
  int sinc_stride;    /* 10 */
  int conv_channels;  /* 60 (Conv1d(80,60,5), Conv1d(60,60,5)) */
  int conv_kernel;    /* 5 */
  int lstm_hidden;    /* 128, bidirectional */
  int lstm_layers;    /* 4 */
  int linear_dim;     /* 128 */
  int linear_layers;  /* 2 */
  int num_classes;    /* 7 powerset classes (<= 3 speakers, <= 2 at once) */
} rvb_seg_config;

RVB_API rvb_seg_model* rvb_seg_create(const rvb_seg_config* cfg);
/* fp32 host tensors under pyannote's state_dict names: sincnet.wav_norm1d.{weight,bias},
 * sincnet.conv1d.0.filterbank.{low_hz_,band_hz_}, sincnet.norm1d.{0,1,2}.{weight,bias}, sincnet.conv1d.{1,2}.{weight,bias},
 * lstm.{weight_ih,weight_hh,bias_ih,bias_hh}_l{k}[_reverse], linear.{i}.{weight,bias}, classifier.{weight,bias} */
RVB_API int rvb_seg_set_tensor(rvb_seg_model* m, const char* name, const float* host, long long count);
RVB_API int rvb_seg_finalize(rvb_seg_model* m);
RVB_API void rvb_seg_destroy(rvb_seg_model* m);
/* output frames for a window of num_samples (160000 -> 589) */
RVB_API int rvb_seg_num_frames(const rvb_seg_model* m, int num_samples);
/* d_wave (B, num_samples) fp32 -> d_logp (B, frames, num_classes) fp32 log-probabilities.
 * d_sincnet (optional, B x frames x conv_channels): the SincNet output, for staged parity tests. */
RVB_API int rvb_seg_forward(rvb_seg_model* m, const float* d_wave, int B, int num_samples, float* d_logp,
                            float* d_sincnet, void* stream);

/* ---- WeSpeaker ResNet34 speaker embedding ------------------------------------------------------------------------
 * waveform window in [-1, 1] -> x 2^15 -> Kaldi fbank (80 mel, hamming window, 25 / 10 ms, no dither) -> minus the mean
 * over time -> ResNet34 (BasicBlock [3, 4, 6, 3], m_channels .. 8 m_channels, BatchNorm folded, ReLU) -> weighted
 * statistics pooling (mean, std over time per (channel, frequency)) -> Linear(embed_dim).
 * The trunk runs ONCE per window; the S weight rows of a window (the local speakers' activity masks, nearest-
 * interpolated to the trunk's frame rate like pyannote's StatsPool) only change the pooling. */
typedef struct rvb_emb_model rvb_emb_model;

typedef struct rvb_emb_config {
  int sample_rate;   /* 16000 */
  int num_mel_bins;  /* 80 */
  int m_channels;    /* 32 */
  int embed_dim;     /* 256 */
  int blocks[4];     /* 3, 4, 6, 3 */
} rvb_emb_config;

RVB_API rvb_emb_model* rvb_emb_create(const rvb_emb_config* cfg);
/* fp32 host tensors under pyannote's state_dict names: resnet.conv1.weight, resnet.bn1.{weight,bias,running_mean,
 * running_var}, resnet.layer{1..4}.{i}.{conv1,conv2}.weight, .bn{1,2}.*, .shortcut.0.weight, .shortcut.1.*,
 * resnet.seg_1.{weight,bias} */
RVB_API int rvb_emb_set_tensor(rvb_emb_model* m, const char* name, const float* host, long long count);
RVB_API int rvb_emb_finalize(rvb_emb_model* m);
RVB_API void rvb_emb_destroy(rvb_emb_model* m);
/* fbank frames of a window (160000 samples -> 998) */
RVB_API int rvb_emb_num_frames(const rvb_emb_model* m, int num_samples);
/* d_wave (B, num_samples) fp32 in [-1, 1]; d_weights (B, S, Tw) fp32 pooling weights or NULL (S = 1, unweighted);
 * d_emb (B, S, embed_dim) fp32.  d_fbank (optional, B x frames x num_mel_bins): the mean-normalised features. */
RVB_API int rvb_emb_forward(rvb_emb_model* m, const float* d_wave, int B, int num_samples, const float* d_weights, int S,
                            int Tw, float* d_emb, float* d_fbank, void* stream);

/* ---- centroid-linkage agglomerative clustering ---------------------------------------------------------------------
 * scipy.cluster.hierarchy.linkage(emb, method="centroid", metric="euclidean") on the device: the same Z, bit for bit,
 * whenever no two candidate merge heights tie.  Ties go to the smallest height, then the smallest slot pair (a, b)
 * (scipy's heap may choose differently there).  Z rows come in merge order, unsorted (centroid linkage has inversions).
 * The condensed distance matrix, n (n - 1) / 2 doubles, lives in the caller's workspace; nothing else bounds n. */
/* bytes of workspace for n embeddings; -1 when n < 2 or n is beyond any device */
RVB_API long long rvb_centroid_linkage_workspace_bytes(int n);
/* d_emb (n, dim) fp64, unit-normalised; d_Z (n - 1, 4) fp64 (cluster, cluster, height, size).  d_dist (optional,
 * n (n - 1) / 2 fp64): the pairwise distances in scipy's pdist order, before any merge. */
RVB_API int rvb_centroid_linkage(const double* d_emb, int n, int dim, double* d_Z, double* d_dist, void* d_workspace,
                                 long long workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RVB_DIAR_H_ */
