// reverb_b200 — compressed WAV decoding on the GPU: G.711 µ-law / A-law and IMA / Microsoft ADPCM, over the data
// chunk uploaded once (DESIGN.md §4l).
//
//   g711_kernel   one thread per 4 input bytes: a per-byte expansion to int16, stored planar
//   ima_kernel    one thread per (block, channel): predictor and step index from the block header, then the IMA
//                 shift-add recurrence over 4-byte groups of 8 nibbles (low nibble first)
//   ms_kernel     one thread per (block, channel): predictor index, delta and two samples from the block header, then
//                 the two-tap prediction with adaptive delta (high nibble first; in stereo high = channel 0)
// The host validates the fmt chunk and the frame count; the kernels still never read outside their block or the data
// span, and never write past `frames`.  An invalid header (IMA step index > 88, MS predictor index >= n_coef) is packed
// into one 64-bit word as (block << 8) | status and kept by atomicMin, so the lowest failing block is reported.
#include <algorithm>
#include <climits>
#include <cstring>

#include "host_mem.h"
#include "../../include/rvb_b200.h"

namespace rvb {
// a named namespace, so the kernels' symbol names (torch.profiler rows) are the same in every build
namespace wav_codec {

enum { kTagMsAdpcm = 0x0002, kTagAlaw = 0x0006, kTagMulaw = 0x0007, kTagImaAdpcm = 0x0011 };
enum { kOk = 0, kBadStepIndex = 1, kBadPredictor = 2 };
constexpr unsigned long long kNoError = ~0ull;

__device__ __forceinline__ int ulaw_sample(unsigned b) {
  const unsigned x = ~b & 0xFF;
  const int mag = (int)(((((x & 15) << 3) + 0x84) << ((x >> 4) & 7)) - 0x84);
  return (x & 0x80) ? -mag : mag;
}

__device__ __forceinline__ int alaw_sample(unsigned b) {
  const unsigned x = b ^ 0x55;
  const unsigned m = x & 15, e = (x >> 4) & 7;
  const int mag = (int)(e == 0 ? (m << 4) + 8 : ((m << 4) + 0x108) << (e - 1));
  return (x & 0x80) ? mag : -mag;
}

__device__ __forceinline__ int rd16(const uint8_t* p) { return (short)(__ldg(p) | (__ldg(p + 1) << 8)); }

__device__ __forceinline__ void report(unsigned long long* err, long long block, int status) {
  atomicMin(err, ((unsigned long long)block << 8) | (unsigned)status);
}

// bytes [4t, 4t + 4) of the interleaved data; sample i is frame i / nch of channel i % nch
__global__ void __launch_bounds__(256)
g711_kernel(const uint8_t* __restrict__ b, int nch, long long frames, int alaw, short* __restrict__ out) {
  const long long total = frames * nch;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; 4 * t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const long long i0 = 4 * t;
    long long f = i0 / nch;
    int c = (int)(i0 - f * nch);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (i0 + j >= total) break;
      const unsigned v = __ldg(b + i0 + j);
      out[(size_t)c * frames + f] = (short)(alaw ? alaw_sample(v) : ulaw_sample(v));
      if (++c == nch) c = 0, ++f;
    }
  }
}

__constant__ short kImaStep[89] = {
    7,     8,     9,     10,    11,    12,    13,    14,    16,    17,    19,    21,    23,    25,    28,
    31,    34,    37,    41,    45,    50,    55,    60,    66,    73,    80,    88,    97,    107,   118,
    130,   143,   157,   173,   190,   209,   230,   253,   279,   307,   337,   371,   408,   449,   494,
    544,   598,   658,   724,   796,   876,   963,   1060,  1166,  1282,  1411,  1552,  1707,  1878,  2066,
    2272,  2499,  2749,  3024,  3327,  3660,  4026,  4428,  4871,  5358,  5894,  6484,  7132,  7845,  8630,
    9493,  10442, 11487, 12635, 13899, 15289, 16818, 18500, 20350, 22385, 24623, 27086, 29794, 32767};

// one thread per (block, channel); a unit past the last block holding output frames does nothing
__global__ void __launch_bounds__(128)
ima_kernel(const uint8_t* __restrict__ b, long long n_bytes, int nch, int block_align, int spb, long long frames,
           long long n_units, short* __restrict__ out, unsigned long long* __restrict__ err) {
  __shared__ int step_tab[89];  // divergent step indices: a shared-memory lookup, not a serialised constant read
  for (int i = threadIdx.x; i < 89; i += blockDim.x) step_tab[i] = kImaStep[i];
  __syncthreads();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_units) return;
  const long long blk = t / nch;
  const int c = (int)(t - blk * nch);
  const long long base = blk * block_align;
  const long long avail = min((long long)block_align, n_bytes - base);
  const int hdr = 4 * nch;
  if (avail < hdr) return;  // unreachable for a frame count the bytes hold
  const uint8_t* p = b + base;
  int pred = rd16(p + 4 * c);
  int idx = __ldg(p + 4 * c + 2);
  if (idx > 88) {
    report(err, blk, kBadStepIndex);
    return;
  }
  const long long f0 = blk * spb;
  short* o = out + (size_t)c * frames + f0;
  const int n_out = (int)min((long long)spb, frames - f0);
  o[0] = (short)pred;
  const int groups = (int)min((long long)(n_out + 6) / 8, (avail - hdr) / hdr);
  for (int g = 0; g < groups; ++g) {
    const uint8_t* q = p + (size_t)hdr * (1 + g) + 4 * c;
    const unsigned w = __ldg(q) | (__ldg(q + 1) << 8) | (__ldg(q + 2) << 16) | ((unsigned)__ldg(q + 3) << 24);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int nib = (w >> (4 * k)) & 15;
      const int step = step_tab[idx];
      int diff = step >> 3;
      if (nib & 4) diff += step;
      if (nib & 2) diff += step >> 1;
      if (nib & 1) diff += step >> 2;
      pred = (nib & 8) ? pred - diff : pred + diff;
      pred = max(-32768, min(32767, pred));
      idx += (nib & 4) ? 2 * (nib & 3) + 2 : -1;
      idx = max(0, min(88, idx));
      const int s = 1 + 8 * g + k;
      if (s < n_out) o[s] = (short)pred;
    }
  }
}

__constant__ short kMsAdapt[16] = {230, 230, 230, 230, 307, 409, 512, 614, 768, 614, 512, 409, 307, 230, 230, 230};

struct MsCoefs {
  short c[512];  // n_coef pairs (c1, c2)
};

__global__ void __launch_bounds__(128)
ms_kernel(const uint8_t* __restrict__ b, long long n_bytes, int nch, int block_align, int spb, int n_coef,
          const MsCoefs coefs, long long frames, long long n_units, short* __restrict__ out,
          unsigned long long* __restrict__ err) {
  __shared__ int adapt_tab[16];
  if (threadIdx.x < 16) adapt_tab[threadIdx.x] = kMsAdapt[threadIdx.x];
  __syncthreads();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_units) return;
  const long long blk = t / nch;
  const int c = (int)(t - blk * nch);
  const long long base = blk * block_align;
  const long long avail = min((long long)block_align, n_bytes - base);
  const int hdr = 7 * nch;
  if (avail < hdr) return;  // unreachable for a frame count the bytes hold
  const uint8_t* p = b + base;
  const int pi = __ldg(p + c);
  if (pi >= n_coef) {
    report(err, blk, kBadPredictor);
    return;
  }
  const int c1 = coefs.c[2 * pi], c2 = coefs.c[2 * pi + 1];
  int delta = rd16(p + nch + 2 * c);
  int s1 = rd16(p + 3 * nch + 2 * c), s2 = rd16(p + 5 * nch + 2 * c);
  const long long f0 = blk * spb;
  short* o = out + (size_t)c * frames + f0;
  const int n_out = (int)min(min((long long)spb, frames - f0), 2 + (avail - hdr) * 2 / nch);
  o[0] = (short)s2;
  if (n_out > 1) o[1] = (short)s1;
  for (int s = 2; s < n_out; ++s) {
    const int k = (s - 2) * nch + c;  // nibble index in the block's data, high nibble of each byte first
    const int byte = __ldg(p + hdr + (k >> 1));
    const int nib = (k & 1) ? byte & 15 : byte >> 4;
    // C division truncates toward zero; an arithmetic >> 8 would round negative predictions down
    const int pred = (int)(((long long)s1 * c1 + (long long)s2 * c2) / 256);
    const int v = max(-32768, min(32767, pred + ((nib ^ 8) - 8) * delta));
    delta = max(16, (adapt_tab[nib] * delta) >> 8);
    delta = min(delta, INT_MAX / 768);  // keeps adapt * delta inside int for any input
    s2 = s1;
    s1 = v;
    o[s] = (short)v;
  }
}

bool codec_ok(const rvb_wav_codec& w) {
  const int ch = w.channels, ba = w.block_align, spb = w.samples_per_block;
  switch (w.format_tag) {
    case kTagMulaw:
    case kTagAlaw:
      return ch >= 1 && ba == ch;
    case kTagImaAdpcm:
      return ch >= 1 && spb >= 1 && (spb - 1) % 8 == 0 && (long long)ba == 4LL * ch * (1 + (spb - 1) / 8);
    case kTagMsAdpcm:
      return (ch == 1 || ch == 2) && ba >= 7 * ch && w.n_coef >= 7 && w.n_coef <= 256 &&
             spb == 2 + (ba - 7 * ch) * 2 / ch;
    default:
      return false;
  }
}

// frames per channel the data span holds: full blocks, then what a trailing partial block with a whole header holds
long long frame_capacity(const rvb_wav_codec& w, long long n_bytes) {
  const int ch = w.channels;
  if (w.format_tag == kTagMulaw || w.format_tag == kTagAlaw) return n_bytes / ch;
  const long long full = n_bytes / w.block_align, rem = n_bytes % w.block_align;
  long long part = 0;
  if (w.format_tag == kTagImaAdpcm && rem >= 4 * ch) part = 1 + 8 * ((rem - 4 * ch) / (4 * ch));
  if (w.format_tag == kTagMsAdpcm && rem >= 7 * ch) part = 2 + (rem - 7 * ch) * 2 / ch;
  return full * w.samples_per_block + part;
}

static thread_local HostPinned g_wav_pin;

}  // namespace wav_codec
}  // namespace rvb

RVB_API int rvb_wav_decode(const void* d_data, long long n_bytes, const rvb_wav_codec* info, long long frames,
                           void* d_out, int* h_bad_block, int* h_bad_status, void* stream_) {
  using namespace rvb;
  using namespace rvb::wav_codec;
  RVB_REQUIRE(d_data && d_out && info && h_bad_block && h_bad_status && n_bytes >= 0 && frames >= 1,
              "rvb_wav_decode: bad arguments");
  RVB_REQUIRE(codec_ok(*info),
              "rvb_wav_decode: invalid codec (format tag 0x%04x, %d channels, block_align %d, %d samples per block, "
              "%d coefficient pairs)",
              info->format_tag, info->channels, info->block_align, info->samples_per_block, info->n_coef);
  const long long cap = frame_capacity(*info, n_bytes);
  RVB_REQUIRE(frames <= cap, "rvb_wav_decode: %lld frames requested, the %lld bytes hold %lld", frames, n_bytes, cap);
  cudaStream_t stream = (cudaStream_t)stream_;
  const uint8_t* b = static_cast<const uint8_t*>(d_data);
  short* out = static_cast<short*>(d_out);
  const int nch = info->channels;
  *h_bad_block = -1;
  *h_bad_status = 0;
  if (info->format_tag == kTagMulaw || info->format_tag == kTagAlaw) {
    const long long quads = (frames * nch + 3) / 4;
    const unsigned grid = (unsigned)std::min<long long>((quads + 255) / 256, 132 * 32);
    g711_kernel<<<grid, 256, 0, stream>>>(b, nch, frames, info->format_tag == kTagAlaw, out);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
    RVB_CHECK_CUDA(cudaStreamSynchronize(stream));
    return 0;
  }
  const int spb = info->samples_per_block;
  const long long n_units = (frames + spb - 1) / spb * nch;
  const unsigned grid = (unsigned)((n_units + 127) / 128);
  unsigned long long* err = nullptr;  // stream-ordered, so it lives on the stream's device
  RVB_CHECK_CUDA(cudaMallocAsync((void**)&err, sizeof(unsigned long long), stream));
  RVB_CHECK_CUDA(cudaMemsetAsync(err, 0xFF, sizeof(unsigned long long), stream));
  if (info->format_tag == kTagImaAdpcm) {
    ima_kernel<<<grid, 128, 0, stream>>>(b, n_bytes, nch, info->block_align, spb, frames, n_units, out, err);
  } else {
    MsCoefs coefs;
    memcpy(coefs.c, info->coef, sizeof(coefs.c));
    ms_kernel<<<grid, 128, 0, stream>>>(b, n_bytes, nch, info->block_align, spb, info->n_coef, coefs, frames, n_units,
                                        out, err);
  }
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  if (g_wav_pin.ensure(sizeof(unsigned long long))) return -1;
  unsigned long long* h_err = g_wav_pin.as<unsigned long long>();
  RVB_CHECK_CUDA(cudaMemcpyAsync(h_err, err, sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
  RVB_CHECK_CUDA(cudaFreeAsync(err, stream));
  RVB_CHECK_CUDA(cudaStreamSynchronize(stream));
  if (*h_err != kNoError) {
    *h_bad_block = (int)(*h_err >> 8);
    *h_bad_status = (int)(*h_err & 0xFF);
  }
  return 0;
}
