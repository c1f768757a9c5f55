// reverb_b200 — Kaldi-compatible 80-bin log-mel filterbank, one fused kernel (sm_90a).
//
// Replaces `torchaudio.compliance.kaldi.fbank(waveform, num_mel_bins=80, frame_length=25, frame_shift=10,
// dither=0.0, energy_floor=0.0, sample_frequency=16000)` as called by the reference at
// asr/wenet/cli/reverb.py:130-138 (torchaudio kaldi.py:514-645): snip_edges framing (400/160), per-frame DC removal,
// pre-emphasis 0.97 (replicate-left), povey window, zero-pad to 512, |rFFT|^2, 80 triangular mel bins
// (20 Hz .. 8 kHz, mel domain), log(max(., eps)).  Input samples are int16-VALUED (not normalised).
//
// One warp per frame (4 consecutive frames per warp, 8 warps per CTA): the frame lives in shared memory / registers from
// load to mel; the 512-point real FFT is a register-resident 8 x 8 x 4 complex FFT of the packed frame (see
// fbank_kernel).  HBM traffic = 4 B/sample in (2 B for the int16 entry point) + 320 B/frame out; everything else is
// on chip.
#include <math.h>

#include <mutex>
#include <vector>

#include "kernels.h"

namespace rvb {

constexpr int FB_WIN = 400, FB_SHIFT = 160, FB_NFFT = 512, FB_NBIN = 80, FB_MAXW = 64;
constexpr int FB_WARPS = 8;

struct FbankTables {
  float* window = nullptr;   // [400] povey
  float* window_hamming = nullptr;   // [400] hamming (WeSpeaker embedding front-end, diar_emb.cu)
  float2* twiddle = nullptr; // [256] (cos, -sin)(2 pi k / 512)
  float2* tw256 = nullptr;   // [256] (cos, -sin)(2 pi j / 256)
  float* mel_w = nullptr;    // [80][FB_MAXW]
  int* mel_start = nullptr;  // [80]
  int* mel_len = nullptr;    // [80]
};
// one table set per device (a process may hold models on several GPUs); entries are written once under the mutex
constexpr int FB_MAXDEV = 64;
static FbankTables g_fb_dev[FB_MAXDEV];
static std::mutex g_fb_mutex;

static int init_fbank_tables(const FbankTables** out) {
  std::lock_guard<std::mutex> lock(g_fb_mutex);
  int dev = 0;
  RVB_CHECK_CUDA(cudaGetDevice(&dev));
  RVB_REQUIRE(dev >= 0 && dev < FB_MAXDEV, "fbank: device index %d out of range", dev);
  *out = &g_fb_dev[dev];
  if (g_fb_dev[dev].window != nullptr) return 0;
  FbankTables g_fb;  // published to g_fb_dev[dev] only when complete
  std::vector<float> win(FB_WIN);
  for (int i = 0; i < FB_WIN; ++i) {
    double h = 0.5 - 0.5 * cos(2.0 * M_PI * i / (FB_WIN - 1));
    win[i] = (float)pow(h, 0.85);
  }
  std::vector<float> win_h(FB_WIN);
  for (int i = 0; i < FB_WIN; ++i) win_h[i] = (float)(0.54 - 0.46 * cos(2.0 * M_PI * i / (FB_WIN - 1)));
  std::vector<float2> tw(FB_NFFT / 2);
  for (int k = 0; k < FB_NFFT / 2; ++k) {
    double a = 2.0 * M_PI * k / FB_NFFT;
    tw[k] = make_float2((float)cos(a), (float)(-sin(a)));
  }
  std::vector<float2> tw2(FB_NFFT / 2);
  for (int k = 0; k < FB_NFFT / 2; ++k) {
    double a = 2.0 * M_PI * k / (FB_NFFT / 2);
    tw2[k] = make_float2((float)cos(a), (float)(-sin(a)));
  }
  // mel banks, float32 arithmetic like torchaudio's get_mel_banks (kaldi.py:436-510)
  const float low = 20.0f, high = 8000.0f, bin_width = 16000.0f / FB_NFFT;
  const float mlow = 1127.0f * logf(1.0f + low / 700.0f), mhigh = 1127.0f * logf(1.0f + high / 700.0f);
  const float delta = (mhigh - mlow) / (FB_NBIN + 1);
  std::vector<float> w(FB_NBIN * FB_MAXW, 0.f);
  std::vector<int> st(FB_NBIN, 0), ln(FB_NBIN, 0);
  for (int b = 0; b < FB_NBIN; ++b) {
    const float left = mlow + b * delta, center = mlow + (b + 1.0f) * delta, right = mlow + (b + 2.0f) * delta;
    int first = -1, last = -1;
    std::vector<float> row(FB_NFFT / 2, 0.f);
    for (int k = 0; k < FB_NFFT / 2; ++k) {  // Nyquist bin (256) has weight 0 (kaldi.py:627)
      float mel = 1127.0f * logf(1.0f + (bin_width * k) / 700.0f);
      float up = (mel - left) / (center - left), down = (right - mel) / (right - center);
      float v = fmaxf(0.0f, fminf(up, down));
      row[k] = v;
      if (v > 0.f) {
        if (first < 0) first = k;
        last = k;
      }
    }
    if (first < 0) { first = 0; last = -1; }
    RVB_REQUIRE(last - first + 1 <= FB_MAXW, "fbank: mel bin %d too wide", b);
    st[b] = first;
    ln[b] = last - first + 1;
    for (int k = first; k <= last; ++k) w[b * FB_MAXW + (k - first)] = row[k];
  }
  RVB_CHECK_CUDA(cudaMalloc(&g_fb.window, sizeof(float) * FB_WIN));
  RVB_CHECK_CUDA(cudaMalloc(&g_fb.window_hamming, sizeof(float) * FB_WIN));
  RVB_CHECK_CUDA(cudaMemcpy(g_fb.window_hamming, win_h.data(), sizeof(float) * FB_WIN, cudaMemcpyHostToDevice));
  RVB_CHECK_CUDA(cudaMalloc(&g_fb.twiddle, sizeof(float2) * FB_NFFT / 2));
  RVB_CHECK_CUDA(cudaMalloc(&g_fb.tw256, sizeof(float2) * FB_NFFT / 2));
  RVB_CHECK_CUDA(cudaMemcpy(g_fb.tw256, tw2.data(), sizeof(float2) * FB_NFFT / 2, cudaMemcpyHostToDevice));
  RVB_CHECK_CUDA(cudaMalloc(&g_fb.mel_w, sizeof(float) * FB_NBIN * FB_MAXW));
  RVB_CHECK_CUDA(cudaMalloc(&g_fb.mel_start, sizeof(int) * FB_NBIN));
  RVB_CHECK_CUDA(cudaMalloc(&g_fb.mel_len, sizeof(int) * FB_NBIN));
  RVB_CHECK_CUDA(cudaMemcpy(g_fb.window, win.data(), sizeof(float) * FB_WIN, cudaMemcpyHostToDevice));
  RVB_CHECK_CUDA(cudaMemcpy(g_fb.twiddle, tw.data(), sizeof(float2) * FB_NFFT / 2, cudaMemcpyHostToDevice));
  RVB_CHECK_CUDA(cudaMemcpy(g_fb.mel_w, w.data(), sizeof(float) * FB_NBIN * FB_MAXW, cudaMemcpyHostToDevice));
  RVB_CHECK_CUDA(cudaMemcpy(g_fb.mel_start, st.data(), sizeof(int) * FB_NBIN, cudaMemcpyHostToDevice));
  RVB_CHECK_CUDA(cudaMemcpy(g_fb.mel_len, ln.data(), sizeof(int) * FB_NBIN, cudaMemcpyHostToDevice));
  g_fb_dev[dev] = g_fb;
  return 0;
}

__device__ __forceinline__ float ld_sample(const float* p, long long i) { return p[i]; }
__device__ __forceinline__ float ld_sample(const short* p, long long i) { return (float)p[i]; }

// ---- small complex helpers -------------------------------------------------------------------------------------
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cmul(float2 a, float2 w) { return make_float2(a.x * w.x - a.y * w.y, a.x * w.y + a.y * w.x); }
__device__ __forceinline__ float2 mul_negi(float2 a) { return make_float2(a.y, -a.x); }  // a * (-i)

// forward 4-point DFT (W4 = -i), natural order in and out
__device__ __forceinline__ void dft4(float2 x0, float2 x1, float2 x2, float2 x3, float2& y0, float2& y1, float2& y2,
                                     float2& y3) {
  const float2 e0 = cadd(x0, x2), e1 = csub(x0, x2), o0 = cadd(x1, x3), o1 = csub(x1, x3);
  y0 = cadd(e0, o0);
  y2 = csub(e0, o0);
  y1 = make_float2(e1.x + o1.y, e1.y - o1.x);  // e1 - i o1
  y3 = make_float2(e1.x - o1.y, e1.y + o1.x);  // e1 + i o1
}

// forward 8-point DFT in registers (radix-2 split into two 4-point DFTs), natural order in and out
__device__ __forceinline__ void dft8(float2* a) {
  float2 e[4], o[4];
  dft4(a[0], a[2], a[4], a[6], e[0], e[1], e[2], e[3]);
  dft4(a[1], a[3], a[5], a[7], o[0], o[1], o[2], o[3]);
  const float h = 0.70710678118654752f;
  const float2 t0 = o[0];
  const float2 t1 = make_float2(h * (o[1].x + o[1].y), h * (o[1].y - o[1].x));    // o1 * W8^1
  const float2 t2 = mul_negi(o[2]);                                                 // o2 * W8^2
  const float2 t3 = make_float2(h * (o[3].y - o[3].x), -h * (o[3].x + o[3].y));   // o3 * W8^3
  a[0] = cadd(e[0], t0);
  a[4] = csub(e[0], t0);
  a[1] = cadd(e[1], t1);
  a[5] = csub(e[1], t1);
  a[2] = cadd(e[2], t2);
  a[6] = csub(e[2], t2);
  a[3] = cadd(e[3], t3);
  a[7] = csub(e[3], t3);
}

// One warp per frame, FB_FPW consecutive frames per warp.  The 512-point REAL FFT of the windowed frame is computed as
// a 256-point complex FFT of z[m] = y[2m] + i y[2m+1] followed by the real-FFT unpacking — and the 256-point FFT
// itself is 8 x 8 x 4 (Cooley-Tukey): two 8-point DFTs in REGISTERS per lane with one shared-memory exchange between
// them (conflict-free padded layout), the last radix-4 step across the 4 neighbouring lanes with shuffles.  Per frame and lane:
// 16 + 16 shared-memory accesses for the FFT instead of the 360 of a radix-2 shared-memory FFT on the full 512
// complex points.
//   n = 32 n1 + n2, k = k1 + 8 k2:   Z[k1 + 8 k2] = sum_n2 W256^(n2 k1) W32^(n2 k2) [ sum_n1 z[32 n1 + n2] W8^(n1 k1) ]
//   n2 = 4 a + b,   k2 = c + 8 d:    (32-point)   = sum_b W32^(b c) W4^(b d)   [ sum_a  y[4 a + b]     W8^(a c)  ]
constexpr int FB_FPW = 4;      // frames per warp
constexpr int FB_YS = 36;      // row stride of the exchange buffer: bank = 4 k1 + b (+ 4 a): conflict-free both ways
__device__ __forceinline__ int zidx(int k) { return k + 8 * (k >> 6); }  // conflict-free layout of the spectrum Z[0..255]

template <typename TIn>
__global__ void __launch_bounds__(FB_WARPS * 32)
fbank_kernel(const TIn* __restrict__ wave_all, long long wave_stride, long long n_frames, float* __restrict__ feats_all,
             const float* __restrict__ window, const float2* __restrict__ tw512, const float2* __restrict__ tw256,
             const float* __restrict__ mel_w, const int* __restrict__ mel_start, const int* __restrict__ mel_len) {
  __shared__ __align__(16) float s_x[FB_WARPS][FB_NFFT];      // windowed frame, later the power spectrum
  __shared__ float s_re[FB_WARPS][8 * FB_YS];                 // exchange buffer Y[k1][n2], later Z (zidx layout)
  __shared__ float s_im[FB_WARPS][8 * FB_YS];
  __shared__ float2 s_tw512[FB_NFFT / 2];                     // W512^k = (cos, -sin)(2 pi k / 512), k < 256
  __shared__ float2 s_tw256[FB_NFFT / 2];                     // W256^j, j < 256
  for (int i = threadIdx.x; i < FB_NFFT / 2; i += blockDim.x) {
    s_tw512[i] = tw512[i];
    s_tw256[i] = tw256[i];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const TIn* wave = wave_all + (long long)blockIdx.y * wave_stride;      // blockIdx.y = recording in the batch
  float* feats = feats_all + (long long)blockIdx.y * n_frames * FB_NBIN;
  float* xs = s_x[warp];
  float* yre = s_re[warp];
  float* yim = s_im[warp];
  const long long frame0 = ((long long)blockIdx.x * FB_WARPS + warp) * FB_FPW;
#pragma unroll 1
  for (int fi = 0; fi < FB_FPW; ++fi) {
    const long long frame = frame0 + fi;
    if (frame >= n_frames) return;
    const TIn* src = wave + frame * FB_SHIFT;
    // 1. load + DC removal (kaldi.py remove_dc_offset: per-frame mean)
    float x[13];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < 13; ++i) {
      const int j = lane + 32 * i;
      x[i] = (j < FB_WIN) ? ld_sample(src, j) : 0.f;
      sum += x[i];
    }
    const float mean = warp_sum(sum) / (float)FB_WIN;
    __syncwarp();  // the previous frame's mel loop has finished reading xs
#pragma unroll
    for (int i = 0; i < 13; ++i) {
      const int j = lane + 32 * i;
      if (j < FB_WIN) xs[j] = x[i] - mean;  // centred frame
    }
    __syncwarp();
    // 2. pre-emphasis (replicate-left) + povey window, zero padded to 512, in place via registers
    float y[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int j = lane + 32 * i;
      float v = 0.f;
      if (j < FB_WIN) {
        const float cur = xs[j];
        const float prev = xs[j > 0 ? j - 1 : 0];
        v = (cur - 0.97f * prev) * __ldg(window + j);
      }
      y[i] = v;
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 16; ++i) xs[lane + 32 * i] = y[i];
    __syncwarp();
    // 3a. lane = n2: 8-point DFT over n1 of z[32 n1 + n2], twiddle W256^(n2 k1), exchange
    float2 a[8];
    const float2* zs = reinterpret_cast<const float2*>(xs);
#pragma unroll
    for (int n1 = 0; n1 < 8; ++n1) a[n1] = zs[32 * n1 + lane];
    dft8(a);
#pragma unroll
    for (int k1 = 0; k1 < 8; ++k1) {
      const float2 v = (k1 == 0) ? a[0] : cmul(a[k1], s_tw256[lane * k1]);
      yre[k1 * FB_YS + lane] = v.x;
      yim[k1 * FB_YS + lane] = v.y;
    }
    __syncwarp();
    // 3b. lane = (k1, b): 8-point DFT over a of Y[k1][4 a + b], twiddle W32^(b c) = W256^(8 b c)
    const int k1 = lane >> 2, b = lane & 3;
#pragma unroll
    for (int q = 0; q < 8; ++q) a[q] = make_float2(yre[k1 * FB_YS + 4 * q + b], yim[k1 * FB_YS + 4 * q + b]);
    dft8(a);
#pragma unroll
    for (int c = 1; c < 8; ++c) a[c] = cmul(a[c], s_tw256[8 * b * c]);
    // 3c. 4-point DFT over b across the 4 neighbouring lanes (two shuffle stages); lane b ends with d = bitrev2(b)
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      float2 v = a[c];
      float2 t = make_float2(__shfl_xor_sync(0xffffffffu, v.x, 2), __shfl_xor_sync(0xffffffffu, v.y, 2));
      v = (b & 2) ? csub(t, v) : cadd(v, t);
      if (b == 3) v = mul_negi(v);
      t = make_float2(__shfl_xor_sync(0xffffffffu, v.x, 1), __shfl_xor_sync(0xffffffffu, v.y, 1));
      a[c] = (b & 1) ? csub(t, v) : cadd(v, t);
    }
    __syncwarp();  // all lanes have read Y: the buffer becomes Z
    const int dd = ((b & 1) << 1) | (b >> 1);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int k = k1 + 8 * c + 64 * dd;
      yre[zidx(k)] = a[c].x;
      yim[zidx(k)] = a[c].y;
    }
    __syncwarp();
    // 4. real-FFT unpacking + power spectrum, bins 0..255 (the Nyquist bin carries zero mel weight, kaldi.py:627):
    //    X[k] = (Z[k] + conj Z[256-k]) / 2 + W512^k (Z[k] - conj Z[256-k]) / (2i),  Z[256] = Z[0]
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int k = lane + 32 * i;
      const int kr = (256 - k) & 255;
      const float2 zk = make_float2(yre[zidx(k)], yim[zidx(k)]);
      const float2 zr = make_float2(yre[zidx(kr)], -yim[zidx(kr)]);   // conj Z[256 - k]
      const float2 ze = make_float2(0.5f * (zk.x + zr.x), 0.5f * (zk.y + zr.y));
      const float2 df = make_float2(0.5f * (zk.x - zr.x), 0.5f * (zk.y - zr.y));
      const float2 zo = make_float2(df.y, -df.x);                      // df / i
      const float2 xk = cadd(ze, cmul(zo, s_tw512[k]));
      xs[k] = xk.x * xk.x + xk.y * xk.y;
    }
    __syncwarp();
    // 5. mel + log
    for (int mb = lane; mb < FB_NBIN; mb += 32) {
      const int st = __ldg(mel_start + mb), ln = __ldg(mel_len + mb);
      float acc = 0.f;
      for (int k = 0; k < ln; ++k) acc = fmaf(xs[st + k], __ldg(mel_w + mb * FB_MAXW + k), acc);
      feats[frame * FB_NBIN + mb] = logf(fmaxf(acc, 1.1920928955078125e-07f));
    }
  }
}

template <typename TIn>
static int launch_fbank_t(const TIn* wave, long long n_samples, float* feats, long long n_frames, cudaStream_t stream,
                          int batch = 1, long long wave_stride = 0, int window_type = 0) {
  const FbankTables* fb = nullptr;
  if (init_fbank_tables(&fb)) return -1;
  const FbankTables& g_fb = *fb;
  long long expect = n_samples < FB_WIN ? 0 : 1 + (n_samples - FB_WIN) / FB_SHIFT;
  RVB_REQUIRE(n_frames <= expect, "fbank: %lld frames requested but only %lld fit %lld samples", n_frames, expect,
              n_samples);
  if (n_frames <= 0) return 0;
  const long long blocks = (n_frames + FB_WARPS * FB_FPW - 1) / (FB_WARPS * FB_FPW);
  dim3 grid((unsigned)blocks, (unsigned)batch);
  fbank_kernel<TIn><<<grid, FB_WARPS * 32, 0, stream>>>(wave, wave_stride, n_frames, feats, window_type == 1 ? g_fb.window_hamming : g_fb.window, g_fb.twiddle,
                                                       g_fb.tw256, g_fb.mel_w, g_fb.mel_start, g_fb.mel_len);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

int launch_fbank(const float* wave, long long n_samples, float* feats, long long n_frames, cudaStream_t stream) {
  return launch_fbank_t<float>(wave, n_samples, feats, n_frames, stream);
}
int launch_fbank_i16(const short* wave, long long n_samples, float* feats, long long n_frames, cudaStream_t stream) {
  return launch_fbank_t<short>(wave, n_samples, feats, n_frames, stream);
}
int launch_fbank_batch(const void* wave, int is_i16, int batch, long long wave_stride, long long n_samples,
                       float* feats, long long n_frames, cudaStream_t stream, int window_type) {
  RVB_REQUIRE(batch >= 1 && batch <= 65535 && wave_stride >= n_samples, "fbank_batch: bad batch/stride");
  if (is_i16)
    return launch_fbank_t<short>(reinterpret_cast<const short*>(wave), n_samples, feats, n_frames, stream, batch,
                                 wave_stride, window_type);
  return launch_fbank_t<float>(reinterpret_cast<const float*>(wave), n_samples, feats, n_frames, stream, batch,
                               wave_stride, window_type);
}

}  // namespace rvb
