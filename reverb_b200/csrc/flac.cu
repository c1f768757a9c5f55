// reverb_b200 — FLAC decoding on the GPU (RFC 9639), frame-parallel over the file's bytes uploaded once.
//
// Passes (DESIGN.md §4k):
//   flac_sync_kernel     every byte offset: 14-bit sync code, no reserved field values, matching header CRC-8 ->
//                        candidate (offset, coded number, block size, blocking strategy) appended to a list
//   host (rvb_flac_index) sorts the candidates and keeps the chain whose coded numbers are consecutive from the frame at
//                        the end of the metadata; a prefix sum of block sizes gives each frame's first sample
//   flac_parse_kernel    one thread per frame: header, every subframe's type / wasted bits / warm-up samples /
//                        predictor, Rice or escaped residuals into the sample buffer, CRC-16 checked
//   flac_predict_kernel  one thread per (frame, channel): CONSTANT, FIXED 0-4 and LPC 1-32 restored in place, wasted
//                        bits undone
//   flac_store_kernel    one thread per sample: inter-channel decorrelation, left-justified int16 / int32 store
// Every bit read is bounds-checked against the frame's span; a frame that fails any check writes a status code and
// the lowest failing frame index is reported (no concealment).  Samples of streams up to 24 bits are held in int32,
// wider ones (and the 33-bit side channel of 32-bit audio) in int64; predictor sums are always 64-bit.
#include <algorithm>
#include <vector>

#include "host_mem.h"
#include "../../include/rvb_b200.h"

namespace rvb {
// a named namespace, so the kernels' symbol names (torch.profiler rows) are the same in every build
namespace flac {

// candidate frame header found by the sync pass
struct FlacCand {
  long long off;
  long long num;  // frame number (fixed blocking) or first sample number (variable blocking)
  int bs;
  int var;
};
// a frame of the index chain: bytes [off, end), samples [sample0, sample0 + bs) of every channel
struct FlacFrame {
  long long off, end, sample0;
  int bs, pad;
};
// per-frame result of the parse pass
struct FlacFrameOut {
  long long err_off;  // byte offset the status refers to
  int status;         // k* below
  int chan_assign;    // 0-7 independent, 8 left/side, 9 side/right, 10 mid/side
};
struct SubDesc {
  long long cval;  // CONSTANT value
  int type;        // 0 CONSTANT, 1 VERBATIM, 2 FIXED / LPC (coefficients below)
  int order, shift, wasted;
  int coef[32];
};
struct IndexHeader {
  int n_cand;
  int pad;
};

enum {
  kOk = 0,
  kBadHeader = 1,    // header fails its syntax or CRC-8 check
  kMismatch = 2,     // header disagrees with STREAMINFO or the index
  kBadSubframe = 3,  // reserved subframe type, bad padding bit, order or wasted bits out of range
  kBadResidual = 4,  // reserved coding method, partition order or escape out of range, Rice value beyond 32 bits
  kTruncated = 5,    // a read runs past the frame's span
  kBadCrc16 = 6,     // frame CRC-16 mismatch
  kTrailing = 7,     // the frame ends before the next frame (or the file) begins
};

constexpr int kMaxCand = 1 << 30;

__host__ __device__ inline long long cand_capacity(long long n_bytes) {
  // a frame is at least 10 bytes (6-byte header, 2-byte subframe, CRC-16); random data yields a sync candidate about
  // once every 2^22 bytes, so n/8 leaves room for either
  return n_bytes / 8 + 64;
}

__device__ __forceinline__ uint8_t crc8_byte(uint8_t crc, uint8_t b) {
  crc ^= b;
#pragma unroll
  for (int i = 0; i < 8; ++i) crc = (uint8_t)((crc & 0x80) ? (crc << 1) ^ 0x07 : crc << 1);
  return crc;
}

struct Hdr {
  long long num;
  int bs, rate, nch, chan_assign, bps, var, len;
};

// parses and CRC-8 checks the frame header at b[off]; rate / bps = 0 stand for "from STREAMINFO"
__device__ bool parse_header(const uint8_t* __restrict__ b, long long off, long long n, Hdr* h) {
  if (off + 6 > n) return false;
  const uint8_t* p = b + off;
  if (p[0] != 0xFF || (p[1] & 0xFE) != 0xF8) return false;
  h->var = p[1] & 1;
  const int bs_code = p[2] >> 4, rate_code = p[2] & 15, ch_code = p[3] >> 4, bps_code = (p[3] >> 1) & 7;
  if (bs_code == 0 || rate_code == 15 || ch_code >= 11 || bps_code == 3 || (p[3] & 1)) return false;
  long long pos = 4;
  // coded number: UTF-8-like, up to 6 bytes for frame numbers (31 bits), 7 for sample numbers (36 bits)
  const int b0 = p[pos++];
  int extra;
  long long v;
  if (b0 < 0x80) extra = 0, v = b0;
  else if (b0 < 0xC0) return false;
  else if (b0 < 0xE0) extra = 1, v = b0 & 0x1F;
  else if (b0 < 0xF0) extra = 2, v = b0 & 0x0F;
  else if (b0 < 0xF8) extra = 3, v = b0 & 0x07;
  else if (b0 < 0xFC) extra = 4, v = b0 & 0x03;
  else if (b0 < 0xFE) extra = 5, v = b0 & 0x01;
  else if (b0 == 0xFE) extra = 6, v = 0;
  else return false;
  if (extra == 6 && !h->var) return false;
  if (off + pos + extra + 5 > n) return false;
  for (int i = 0; i < extra; ++i) {
    const int c = p[pos++];
    if ((c & 0xC0) != 0x80) return false;
    v = (v << 6) | (c & 0x3F);
  }
  h->num = v;
  if (bs_code == 1) h->bs = 192;
  else if (bs_code <= 5) h->bs = 144 << bs_code;
  else if (bs_code == 6) h->bs = p[pos++] + 1;
  else if (bs_code == 7) {
    h->bs = ((p[pos] << 8) | p[pos + 1]) + 1;
    pos += 2;
  } else h->bs = 1 << bs_code;
  if (h->bs > 65535) return false;
  static constexpr int kRates[12] = {0, 88200, 176400, 192000, 8000, 16000, 22050, 24000, 32000, 44100, 48000, 96000};
  if (rate_code < 12) h->rate = kRates[rate_code];
  else if (rate_code == 12) h->rate = p[pos++] * 1000;
  else {
    h->rate = ((p[pos] << 8) | p[pos + 1]) * (rate_code == 14 ? 10 : 1);
    pos += 2;
  }
  h->chan_assign = ch_code;
  h->nch = ch_code < 8 ? ch_code + 1 : 2;
  static constexpr int kBps[8] = {0, 8, 12, 0, 16, 20, 24, 32};
  h->bps = kBps[bps_code];
  uint8_t crc = 0;
  for (long long i = 0; i < pos; ++i) crc = crc8_byte(crc, p[i]);
  if (crc != p[pos]) return false;
  h->len = (int)pos + 1;
  return true;
}

__global__ void __launch_bounds__(256)
flac_sync_kernel(const uint8_t* __restrict__ b, long long n, FlacCand* __restrict__ cand, int* __restrict__ n_cand,
                 long long cap) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i + 1 < n; i += (long long)gridDim.x * blockDim.x) {
    if (b[i] != 0xFF || (b[i + 1] & 0xFE) != 0xF8) continue;
    Hdr h;
    if (!parse_header(b, i, n, &h)) continue;
    const int k = atomicAdd(n_cand, 1);
    if (k < cap) cand[k] = FlacCand{i, h.num, h.bs, h.var};
  }
}

// MSB-first bit reader over bytes [pos, end) with a 64-bit cache; any read past `end` sets `bad` and returns 0
struct BitReader {
  const uint8_t* b;
  long long nb, end;  // next byte to load, end of the span
  unsigned long long cache;
  int cbits;
  bool bad;
  __device__ void init(const uint8_t* bytes, long long pos, long long end_) {
    b = bytes, nb = pos, end = end_, cache = 0, cbits = 0, bad = false;
  }
  __device__ __forceinline__ void refill() {
    while (cbits <= 56 && nb < end) {
      cache |= (unsigned long long)__ldg(b + nb++) << (56 - cbits);
      cbits += 8;
    }
  }
  // n <= 56 bits, unsigned
  __device__ __forceinline__ unsigned long long read(int n) {
    if (n == 0) return 0;
    if (cbits < n) {
      refill();
      if (cbits < n) {
        bad = true;
        return 0;
      }
    }
    const unsigned long long v = cache >> (64 - n);
    cache <<= n;
    cbits -= n;
    return v;
  }
  __device__ __forceinline__ long long read_signed(int n) {
    if (n == 0) return 0;
    return (long long)(read(n) << (64 - n)) >> (64 - n);
  }
  // count of 0 bits before the next 1 bit (consumed); stops with `bad` at the span's end
  __device__ __forceinline__ long long unary() {
    long long zeros = 0;
    for (;;) {
      if (cbits == 0) {
        refill();
        if (cbits == 0) {
          bad = true;
          return 0;
        }
      }
      const int lz = cache ? __clzll((long long)cache) : 64;
      if (lz >= cbits) {
        zeros += cbits;
        cache = 0;
        cbits = 0;
        continue;
      }
      cache <<= lz + 1;
      cbits -= lz + 1;
      return zeros + lz;
    }
  }
  __device__ long long byte_pos() const { return nb - cbits / 8; }
  __device__ void align() {
    const int r = cbits & 7;
    cache <<= r;
    cbits -= r;
  }
};

template <typename S>
__device__ int read_residual(BitReader& br, S* __restrict__ x, int bs, int order) {
  const int method = (int)br.read(2);
  if (method >= 2) return kBadResidual;
  const int pw = method ? 5 : 4, esc = method ? 31 : 15;
  const int po = (int)br.read(4);
  if (br.bad) return kTruncated;
  const int parts = 1 << po;
  if (bs & (parts - 1)) return kBadResidual;
  const int psize = bs >> po;
  if (psize < order) return kBadResidual;
  int i = order;
  for (int p = 0; p < parts; ++p) {
    const int k = (int)br.read(pw);
    const int cnt = p == 0 ? psize - order : psize;
    if (k == esc) {
      const int nb = (int)br.read(5);
      for (int j = 0; j < cnt; ++j) x[i++] = (S)br.read_signed(nb);
    } else {
      for (int j = 0; j < cnt; ++j) {
        const long long q = br.unary();
        if (q >> (32 - k)) return br.bad ? kTruncated : kBadResidual;  // (q << k) | r must fit in 32 bits
        const unsigned u = ((unsigned)q << k) | (unsigned)br.read(k);
        x[i++] = (S)(int)((u >> 1) ^ (0u - (u & 1u)));
      }
    }
    if (br.bad) return kTruncated;
  }
  return kOk;
}

// one thread per frame
template <typename S>
__global__ void __launch_bounds__(64)
flac_parse_kernel(const uint8_t* __restrict__ b, long long n, rvb_flac_info info, const FlacFrame* __restrict__ frames,
                  int n_frames, long long total, SubDesc* __restrict__ desc, S* __restrict__ samples,
                  FlacFrameOut* __restrict__ fout, int* __restrict__ first_bad) {
  __shared__ unsigned short crc16[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    unsigned c = (unsigned)i << 8;
    for (int k = 0; k < 8; ++k) c = (c & 0x8000) ? (c << 1) ^ 0x8005 : c << 1;
    crc16[i] = (unsigned short)c;
  }
  __syncthreads();
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_frames) return;
  const FlacFrame fr = frames[f];
  const int nch = info.channels;
  int status = kOk;
  long long err_off = fr.off;
  Hdr h;
  if (!parse_header(b, fr.off, fr.end, &h)) status = kBadHeader;
  else if (h.bs != fr.bs || h.nch != nch || (h.bps && h.bps != info.bits_per_sample) ||
           (h.rate && h.rate != info.sample_rate))
    status = kMismatch;
  BitReader br;
  br.init(b, fr.off + (status == kOk ? h.len : 0), fr.end);
  for (int c = 0; c < nch && status == kOk; ++c) {
    SubDesc& d = desc[(size_t)f * nch + c];
    S* x = samples + (size_t)c * total + fr.sample0;
    const bool side = (h.chan_assign == 8 || h.chan_assign == 10) ? c == 1 : h.chan_assign == 9 && c == 0;
    int sbps = info.bits_per_sample + (side ? 1 : 0);
    const int pad = (int)br.read(1), type = (int)br.read(6), has_wasted = (int)br.read(1);
    int wasted = 0;
    if (has_wasted) wasted = (int)br.unary() + 1;
    if (br.bad) {
      status = kTruncated;
      break;
    }
    if (pad || wasted >= sbps) {
      status = kBadSubframe;
      break;
    }
    sbps -= wasted;
    d.wasted = wasted;
    d.shift = 0;
    d.order = 0;
    if (type == 0) {
      d.type = 0;
      d.cval = br.read_signed(sbps);
    } else if (type == 1) {
      d.type = 1;
      for (int i = 0; i < fr.bs; ++i) x[i] = (S)br.read_signed(sbps);
    } else if ((type >= 8 && type <= 12) || type >= 32) {
      const bool lpc = type >= 32;
      const int order = lpc ? type - 31 : type - 8;
      if (order > fr.bs) {
        status = kBadSubframe;
        break;
      }
      d.type = 2;
      d.order = order;
      for (int i = 0; i < order; ++i) x[i] = (S)br.read_signed(sbps);
      if (lpc) {
        const int prec = (int)br.read(4) + 1;
        const int shift = (int)br.read_signed(5);
        if (prec == 16 || shift < 0) {
          status = br.bad ? kTruncated : kBadSubframe;
          break;
        }
        d.shift = shift;
        for (int i = 0; i < order; ++i) d.coef[i] = (int)br.read_signed(prec);
      } else {
        // FIXED predictors as integer LPC coefficients with shift 0 (RFC 9639 §9.2.5)
        static constexpr int kFixed[5][4] = {{0, 0, 0, 0}, {1, 0, 0, 0}, {2, -1, 0, 0}, {3, -3, 1, 0}, {4, -6, 4, -1}};
        for (int i = 0; i < order; ++i) d.coef[i] = kFixed[order][i];
      }
      if (br.bad) {
        status = kTruncated;
        break;
      }
      status = read_residual(br, x, fr.bs, order);
    } else {
      status = kBadSubframe;
    }
    if (status == kOk && br.bad) status = kTruncated;
  }
  if (status == kOk) {
    br.align();
    const long long body_end = br.byte_pos();
    const unsigned want = (unsigned)br.read(16);
    if (br.bad) status = kTruncated;
    else {
      unsigned crc = 0;
      for (long long i = fr.off; i < body_end; ++i) crc = ((crc << 8) ^ crc16[((crc >> 8) ^ __ldg(b + i)) & 0xFF]) & 0xFFFF;
      if (crc != want) status = kBadCrc16, err_off = fr.off;
      else if (body_end + 2 != fr.end) status = kTrailing, err_off = body_end + 2;
    }
  } else if (status == kTruncated) {
    err_off = fr.end;
  }
  fout[f] = FlacFrameOut{err_off, status, status == kOk ? h.chan_assign : 0};
  if (status != kOk) atomicMin(first_bad, f);
}

// one thread per (frame, channel): prediction restored in place, then wasted bits
template <int N, typename S>
__device__ void lpc_restore(S* __restrict__ x, int bs, int order, const int* __restrict__ coef, int shift) {
  int c[N];
  S h[N];  // h[j] = x[i - 1 - j]
#pragma unroll
  for (int j = 0; j < N; ++j) {
    c[j] = j < order ? coef[j] : 0;
    h[j] = j < order ? x[order - 1 - j] : (S)0;
  }
  for (int i = order; i < bs; ++i) {
    long long acc = 0;
#pragma unroll
    for (int j = 0; j < N; ++j) acc += (long long)c[j] * (long long)h[j];
    const S v = (S)((long long)x[i] + (acc >> shift));
    x[i] = v;
#pragma unroll
    for (int j = N - 1; j > 0; --j) h[j] = h[j - 1];
    h[0] = v;
  }
}

template <typename S>
__global__ void __launch_bounds__(128)
flac_predict_kernel(const FlacFrame* __restrict__ frames, int n_frames, int nch, long long total,
                    const SubDesc* __restrict__ desc, const FlacFrameOut* __restrict__ fout, S* __restrict__ samples) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)n_frames * nch) return;
  const int f = (int)(t / nch), c = (int)(t % nch);
  if (fout[f].status != kOk) return;
  const FlacFrame fr = frames[f];
  const SubDesc& d = desc[t];
  S* x = samples + (size_t)c * total + fr.sample0;
  if (d.type == 0) {
    const S v = (S)d.cval;
    for (int i = 0; i < fr.bs; ++i) x[i] = v;
  } else if (d.type == 2 && d.order > 0) {
    if (d.order <= 8) lpc_restore<8>(x, fr.bs, d.order, d.coef, d.shift);
    else if (d.order <= 16) lpc_restore<16>(x, fr.bs, d.order, d.coef, d.shift);
    else lpc_restore<32>(x, fr.bs, d.order, d.coef, d.shift);
  }
  if (d.wasted)
    for (int i = 0; i < fr.bs; ++i) x[i] = (S)(long long)((unsigned long long)(long long)x[i] << d.wasted);
}

// grid (frames, sample tiles): decorrelate the channels and store left-justified samples
template <typename S, typename T>
__global__ void __launch_bounds__(256)
flac_store_kernel(const FlacFrame* __restrict__ frames, int nch, long long total, const FlacFrameOut* __restrict__ fout,
                  const S* __restrict__ samples, int lshift, T* __restrict__ out) {
  const int f = blockIdx.x;
  const FlacFrameOut fo = fout[f];
  if (fo.status != kOk) return;
  const FlacFrame fr = frames[f];
  for (int i = blockIdx.y * blockDim.x + threadIdx.x; i < fr.bs; i += gridDim.y * blockDim.x) {
    const long long s = fr.sample0 + i;
    if (fo.chan_assign < 8) {
      for (int c = 0; c < nch; ++c)
        out[(size_t)c * total + s] = (T)((unsigned long long)(long long)samples[(size_t)c * total + s] << lshift);
      continue;
    }
    const long long a = samples[s], d = samples[(size_t)total + s];
    long long l, r;
    if (fo.chan_assign == 8) l = a, r = a - d;        // left / side
    else if (fo.chan_assign == 9) l = a + d, r = d;   // side / right (a = side, d = right)
    else {                                            // mid / side: the side's LSB restores the mid's
      const long long m = (long long)((unsigned long long)a << 1) | (d & 1);
      l = (m + d) >> 1, r = (m - d) >> 1;
    }
    out[s] = (T)((unsigned long long)l << lshift);
    out[(size_t)total + s] = (T)((unsigned long long)r << lshift);
  }
}

// workspace of rvb_flac_decode, in this order
struct DecodeLayout {
  size_t fout, first_bad, desc, samples, total;
};
DecodeLayout decode_layout(int n_frames, long long total, const rvb_flac_info& info) {
  auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
  DecodeLayout L;
  L.fout = 0;
  L.first_bad = up((size_t)n_frames * sizeof(FlacFrameOut));
  L.desc = L.first_bad + 256;
  L.samples = L.desc + up((size_t)n_frames * info.channels * sizeof(SubDesc));
  L.total = L.samples + up((size_t)info.channels * total * (info.bits_per_sample > 24 ? 8 : 4));
  return L;
}

bool info_ok(const rvb_flac_info* info) {
  return info && info->channels >= 1 && info->channels <= 8 && info->bits_per_sample >= 4 &&
         info->bits_per_sample <= 32 && info->sample_rate > 0;
}

size_t index_cand_off() { return 256; }
size_t index_frames_off(long long n_bytes) {
  return index_cand_off() + (((size_t)cand_capacity(n_bytes) * sizeof(FlacCand) + 255) & ~(size_t)255);
}

static thread_local HostPinned g_flac_pin;

template <typename S>
int flac_decode_impl(const uint8_t* d_bytes, long long n_bytes, const rvb_flac_info& info, const FlacFrame* frames,
                     int n_frames, long long total, char* ws, void* d_out, int* h_bad_frame, long long* h_bad_offset,
                     int* h_bad_status, cudaStream_t stream) {
  const DecodeLayout L = decode_layout(n_frames, total, info);
  FlacFrameOut* fout = reinterpret_cast<FlacFrameOut*>(ws + L.fout);
  int* first_bad = reinterpret_cast<int*>(ws + L.first_bad);
  SubDesc* desc = reinterpret_cast<SubDesc*>(ws + L.desc);
  S* samples = reinterpret_cast<S*>(ws + L.samples);
  const int nch = info.channels;
  RVB_CHECK_CUDA(cudaMemsetAsync(first_bad, 0x7F, sizeof(int), stream));
  flac_parse_kernel<S><<<(n_frames + 63) / 64, 64, 0, stream>>>(d_bytes, n_bytes, info, frames, n_frames, total, desc,
                                                                 samples, fout, first_bad);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  const long long threads = (long long)n_frames * nch;
  flac_predict_kernel<S><<<(unsigned)((threads + 127) / 128), 128, 0, stream>>>(frames, n_frames, nch, total, desc, fout,
                                                                                samples);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  const int tiles = std::min(256, std::max(1, (info.max_block_size + 255) / 256));
  const dim3 grid((unsigned)n_frames, (unsigned)tiles);
  if (info.bits_per_sample <= 16)
    flac_store_kernel<S, short><<<grid, 256, 0, stream>>>(frames, nch, total, fout, samples, 16 - info.bits_per_sample,
                                                          static_cast<short*>(d_out));
  else
    flac_store_kernel<S, int><<<grid, 256, 0, stream>>>(frames, nch, total, fout, samples, 32 - info.bits_per_sample,
                                                        static_cast<int*>(d_out));
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  // first failing frame, then its record: 16 bytes apart in one page-locked buffer
  if (g_flac_pin.ensure(16 + sizeof(FlacFrameOut))) return -1;
  int* h_first = g_flac_pin.as<int>();
  FlacFrameOut* h_fo = reinterpret_cast<FlacFrameOut*>(g_flac_pin.as<char>() + 16);
  RVB_CHECK_CUDA(cudaMemcpyAsync(h_first, first_bad, sizeof(int), cudaMemcpyDeviceToHost, stream));
  RVB_CHECK_CUDA(cudaStreamSynchronize(stream));
  *h_bad_frame = -1;
  *h_bad_offset = -1;
  *h_bad_status = 0;
  if (*h_first < n_frames) {
    const int bad = *h_first;
    RVB_CHECK_CUDA(cudaMemcpyAsync(h_fo, fout + bad, sizeof(FlacFrameOut), cudaMemcpyDeviceToHost, stream));
    RVB_CHECK_CUDA(cudaStreamSynchronize(stream));
    *h_bad_frame = bad;
    *h_bad_offset = h_fo->err_off;
    *h_bad_status = h_fo->status;
  }
  return 0;
}

}  // namespace flac
}  // namespace rvb

RVB_API long long rvb_flac_index_workspace_bytes(long long n_bytes) {
  if (n_bytes < 0) return -1;
  return (long long)(rvb::flac::index_frames_off(n_bytes) + (size_t)rvb::flac::cand_capacity(n_bytes) * sizeof(rvb::flac::FlacFrame));
}

RVB_API int rvb_flac_index(const void* d_bytes, long long n_bytes, long long audio_offset, const rvb_flac_info* info,
                           void* d_workspace, long long workspace_bytes, int* h_n_frames, long long* h_total_samples,
                           void* stream_) {
  using namespace rvb;
  using namespace rvb::flac;
  cudaStream_t stream = (cudaStream_t)stream_;
  RVB_REQUIRE(d_bytes && d_workspace && h_n_frames && h_total_samples && n_bytes >= 0 && audio_offset >= 0 &&
                  audio_offset <= n_bytes && info_ok(info),
              "rvb_flac_index: bad arguments");
  const long long need = rvb_flac_index_workspace_bytes(n_bytes);
  RVB_REQUIRE(workspace_bytes >= need, "rvb_flac_index: %lld bytes need %lld bytes of workspace, %lld given", n_bytes,
              need, workspace_bytes);
  const long long cap = std::min<long long>(cand_capacity(n_bytes), kMaxCand);
  char* ws = static_cast<char*>(d_workspace);
  IndexHeader* hdr = reinterpret_cast<IndexHeader*>(ws);
  FlacCand* cand = reinterpret_cast<FlacCand*>(ws + index_cand_off());
  FlacFrame* frames = reinterpret_cast<FlacFrame*>(ws + index_frames_off(n_bytes));
  *h_n_frames = 0;
  *h_total_samples = 0;
  RVB_CHECK_CUDA(cudaMemsetAsync(hdr, 0, sizeof(IndexHeader), stream));
  const long long span = n_bytes - audio_offset;
  if (span > 1) {
    const unsigned grid = (unsigned)std::min<long long>((span + 255) / 256, 132 * 16);
    flac_sync_kernel<<<grid, 256, 0, stream>>>(static_cast<const uint8_t*>(d_bytes) + audio_offset, span, cand,
                                               &hdr->n_cand, cap);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
  }
  if (g_flac_pin.ensure(sizeof(IndexHeader))) return -1;
  RVB_CHECK_CUDA(cudaMemcpyAsync(g_flac_pin.p, hdr, sizeof(IndexHeader), cudaMemcpyDeviceToHost, stream));
  RVB_CHECK_CUDA(cudaStreamSynchronize(stream));
  const int n_cand = g_flac_pin.as<IndexHeader>()->n_cand;
  if (n_cand > cap) {
    *h_n_frames = -1;  // more sync candidates than any FLAC stream of this size can hold
    return 0;
  }
  if (n_cand == 0) return 0;
  std::vector<FlacCand> c(n_cand);
  if (g_flac_pin.ensure((size_t)n_cand * std::max(sizeof(FlacCand), sizeof(FlacFrame)))) return -1;
  RVB_CHECK_CUDA(cudaMemcpyAsync(g_flac_pin.p, cand, (size_t)n_cand * sizeof(FlacCand), cudaMemcpyDeviceToHost, stream));
  RVB_CHECK_CUDA(cudaStreamSynchronize(stream));
  memcpy(c.data(), g_flac_pin.p, (size_t)n_cand * sizeof(FlacCand));
  std::sort(c.begin(), c.end(), [](const FlacCand& a, const FlacCand& b) { return a.off < b.off; });
  // the chain: the frame right after the metadata, then each next candidate of the same blocking strategy whose
  // coded number continues it.  Candidates in between are sync patterns inside frame data.
  if (c[0].off != 0) return 0;
  std::vector<FlacFrame> fr;
  fr.reserve(n_cand);
  long long sample0 = 0;
  size_t cur = 0;
  for (;;) {
    const FlacCand& a = c[cur];
    fr.push_back(FlacFrame{audio_offset + a.off, n_bytes, sample0, a.bs, 0});
    sample0 += a.bs;
    const long long want = a.var ? a.num + a.bs : a.num + 1;
    size_t nxt = cur + 1;
    while (nxt < c.size() && !(c[nxt].var == a.var && c[nxt].num == want)) ++nxt;
    if (nxt == c.size()) break;
    fr.back().end = audio_offset + c[nxt].off;
    cur = nxt;
  }
  FlacFrame* h_fr = g_flac_pin.as<FlacFrame>();
  memcpy(h_fr, fr.data(), fr.size() * sizeof(FlacFrame));
  RVB_CHECK_CUDA(cudaMemcpyAsync(frames, h_fr, fr.size() * sizeof(FlacFrame), cudaMemcpyHostToDevice, stream));
  RVB_CHECK_CUDA(cudaStreamSynchronize(stream));
  *h_n_frames = (int)fr.size();
  *h_total_samples = sample0;
  return 0;
}

RVB_API long long rvb_flac_decode_workspace_bytes(int n_frames, long long total_samples, const rvb_flac_info* info) {
  if (n_frames < 1 || total_samples < 1 || !rvb::flac::info_ok(info)) return -1;
  return (long long)rvb::flac::decode_layout(n_frames, total_samples, *info).total;
}

RVB_API int rvb_flac_decode(const void* d_bytes, long long n_bytes, const rvb_flac_info* info,
                            const void* d_index_workspace, int n_frames, long long total_samples, void* d_workspace,
                            long long workspace_bytes, void* d_out, int* h_bad_frame, long long* h_bad_offset,
                            int* h_bad_status, void* stream_) {
  using namespace rvb;
  using namespace rvb::flac;
  RVB_REQUIRE(d_bytes && d_index_workspace && d_workspace && d_out && h_bad_frame && h_bad_offset && h_bad_status &&
                  n_frames >= 1 && total_samples >= 1 && info_ok(info),
              "rvb_flac_decode: bad arguments");
  const long long need = rvb_flac_decode_workspace_bytes(n_frames, total_samples, info);
  RVB_REQUIRE(workspace_bytes >= need, "rvb_flac_decode: %d frames of %lld samples need %lld bytes of workspace, %lld given",
              n_frames, total_samples, need, workspace_bytes);
  RVB_REQUIRE(n_frames <= cand_capacity(n_bytes), "rvb_flac_decode: %d frames exceed the index of %lld bytes", n_frames,
              n_bytes);
  const FlacFrame* frames =
      reinterpret_cast<const FlacFrame*>(static_cast<const char*>(d_index_workspace) + index_frames_off(n_bytes));
  const uint8_t* b = static_cast<const uint8_t*>(d_bytes);
  char* ws = static_cast<char*>(d_workspace);
  cudaStream_t stream = (cudaStream_t)stream_;
  if (info->bits_per_sample > 24)
    return flac_decode_impl<long long>(b, n_bytes, *info, frames, n_frames, total_samples, ws, d_out, h_bad_frame,
                                       h_bad_offset, h_bad_status, stream);
  return flac_decode_impl<int>(b, n_bytes, *info, frames, n_frames, total_samples, ws, d_out, h_bad_frame, h_bad_offset,
                               h_bad_status, stream);
}
