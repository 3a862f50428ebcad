// Shared declarations for libb200audio (sm_90a).  No torch headers anywhere in csrc/.
#pragma once
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include "../../include/b200audio.h"

namespace b200a {

constexpr uint32_t kWsMagic = 0xB200A0D1u;
constexpr int kMaxStages = 16;
constexpr int kMaxFft = 8192;
constexpr float kKaldiEps = 1.1920928955078125e-07f;  // numeric_limits<float>::epsilon(), kaldi.py:21-22

// Device-side header at the start of a front-end workspace.
struct WsHeader {
  uint32_t magic;
  int32_t n_fft;
  int32_t n_bins;
  int32_t n_mels;
  int32_t n_mfcc;
  float scale;  // frame_length / window normalisation folded into one factor
  int32_t reserved[10];
};
static_assert(sizeof(WsHeader) == 64, "header is 64 bytes");

// Byte offsets of the tables inside a front-end workspace (host + device agree via this struct).
struct WsLayout {
  size_t header, window, twiddle, bands, fb, dct, total;
};

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

inline WsLayout ws_layout(const b200a_frontend_desc& d) {
  WsLayout l{};
  const size_t n_bins = d.onesided ? d.n_fft / 2 + 1 : d.n_fft;
  size_t off = 0;
  l.header = off;
  off = align_up(off + sizeof(WsHeader), 256);
  l.window = off;
  off = align_up(off + sizeof(float) * d.n_fft, 256);
  l.twiddle = off;
  off = align_up(off + sizeof(float2) * d.n_fft, 256);
  l.bands = off;
  off = align_up(off + sizeof(int2) * (d.n_mels > 0 ? d.n_mels : 1), 256);
  l.fb = off;
  off = align_up(off + sizeof(float) * n_bins * (d.n_mels > 0 ? d.n_mels : 0), 256);
  l.dct = off;
  off = align_up(off + sizeof(float) * (size_t)(d.n_mels > 0 ? d.n_mels : 0) * (d.n_mfcc > 0 ? d.n_mfcc : 0), 256);
  l.total = off;
  return l;
}

// SMs of the current device (persistent grids are sized to one wave of it); -1 if the query fails
inline int device_sm_count() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      n <= 0)
    return -1;
  return n;
}

inline int launch_status() { return cudaGetLastError() == cudaSuccess ? B200A_OK : B200A_ECUDA; }

// ---- device helpers -----------------------------------------------------------------------
// Index into the raw waveform row for sample i of the (constant `pad`-extended, then centre
// padded) signal; returns -1 for a zero sample.  Mirrors b200a_pad_index on the host.
__device__ __forceinline__ int64_t source_index(int64_t i, int64_t length, int pad, int half, int pad_mode) {
  const int64_t ext = length + 2 * (int64_t)pad;  // length after the constant pre-padding
  int64_t j = i - half;                           // index into the pre-padded signal
  if (j < 0 || j >= ext) {
    if (pad_mode == B200A_PAD_CONSTANT) return -1;
    if (pad_mode == B200A_PAD_REFLECT) {
      j = j < 0 ? -j : 2 * (ext - 1) - j;
    } else if (pad_mode == B200A_PAD_REPLICATE) {
      j = j < 0 ? 0 : ext - 1;
    } else {
      j %= ext;
      if (j < 0) j += ext;
    }
  }
  const int64_t s = j - pad;
  return (s >= 0 && s < length) ? s : -1;
}

// dL/dX of |X|^p for the upstream value s, as torch differentiates abs().pow(p): p |X|^(p-2) X s.  At X = 0 it is 0 for
// p >= 1 and NaN for p < 1 (0^(p-1) = inf times sgn(0) = 0).
__device__ __forceinline__ float2 power_vjp(float re, float im, float p, float s) {
  if (p == 2.f) return make_float2(2.f * re * s, 2.f * im * s);
  const float mag = hypotf(re, im);
  if (mag == 0.f) return p < 1.f ? make_float2(CUDART_NAN_F, CUDART_NAN_F) : make_float2(0.f, 0.f);
  const float c = (p == 1.f ? s : p * powf(mag, p - 1.f) * s) / mag;
  return make_float2(re * c, im * c);
}

// The overlap-added squared window at sample s of an iSTFT of `frames` frames, formed exactly as istft_ola_kernel forms
// it (float, fmaf, frames in ascending order); 0 where no frame covers s.
__device__ __forceinline__ float istft_envelope(const float* window, int n_fft, int hop, int64_t frames, int64_t s) {
  const int64_t t_lo = s - n_fft + 1 <= 0 ? 0 : (s - n_fft + hop) / hop;  // ceil((s - n_fft + 1) / hop)
  int64_t t_hi = s / hop;
  if (t_hi > frames - 1) t_hi = frames - 1;
  float env = 0.f;
  for (int64_t t = t_lo; t <= t_hi; ++t) {
    const float w = window[s - t * hop];
    env = fmaf(w, w, env);
  }
  return env;
}

// The filters [x, y) with a non-zero weight at bin k, from each filter's non-zero bin range bands[m] = [x, y); (0, 0)
// when none is.
__device__ __forceinline__ int2 filter_range(const int2* bands, int n_mels, int k) {
  int lo = n_mels, hi = 0;
  for (int m = 0; m < n_mels; ++m) {
    const int2 b = bands[m];
    if (b.x <= k && k < b.y) {
      lo = min(lo, m);
      hi = m + 1;
    }
  }
  return hi > lo ? make_int2(lo, hi) : make_int2(0, 0);
}

__device__ __forceinline__ void atomic_max_f32(float* addr, float v) {
  // total order trick: non-negative floats compare like ints, negative like reversed uints
  if (v >= 0.f) {
    atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
  } else {
    atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
  }
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace b200a
