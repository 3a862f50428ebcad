// vad (functional/filtering.py:1414-1702): SoX's voice-activity trim.  The reference loops over 50 ms measurement
// frames and, inside, over channels; each step is a windowed rFFT, a smoothing of the magnitude spectrum, an adaptive
// noise estimate, a second rFFT of the noise-reduced spectrum ("cepstrum") and its band power.  Here a call runs in
// chunks of frames.  The two FFTs are front-end passes (b200a_frontend_run: POWER with power 1, then MEL with a
// one-column indicator bank over the lifter band); between them the walk kernel below carries the per-(channel, bin)
// recurrences over the chunk's frames, and after them the trigger kernel turns band powers into measures, runs the
// reference's trigger and flush rules and writes the trim start.  State carried from chunk to chunk lives in the
// workspace and is carried exactly.
//
// Every float32 step of the walk is one rounded operation in the reference's order (__fmul_rn / __fadd_rn /
// __fsqrt_rn: no FMA contraction), because the reference runs each step as a separate float32 tensor op.
#include <cmath>

#include "common.cuh"

namespace b200a {
namespace {

constexpr int kWalkThreads = 128;
constexpr int kWalkPrefetch = 8;  // frames of |X| loaded ahead by each walk thread
constexpr int kTriggerThreads = 256;
constexpr int64_t kVadMaxChunk = 1 << 20;  // frames per call: 14.5 hours at the default 20 Hz

// Workspace, 256-byte aligned sections:
//   status int64 [2]                 {first triggering frame or -1, trim start}: the 16 bytes the caller reads back
//   spec   float [C][B]              smoothed spectrum over the band [s0, s1), B = s1 - s0
//   noise  float [C][B]              noise estimate
//   mean   float [C]                 mean measure
//   ring   float [C][measures_len]   the last measures_len measures, at frame % measures_len
//   addend float [C][chunk]          float32(meas * (1 - trigger_mult)) of the chunk's frames
//   first  int32 [C]                 each channel's first triggering frame in the chunk (chunk when none)
struct VadLayout {
  size_t status, spec, noise, mean, ring, addend, first, total;
};

VadLayout vad_layout(const b200a_vad_desc& d, int64_t chunk) {
  const size_t c = (size_t)d.channels, band = (size_t)(d.spectrum_end - d.spectrum_start);
  VadLayout l{};
  size_t off = 0;
  l.status = off;
  off = align_up(off + 2 * sizeof(int64_t), 256);
  l.spec = off;
  off = align_up(off + sizeof(float) * c * band, 256);
  l.noise = off;
  off = align_up(off + sizeof(float) * c * band, 256);
  l.mean = off;
  off = align_up(off + sizeof(float) * c, 256);
  l.ring = off;
  off = align_up(off + sizeof(float) * c * (size_t)d.measures_len, 256);
  l.addend = off;
  off = align_up(off + sizeof(float) * c * (size_t)chunk, 256);
  l.first = off;
  off = align_up(off + sizeof(int32_t) * c, 256);
  l.total = off;
  return l;
}

int validate_vad(const b200a_vad_desc* d, int64_t chunk) {
  if (d == nullptr || chunk < 1 || d->channels < 1 || d->period < 1 || d->measures_len < 1) return B200A_EINVAL;
  if (chunk > kVadMaxChunk) return B200A_EUNSUPPORTED;
  const int dft = d->dft_len;
  if (dft < 16 || (dft & (dft - 1)) != 0) return B200A_EINVAL;
  if (dft > kMaxFft) return B200A_EUNSUPPORTED;
  if (d->spectrum_start < 1 || d->spectrum_start > d->spectrum_end || d->spectrum_end > dft / 2) return B200A_EINVAL;
  if (d->cepstrum_start < 0 || d->cepstrum_start >= d->cepstrum_end || d->cepstrum_end > dft / 4) return B200A_EINVAL;
  if (d->channels > 65535) return B200A_EUNSUPPORTED;  // grid.y of the walk
  return B200A_OK;
}

// One thread per (channel, bin of [s0, s1)), walking the chunk's frames in order: the smoothing of |X| and the noise
// tracker of _measure (filtering.py:1448-1471), then r * cepstrum_window into the bin's slot of the frame's cepstrum
// row.  Loads of |X| are coalesced across bins and issued kWalkPrefetch frames at a time.
__global__ void __launch_bounds__(kWalkThreads) vad_walk_kernel(b200a_vad_desc d, int64_t chunk, int64_t frame0,
                                                                int frames, const float* __restrict__ spectrum,
                                                                const float* __restrict__ cep_window,
                                                                float* __restrict__ rows, float* spec_state,
                                                                float* noise_state) {
  const int band = d.spectrum_end - d.spectrum_start;
  const int i = blockIdx.x * kWalkThreads + threadIdx.x;
  if (i >= band) return;
  const int c = blockIdx.y;
  const int n_bins = d.dft_len / 2 + 1, half = d.dft_len / 2;
  const int k = d.spectrum_start + i;
  float s = 0.f, n = 0.f;
  if (frame0 > 0) {
    s = spec_state[(size_t)c * band + i];
    n = noise_state[(size_t)c * band + i];
  }
  const float cw = cep_window[i];
  const float up = (float)d.noise_up_mult, down = (float)d.noise_down_mult, nra = (float)d.noise_reduction_amount;
  const float smooth = (float)d.measure_smooth_mult, smooth_c = (float)(1.0 - d.measure_smooth_mult);
  const float* x = spectrum + (size_t)c * frames * n_bins + k;
  float* out = rows + (size_t)c * chunk * half + k;
  for (int f0 = 0; f0 < frames; f0 += kWalkPrefetch) {
    float xv[kWalkPrefetch];
#pragma unroll
    for (int u = 0; u < kWalkPrefetch; ++u) xv[u] = f0 + u < frames ? __ldg(x + (size_t)(f0 + u) * n_bins) : 0.f;
#pragma unroll
    for (int u = 0; u < kWalkPrefetch; ++u) {
      const int f = f0 + u;
      if (f >= frames) break;
      const int64_t g = frame0 + f;
      // boot_count: the frame index while it is <= boot_count_max (forever when that is negative), then -1
      const bool boot = d.boot_count_max < 0 || g <= d.boot_count_max;
      float mult = smooth, mult_c = smooth_c;
      if (boot) {
        const double b = (double)g / (1.0 + (double)g);  // python float, rounded to float32 by the tensor op
        mult = (float)b;
        mult_c = (float)(1.0 - b);
      }
      s = __fadd_rn(__fmul_rn(s, mult), __fmul_rn(xv[u], mult_c));
      const float dd = __fmul_rn(s, s);
      const float nm = boot ? 0.f : (dd > n ? up : down);
      n = __fadd_rn(__fmul_rn(n, nm), __fmul_rn(dd, __fsub_rn(1.f, nm)));
      const float v = __fsub_rn(dd, __fmul_rn(nra, n));
      const float r = __fsqrt_rn(v != v ? v : fmaxf(0.f, v));  // torch.max propagates NaN
      out[(size_t)f * half] = __fmul_rn(r, cw);
    }
  }
  spec_state[(size_t)c * band + i] = s;
  noise_state[(size_t)c * band + i] = n;
}

// meas = max(0, 21 + log(P / (c1 - c0))) in double, 0 for P <= 0 (filtering.py:1480-1482)
__device__ __forceinline__ double measure_of(float p, int lifter_bins) {
  const double pd = (double)p;
  if (!(pd > 0.0)) return 0.0;
  const double v = 21.0 + log(pd / (double)lifter_bins);
  return v > 0.0 ? v : 0.0;
}

// One CTA.  (1) measures of every (channel, frame) of the chunk, stored as float32, and the float32 addend of the mean
// update; (2) per channel, the float32 mean recurrence and its first frame with mean >= trigger_level; (3) the first
// (frame, channel) in the reference's frame-major order; (4) the flush scan (filtering.py:1671-1685) of that channel and
// every later one at that frame; (5) the status, or the carried ring when nothing triggered.
__global__ void __launch_bounds__(kTriggerThreads) vad_trigger_kernel(b200a_vad_desc d, int64_t chunk, int64_t frame0,
                                                                      int frames, const float* __restrict__ power,
                                                                      float* __restrict__ measures, int64_t* status,
                                                                      float* mean_state, float* ring, float* addend,
                                                                      int32_t* first) {
  const int C = d.channels, n = d.measures_len;
  const int lifter_bins = d.cepstrum_end - d.cepstrum_start;
  const double tm_c = 1.0 - d.trigger_mult;
  const float tm = (float)d.trigger_mult, level = (float)d.trigger_level;
  for (int64_t e = threadIdx.x; e < (int64_t)C * frames; e += blockDim.x) {
    const int c = (int)(e / frames), f = (int)(e % frames);
    const double m = measure_of(power[e], lifter_bins);
    measures[e] = (float)m;
    addend[(size_t)c * chunk + f] = (float)(m * tm_c);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float mean = frame0 > 0 ? mean_state[c] : 0.f;
    int hit = frames;
    for (int f = 0; f < frames; ++f) {
      mean = __fadd_rn(__fmul_rn(mean, tm), addend[(size_t)c * chunk + f]);
      if (mean >= level) {
        hit = f;
        break;
      }
    }
    mean_state[c] = mean;
    first[c] = hit;
  }
  __syncthreads();
  __shared__ int s_frame, s_channel;
  if (threadIdx.x == 0) {
    int fs = frames, cs = C;
    for (int c = 0; c < C; ++c) {
      if (first[c] < fs) {
        fs = first[c];
        cs = c;
      }
    }
    s_frame = fs;
    s_channel = cs;
  }
  __syncthreads();
  const int fs = s_frame, cs = s_channel;
  if (fs < frames) {
    // channels cs.. at frame fs: the newest n measures, zeros before frame 0
    const int64_t g_hit = frame0 + fs;
    for (int c = cs + threadIdx.x; c < C; c += blockDim.x) {
      int j_trigger = n, j_zero = n;
      for (int j = 0; j < n; ++j) {
        const int64_t g = g_hit - j;
        const float m = g < 0 ? 0.f : g >= frame0 ? measures[(size_t)c * frames + (g - frame0)] : ring[(size_t)c * n + g % n];
        if (m >= level && j <= j_trigger + d.gap_len) {
          j_zero = j_trigger = j;
        } else if (m == 0.f && j_trigger >= j_zero) {
          j_zero = j;
        }
      }
      first[c] = min(n - 1, j_zero);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int flush = 0;  // num_measures_to_flush = min(max(num_measures_to_flush, j), n) over channels cs..C-1
      for (int c = cs; c < C; ++c) flush = min(max(flush, (int)first[c]), n);
      const int64_t start = g_hit * d.period - d.fixed_pre_trigger - (int64_t)flush * d.period;
      status[0] = g_hit;
      status[1] = start > 0 ? start : 0;
    }
    return;
  }
  if (threadIdx.x == 0) {
    status[0] = -1;
    status[1] = 0;
  }
  const int keep = frames < n ? frames : n;
  for (int64_t e = threadIdx.x; e < (int64_t)C * keep; e += blockDim.x) {
    const int c = (int)(e / keep), f = frames - keep + (int)(e % keep);
    ring[(size_t)c * n + (frame0 + f) % n] = measures[(size_t)c * frames + f];
  }
  // every frame of [frame0 + frames - n, frame0 + frames) is now in the ring: the older ones were stored by the chunk
  // that ran them, and the scan reads frames before 0 as zeros without touching the ring
}

}  // namespace

size_t vad_workspace_bytes_impl(const b200a_vad_desc* d, int64_t chunk) {
  if (validate_vad(d, chunk) != B200A_OK) return 0;
  return vad_layout(*d, chunk).total;
}

static int check_chunk_call(const b200a_vad_desc* d, int64_t chunk, int64_t frame0, int64_t frames, size_t ws_bytes) {
  const int rc = validate_vad(d, chunk);
  if (rc != B200A_OK) return rc;
  if (frame0 < 0 || frames < 0 || frames > chunk) return B200A_EINVAL;
  if (ws_bytes < vad_layout(*d, chunk).total) return B200A_EWORKSPACE;
  return B200A_OK;
}

int vad_walk_impl(const b200a_vad_desc* d, int64_t chunk, int64_t frame0, int64_t frames, const float* spectrum,
                  const float* cepstrum_window, float* rows, void* ws, size_t ws_bytes, cudaStream_t stream) {
  const int rc = check_chunk_call(d, chunk, frame0, frames, ws_bytes);
  if (rc != B200A_OK) return rc;
  if (spectrum == nullptr || cepstrum_window == nullptr || rows == nullptr || ws == nullptr) return B200A_EINVAL;
  const int band = d->spectrum_end - d->spectrum_start;
  if (frames == 0 || band == 0) return B200A_OK;
  const VadLayout l = vad_layout(*d, chunk);
  const dim3 grid((band + kWalkThreads - 1) / kWalkThreads, d->channels);
  vad_walk_kernel<<<grid, kWalkThreads, 0, stream>>>(*d, chunk, frame0, (int)frames, spectrum, cepstrum_window, rows,
                                                     ws_at<float>(ws, l.spec), ws_at<float>(ws, l.noise));
  return launch_status();
}

int vad_trigger_impl(const b200a_vad_desc* d, int64_t chunk, int64_t frame0, int64_t frames, const float* power,
                     float* measures, void* ws, size_t ws_bytes, cudaStream_t stream) {
  const int rc = check_chunk_call(d, chunk, frame0, frames, ws_bytes);
  if (rc != B200A_OK) return rc;
  if (power == nullptr || measures == nullptr || ws == nullptr) return B200A_EINVAL;
  if (frames == 0) return B200A_OK;
  const VadLayout l = vad_layout(*d, chunk);
  vad_trigger_kernel<<<1, kTriggerThreads, 0, stream>>>(*d, chunk, frame0, (int)frames, power, measures,
                                                        ws_at<int64_t>(ws, l.status), ws_at<float>(ws, l.mean),
                                                        ws_at<float>(ws, l.ring), ws_at<float>(ws, l.addend),
                                                        ws_at<int32_t>(ws, l.first));
  return launch_status();
}

}  // namespace b200a
