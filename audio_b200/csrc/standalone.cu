// Stand-alone stages: MelScale on an existing spectrogram, AmplitudeToDB, fill.
// These exist so the drop-in MelScale / AmplitudeToDB modules work on their own; the fused
// front-end kernels never call them.
// Reference: transforms/_transforms.py:403-415 (MelScale.forward), functional.py:356-404.
#include <cmath>

#include "common.cuh"

namespace b200a {

// Lanes run along the frame axis (contiguous in the reference's logical (bins, frames) layout).
__global__ void __launch_bounds__(256)
apply_fbank_kernel(const float* __restrict__ spec, int64_t n_bins, int64_t frames, int64_t stride_row,
                   int64_t stride_bin, int64_t stride_frame, const float* __restrict__ fb, int n_filters,
                   float* __restrict__ out) {
  const int64_t row = blockIdx.y;
  const int64_t t = (int64_t)blockIdx.x * 32 + (threadIdx.x & 31);
  if (t >= frames) return;
  const float* s = spec + row * stride_row + t * stride_frame;
  for (int m = threadIdx.x >> 5; m < n_filters; m += blockDim.x >> 5) {
    float acc = 0.f;
    for (int64_t k = 0; k < n_bins; ++k) acc = fmaf(s[k * stride_bin], fb[k * n_filters + m], acc);
    out[(row * frames + t) * n_filters + m] = acc;
  }
}

__global__ void __launch_bounds__(256)
to_db_kernel(const float* __restrict__ x, int64_t group_elems, float mult, float amin, float offset,
             float* group_max, float* __restrict__ out) {
  const int64_t g = blockIdx.y;
  const float* xi = x + g * group_elems;
  float* oi = out + g * group_elems;
  float local = -CUDART_INF_F;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < group_elems; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = db_value(xi[i], mult, amin, offset);
    oi[i] = v;
    local = fmaxf(local, v);
  }
  if (group_max != nullptr) {
    local = warp_max(local);
    if ((threadIdx.x & 31) == 0 && local > -CUDART_INF_F) atomic_max_f32(group_max + g, local);
  }
}

__global__ void __launch_bounds__(256)
clamp_floor_kernel(float* __restrict__ y, int64_t group_elems, const float* __restrict__ group_max, float top_db) {
  const int64_t g = blockIdx.y;
  const float floor_v = group_max[g] - top_db;
  float* yi = y + g * group_elems;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < group_elems; i += (int64_t)gridDim.x * blockDim.x)
    yi[i] = fmaxf(yi[i], floor_v);
}

// out[i] = pairs[i][0] / pairs[i][1]  (SpectralCentroid: sum f|X| / sum |X|, functional.py:1257-1299)
__global__ void ratio_kernel(const float2* __restrict__ pairs, int64_t n, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float2 v = pairs[i];
    out[i] = v.x / v.y;
  }
}

__global__ void fill_kernel(float* dst, int64_t n, float v) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = v;
}

int ratio_impl(const float* pairs, int64_t n, float* out, cudaStream_t stream) {
  if (n <= 0) return B200A_OK;
  ratio_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float2*>(pairs), n, out);
  return launch_status();
}

int fill_impl(float* dst, int64_t n, float v, cudaStream_t stream) {
  if (n <= 0) return B200A_OK;
  fill_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(dst, n, v);
  return launch_status();
}

int apply_fbank_impl(const float* spec, int64_t rows, int64_t n_bins, int64_t frames, int64_t stride_row,
                     int64_t stride_bin, int64_t stride_frame, const float* fb, int n_filters, float* out,
                     cudaStream_t stream) {
  if (rows == 0 || frames == 0) return B200A_OK;
  if (rows > 65535) return B200A_EUNSUPPORTED;
  dim3 grid((unsigned)((frames + 31) / 32), (unsigned)rows);
  apply_fbank_kernel<<<grid, 256, 0, stream>>>(spec, n_bins, frames, stride_row, stride_bin, stride_frame, fb, n_filters, out);
  return launch_status();
}

int amplitude_to_db_impl(const float* x, int64_t groups, int64_t group_elems, float mult, float amin, float offset,
                         float top_db, float* scratch, float* out, cudaStream_t stream) {
  if (groups == 0 || group_elems == 0) return B200A_OK;
  if (groups > 65535) return B200A_EUNSUPPORTED;
  const bool clamp = top_db >= 0.f;
  if (clamp) {
    if (scratch == nullptr) return B200A_EINVAL;
    int rc = fill_impl(scratch, groups, -INFINITY, stream);
    if (rc != B200A_OK) return rc;
  }
  const int64_t bx = sm_capped_grid((group_elems + 255) / 256, 8);  // 8 CTAs per SM, grid-stride beyond
  if (bx < 0) return B200A_ECUDA;
  dim3 grid((unsigned)bx, (unsigned)groups);
  to_db_kernel<<<grid, 256, 0, stream>>>(x, group_elems, mult, amin, offset, clamp ? scratch : nullptr, out);
  if (clamp) clamp_floor_kernel<<<grid, 256, 0, stream>>>(out, group_elems, scratch, top_db);
  return launch_status();
}

// x[r][t][c] -= mean over t.  One CTA per (matrix, group of 32 columns): warp w sums frames w, w+8, ... of its
// 32 columns (coalesced rows), the partial sums meet in shared memory, then the same sweep subtracts.
__global__ void __launch_bounds__(256) subtract_column_mean_kernel(float* __restrict__ x, int64_t frames, int64_t width,
                                                                   int64_t col_groups) {
  __shared__ float s_part[8][32];
  const int64_t r = blockIdx.x / col_groups, cg = blockIdx.x - r * col_groups;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t c = cg * 32 + lane;
  float* base = x + r * frames * width;
  float sum = 0.f;
  if (c < width)
    for (int64_t t = warp; t < frames; t += 8) sum += base[t * width + c];
  s_part[warp][lane] = sum;
  __syncthreads();
  float mean = 0.f;
  for (int w = 0; w < 8; ++w) mean += s_part[w][lane];
  mean /= (float)frames;
  if (c < width)
    for (int64_t t = warp; t < frames; t += 8) base[t * width + c] -= mean;
}

int subtract_column_mean_impl(float* x, int64_t rows, int64_t frames, int64_t width, cudaStream_t stream) {
  const int64_t col_groups = (width + 31) / 32;
  const int64_t grid = rows * col_groups;
  if (grid > 0x7fffffffLL) return B200A_EUNSUPPORTED;
  subtract_column_mean_kernel<<<(unsigned)grid, 256, 0, stream>>>(x, frames, width, col_groups);
  return launch_status();
}

// Griffin-Lim phase step (functional.py:330-341): proj = mag^(1/power) * angles,
//   angles = d / (|d| + 1e-16), d = rebuilt - momentum * tprev   (angles = 1 when there is no rebuilt yet).
// mag: logical [rows][bins][frames] with element strides; rebuilt / tprev / proj: frame-major [rows][frames][bins] complex.
__global__ void __launch_bounds__(256) griffinlim_update_kernel(const float* __restrict__ mag, int64_t ms_row, int64_t ms_bin,
                                                                int64_t ms_frame, float inv_power,
                                                                const float2* __restrict__ rebuilt,
                                                                const float2* __restrict__ tprev, float momentum, int normalize,
                                                                float2* __restrict__ proj, int64_t bins, int64_t frames,
                                                                int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = i % bins, rt = i / bins;
    const int64_t t = rt % frames, r = rt / frames;
    float m = mag[r * ms_row + k * ms_bin + t * ms_frame];
    m = inv_power == 1.f ? m : (inv_power == 0.5f ? sqrtf(m) : powf(m, inv_power));
    float2 a = make_float2(1.f, 0.f);
    if (rebuilt != nullptr) {
      float2 d = rebuilt[i];
      if (tprev != nullptr) {
        const float2 p = tprev[i];
        d.x -= momentum * p.x;
        d.y -= momentum * p.y;
      }
      const float inv = normalize ? 1.f / (hypotf(d.x, d.y) + 1e-16f) : 1.f;
      a = make_float2(d.x * inv, d.y * inv);
    }
    proj[i] = make_float2(m * a.x, m * a.y);
  }
}

int griffinlim_update_impl(const float* mag, int64_t ms_row, int64_t ms_bin, int64_t ms_frame, float inv_power,
                           const float* rebuilt, const float* tprev, float momentum, int normalize, float* proj,
                           int64_t rows, int64_t bins, int64_t frames, cudaStream_t stream) {
  const int64_t total = rows * bins * frames;
  const int64_t grid = sm_capped_grid((total + 255) / 256, 16);  // 16 CTAs per SM, grid-stride beyond
  if (grid < 0) return B200A_ECUDA;
  griffinlim_update_kernel<<<(unsigned)grid, 256, 0, stream>>>(mag, ms_row, ms_bin, ms_frame, inv_power,
                                                              reinterpret_cast<const float2*>(rebuilt),
                                                              reinterpret_cast<const float2*>(tprev), momentum, normalize,
                                                              reinterpret_cast<float2*>(proj), bins, frames, total);
  return launch_status();
}

// The time grid of F.phase_vocoder (torch.arange(0, frames_in, rate, dtype=float32)): step t sits at ts = float(rate * t)
// of the input; its neighbours are frames trunc(ts) and trunc(ts + 1), the latter computed in float (so not always
// i0 + 1: it is i0 + 2 when ts + 1 rounds up to the next integer); alpha = ts mod 1.  The forward and its adjoint both
// take their neighbours from here, so they make the same decisions bit for bit.
struct VocoderStep {
  int64_t i0, i1;
  float alpha;
};

__device__ __forceinline__ VocoderStep vocoder_step(double rate, int64_t t) {
  const float ts = (float)(rate * (double)t);
  VocoderStep s;
  s.alpha = fmodf(ts, 1.0f);
  s.i0 = (int64_t)ts;
  s.i1 = (int64_t)(ts + 1.0f);
  return s;
}

// F.phase_vocoder (functional.py:713-803): one thread per (row, bin) walks the output frames in order, carrying the
// accumulated phase (the reference's cumsum); consecutive threads are consecutive bins of the frame-major output.
// Step t' interpolates frames vocoder_step(t').i0 / .i1 (frames >= frames_in are the two zero frames the reference pads).
__global__ void __launch_bounds__(128) phase_vocoder_kernel(const float2* __restrict__ spec, int64_t s_row, int64_t s_bin,
                                                            int64_t s_frame, int64_t bins, int64_t frames_in, double rate,
                                                            const float* __restrict__ phase_advance,
                                                            float2* __restrict__ out, int64_t frames_out) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = blockIdx.y;
  if (k >= bins) return;
  const float2* sp = spec + r * s_row + k * s_bin;
  float2* o = out + r * frames_out * bins + k;
  const float pa = phase_advance[k];
  const float2 first = sp[0];
  // the accumulated phase grows to thousands of radians: carried in double so that its round-off (1e-3 rad in the
  // reference's float32 cumsum) does not reach the output
  double acc = (double)atan2f(first.y, first.x);  // phase_0
  // the neighbours of step t + 1 are fetched before step t's arithmetic, so the global-load latency of the walk hides
  // behind the transcendental chain instead of adding to it
  auto fetch = [&](int64_t t, float& alpha, float2& z0, float2& z1) {
    const VocoderStep s = vocoder_step(rate, t);
    alpha = s.alpha;
    z0 = (t < frames_out && s.i0 < frames_in) ? sp[s.i0 * s_frame] : make_float2(0.f, 0.f);
    z1 = (t < frames_out && s.i1 < frames_in) ? sp[s.i1 * s_frame] : make_float2(0.f, 0.f);
  };
  float alpha, alpha_n;
  float2 z0, z1, z0n, z1n;
  fetch(0, alpha, z0, z1);
  for (int64_t t = 0; t < frames_out; ++t) {
    fetch(t + 1, alpha_n, z0n, z1n);
    const float n0 = hypotf(z0.x, z0.y), n1 = hypotf(z1.x, z1.y);
    const float mag = alpha * n1 + (1.f - alpha) * n0;
    float sn, cs;
    sincosf((float)(acc - 6.283185307179586 * rint(acc / 6.283185307179586)), &sn, &cs);
    o[t * bins] = make_float2(mag * cs, mag * sn);
    // the expected advance reaches hundreds of radians at the top bins: subtract and wrap in double as well
    double ph = (double)atan2f(z1.y, z1.x) - (double)atan2f(z0.y, z0.x) - (double)pa;
    ph -= 6.283185307179586 * rint(ph / 6.283185307179586);
    acc += ph + (double)pa;
    alpha = alpha_n;
    z0 = z0n;
    z1 = z1n;
  }
}

int phase_vocoder_impl(const float* spec, int64_t s_row, int64_t s_bin, int64_t s_frame, int64_t rows, int64_t bins,
                       int64_t frames_in, double rate, const float* phase_advance, float* out, int64_t frames_out,
                       cudaStream_t stream) {
  if (rows > 65535) return B200A_EUNSUPPORTED;
  phase_vocoder_kernel<<<dim3((unsigned)((bins + 127) / 128), (unsigned)rows), 128, 0, stream>>>(
      reinterpret_cast<const float2*>(spec), s_row, s_bin, s_frame, bins, frames_in, rate, phase_advance,
      reinterpret_cast<float2*>(out), frames_out);
  return launch_status();
}

// Adjoint of phase_vocoder_kernel (include/b200audio.h has the formula).  One thread per (row, bin), as the forward,
// walks the output frames backwards, t = frames_out - 1 ... 0, carrying the suffix sum S of a_t = dL/dphi_t (the
// adjoint of the phase cumsum) and the pending accumulators M (magnitude) and P (phase) of the input frames the walk
// can still reach: frames top, top - 1, top - 2 with top = min(frames_in - 1, i1(t)), since i1 - i0 is 1 or 2 and both
// only decrease along the walk.  A frame is written once, when the walk passes below it; frames no step touches are
// written as 0.  S, M and P are double: S sums frames_out terms, and the forward carries its phase in double too.
__global__ void __launch_bounds__(128) phase_vocoder_backward_kernel(
    const float2* __restrict__ spec, int64_t s_row, int64_t s_bin, int64_t s_frame, int64_t bins, int64_t frames_in,
    double rate, const float2* __restrict__ out, const float2* __restrict__ grad, int64_t g_row, int64_t g_bin,
    int64_t g_frame, float2* __restrict__ grad_spec, int64_t frames_out) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = blockIdx.y;
  if (k >= bins) return;
  const float2* sp = spec + r * s_row + k * s_bin;
  const float2* o = out + r * frames_out * bins + k;
  const float2* g = grad + r * g_row + k * g_bin;
  float2* gx = grad_spec + r * frames_in * bins + k;
  // grad_X = sgn(X) M + i X / |X|^2 P = (X / |X|) (M + i P / |X|); exactly 0 at X = 0 (torch's abs / angle backward)
  auto flush = [&](int64_t i, double m, double p) {
    const float2 x = sp[i * s_frame];
    const double n2 = (double)x.x * x.x + (double)x.y * x.y;
    float2 v = make_float2(0.f, 0.f);
    if (n2 > 0.0) {
      const double inv = 1.0 / sqrt(n2), cr = x.x * inv, ci = x.y * inv, q = p * inv;
      v = make_float2((float)(cr * m - ci * q), (float)(ci * m + cr * q));
    }
    gx[i * bins] = v;
  };
  double S = 0.0;
  double m0 = 0.0, p0 = 0.0, m1 = 0.0, p1 = 0.0, m2 = 0.0, p2 = 0.0;  // pending frames top, top - 1, top - 2
  int64_t top = frames_in - 1;
  auto add = [&](int64_t i, double dm, double dp) {  // contributions to the pad frames (i > top) are dropped
    const int64_t d = top - i;
    if (d == 0) {
      m0 += dm;
      p0 += dp;
    } else if (d == 1) {
      m1 += dm;
      p1 += dp;
    } else if (d == 2) {
      m2 += dm;
      p2 += dp;
    }
  };
  // g_t and o_t of the next step are fetched before this step's arithmetic, as the forward prefetches its neighbours
  float2 gn = g[(frames_out - 1) * g_frame], on = o[(frames_out - 1) * bins];
  for (int64_t t = frames_out - 1; t >= 0; --t) {
    const float2 gt = gn, ot = on;
    if (t > 0) {
      gn = g[(t - 1) * g_frame];
      on = o[(t - 1) * bins];
    }
    const VocoderStep st = vocoder_step(rate, t);
    while (top > st.i1) {  // no step t' <= t reaches these frames any more
      flush(top, m0, p0);
      m0 = m1;
      p0 = p1;
      m1 = m2;
      p1 = p2;
      m2 = 0.0;
      p2 = 0.0;
      --top;
    }
    // torch's polar_backward on the result: a = Re(conj(g) i o), m = Re(conj(g) sgn(o))
    const double a = (double)gt.y * ot.x - (double)gt.x * ot.y;
    const double on2 = (double)ot.x * ot.x + (double)ot.y * ot.y;
    const double m = on2 > 0.0 ? ((double)gt.x * ot.x + (double)gt.y * ot.y) / sqrt(on2) : 0.0;
    const double al = (double)st.alpha;
    // mag_t = alpha n(i1) + (1 - alpha) n(i0); psi_t (which reaches phi_u for u > t, so it sees S_{t+1}) adds
    // angle(i1) - angle(i0)
    add(st.i1, al * m, S);
    add(st.i0, (1.0 - al) * m, -S);
    S += a;
  }
  p0 += top == 0 ? S : 0.0;  // phi_0 = angle(X_0): frame 0 gets S_0
  p1 += top == 1 ? S : 0.0;
  while (top >= 0) {
    flush(top, m0, p0);
    m0 = m1;
    p0 = p1;
    m1 = m2;
    p1 = p2;
    m2 = 0.0;
    p2 = 0.0;
    --top;
  }
}

int phase_vocoder_backward_impl(const float* spec, int64_t s_row, int64_t s_bin, int64_t s_frame, int64_t rows,
                                int64_t bins, int64_t frames_in, double rate, const float* out, const float* grad,
                                int64_t g_row, int64_t g_bin, int64_t g_frame, float* grad_spec, int64_t frames_out,
                                cudaStream_t stream) {
  if (rows > 65535) return B200A_EUNSUPPORTED;
  phase_vocoder_backward_kernel<<<dim3((unsigned)((bins + 127) / 128), (unsigned)rows), 128, 0, stream>>>(
      reinterpret_cast<const float2*>(spec), s_row, s_bin, s_frame, bins, frames_in, rate,
      reinterpret_cast<const float2*>(out), reinterpret_cast<const float2*>(grad), g_row, g_bin, g_frame,
      reinterpret_cast<float2*>(grad_spec), frames_out);
  return launch_status();
}

}  // namespace b200a
