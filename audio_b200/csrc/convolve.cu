// fftconvolve (functional/functional.py:2222-2258) as uniformly partitioned overlap-save, and its gradients.
//
// The shorter operand is the filter h (K taps), the longer the signal s (S samples).  The block size B is a power of
// two chosen from K alone (next power of two, clamped to [256, 2048]); every FFT is 2B points long, a real FFT done as
// one B-point complex FFT on the even/odd sample pairs.  A spectrum is stored packed: B float2, slot 0 holding the
// real bins 0 and B, slot k the complex bin k.
//   H_p  = FFT(h[pB, (p+1)B) zero-padded) / 2B               p < P = ceil(K / B), once per distinct filter row
//   S_j  = FFT(s[(j-1)B, (j+1)B))                            zeros outside [0, S), once per distinct signal row
//   out block k = second half of IFFT(sum_p S_{k-p} H_p)     only the blocks that meet [start, start + L)
// Gradients, with g placed at `start` in the full-length range and zero elsewhere:
//   G_j  = FFT(g[jB, (j+2)B)),  S^_q = FFT(s[qB, (q+1)B) zero-padded) / 2B
//   ds block q = first half of IFFT(sum_p G_{q+p} conj(H_p))      (the correlation with h)
//   dh_p       = first half of IFFT(sum_q G_{q+p} conj(S^_q))     (the correlation with s)
// Every sum runs in a fixed order and nothing is atomic, so reruns are bit-identical and a row's result does not depend
// on the other rows.
#include "common.cuh"

namespace b200a {
namespace {

constexpr int kMinLogB = 8, kMaxLogB = 11;
constexpr int64_t kMaxParts = B200A_FFTCONVOLVE_MAX_PARTITIONS;

inline int block_log2(int64_t k) {
  int l = kMinLogB;
  while (l < kMaxLogB && (int64_t(1) << l) < k) ++l;
  return l;
}

inline size_t up256(size_t v) { return (v + 255) & ~size_t(255); }

// Block geometry of one call; output blocks [k0, k0 + nk), forward signal spectra j in [j0, j0 + nj), backward signal
// blocks q < nq and gradient windows j < ng = nq + P - 1.
struct Geo {
  int logb;
  int64_t B, S, K, P;
  bool swap;  // x is the filter (N < M)
  int64_t k0, nk, j0, nj, nq, ng;
};

Geo make_geo(const b200a_fftconvolve_desc& d) {
  Geo g{};
  g.swap = d.n < d.m;
  g.S = g.swap ? d.m : d.n;
  g.K = g.swap ? d.n : d.m;
  g.logb = block_log2(g.K);
  g.B = int64_t(1) << g.logb;
  g.P = (g.K + g.B - 1) / g.B;
  if (d.out_len > 0) {
    g.k0 = d.start / g.B;
    const int64_t k1 = (d.start + d.out_len - 1) / g.B;
    g.nk = k1 - g.k0 + 1;
    g.j0 = g.k0 - g.P + 1 > 0 ? g.k0 - g.P + 1 : 0;
    const int64_t jmax = (g.S - 1) / g.B + 1;  // the last window that meets [0, S)
    const int64_t j1 = k1 < jmax ? k1 : jmax;
    g.nj = j1 >= g.j0 ? j1 - g.j0 + 1 : 0;
  }
  g.nq = (g.S + g.B - 1) / g.B;
  g.ng = g.nq + g.P - 1;
  return g;
}

// Workspace, 256-byte aligned sections:
//   tw    float2 [B]               W_2B^k = exp(-i pi k / B), k < B
//   H     float2 [filter rows][P][B]
//   S     float2 [signal rows][nj][B]     (forward) the signal windows
//   G     float2 [rows][ng][B]            (backward) the gradient windows
//   Sh    float2 [signal rows][nq][B]     (backward) the zero-padded signal blocks
struct ConvLayout {
  size_t tw, h, s, g, sh, total;
};

ConvLayout conv_layout(const b200a_fftconvolve_desc& d, const Geo& g, bool backward) {
  const int64_t frows = g.swap ? d.x_rows : d.y_rows, srows = g.swap ? d.y_rows : d.x_rows;
  const size_t spec = (size_t)g.B * sizeof(float2);
  ConvLayout l{};
  size_t o = 0;
  l.tw = o, o += up256(spec);
  l.h = o, o += up256((size_t)frows * g.P * spec);
  if (!backward) {
    l.s = o, o += up256((size_t)srows * g.nj * spec);
  } else {
    l.g = o, o += up256((size_t)d.rows * g.ng * spec);
    l.sh = o, o += up256((size_t)srows * g.nq * spec);
  }
  l.total = o;
  return l;
}

// ---- the B-point complex FFT in shared memory: Stockham radix-4 stages (+ one radix-2 stage for odd log2 B) -------
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 conjf2(float2 a) { return make_float2(a.x, -a.y); }

// W_2B^e for e in [0, 2B), conjugated for the inverse transform
__device__ __forceinline__ float2 twiddle(const float2* __restrict__ tw, int e, int B, bool inverse) {
  float2 w = e < B ? __ldg(tw + e) : make_float2(-__ldg(tw + e - B).x, -__ldg(tw + e - B).y);
  return inverse ? conjf2(w) : w;
}

// In place on buf[0, B): the unnormalised DFT (inverse: exponent sign +).  B / 4 threads; ends with a barrier.
template <int LOGB>
__device__ void fft_smem(float2* buf, const float2* __restrict__ tw, bool inverse) {
  constexpr int B = 1 << LOGB, Q = B / 4;
  const int j = threadIdx.x;
#pragma unroll 1
  for (int ns = 1; ns * 4 <= B; ns *= 4) {
    const int k = j & (ns - 1);
    const int step = B / (2 * ns);  // W_(4 ns)^(k r) = W_2B^(k r step)
    float2 v[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) v[r] = buf[j + r * Q];
#pragma unroll
    for (int r = 1; r < 4; ++r) v[r] = cmul(v[r], twiddle(tw, k * r * step, B, inverse));
    const float2 a = cadd(v[0], v[2]), b = csub(v[0], v[2]), c = cadd(v[1], v[3]), dd = csub(v[1], v[3]);
    const float2 mid = inverse ? make_float2(-dd.y, dd.x) : make_float2(dd.y, -dd.x);  // -/+ i (v1 - v3)
    __syncthreads();
    const int base = (j - k) * 4 + k;
    buf[base] = cadd(a, c);
    buf[base + ns] = cadd(b, mid);
    buf[base + 2 * ns] = csub(a, c);
    buf[base + 3 * ns] = csub(b, mid);
    __syncthreads();
  }
  if constexpr (LOGB % 2 == 1) {  // ns = B / 2: butterflies (k, k + B/2) in place, twiddle W_2B^(2k)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int k = j + h * Q;
      const float2 v0 = buf[k], v1 = cmul(buf[k + B / 2], twiddle(tw, 2 * k, B, inverse));
      buf[k] = cadd(v0, v1);
      buf[k + B / 2] = csub(v0, v1);
    }
    __syncthreads();
  }
}

// A packed spectrum's product of bins: slot 0 holds two real bins, the others one complex bin each
__device__ __forceinline__ float2 bin_mac(float2 acc, float2 a, float2 b, bool conj_b, bool slot0) {
  if (slot0) return make_float2(fmaf(a.x, b.x, acc.x), fmaf(a.y, b.y, acc.y));
  if (conj_b) b = conjf2(b);
  return make_float2(fmaf(a.x, b.x, fmaf(-a.y, b.y, acc.x)), fmaf(a.x, b.y, fmaf(a.y, b.x, acc.y)));
}

// ---- window spectra: one CTA per (row, window) ---------------------------------------------------------------------
struct SegParams {
  const float* src;          // row r at src + r * row_stride (unit element stride)
  int64_t row_stride, len;   // samples [0, len) exist, zeros elsewhere
  int64_t off0;              // first sample of window 0 (may be negative); window w starts at off0 + w B
  int64_t nseg;              // windows per row
  int win;                   // samples read per window: B (zero-padded) or 2B
  float scale;
  const float2* tw;
  float2* out;               // [rows][nseg][B]
};

template <int LOGB>
__global__ void __launch_bounds__((1 << LOGB) / 4) conv_spectra_kernel(const SegParams p) {
  constexpr int B = 1 << LOGB, Q = B / 4;
  __shared__ float2 buf[B];
  const int64_t row = blockIdx.x / p.nseg, w = blockIdx.x - row * p.nseg;
  const float* src = p.src + row * p.row_stride;
  const int64_t o = p.off0 + w * B;
  for (int n = threadIdx.x; n < B; n += Q) {
    const int64_t i0 = o + 2 * n, i1 = i0 + 1;
    const float a = (2 * n < p.win && i0 >= 0 && i0 < p.len) ? src[i0] : 0.f;
    const float b = (2 * n + 1 < p.win && i1 >= 0 && i1 < p.len) ? src[i1] : 0.f;
    buf[n] = make_float2(a, b);
  }
  __syncthreads();
  fft_smem<LOGB>(buf, p.tw, false);
  // Z = DFT_B(x_even + i x_odd):  X[k] = (Z[k] + conj Z[B-k]) / 2 - i W_2B^k (Z[k] - conj Z[B-k]) / 2
  float2* out = p.out + (size_t)blockIdx.x * B;
  for (int k = threadIdx.x; k <= B / 2; k += Q) {
    if (k == 0) {
      const float2 z = buf[0];
      out[0] = make_float2((z.x + z.y) * p.scale, (z.x - z.y) * p.scale);
      continue;
    }
    const float2 zk = buf[k], zm = buf[B - k];
    const float2 w = __ldg(p.tw + k);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h == 1 && k == B / 2) break;
      const float2 a = h == 0 ? zk : zm, b = h == 0 ? zm : zk;
      const float2 wk = h == 0 ? w : make_float2(-w.x, w.y);  // W_2B^(B-k) = -conj W_2B^k
      const float2 fe = make_float2(0.5f * (a.x + b.x), 0.5f * (a.y - b.y));
      const float2 fo = make_float2(0.5f * (a.y + b.y), -0.5f * (a.x - b.x));  // (a - conj b) / 2i
      const float2 x = cadd(fe, cmul(wk, fo));
      out[h == 0 ? k : B - k] = make_float2(x.x * p.scale, x.y * p.scale);
    }
  }
}

// ---- products of spectra and the inverse transform -----------------------------------------------------------------
// buf holds a packed Hermitian spectrum Y; leaves z with z[n] = 2B (y[2n] + i y[2n+1]), y = IDFT_2B(Y).
template <int LOGB>
__device__ void inverse_real(float2* buf, const float2* __restrict__ tw) {
  constexpr int B = 1 << LOGB, Q = B / 4;
  __syncthreads();
  // Z'[k] = (Y[k] + conj Y[B-k]) + i W_2B^-k (Y[k] - conj Y[B-k]); each thread owns the pair (k, B - k)
  for (int k = threadIdx.x; k <= B / 2; k += Q) {
    if (k == 0) {
      const float2 y = buf[0];
      buf[0] = make_float2(y.x + y.y, y.x - y.y);
      continue;
    }
    const float2 yk = buf[k], ym = buf[B - k];
    const float2 w = __ldg(tw + k);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h == 1 && k == B / 2) break;
      const float2 a = h == 0 ? yk : ym, b = h == 0 ? ym : yk;
      const float2 wi = h == 0 ? conjf2(w) : make_float2(-w.x, -w.y);  // W_2B^-(B-k) = -W_2B^k
      const float2 e = make_float2(a.x + b.x, a.y - b.y), o = make_float2(a.x - b.x, a.y + b.y);
      const float2 io = cmul(wi, o);
      buf[h == 0 ? k : B - k] = make_float2(e.x - io.y, e.y + io.x);
    }
  }
  __syncthreads();
  fft_smem<LOGB>(buf, tw, true);
}

// out[n] = a[n] * c[n] summed in a fixed order (FWD: windows blk - q of a, BWD: windows blk + q of a times conj c), then
// the inverse transform and one half of each block written out.
//   forward        : a = S (row a_index[r]), c = H (row c_index[r]), q < P,  second half -> out block k
//   signal gradient: a = G (row r),           c = H (row c_index[r]), q < P,  first half  -> ds block q
//   filter gradient: a = G (row r),           c = S^ (row c_index[r]), q < nq, first half -> dh_p
struct BlockParams {
  const float2* a;
  const float2* c;
  const int64_t* a_index;  // null: row r of `a` belongs to output row r
  const int64_t* c_index;
  int64_t na, a0;          // windows per row of `a` and the window index of its first
  int64_t nc;              // spectra per row of `c`, all summed
  int64_t nblk, blk0;      // blocks per output row and the first
  const float2* tw;
  float* out;              // row r at out + r * out_len
  int64_t out_len, out_off;  // block b covers out[b B - out_off, (b + 1) B - out_off), clipped to [0, out_len)
};

template <int LOGB, bool BWD>
__global__ void __launch_bounds__((1 << LOGB) / 4) conv_block_kernel(const BlockParams p) {
  constexpr int B = 1 << LOGB, Q = B / 4;
  __shared__ float2 buf[B];
  const int64_t row = blockIdx.x / p.nblk;
  const int64_t blk = p.blk0 + (blockIdx.x - row * p.nblk);
  const int64_t arow = p.a_index == nullptr ? row : p.a_index[row];
  const float2* as = p.a + (size_t)arow * p.na * B;
  const float2* cs = p.c + (size_t)p.c_index[row] * p.nc * B;
  float2 acc[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) acc[i] = make_float2(0.f, 0.f);
  for (int64_t q = 0; q < p.nc; ++q) {
    const int64_t j = (BWD ? blk + q : blk - q) - p.a0;
    if (j < 0 || j >= p.na) continue;
    const float2* ap = as + (size_t)j * B;
    const float2* cp = cs + (size_t)q * B;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = threadIdx.x + i * Q;
      acc[i] = bin_mac(acc[i], __ldg(ap + k), __ldg(cp + k), BWD, k == 0);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) buf[threadIdx.x + i * Q] = acc[i];
  inverse_real<LOGB>(buf, p.tw);
  // z[n] = (y[2n], y[2n+1]): the forward keeps samples [B, 2B) of the window, the gradients [0, B)
  float* out = p.out + row * p.out_len;
  const int64_t first = blk * B - p.out_off;
  for (int t = threadIdx.x; t < B; t += Q) {
    const int64_t i = first + t;
    if (i < 0 || i >= p.out_len) continue;
    const float2 z = buf[(BWD ? 0 : B / 2) + t / 2];
    out[i] = (t & 1) ? z.y : z.x;
  }
}

__global__ void conv_twiddle_kernel(float2* tw, int B) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= B) return;
  double s, c;
  sincospi((double)k / B, &s, &c);
  tw[k] = make_float2((float)c, (float)-s);
}

// Filter and signal operands of a call: rows, stride and length of each.
struct Operands {
  const float* f;
  const float* s;
  int64_t f_rows, s_rows, f_stride, s_stride;
  const int64_t* f_index;
  const int64_t* s_index;
};

Operands operands(const b200a_fftconvolve_desc& d, const Geo& g, const float* x, const float* y) {
  if (g.swap) return {x, y, d.x_rows, d.y_rows, d.x_stride, d.y_stride, d.x_index, d.y_index};
  return {y, x, d.y_rows, d.x_rows, d.y_stride, d.x_stride, d.y_index, d.x_index};
}

template <int LOGB>
int spectra(const float* src, int64_t rows, int64_t stride, int64_t len, int64_t off0, int64_t nseg, int win,
            float scale, const float2* tw, float2* out, cudaStream_t stream) {
  if (rows == 0 || nseg == 0) return B200A_OK;
  const SegParams sp{src, stride, len, off0, nseg, win, scale, tw, out};
  // static shared memory only: launched directly (launch_kernel raises the dynamic limit to the whole 227 KB)
  conv_spectra_kernel<LOGB><<<(unsigned)(rows * nseg), (1 << LOGB) / 4, 0, stream>>>(sp);
  return launch_status();
}

template <int LOGB>
int run_logb(const b200a_fftconvolve_desc& d, const Geo& g, const ConvLayout& l, const float* x, const float* y,
             float* out, void* ws, cudaStream_t stream) {
  constexpr int B = 1 << LOGB;
  const Operands o = operands(d, g, x, y);
  float2* tw = ws_at<float2>(ws, l.tw);
  float2* hs = ws_at<float2>(ws, l.h);
  float2* ss = ws_at<float2>(ws, l.s);
  conv_twiddle_kernel<<<(B + 255) / 256, 256, 0, stream>>>(tw, B);
  int rc = launch_status();
  if (rc == B200A_OK) rc = spectra<LOGB>(o.f, o.f_rows, o.f_stride, g.K, 0, g.P, B, 1.f / (2 * B), tw, hs, stream);
  if (rc == B200A_OK)
    rc = spectra<LOGB>(o.s, o.s_rows, o.s_stride, g.S, (g.j0 - 1) * B, g.nj, 2 * B, 1.f, tw, ss, stream);
  if (rc != B200A_OK) return rc;
  const BlockParams bp{ss, hs, o.s_index, o.f_index, g.nj, g.j0, g.P, g.nk, g.k0, tw, out, d.out_len, d.start};
  conv_block_kernel<LOGB, false><<<(unsigned)(d.rows * g.nk), B / 4, 0, stream>>>(bp);
  return launch_status();
}

template <int LOGB>
int backward_logb(const b200a_fftconvolve_desc& d, const Geo& g, const ConvLayout& l, const float* x, const float* y,
                  const float* grad, float* grad_x, float* grad_y, void* ws, cudaStream_t stream) {
  constexpr int B = 1 << LOGB;
  const Operands o = operands(d, g, x, y);
  float2* tw = ws_at<float2>(ws, l.tw);
  float2* hs = ws_at<float2>(ws, l.h);
  float2* gs = ws_at<float2>(ws, l.g);
  float2* sh = ws_at<float2>(ws, l.sh);
  float* ds = g.swap ? grad_y : grad_x;
  float* dh = g.swap ? grad_x : grad_y;
  conv_twiddle_kernel<<<(B + 255) / 256, 256, 0, stream>>>(tw, B);
  int rc = launch_status();
  const float inv = 1.f / (2 * B);
  if (rc == B200A_OK) rc = spectra<LOGB>(o.f, o.f_rows, o.f_stride, g.K, 0, g.P, B, inv, tw, hs, stream);
  if (rc == B200A_OK) rc = spectra<LOGB>(o.s, o.s_rows, o.s_stride, g.S, 0, g.nq, B, inv, tw, sh, stream);
  // g at `start` of the full range: window j of g_full starts at jB, at jB - start in the grad row
  if (rc == B200A_OK) rc = spectra<LOGB>(grad, d.rows, d.out_len, d.out_len, -d.start, g.ng, 2 * B, 1.f, tw, gs, stream);
  if (rc != B200A_OK) return rc;
  const BlockParams bs{gs, hs, nullptr, o.f_index, g.ng, 0, g.P, g.nq, 0, tw, ds, g.S, 0};
  conv_block_kernel<LOGB, true><<<(unsigned)(d.rows * g.nq), B / 4, 0, stream>>>(bs);
  rc = launch_status();
  if (rc != B200A_OK) return rc;
  const BlockParams bh{gs, sh, nullptr, o.s_index, g.ng, 0, g.nq, g.P, 0, tw, dh, g.K, 0};
  conv_block_kernel<LOGB, true><<<(unsigned)(d.rows * g.P), B / 4, 0, stream>>>(bh);
  return launch_status();
}

// B200A_OK with `work` false when there is nothing to enqueue
int check_desc(const b200a_fftconvolve_desc* d, bool& work) {
  work = false;
  if (d == nullptr || d->n < 1 || d->m < 1 || d->rows < 0 || d->x_rows < 1 || d->y_rows < 1 || d->out_len < 0 ||
      d->start < 0 || d->x_stride < 0 || d->y_stride < 0)
    return B200A_EINVAL;
  const int64_t full = d->n + d->m - 1;
  if (full > INT32_MAX) return B200A_EUNSUPPORTED;
  if (d->start + d->out_len > full) return B200A_EINVAL;
  const Geo g = make_geo(*d);
  if (g.P > kMaxParts) return B200A_EUNSUPPORTED;
  if (d->rows * (g.nk > g.ng ? g.nk : g.ng) > INT32_MAX || (g.swap ? d->y_rows : d->x_rows) * g.ng > INT32_MAX)
    return B200A_EUNSUPPORTED;  // grid.x
  work = d->rows > 0 && d->out_len > 0;
  if (work && (d->x_index == nullptr || d->y_index == nullptr)) return B200A_EINVAL;
  return B200A_OK;
}

}  // namespace

size_t fftconvolve_workspace_bytes_impl(const b200a_fftconvolve_desc* d, bool backward) {
  bool work = false;
  if (check_desc(d, work) != B200A_OK) return 0;
  return conv_layout(*d, make_geo(*d), backward).total;
}

int fftconvolve_run_impl(const b200a_fftconvolve_desc* d, const float* x, const float* y, float* out, void* ws,
                         size_t ws_bytes, cudaStream_t stream) {
  bool work = false;
  const int rc = check_desc(d, work);
  if (rc != B200A_OK || !work) return rc;
  if (x == nullptr || y == nullptr || out == nullptr || ws == nullptr) return B200A_EINVAL;
  const Geo g = make_geo(*d);
  const ConvLayout l = conv_layout(*d, g, false);
  if (ws_bytes < l.total) return B200A_EWORKSPACE;
  switch (g.logb) {
    case 8: return run_logb<8>(*d, g, l, x, y, out, ws, stream);
    case 9: return run_logb<9>(*d, g, l, x, y, out, ws, stream);
    case 10: return run_logb<10>(*d, g, l, x, y, out, ws, stream);
    default: return run_logb<11>(*d, g, l, x, y, out, ws, stream);
  }
}

int fftconvolve_backward_impl(const b200a_fftconvolve_desc* d, const float* x, const float* y, const float* grad,
                              float* grad_x, float* grad_y, void* ws, size_t ws_bytes, cudaStream_t stream) {
  bool work = false;
  const int rc = check_desc(d, work);
  if (rc != B200A_OK || d->rows == 0) return rc;
  if (grad_x == nullptr || grad_y == nullptr) return B200A_EINVAL;
  if (!work) {  // empty output: both gradients are zero
    if (cudaMemsetAsync(grad_x, 0, (size_t)d->rows * d->n * 4, stream) != cudaSuccess ||
        cudaMemsetAsync(grad_y, 0, (size_t)d->rows * d->m * 4, stream) != cudaSuccess)
      return B200A_ECUDA;
    return B200A_OK;
  }
  if (x == nullptr || y == nullptr || grad == nullptr || ws == nullptr) return B200A_EINVAL;
  const Geo g = make_geo(*d);
  const ConvLayout l = conv_layout(*d, g, true);
  if (ws_bytes < l.total) return B200A_EWORKSPACE;
  switch (g.logb) {
    case 8: return backward_logb<8>(*d, g, l, x, y, grad, grad_x, grad_y, ws, stream);
    case 9: return backward_logb<9>(*d, g, l, x, y, grad, grad_x, grad_y, ws, stream);
    case 10: return backward_logb<10>(*d, g, l, x, y, grad, grad_x, grad_y, ws, stream);
    default: return backward_logb<11>(*d, g, l, x, y, grad, grad_x, grad_y, ws, stream);
  }
}

}  // namespace b200a
