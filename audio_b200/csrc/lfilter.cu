// lfilter (functional/filtering.py:1032-1099) and its gradients as a chunked linear scan.  The reference runs one
// thread per row over all samples; here a row is cut into tiles of kTileChunks chunks of kChunk samples.  Each thread
// runs the recurrence serially over one chunk staged in shared memory, and chunks are joined through the N-sample
// output history s = (y[t-1], ..., y[t-N]):  s_{c+1} = M^L s_c + z_c, with z_c the chunk's end history from a zero
// start and M the companion matrix of the normalised denominator.  M, its powers and every carry are DOUBLE, built from
// the float32 a^ promoted to double (so the carries match the recurrence the chunks actually run); a chunk's starting
// history is rounded to float32 once.  Launches per call: prep (a^, b^, powers of M) -> per-tile aggregates with an
// in-tile Kogge-Stone scan -> a fixed-order scan over each row's tiles -> the chunks re-run from their true histories.
#include <cmath>

#include "common.cuh"
#include "ptx.cuh"

namespace b200a {
namespace {

constexpr int kMaxOrder = B200A_LFILTER_MAX_ORDER;
constexpr int kChunk = 32;                       // samples per thread (L); a function of nothing, so of N alone
constexpr int kTileChunks = 128;                 // threads (chunks) per tile CTA
constexpr int kTile = kChunk * kTileChunks;      // samples per tile
constexpr int kLevels = 7;                       // log2(kTileChunks): Kogge-Stone steps of the in-tile scan
constexpr int kPowers = kLevels + 1;             // M^(L 2^j), j = 0..kLevels; the last carries a whole tile
constexpr int kPitch = kChunk + 1;               // odd chunk pitch: lane c reads bank (c + k) % 32 at step k
constexpr int kCoefStride = 2 * (kMaxOrder + 1) + 2;  // floats per filter: a^[17] | b^[17] | pad
constexpr int kRedThreads = 256;
static_assert(kTileChunks == 1 << kLevels, "tile = 2^levels chunks");
static_assert(kChunk == 32, "M^L is built by five squarings");

// The padded state size the kernels are compiled for: orders round up to 1, 2, 4, 8, 16 with zero coefficients.
inline int padded_order(int n) { return n == 0 ? 0 : n <= 1 ? 1 : n <= 2 ? 2 : n <= 4 ? 4 : n <= 8 ? 8 : 16; }

// Workspace, 256-byte aligned sections:
//   coef  float  [F][kCoefStride]        a^ and b^ (zero past the order)
//   pows  double [F][kPowers][NP*NP]     M^(L 2^j)
//   carry double [rows][tiles][NP]       tile aggregates, then the tiles' starting histories
//   (backward) u    float  [rows][length]           the IIR adjoint of the masked gradient
//   (backward) part double [rows][tiles][2 NP + 1]  per-(row, tile) correlation partials: d a^_1..N | d b^_0..N
//   (backward) gnorm double [F][2 NP + 1]           the reduced normalised gradients
struct LfLayout {
  size_t coef, pows, carry, u, part, gnorm, total;
};

inline size_t up256(size_t v) { return (v + 255) & ~size_t(255); }

LfLayout lf_layout(int64_t rows, int64_t length, int np, int n_filters, bool backward) {
  const int64_t tiles = (length + kTile - 1) / kTile;
  LfLayout l{};
  size_t o = 0;
  l.coef = o, o += up256((size_t)n_filters * kCoefStride * 4);
  l.pows = o, o += up256((size_t)n_filters * kPowers * np * np * 8);
  l.carry = o, o += up256((size_t)rows * tiles * np * 8);
  if (backward) {
    l.u = o, o += up256((size_t)rows * length * 4);
    l.part = o, o += up256((size_t)rows * tiles * (2 * np + 1) * 8);
    l.gnorm = o, o += up256((size_t)n_filters * (2 * np + 1) * 8);
  }
  l.total = o;
  return l;
}

struct LfParams {
  const float* x;        // input rows (unit element stride)
  const float* mask_y;   // adjoint pass: the forward's unclamped y gating x by the clamp mask (contiguous), or null
  const float* coef;
  const double* pows;
  double* carry;
  float* y;              // output rows, contiguous [rows][length]
  float* y_raw;          // unclamped copy, or null
  int64_t s_batch, s_filter, length, tiles, rows;
  int n_filters;
  int reverse;           // 1: the recurrence runs from length-1 downward
  int fir;               // 0: IIR only (the adjoint: v = x)
  int clamp;
};

__device__ inline const float* row_ptr(const float* base, int64_t row, int n_filters, int64_t s_batch,
                                       int64_t s_filter) {
  const int64_t bi = row / n_filters;
  return base + bi * s_batch + (row - bi * n_filters) * s_filter;
}

__device__ inline int64_t phys(int64_t tau, int64_t length, int reverse) { return reverse ? length - 1 - tau : tau; }

// torch.clamp(y, -1, 1): NaN passes through
__device__ inline float clamp1(float v) { return v < -1.f ? -1.f : (v > 1.f ? 1.f : v); }

// ---- prep: a^, b^ and the powers of M, one CTA per filter ---------------------------------------------------------
template <int NP>
__global__ void __launch_bounds__(256) lfilter_prep_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                           int n_order, float* coef, double* pows) {
  __shared__ double sa[kMaxOrder * kMaxOrder];
  __shared__ float sah[kMaxOrder + 1];
  const int f = blockIdx.x, tid = threadIdx.x;
  const float a0 = a[(int64_t)f * n_order];
  if (tid <= kMaxOrder) {
    const float ah = tid < n_order ? __fdiv_rn(a[(int64_t)f * n_order + tid], a0) : 0.f;
    const float bh = tid < n_order ? __fdiv_rn(b[(int64_t)f * n_order + tid], a0) : 0.f;
    coef[f * kCoefStride + tid] = ah;
    coef[f * kCoefStride + kMaxOrder + 1 + tid] = bh;
    sah[tid] = ah;
  }
  if constexpr (NP > 0) {
    __syncthreads();
    const int i = tid / NP, j = tid % NP;
    const bool mine = tid < NP * NP;
    // s' = M s + e0 v:  s'_0 = -sum_j a^_{j+1} s_j,  s'_i = s_{i-1}
    if (mine) sa[tid] = i == 0 ? -(double)sah[j + 1] : (i == j + 1 ? 1.0 : 0.0);
    __syncthreads();
    double* out = pows + (size_t)f * kPowers * NP * NP;
    for (int sq = 0; sq < 5 + kLevels; ++sq) {  // M^2, ..., M^32 = M^L, then M^(L 2^j)
      double acc = 0.0;
      if (mine)
        for (int k = 0; k < NP; ++k) acc = fma(sa[i * NP + k], sa[k * NP + j], acc);
      __syncthreads();
      if (mine) {
        sa[tid] = acc;
        if (sq >= 4) out[(sq - 4) * NP * NP + tid] = acc;
      }
      __syncthreads();
    }
  }
}

// ---- the tile pass: aggregates (FINAL = false) or the output (FINAL = true) ----------------------------------------
template <int NP>
__host__ __device__ constexpr int vec_pitch() { return NP > 0 ? (NP | 1) : 0; }  // odd: conflict-free double rows

template <int NP>
__host__ __device__ constexpr size_t tile_smem() {
  return (size_t)kTileChunks * vec_pitch<NP>() * 8 + (size_t)kPowers * NP * NP * 8 +
         ((NP > 0 ? NP : 1) + kTileChunks * kPitch) * 4;
}

template <int NP, bool FINAL>
__global__ void __launch_bounds__(kTileChunks, NP >= 8 ? 2 : 8) lfilter_tile_kernel(const LfParams p) {
  constexpr int NA = NP > 0 ? NP : 1;
  constexpr int VP = vec_pitch<NP>();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* sv = reinterpret_cast<double*>(smem_raw);  // [kTileChunks][VP] scan vectors
  double* spow = sv + kTileChunks * VP;              // [kPowers][NP*NP]
  float* halo = reinterpret_cast<float*>(spow + kPowers * NP * NP);  // [NA]: the NP samples before the tile
  float* body = halo + NA;                           // [kTileChunks][kPitch]
  const int c = threadIdx.x;
  const int64_t row = blockIdx.x / p.tiles, tile = blockIdx.x - row * p.tiles;
  const int64_t t0 = tile * kTile, T = p.length;
  const int f = (int)(row % p.n_filters);
  const float* src = row_ptr(p.x, row, p.n_filters, p.s_batch, p.s_filter);

  // stage logical samples [t0 - NP, t0 + kTile): asynchronous 4-byte copies, coalesced along the row (either way)
  if (p.mask_y == nullptr) {
    if (c < NP) {
      const int64_t tau = t0 - NP + c;
      if (p.fir && tau >= 0) cp_async4(halo + c, src + phys(tau, T, p.reverse));
      else halo[c] = 0.f;
    }
    for (int i = c; i < kTile; i += kTileChunks) {
      float* dst = body + (i / kChunk) * kPitch + i % kChunk;
      const int64_t tau = t0 + i;
      if (tau < T) cp_async4(dst, src + phys(tau, T, p.reverse));
      else *dst = 0.f;
    }
    cp_async_wait_all();
  } else {  // the adjoint's input: grad gated by the forward's clamp mask (torch.clamp's inclusive rule; NaN -> 0)
    const float* my = p.mask_y + row * T;
    if (c < NP) halo[c] = 0.f;
    for (int i = c; i < kTile; i += kTileChunks) {
      const int64_t tau = t0 + i;
      float v = 0.f;
      if (tau < T) {
        const int64_t q = phys(tau, T, p.reverse);
        const float yv = my[q];
        v = (yv >= -1.f && yv <= 1.f) ? src[q] : 0.f;
      }
      body[(i / kChunk) * kPitch + i % kChunk] = v;
    }
  }
  if constexpr (NP > 0)
    for (int i = c; i < kPowers * NP * NP; i += kTileChunks) spow[i] = p.pows[(size_t)f * kPowers * NP * NP + i];
  __syncthreads();

  const float* cf = p.coef + f * kCoefStride;
  float ah[NA], bh[NP + 1];
#pragma unroll
  for (int j = 0; j < NP; ++j) ah[j] = __ldg(cf + 1 + j);
#pragma unroll
  for (int j = 0; j <= NP; ++j) bh[j] = __ldg(cf + kMaxOrder + 1 + j);
  float xw[NA];  // xw[j] = x[tau - 1 - j] of this chunk's first sample (the FIR halo)
#pragma unroll
  for (int j = 0; j < NA; ++j) {
    const int i = c * kChunk - 1 - j;
    xw[j] = j >= NP ? 0.f : (i >= 0 ? body[(i / kChunk) * kPitch + i % kChunk] : halo[NP + i]);
  }
  __syncthreads();  // every halo is in registers before the chunks are overwritten with v

  float* mine = body + c * kPitch;
  // The zero-start end history z_c runs in DOUBLE on the float32 v: from a zero start a resonant section's chunk
  // response can be many times |y| (the homogeneous part cancels it later), and float32 rounding at that magnitude
  // would dominate the carries.
  double yw[NA];  // yw[j] = z[tau - 1 - j]
#pragma unroll
  for (int j = 0; j < NA; ++j) yw[j] = 0.0;
#pragma unroll 4
  for (int k = 0; k < kChunk; ++k) {
    const float xv = mine[k];
    float v = xv;
    if (p.fir) {
      v = bh[0] * xv;
#pragma unroll
      for (int j = 0; j < NP; ++j) v = fmaf(bh[j + 1], xw[j], v);
#pragma unroll
      for (int j = NA - 1; j > 0; --j) xw[j] = xw[j - 1];
      xw[0] = xv;
    }
    mine[k] = v;
    double yv = v;
#pragma unroll
    for (int j = 0; j < NP; ++j) yv = fma(-(double)ah[j], yw[j], yv);
#pragma unroll
    for (int j = NA - 1; j > 0; --j) yw[j] = yw[j - 1];
    yw[0] = yv;
  }

  float start[NA];
#pragma unroll
  for (int j = 0; j < NA; ++j) start[j] = 0.f;
  if constexpr (NP > 0) {
    // inclusive scan over the tile's chunks of w_c = z_c (+ M^L S_tile for chunk 0 in the final pass)
    double w[NP];
#pragma unroll
    for (int j = 0; j < NP; ++j) w[j] = yw[j];
    const double* cin = p.carry + ((size_t)row * p.tiles + tile) * NP;
    if (FINAL && c == 0 && tile > 0) {
#pragma unroll
      for (int i = 0; i < NP; ++i) {
        double acc = w[i];
#pragma unroll
        for (int j = 0; j < NP; ++j) acc = fma(spow[i * NP + j], cin[j], acc);
        w[i] = acc;
      }
    }
#pragma unroll 1
    for (int lvl = 0; lvl < kLevels; ++lvl) {
      const int d = 1 << lvl;
#pragma unroll
      for (int j = 0; j < NP; ++j) sv[c * VP + j] = w[j];
      __syncthreads();
      if (c >= d) {
        double prev[NP];
#pragma unroll
        for (int j = 0; j < NP; ++j) prev[j] = sv[(c - d) * VP + j];
        const double* P = spow + lvl * NP * NP;
#pragma unroll
        for (int i = 0; i < NP; ++i) {
          double acc = w[i];
#pragma unroll
          for (int j = 0; j < NP; ++j) acc = fma(P[i * NP + j], prev[j], acc);
          w[i] = acc;
        }
      }
      __syncthreads();
    }
    if constexpr (!FINAL) {
      if (c == kTileChunks - 1 && tile < p.tiles - 1) {
        double* cout = p.carry + ((size_t)row * p.tiles + tile) * NP;
#pragma unroll
        for (int j = 0; j < NP; ++j) cout[j] = w[j];
      }
      return;
    } else {
#pragma unroll
    for (int j = 0; j < NP; ++j) sv[c * VP + j] = w[j];
    __syncthreads();
    if (c > 0) {
#pragma unroll
      for (int j = 0; j < NP; ++j) start[j] = (float)sv[(c - 1) * VP + j];
    } else if (tile > 0) {
#pragma unroll
      for (int j = 0; j < NP; ++j) start[j] = (float)cin[j];
    }
    }
  }
  if constexpr (FINAL) {
    // the chunk again, from its true starting history; y overwrites v in place
#pragma unroll 4
    for (int k = 0; k < kChunk; ++k) {
      float yv = mine[k];
#pragma unroll
      for (int j = 0; j < NP; ++j) yv = fmaf(-ah[j], start[j], yv);
#pragma unroll
      for (int j = NA - 1; j > 0; --j) start[j] = start[j - 1];
      start[0] = yv;
      mine[k] = yv;
    }
    __syncthreads();
    float* yrow = p.y + row * T;
    float* rrow = p.y_raw == nullptr ? nullptr : p.y_raw + row * T;
    for (int i = c; i < kTile; i += kTileChunks) {
      const int64_t tau = t0 + i;
      if (tau >= T) break;
      const int64_t q = phys(tau, T, p.reverse);
      const float v = body[(i / kChunk) * kPitch + i % kChunk];
      yrow[q] = p.clamp ? clamp1(v) : v;
      if (rrow != nullptr) rrow[q] = v;
    }
  }
}

// ---- the fixed-order scan over each row's tiles: one warp per row, lane i owns component i ------------------------
template <int NP>
__global__ void __launch_bounds__(256) lfilter_carry_kernel(const double* __restrict__ pows, double* carry, int64_t rows,
                                                            int64_t tiles, int n_filters) {
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;  // whole warps leave together
  const int f = (int)(row % n_filters);
  const double* P = pows + ((size_t)f * kPowers + kLevels) * NP * NP;  // M^(L kTileChunks): one whole tile
  double prow[NP];
#pragma unroll
  for (int j = 0; j < NP; ++j) prow[j] = lane < NP ? P[lane * NP + j] : 0.0;
  double* cr = carry + (size_t)row * tiles * NP;
  double s = 0.0;
  for (int64_t t = 0; t < tiles; ++t) {
    const double agg = (lane < NP && t + 1 < tiles) ? cr[t * NP + lane] : 0.0;
    if (lane < NP) cr[t * NP + lane] = s;  // S_t: the history entering tile t
    double acc = agg;
#pragma unroll
    for (int j = 0; j < NP; ++j) acc = fma(prow[j], __shfl_sync(0xffffffffu, s, j), acc);
    s = acc;
  }
}

// ---- backward: grad_x (the FIR adjoint) and per-(row, tile) correlation partials ----------------------------------
template <int NP>
__host__ __device__ constexpr size_t grad_smem() {
  return (size_t)3 * (kTile + (NP > 0 ? NP : 1)) * 4 > (size_t)(2 * NP + 1) * kTileChunks * 8
             ? (size_t)3 * (kTile + (NP > 0 ? NP : 1)) * 4
             : (size_t)(2 * NP + 1) * kTileChunks * 8;
}

// In the forward's logical order tau (phys = reverse ? T-1-tau : tau): grad_x[tau] = sum_k b^_k u[tau+k],
// d a^_k += -u[tau] y[tau-k] (k >= 1), d b^_k += u[tau] x[tau-k].
template <int NP>
__global__ void __launch_bounds__(kTileChunks) lfilter_grad_kernel(const LfParams p, const float* __restrict__ yraw,
                                                                   const float* __restrict__ u, float* grad_x,
                                                                   double* part) {
  constexpr int NA = NP > 0 ? NP : 1;
  constexpr int NQ = 2 * NP + 1;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* su = reinterpret_cast<float*>(smem_raw);  // [kTile + NA]: u[t0 .. t0 + kTile + NP)
  float* sx = su + kTile + NA;                     // [NA + kTile]: x[t0 - NP .. t0 + kTile)
  float* sy = sx + kTile + NA;                     // [NA + kTile]: y likewise
  const int c = threadIdx.x;
  const int64_t row = blockIdx.x / p.tiles, tile = blockIdx.x - row * p.tiles;
  const int64_t t0 = tile * kTile, T = p.length;
  const int f = (int)(row % p.n_filters);
  const float* xs = row_ptr(p.x, row, p.n_filters, p.s_batch, p.s_filter);
  const float* ys = yraw + row * T;
  const float* us = u + row * T;
  for (int i = c; i < kTile + NA; i += kTileChunks) {
    const int64_t tu = t0 + i, tp = t0 - NA + i;
    su[i] = (i < kTile + NP && tu < T) ? us[phys(tu, T, p.reverse)] : 0.f;
    const bool okp = tp >= 0 && tp < T && i >= NA - NP;
    sx[i] = okp ? xs[phys(tp, T, p.reverse)] : 0.f;
    sy[i] = okp ? ys[phys(tp, T, p.reverse)] : 0.f;
  }
  __syncthreads();
  const float* cf = p.coef + f * kCoefStride;
  float bh[NP + 1];
#pragma unroll
  for (int j = 0; j <= NP; ++j) bh[j] = __ldg(cf + kMaxOrder + 1 + j);
  double acc[NQ];
#pragma unroll
  for (int q = 0; q < NQ; ++q) acc[q] = 0.0;
  float* gx = grad_x == nullptr ? nullptr : grad_x + row * T;
  for (int i = c; i < kTile; i += kTileChunks) {
    const int64_t tau = t0 + i;
    if (tau >= T) break;
    const float uv = su[i];
    float g = bh[0] * uv;
#pragma unroll
    for (int k = 1; k <= NP; ++k) g = fmaf(bh[k], su[i + k], g);
    if (gx != nullptr) gx[phys(tau, T, p.reverse)] = g;
#pragma unroll
    for (int k = 1; k <= NP; ++k) acc[k - 1] -= (double)uv * (double)sy[NA + i - k];
#pragma unroll
    for (int k = 0; k <= NP; ++k) acc[NP + k] += (double)uv * (double)sx[NA + i - k];
  }
  __syncthreads();
  double* red = reinterpret_cast<double*>(smem_raw);  // [NQ][kTileChunks]
#pragma unroll
  for (int q = 0; q < NQ; ++q) red[q * kTileChunks + c] = acc[q];
  __syncthreads();
  if (c < NQ) {
    double s = 0.0;
    for (int i = 0; i < kTileChunks; ++i) s += red[c * kTileChunks + i];
    part[((size_t)row * p.tiles + tile) * NQ + c] = s;
  }
}

// d a^ / d b^ of filter f, component q: the partials of rows f, f + F, ... and their tiles, in a fixed order
__global__ void __launch_bounds__(kRedThreads) lfilter_reduce_kernel(const double* __restrict__ part, int64_t rows,
                                                                     int64_t tiles, int n_filters, int nq,
                                                                     double* gnorm) {
  __shared__ double red[kRedThreads];
  const int f = blockIdx.x / nq, q = blockIdx.x - f * nq;
  const int64_t per = (rows / n_filters) * tiles;  // rows = batch * n_filters
  double s = 0.0;
  for (int64_t m = threadIdx.x; m < per; m += kRedThreads) {
    const int64_t bi = m / tiles, t = m - bi * tiles;
    s += part[((size_t)(bi * n_filters + f) * tiles + t) * nq + q];
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = kRedThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) gnorm[(size_t)f * nq + q] = red[0];
}

// through a0: d a_k = d a^_k / a0 (k >= 1), d b_k = d b^_k / a0, d a_0 = -(sum_{k>=1} d a^_k a^_k + sum_k d b^_k b^_k) / a0
__global__ void lfilter_coef_grad_kernel(const float* __restrict__ a, const float* __restrict__ coef,
                                         const double* __restrict__ gnorm, int n_order, int np, float* grad_a,
                                         float* grad_b) {
  const int f = blockIdx.x, k = threadIdx.x;
  const int nq = 2 * np + 1;
  const double a0 = (double)a[(int64_t)f * n_order];
  const double* g = gnorm + (size_t)f * nq;
  const float* cf = coef + f * kCoefStride;
  if (k >= n_order) return;
  if (grad_b != nullptr) grad_b[(int64_t)f * n_order + k] = (float)(g[np + k] / a0);
  if (grad_a == nullptr) return;
  if (k > 0) {
    grad_a[(int64_t)f * n_order + k] = (float)(g[k - 1] / a0);
    return;
  }
  double s = 0.0;
  for (int j = 1; j < n_order; ++j) s = fma(g[j - 1], (double)cf[j], s);
  for (int j = 0; j < n_order; ++j) s = fma(g[np + j], (double)cf[kMaxOrder + 1 + j], s);
  grad_a[(int64_t)f * n_order] = (float)(-s / a0);
}

int check_args(const float* a, const float* b, int n_filters, int n_order, const float* x, int64_t batch,
               int64_t length, int64_t s_batch, int64_t s_filter, const void* ws) {
  if (n_order < 1 || n_filters < 1 || batch < 0 || length < 0 || s_batch < 0 || s_filter < 0) return B200A_EINVAL;
  if (n_order - 1 > kMaxOrder) return B200A_EUNSUPPORTED;
  if (batch == 0 || length == 0) return B200A_OK;
  if (a == nullptr || b == nullptr || x == nullptr || ws == nullptr) return B200A_EINVAL;
  const int64_t tiles = (length + kTile - 1) / kTile;
  if (batch * n_filters * tiles > INT32_MAX) return B200A_EUNSUPPORTED;  // grid.x
  return B200A_OK;
}

template <int NP>
int scan_launch(const LfParams& p, cudaStream_t stream) {
  const int64_t grid = p.rows * p.tiles;
  if constexpr (NP > 0) {
    if (p.tiles > 1) {  // one tile: the first tile starts from a zero history, nothing to carry
      int rc = launch_kernel(lfilter_tile_kernel<NP, false>, grid, kTileChunks, tile_smem<NP>(), stream, p);
      if (rc != B200A_OK) return rc;
      rc = launch_kernel(lfilter_carry_kernel<NP>, (p.rows + 7) / 8, 256, 0, stream, p.pows, p.carry, p.rows, p.tiles,
                         p.n_filters);
      if (rc != B200A_OK) return rc;
    }
  }
  return launch_kernel(lfilter_tile_kernel<NP, true>, grid, kTileChunks, tile_smem<NP>(), stream, p);
}

template <int NP>
int run_np(const float* a, const float* b, int n_order, LfParams p, cudaStream_t stream) {
  lfilter_prep_kernel<NP><<<p.n_filters, 256, 0, stream>>>(a, b, n_order, const_cast<float*>(p.coef),
                                                          const_cast<double*>(p.pows));
  int rc = launch_status();
  return rc != B200A_OK ? rc : scan_launch<NP>(p, stream);
}

template <int NP>
int backward_np(const float* a, int n_order, LfParams p, const float* y_raw, const float* grad, float* grad_x,
                float* grad_a, float* grad_b, float* u, double* part, double* gnorm, cudaStream_t stream) {
  // u: the IIR recurrence in the opposite direction over the masked gradient (b^ unused: fir = 0)
  LfParams q = p;
  q.x = grad, q.s_batch = p.n_filters * p.length, q.s_filter = p.length;
  q.mask_y = p.clamp ? y_raw : nullptr;
  q.y = u, q.y_raw = nullptr, q.fir = 0, q.clamp = 0, q.reverse = !p.reverse;
  int rc = scan_launch<NP>(q, stream);
  if (rc != B200A_OK) return rc;
  rc = launch_kernel(lfilter_grad_kernel<NP>, p.rows * p.tiles, kTileChunks, grad_smem<NP>(), stream, p, y_raw, u,
                     grad_x, part);
  if (rc != B200A_OK || (grad_a == nullptr && grad_b == nullptr)) return rc;
  const int nq = 2 * NP + 1;
  // static shared memory only: launched directly (launch_kernel raises the dynamic limit to the whole 227 KB)
  lfilter_reduce_kernel<<<p.n_filters * nq, kRedThreads, 0, stream>>>(part, p.rows, p.tiles, p.n_filters, nq, gnorm);
  rc = launch_status();
  if (rc != B200A_OK) return rc;
  lfilter_coef_grad_kernel<<<p.n_filters, 32, 0, stream>>>(a, p.coef, gnorm, n_order, NP, grad_a, grad_b);
  return launch_status();
}

LfParams make_params(const float* x, int n_filters, int64_t batch, int64_t length, int64_t s_batch, int64_t s_filter,
                     bool clamp, bool reverse, void* ws, const LfLayout& l) {
  LfParams p{};
  char* base = static_cast<char*>(ws);
  p.x = x;
  p.coef = reinterpret_cast<const float*>(base + l.coef);
  p.pows = reinterpret_cast<const double*>(base + l.pows);
  p.carry = reinterpret_cast<double*>(base + l.carry);
  p.s_batch = s_batch, p.s_filter = s_filter, p.length = length;
  p.tiles = (length + kTile - 1) / kTile;
  p.rows = batch * n_filters;
  p.n_filters = n_filters;
  p.reverse = reverse, p.fir = 1, p.clamp = clamp;
  return p;
}

}  // namespace

size_t lfilter_workspace_bytes_impl(int64_t rows, int64_t length, int n_order, int n_filters, bool backward) {
  if (rows < 0 || length < 0 || n_order < 1 || n_filters < 1 || n_order - 1 > kMaxOrder) return 0;
  return lf_layout(rows, length, padded_order(n_order - 1), n_filters, backward).total;
}

int lfilter_run_impl(const float* a, const float* b, int n_filters, int n_order, const float* x, int64_t batch,
                     int64_t length, int64_t s_batch, int64_t s_filter, bool clamp, bool reverse, float* y,
                     float* y_raw, void* ws, size_t ws_bytes, cudaStream_t stream) {
  int rc = check_args(a, b, n_filters, n_order, x, batch, length, s_batch, s_filter, ws);
  if (rc != B200A_OK || batch == 0 || length == 0) return rc;
  if (y == nullptr) return B200A_EINVAL;
  const int np = padded_order(n_order - 1);
  const LfLayout l = lf_layout(batch * n_filters, length, np, n_filters, false);
  if (ws_bytes < l.total) return B200A_EWORKSPACE;
  LfParams p = make_params(x, n_filters, batch, length, s_batch, s_filter, clamp, reverse, ws, l);
  p.y = y, p.y_raw = y_raw;
  switch (np) {
    case 0: return run_np<0>(a, b, n_order, p, stream);
    case 1: return run_np<1>(a, b, n_order, p, stream);
    case 2: return run_np<2>(a, b, n_order, p, stream);
    case 4: return run_np<4>(a, b, n_order, p, stream);
    case 8: return run_np<8>(a, b, n_order, p, stream);
    default: return run_np<16>(a, b, n_order, p, stream);
  }
}

int lfilter_backward_impl(const float* a, const float* b, int n_filters, int n_order, const float* x, int64_t batch,
                          int64_t length, int64_t s_batch, int64_t s_filter, const float* y_raw, const float* grad,
                          bool clamp, bool reverse, float* grad_x, float* grad_a, float* grad_b, void* ws,
                          size_t ws_bytes, cudaStream_t stream) {
  int rc = check_args(a, b, n_filters, n_order, x, batch, length, s_batch, s_filter, ws);
  if (rc != B200A_OK) return rc;
  if (batch == 0 || length == 0) {
    if (grad_a == nullptr && grad_b == nullptr) return B200A_OK;
    // empty signal: the coefficient gradients are zero
    if (grad_a != nullptr && cudaMemsetAsync(grad_a, 0, (size_t)n_filters * n_order * 4, stream) != cudaSuccess)
      return B200A_ECUDA;
    if (grad_b != nullptr && cudaMemsetAsync(grad_b, 0, (size_t)n_filters * n_order * 4, stream) != cudaSuccess)
      return B200A_ECUDA;
    return B200A_OK;
  }
  if (y_raw == nullptr || grad == nullptr) return B200A_EINVAL;
  const int np = padded_order(n_order - 1);
  const LfLayout l = lf_layout(batch * n_filters, length, np, n_filters, true);
  if (ws_bytes < l.total) return B200A_EWORKSPACE;
  LfParams p = make_params(x, n_filters, batch, length, s_batch, s_filter, clamp, reverse, ws, l);
  char* base = static_cast<char*>(ws);
  float* u = reinterpret_cast<float*>(base + l.u);
  double* part = reinterpret_cast<double*>(base + l.part);
  double* gnorm = reinterpret_cast<double*>(base + l.gnorm);
#define B200A_LF_BACKWARD(NP)                                                                                   \
  lfilter_prep_kernel<NP><<<n_filters, 256, 0, stream>>>(a, b, n_order, const_cast<float*>(p.coef),           \
                                                          const_cast<double*>(p.pows));                        \
  rc = launch_status();                                                                                         \
  return rc != B200A_OK ? rc                                                                                    \
                        : backward_np<NP>(a, n_order, p, y_raw, grad, grad_x, grad_a, grad_b, u, part, gnorm, stream)
  switch (np) {
    case 0: B200A_LF_BACKWARD(0);
    case 1: B200A_LF_BACKWARD(1);
    case 2: B200A_LF_BACKWARD(2);
    case 4: B200A_LF_BACKWARD(4);
    case 8: B200A_LF_BACKWARD(8);
    default: B200A_LF_BACKWARD(16);
  }
#undef B200A_LF_BACKWARD
  return B200A_EINVAL;
}

}  // namespace b200a
