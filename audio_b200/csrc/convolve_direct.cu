// convolve (functional/functional.py:2261-2314) by the direct method, and its gradients.
//
// The shorter operand is the filter h (K taps; y when n == m), the longer the signal s.  For output t = t0 + 8 q + c
// (MMA row q, column c < 8) the full convolution is the banded Toeplitz product
//     out[t] = sum_j A[q][j] B[j][c],   A[q][j] = s[t0 - (K - 1) + 8 q + j],   B[j][c] = h[c + K - 1 - j],
// j < K + 7, with zeros outside the operands, over ceil((K + 7) / 8) k-steps of mma.sync.m16n8k8.  A prep kernel
// splits B into TF32 hi/lo fragments once per distinct filter row (the layout of band_mma.cuh); the main kernel stages
// the signal span of a 2048-output tile in shared memory and contracts it against them.
//
// Precision (TF32 x 3 at float32 grade).  Both splits round to nearest, v = hi + lo with hi = rn_tf32(v) and
// lo = rn_tf32(v - hi), so |v - hi - lo| <= 2^-22 |v| (band_mma.cuh's truncating split leaves up to 2^-20 after the
// three products).  The tensor cores add into their accumulator with truncation, a bias that grows with the number of
// k-steps a chain runs over (up to 513 here), so only the small A_lo B_hi + A_hi B_lo chain stays in the accumulator;
// each step's A_hi B_hi product starts from zero and is added to a float32 sum with round-to-nearest.
//
// Gradients, with g placed at `start` of the full range and zero elsewhere:
//   ds[i] = sum_k g[i + k] h[k]   the main kernel on g with the fragments of the reversed filter (outputs K - 1 ..)
//   dh[k] = sum_i g[i + k] s[i]   per 2048-sample tile of u = i + c:  dh[8 a + c] = sum_u g[u + 8 a] s[u - c], an
//                                 m16n8k8 product with the taps as M (16 rows = 128 taps) and u as the k dimension;
//                                 the tiles' partials are summed in tile order.
// Tile sizes depend on K alone and nothing is atomic, so reruns are bit-identical and a row's result does not depend on
// the other rows.
//
// Shared-memory layout of a staged row: sample i at i + 4 (i / 32) (a 4-float gap every 32 samples).  The 8 A rows one
// fragment load touches start 8 samples apart, so at a linear pitch rows r and r + 4 would share banks; with the gap
// the 8 rows' 4-word windows fall into 32 distinct banks.
#include "common.cuh"
#include "ptx.cuh"

namespace b200a {
namespace {

constexpr int kWarps = 8;
constexpr int kMT = 2;                          // 16-row M tiles per warp, sharing each B fragment load
constexpr int kTile = kWarps * kMT * 128;       // outputs per CTA of the main kernel
constexpr int kGradTile = 2048;                 // u samples per CTA of the filter gradient (256 k-steps)
constexpr int kFragSmemSteps = 64;              // fragments staged in shared memory up to 64 k-steps (32 KB)
constexpr int64_t kMaxTaps = B200A_CONVOLVE_MAX_TAPS;

__host__ __device__ __forceinline__ int skewed(int i) { return i + ((i >> 5) << 2); }
inline size_t up256(size_t v) { return (v + 255) & ~size_t(255); }

__device__ __forceinline__ uint32_t tf32_rn(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return r;
}
// v = hi + lo to 2^-22 |v|, both TF32 rounded to nearest
__device__ __forceinline__ void split_rn(float v, uint32_t& hi, uint32_t& lo) {
  hi = tf32_rn(v);
  lo = tf32_rn(v - __uint_as_float(hi));
}

// One k-step of one M tile: big += A_hi B_hi (a fresh product, added with round-to-nearest), small += A_lo B_hi +
// A_hi B_lo (in the accumulator).  b = (B_hi[k0], B_hi[k1], B_lo[k0], B_lo[k1]) of this lane.
__device__ __forceinline__ void step_x3(const float (&av)[4], const uint4& b, float (&big)[4], float (&small)[4]) {
  uint32_t hi[4], lo[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) split_rn(av[q], hi[q], lo[q]);
  float t[4];
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
      : "=f"(t[0]), "=f"(t[1]), "=f"(t[2]), "=f"(t[3])
      : "r"(hi[0]), "r"(hi[1]), "r"(hi[2]), "r"(hi[3]), "r"(b.x), "r"(b.y), "f"(0.f));
#pragma unroll
  for (int q = 0; q < 4; ++q) big[q] += t[q];
  mma_tf32(small, lo, b.x, b.y);
  mma_tf32(small, hi, b.z, b.w);
}
inline int k_steps(int64_t K) { return (int)((K + 7 + 7) / 8); }  // ceil((K + 7) / 8)

// Filter and signal operands of a call.
struct Operands {
  const float* f;
  const float* s;
  int64_t f_rows, s_rows, f_stride, s_stride;
  const int64_t* f_index;
  const int64_t* s_index;
  int64_t K, S;
};

Operands operands(const b200a_convolve_desc& d, const float* x, const float* y) {
  if (d.n < d.m) return {x, y, d.x_rows, d.y_rows, d.x_stride, d.y_stride, d.x_index, d.y_index, d.n, d.m};
  return {y, x, d.y_rows, d.x_rows, d.y_stride, d.x_stride, d.y_index, d.x_index, d.m, d.n};
}

// Workspace, 256-byte aligned sections:
//   frags    uint4  [filter rows][k_steps(K)][32]      the B fragments (backward: of the reversed filter)
//   partial  float  [rows][grad tiles][K]              (backward) the filter gradient per tile
struct Layout {
  size_t frags, partial, total;
};

inline int64_t grad_tiles(int64_t S) { return (S + 7 + kGradTile - 1) / kGradTile; }

Layout layout(const b200a_convolve_desc& d, bool backward) {
  const Operands o = operands(d, nullptr, nullptr);
  Layout l{};
  l.frags = 0;
  size_t off = up256((size_t)o.f_rows * k_steps(o.K) * 32 * sizeof(uint4));
  l.partial = off;
  if (backward) off += up256((size_t)d.rows * grad_tiles(o.S) * o.K * sizeof(float));
  l.total = off;
  return l;
}

// One CTA per filter row: B[j][c] = h[c + K - 1 - j] (reverse: of the reversed filter) as TF32 hi/lo fragments,
// step s at frags[s * 32 + lane] = (B_hi[k0][n], B_hi[k1][n], B_lo[k0][n], B_lo[k1][n]), n = lane / 4,
// k0 = 8 s + lane % 4, k1 = k0 + 4.
__global__ void __launch_bounds__(256) convolve_frags_kernel(const float* __restrict__ f, int64_t f_stride, int K,
                                                             int nsteps, bool reverse, uint4* frags) {
  const float* h = f + (int64_t)blockIdx.x * f_stride;
  auto b = [&](int n, int k) {
    const int tap = n + K - 1 - k;
    if (tap < 0 || tap >= K) return 0.f;
    return h[reverse ? K - 1 - tap : tap];
  };
  uint4* out = frags + (size_t)blockIdx.x * nsteps * 32;
  for (int i = threadIdx.x; i < nsteps * 32; i += blockDim.x) {
    const int n = (i & 31) >> 2, k0 = 8 * (i >> 5) + (i & 3);
    uint4 v;
    split_rn(b(n, k0), v.x, v.z);
    split_rn(b(n, k0 + 4), v.y, v.w);
    out[i] = v;
  }
}

struct DirectParams {
  const float* sig;          // signal row r at sig + (sig_index ? sig_index[r] : r) * sig_stride, unit time stride
  const int64_t* sig_index;
  int64_t sig_stride;
  int64_t sig_off, sig_len;  // signal sample u is sig[u - sig_off] for 0 <= u - sig_off < sig_len, else 0
  const uint4* frags;        // filter row f_index[r]'s fragments at frags + f_index[r] * nsteps * 32
  const int64_t* f_index;
  int K, nsteps;
  float* out;                // row r at out + r * out_len: full-range outputs [start, start + out_len)
  int64_t out_len, start;
  int64_t tiles;             // output tiles per row
  int span;                  // staged samples per tile
  bool frags_in_smem, pairs; // pairs: float2 stores (even out_len, 8-byte aligned out)
};

// The M tiles of one warp over all k-steps, the fragments read from shared memory (SMEM) or through the read-only
// cache.  base[2 h (+ 1)]: span index of this lane's A entries in rows r (r + 8) of M tile h at k-step 0.
template <bool SMEM>
__device__ __forceinline__ void direct_contract(const uint4* frg, int nsteps, const float* xs,
                                                const int (&base)[2 * kMT], float (&big)[kMT][4],
                                                float (&small)[kMT][4]) {
#pragma unroll 2
  for (int s = 0; s < nsteps; ++s) {
    uint4 b;
    if constexpr (SMEM) b = frg[(size_t)s * 32];
    else b = __ldg(frg + (size_t)s * 32);
#pragma unroll
    for (int h = 0; h < kMT; ++h) {
      const int i0 = base[2 * h] + 8 * s, i1 = base[2 * h + 1] + 8 * s;
      const float av[4] = {xs[skewed(i0)], xs[skewed(i1)], xs[skewed(i0 + 4)], xs[skewed(i1 + 4)]};
      step_x3(av, b, big[h], small[h]);
    }
  }
}

// One CTA per (row, tile of kTile outputs): stage the tile's signal span (kTile + 8 nsteps samples from t0 - (K - 1))
// with 4-byte asynchronous copies, then each warp contracts kMT M tiles and writes its outputs straight to `out`.
__global__ void __launch_bounds__(kWarps * 32) convolve_direct_kernel(const DirectParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint4* s_frags = reinterpret_cast<uint4*>(smem_raw);
  float* xs = reinterpret_cast<float*>(s_frags + (p.frags_in_smem ? (size_t)p.nsteps * 32 : 0));
  const int64_t row = blockIdx.x / p.tiles, tile = blockIdx.x - row * p.tiles;
  const int64_t t0 = p.start + tile * kTile;
  const float* sig = p.sig + (p.sig_index == nullptr ? row : p.sig_index[row]) * p.sig_stride;
  const uint4* frags = p.frags + (size_t)p.f_index[row] * p.nsteps * 32;
  const int64_t u0 = t0 - (p.K - 1) - p.sig_off;  // sig index of span sample 0
  for (int i = threadIdx.x; i < p.span; i += blockDim.x) {
    const int64_t u = u0 + i;
    float* dst = xs + skewed(i);
    if (u >= 0 && u < p.sig_len) cp_async4(dst, sig + u);
    else *dst = 0.f;
  }
  if (p.frags_in_smem)
    for (int i = threadIdx.x; i < p.nsteps * 32; i += blockDim.x) s_frags[i] = frags[i];
  cp_async_wait_all();
  __syncthreads();

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = lane >> 2, c = lane & 3;
  int base[2 * kMT];
#pragma unroll
  for (int h = 0; h < kMT; ++h) {
    base[2 * h] = 128 * (kMT * warp + h) + 8 * r + c;
    base[2 * h + 1] = base[2 * h] + 64;
  }
  float big[kMT][4], small[kMT][4];
#pragma unroll
  for (int h = 0; h < kMT; ++h)
#pragma unroll
    for (int q = 0; q < 4; ++q) big[h][q] = small[h][q] = 0.f;
  if (p.frags_in_smem) direct_contract<true>(s_frags + lane, p.nsteps, xs, base, big, small);
  else direct_contract<false>(frags + lane, p.nsteps, xs, base, big, small);
  // D rows r (+ 8) of M tile h, columns 2c, 2c + 1: outputs t0 + 128 (kMT warp + h) + 8 (r (+ 8)) + 2c (+ 1)
  float* orow = p.out + row * p.out_len;
  const int64_t end = p.start + p.out_len;
#pragma unroll
  for (int h = 0; h < kMT; ++h)
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int64_t t = t0 + base[2 * h + half] + c;
      const float v0 = big[h][2 * half] + small[h][2 * half], v1 = big[h][2 * half + 1] + small[h][2 * half + 1];
      float* o = orow + (t - p.start);
      if (p.pairs && t + 1 < end) {
        *reinterpret_cast<float2*>(o) = make_float2(v0, v1);  // t - start even, out_len even: 8-byte aligned
      } else {
        if (t < end) o[0] = v0;
        if (t + 1 < end) o[1] = v1;
      }
    }
}

struct GradParams {
  const float* grad;         // g row r at grad + r * out_len: full-range samples [start, start + out_len)
  int64_t out_len, start;
  const float* sig;          // signal row s_index[r] at sig + s_index[r] * s_stride, S samples
  const int64_t* s_index;
  int64_t s_stride, S;
  int K, n_mt, parts;        // M tiles of 128 taps; parts: k-step ranges of one M tile on separate warps
  int64_t tiles;             // gradient tiles per row
  int g_span;                // staged g samples: kGradTile + 128 n_mt
  float* partial;            // [rows][tiles][K]
};

// One CTA per (row, tile of kGradTile values of u): dh[8 a + c] over the tile = sum_u A[a][u] B[u][c] with
// A[a][u] = g[u + 8 a] and B[u][c] = s[u - c], both staged skewed and split into hi/lo on the fly.  Warp items are
// (M tile, part); the parts of an M tile are added in part order in shared memory.
__global__ void __launch_bounds__(kWarps * 32) convolve_filter_grad_kernel(const GradParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* gs = reinterpret_cast<float*>(smem_raw);              // skewed [g_span]: g_full[u0 + v]
  float* ss = gs + ((skewed(p.g_span - 1) + 4) & ~3);           // skewed [kGradTile + 8]: s[u0 - 8 + v]
  float* sd = ss + ((skewed(kGradTile + 7) + 4) & ~3);          // [parts][n_mt * 128]
  const int64_t row = blockIdx.x / p.tiles, tile = blockIdx.x - row * p.tiles;
  const int64_t u0 = tile * kGradTile;
  const float* g = p.grad + row * p.out_len;
  const float* s = p.sig + p.s_index[row] * p.s_stride;
  for (int v = threadIdx.x; v < p.g_span; v += blockDim.x) {
    const int64_t i = u0 + v - p.start;
    float* dst = gs + skewed(v);
    if (i >= 0 && i < p.out_len) cp_async4(dst, g + i);
    else *dst = 0.f;
  }
  for (int v = threadIdx.x; v < kGradTile + 8; v += blockDim.x) {
    const int64_t i = u0 - 8 + v;
    float* dst = ss + skewed(v);
    if (i >= 0 && i < p.S) cp_async4(dst, s + i);
    else *dst = 0.f;
  }
  cp_async_wait_all();
  __syncthreads();

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = lane >> 2, c = lane & 3;
  const int steps = kGradTile / 8 / p.parts;
  const int pitch = p.n_mt * 128;
  for (int item = warp; item < p.n_mt * p.parts; item += kWarps) {
    const int mt = item / p.parts, part = item - mt * p.parts;
    float big[4] = {0.f, 0.f, 0.f, 0.f}, small[4] = {0.f, 0.f, 0.f, 0.f};
    const int a0 = 128 * mt + 8 * r + c;  // g index of A[r][c] at k-step 0
#pragma unroll 4
    for (int st = part * steps; st < (part + 1) * steps; ++st) {
      const int k = 8 * st;
      const float av[4] = {gs[skewed(a0 + k)], gs[skewed(a0 + k + 64)], gs[skewed(a0 + k + 4)],
                           gs[skewed(a0 + k + 68)]};
      uint4 b;  // B[k + c (+ 4)][r] = s[u0 + k + c (+ 4) - r]
      split_rn(ss[skewed(k + c + 8 - r)], b.x, b.z);
      split_rn(ss[skewed(k + c + 12 - r)], b.y, b.w);
      step_x3(av, b, big, small);
    }
    // D rows r (+ 8), columns 2c, 2c + 1: taps 128 mt + 8 (r (+ 8)) + 2c (+ 1)
    float* dp = sd + part * pitch + 128 * mt + 8 * r + 2 * c;
    *reinterpret_cast<float2*>(dp) = make_float2(big[0] + small[0], big[1] + small[1]);
    *reinterpret_cast<float2*>(dp + 64) = make_float2(big[2] + small[2], big[3] + small[3]);
  }
  __syncthreads();
  float* out = p.partial + (size_t)blockIdx.x * p.K;
  for (int k = threadIdx.x; k < p.K; k += blockDim.x) {
    float acc = sd[k];
    for (int part = 1; part < p.parts; ++part) acc += sd[part * pitch + k];
    out[k] = acc;
  }
}

// dh[r][k] = sum over the tiles of partial[r][tile][k], in tile order.
__global__ void __launch_bounds__(256) convolve_tile_sum_kernel(const float* __restrict__ partial, int64_t rows,
                                                                int64_t tiles, int K, float* __restrict__ dh) {
  const int64_t n = rows * K;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = e / K, k = e - r * K;
    const float* pp = partial + (size_t)r * tiles * K + k;
    float acc = 0.f;
    for (int64_t t = 0; t < tiles; ++t) acc += pp[(size_t)t * K];
    dh[e] = acc;
  }
}

// Shared memory of convolve_direct_kernel for K taps: the skewed span, and the fragments when they are staged.
inline size_t direct_smem(int K, bool frags_in_smem) {
  const int span = kTile + 8 * k_steps(K);
  return sizeof(float) * (size_t)((skewed(span - 1) + 4) & ~3) +
         (frags_in_smem ? sizeof(uint4) * 32 * (size_t)k_steps(K) : 0);
}

int launch_direct(const float* sig, const int64_t* sig_index, int64_t sig_stride, int64_t sig_off, int64_t sig_len,
                  const uint4* frags, const int64_t* f_index, int K, float* out, int64_t rows, int64_t out_len,
                  int64_t start, cudaStream_t stream) {
  DirectParams p{};
  p.sig = sig;
  p.sig_index = sig_index;
  p.sig_stride = sig_stride;
  p.sig_off = sig_off;
  p.sig_len = sig_len;
  p.frags = frags;
  p.f_index = f_index;
  p.K = K;
  p.nsteps = k_steps(K);
  p.out = out;
  p.out_len = out_len;
  p.start = start;
  p.tiles = (out_len + kTile - 1) / kTile;
  p.span = kTile + 8 * p.nsteps;
  p.frags_in_smem = p.nsteps <= kFragSmemSteps;
  p.pairs = (out_len & 1) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0;
  return launch_kernel(convolve_direct_kernel, rows * p.tiles, kWarps * 32, direct_smem(K, p.frags_in_smem), stream,
                       p);
}

int launch_frags(const Operands& o, bool reverse, uint4* frags, cudaStream_t stream) {
  convolve_frags_kernel<<<(unsigned)o.f_rows, 256, 0, stream>>>(o.f, o.f_stride, (int)o.K, k_steps(o.K), reverse,
                                                                frags);
  return launch_status();
}

// B200A_OK with `work` false when there is nothing to enqueue
int check_desc(const b200a_convolve_desc* d, bool& work) {
  work = false;
  if (d == nullptr || d->n < 1 || d->m < 1 || d->rows < 0 || d->x_rows < 1 || d->y_rows < 1 || d->out_len < 0 ||
      d->start < 0 || d->x_stride < 0 || d->y_stride < 0)
    return B200A_EINVAL;
  const int64_t full = d->n + d->m - 1;
  if (full > INT32_MAX) return B200A_EUNSUPPORTED;
  if (d->start + d->out_len > full) return B200A_EINVAL;
  const Operands o = operands(*d, nullptr, nullptr);
  if (o.K > kMaxTaps) return B200A_EUNSUPPORTED;
  const int64_t out_tiles = (full + kTile - 1) / kTile;  // the most tiles a row of either pass has
  if (d->rows * (out_tiles > grad_tiles(o.S) ? out_tiles : grad_tiles(o.S)) > INT32_MAX || o.f_rows > INT32_MAX)
    return B200A_EUNSUPPORTED;  // grid.x
  work = d->rows > 0 && d->out_len > 0;
  if (work && (d->x_index == nullptr || d->y_index == nullptr)) return B200A_EINVAL;
  return B200A_OK;
}

}  // namespace

size_t convolve_workspace_bytes_impl(const b200a_convolve_desc* d, bool backward) {
  bool work = false;
  if (check_desc(d, work) != B200A_OK) return 0;
  return layout(*d, backward).total;
}

int convolve_run_impl(const b200a_convolve_desc* d, const float* x, const float* y, float* out, void* ws,
                      size_t ws_bytes, cudaStream_t stream) {
  bool work = false;
  const int rc = check_desc(d, work);
  if (rc != B200A_OK || !work) return rc;
  if (x == nullptr || y == nullptr || out == nullptr || ws == nullptr) return B200A_EINVAL;
  const Layout l = layout(*d, false);
  if (ws_bytes < l.total) return B200A_EWORKSPACE;
  const Operands o = operands(*d, x, y);
  uint4* frags = ws_at<uint4>(ws, l.frags);
  int r = launch_frags(o, false, frags, stream);
  if (r != B200A_OK) return r;
  return launch_direct(o.s, o.s_index, o.s_stride, 0, o.S, frags, o.f_index, (int)o.K, out, d->rows, d->out_len,
                       d->start, stream);
}

int convolve_backward_impl(const b200a_convolve_desc* d, const float* x, const float* y, const float* grad,
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
  const Layout l = layout(*d, true);
  if (ws_bytes < l.total) return B200A_EWORKSPACE;
  const Operands o = operands(*d, x, y);
  float* ds = d->n < d->m ? grad_y : grad_x;
  float* dh = d->n < d->m ? grad_x : grad_y;
  uint4* frags = ws_at<uint4>(ws, l.frags);
  float* partial = ws_at<float>(ws, l.partial);
  const int K = (int)o.K;
  // ds: the forward on g (full-range sample u = grad[u - start]) with the reversed filter, outputs [K - 1, K - 1 + S)
  int r = launch_frags(o, true, frags, stream);
  if (r == B200A_OK)
    r = launch_direct(grad, nullptr, d->out_len, d->start, d->out_len, frags, o.f_index, K, ds, d->rows, o.S, K - 1,
                      stream);
  if (r != B200A_OK) return r;
  GradParams p{};
  p.grad = grad;
  p.out_len = d->out_len;
  p.start = d->start;
  p.sig = o.s;
  p.s_index = o.s_index;
  p.s_stride = o.s_stride;
  p.S = o.S;
  p.K = K;
  p.n_mt = (K + 127) / 128;
  p.parts = p.n_mt >= kWarps ? 1 : kWarps / p.n_mt;  // 8, 4, 2, 2, 1, ...: every warp has an item for small K
  p.tiles = grad_tiles(o.S);
  p.g_span = kGradTile + 128 * p.n_mt;
  p.partial = partial;
  const size_t smem = sizeof(float) * ((size_t)((skewed(p.g_span - 1) + 4) & ~3) + ((skewed(kGradTile + 7) + 4) & ~3) +
                                       (size_t)p.parts * p.n_mt * 128);
  r = launch_kernel(convolve_filter_grad_kernel, d->rows * p.tiles, kWarps * 32, smem, stream, p);
  if (r != B200A_OK) return r;
  const int64_t n = d->rows * o.K;
  const unsigned grid = (unsigned)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
  convolve_tile_sum_kernel<<<grid, 256, 0, stream>>>(partial, d->rows, p.tiles, K, dh);
  return launch_status();
}

}  // namespace b200a
