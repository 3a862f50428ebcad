// InverseMelScale (transforms/_transforms.py:418-503): x = relu(lstsq(fb^T, m).solution) for an underdetermined,
// full-rank system, i.e. the minimum-norm solution x = relu(fb G^-1 m) with the Gram matrix G = fb^T fb.  A bin of a
// triangular mel bank touches at most two adjacent filters, so G is banded (tridiagonal for every mel and linear bank).
// The plan factors G = L D L^T once on the host in double precision; per frame the kernels then run one banded solve
// over the n_mels values and a <= (bandwidth + 1)-tap expansion to the n_stft bins.  Memory-bound: the arithmetic is a
// few flops per byte moved.
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"

namespace b200a {
namespace {

constexpr int kBw = B200A_INVERSE_MEL_MAX_BANDWIDTH;  // Gram bandwidth cap (mel and linear banks have 1)
constexpr int kTaps = kBw + 1;                         // nonzero filters per bin: at most bandwidth + 1
constexpr int kMaxMels = B200A_INVERSE_MEL_MAX_MELS;   // shared-memory cap: two 32-frame tiles of n_mels in backward
constexpr int kTileFrames = 32;                        // frames per CTA: one solving warp, one frame per lane
constexpr int kThreads = 256;
constexpr int kGradChunk = 128;                        // bins of masked gradient staged per step of the backward

// The plan blob, 4-byte words.  The strides use the caps, so the layout depends on (n_stft, n_mels) alone:
//   [0..3]       n_stft, n_mels, bandwidth, 0
//   lsub         [n_mels][kBw]    L[i][i - 1 - j] (entries past the bandwidth are 0)
//   inv_d        [n_mels]         1 / D[i]
//   bin_first    [n_stft] int32   first nonzero filter of bin k
//   bin_count    [n_stft] int32   nonzero span length (0: empty bin)
//   bin_vals     [n_stft][kTaps]  fb[k][bin_first[k] + j]
//   filt_first   [n_mels] int32   first nonzero bin of filter m
//   filt_count   [n_mels] int32
struct PlanView {
  const int32_t* hdr;
  const float* lsub;
  const float* inv_d;
  const int32_t* bin_first;
  const int32_t* bin_count;
  const float* bin_vals;
  const int32_t* filt_first;
  const int32_t* filt_count;
};

__host__ __device__ inline int64_t plan_words(int64_t n_stft, int64_t n_mels) {
  return 4 + n_mels * (kBw + 3) + n_stft * (2 + kTaps);
}

template <typename W>
__host__ __device__ inline void plan_layout(W* base, int64_t n_stft, int64_t n_mels, W** lsub, W** inv_d, W** bfirst,
                                            W** bcount, W** bvals, W** ffirst, W** fcount) {
  W* p = base + 4;
  *lsub = p, p += n_mels * kBw;
  *inv_d = p, p += n_mels;
  *bfirst = p, p += n_stft;
  *bcount = p, p += n_stft;
  *bvals = p, p += n_stft * kTaps;
  *ffirst = p, p += n_mels;
  *fcount = p;
}

__device__ inline PlanView plan_view(const void* plan) {
  const uint32_t* base = static_cast<const uint32_t*>(plan);
  const int64_t n_stft = (int32_t)base[0], n_mels = (int32_t)base[1];
  const uint32_t *lsub, *inv_d, *bf, *bc, *bv, *ff, *fc;
  plan_layout(base, n_stft, n_mels, &lsub, &inv_d, &bf, &bc, &bv, &ff, &fc);
  return {reinterpret_cast<const int32_t*>(base),     reinterpret_cast<const float*>(lsub),
          reinterpret_cast<const float*>(inv_d),      reinterpret_cast<const int32_t*>(bf),
          reinterpret_cast<const int32_t*>(bc),       reinterpret_cast<const float*>(bv),
          reinterpret_cast<const int32_t*>(ff),       reinterpret_cast<const int32_t*>(fc)};
}

// Odd pitch: frame t's row starts at t * pitch, so the solving lanes (one frame each) hit distinct banks.
__host__ __device__ inline int tile_pitch(int n_mels) { return n_mels | 1; }

// Mel values of frames [t0, t0 + nt) of one row into z[t][m] through element strides.  Lanes run along whichever
// axis is contiguous in memory, so the frame-major view MelSpectrogram returns and a contiguous (n_mels, T) tensor
// both load coalesced; the odd pitch keeps the transposing writes conflict-free.
__device__ inline void load_tile(float* z, int pitch, const float* src, int n_mels, int nt, int64_t s_mel,
                                 int64_t s_frame) {
  const int total = nt * n_mels;
  if (s_frame == 1 && s_mel != 1) {
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
      const int m = i / nt, t = i - m * nt;
      z[t * pitch + m] = src[m * s_mel + t];
    }
  } else {
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
      const int t = i / n_mels, m = i - t * n_mels;
      z[t * pitch + m] = src[t * s_frame + m * s_mel];
    }
  }
}

// G z = b in place for one frame's row of the tile: forward substitution with the unit lower factor, 1/D, back
// substitution with its transpose.  The last BW values ride in registers, so the dependent chain per step is the FMAs
// alone and the tile / factor loads run ahead of it.  The forward and backward kernels run exactly this code.
template <int BW>
__device__ inline void banded_solve_bw(float* __restrict__ z, const float* __restrict__ lsub,
                                       const float* __restrict__ inv_d, int n) {
  float win[BW + 1];  // win[j] = y[i - 1 - j] (forward) / x[i + 1 + j] (backward); 0 outside the system
#pragma unroll
  for (int j = 0; j <= BW; ++j) win[j] = 0.f;
#pragma unroll 4
  for (int i = 0; i < n; ++i) {
    float acc = z[i];
#pragma unroll
    for (int j = 0; j < BW; ++j) acc = fmaf(-__ldg(lsub + i * kBw + j), win[j], acc);
#pragma unroll
    for (int j = BW; j > 0; --j) win[j] = win[j - 1];
    win[0] = acc;
    z[i] = acc * __ldg(inv_d + i);
  }
#pragma unroll
  for (int j = 0; j <= BW; ++j) win[j] = 0.f;
#pragma unroll 4
  for (int i = n - 1; i >= 0; --i) {
    float acc = z[i];
#pragma unroll
    for (int j = 0; j < BW; ++j)
      if (i + 1 + j < n) acc = fmaf(-__ldg(lsub + (i + 1 + j) * kBw + j), win[j], acc);
#pragma unroll
    for (int j = BW; j > 0; --j) win[j] = win[j - 1];
    win[0] = acc;
    z[i] = acc;
  }
}

__device__ inline void banded_solve(float* z, const PlanView& p, int n, int bw) {
  switch (bw) {
    case 0: banded_solve_bw<0>(z, p.lsub, p.inv_d, n); break;
    case 1: banded_solve_bw<1>(z, p.lsub, p.inv_d, n); break;
    case 2: banded_solve_bw<2>(z, p.lsub, p.inv_d, n); break;
    case 3: banded_solve_bw<3>(z, p.lsub, p.inv_d, n); break;
    default: banded_solve_bw<kBw>(z, p.lsub, p.inv_d, n); break;
  }
}

// Pre-relu value of bin k: sum_j fb[k][first + j] z[first + j], in this order in both kernels (the backward's relu
// mask is bit-identical to the forward's).
__device__ inline float bin_value(const float* zrow, const float (&v)[kTaps], int first, int count) {
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < kTaps; ++j)
    if (j < count) acc = fmaf(v[j], zrow[first + j], acc);
  return acc;
}

// torch.relu: NaN passes through (fmaxf would drop it)
__device__ inline float relu(float x) { return x > 0.f || x != x ? x : 0.f; }

__device__ inline void load_bin(const PlanView& p, int k, int& first, int& count, float (&v)[kTaps]) {
  first = p.bin_first[k];
  count = p.bin_count[k];
#pragma unroll
  for (int j = 0; j < kTaps; ++j) v[j] = p.bin_vals[k * kTaps + j];
}

// Shared prologue of both kernels: which row and frames this CTA owns, then the solved tile z = G^-1 m.
__device__ inline int solved_tile(float* z, const PlanView& p, const float* mel, int64_t frames, int64_t tiles,
                                  int64_t s_row, int64_t s_mel, int64_t s_frame, int64_t& row, int64_t& t0) {
  const int n_mels = p.hdr[1], bw = p.hdr[2], pitch = tile_pitch(n_mels);
  row = blockIdx.x / tiles;
  t0 = (blockIdx.x - row * tiles) * kTileFrames;
  const int nt = frames - t0 < kTileFrames ? (int)(frames - t0) : kTileFrames;
  load_tile(z, pitch, mel + row * s_row + t0 * s_frame, n_mels, nt, s_mel, s_frame);
  __syncthreads();
  if (threadIdx.x < nt) banded_solve(z + threadIdx.x * pitch, p, n_mels, bw);
  __syncthreads();
  return nt;
}

// out[row][t][k] = relu(sum_j fb[k][first_k + j] z[t][first_k + j]), FRAME-MAJOR; warps walk frames, lanes walk bins.
__global__ void __launch_bounds__(kThreads)
inverse_mel_kernel(const void* __restrict__ plan, const float* __restrict__ mel, int64_t frames, int64_t tiles,
                   int64_t s_row, int64_t s_mel, int64_t s_frame, float* __restrict__ out) {
  extern __shared__ float z[];
  const PlanView p = plan_view(plan);
  int64_t row, t0;
  const int nt = solved_tile(z, p, mel, frames, tiles, s_row, s_mel, s_frame, row, t0);
  const int n_stft = p.hdr[0], pitch = tile_pitch(p.hdr[1]);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* dst = out + (row * frames + t0) * n_stft;
  for (int k = lane; k < n_stft; k += 32) {
    int first, count;
    float v[kTaps];
    load_bin(p, k, first, count, v);
    for (int t = warp; t < nt; t += kThreads / 32)
      dst[(int64_t)t * n_stft + k] = relu(bin_value(z + t * pitch, v, first, count));
  }
}

// Mel gradient: u[t][m] = sum_{k in filter m} fb[k][m] [x_k > 0] g[t][k] (fixed order, torch's relu rule: no
// gradient where the output is <= 0), then G w = u with the same factors (G is symmetric); w goes out frame-major.
__global__ void __launch_bounds__(kThreads)
inverse_mel_backward_kernel(const void* __restrict__ plan, const float* __restrict__ mel, int64_t frames, int64_t tiles,
                            int64_t s_row, int64_t s_mel, int64_t s_frame, const float* __restrict__ grad,
                            int64_t g_row, int64_t g_frame, int64_t g_bin, float* __restrict__ grad_mel) {
  extern __shared__ float z[];
  const PlanView p = plan_view(plan);
  int64_t row, t0;
  const int nt = solved_tile(z, p, mel, frames, tiles, s_row, s_mel, s_frame, row, t0);
  const int n_mels = p.hdr[1], bw = p.hdr[2], pitch = tile_pitch(n_mels);
  float* w = z + kTileFrames * pitch;
  float* h = w + kTileFrames * pitch;  // [kTileFrames][kGradChunk + 1]: the masked gradient of one chunk of bins
  const float* g = grad + row * g_row + t0 * g_frame;
  const int n_stft = p.hdr[0];
  for (int i = threadIdx.x; i < nt * n_mels; i += kThreads) w[(i / n_mels) * pitch + i % n_mels] = 0.f;
  // bins in ascending chunks: each (t, m) accumulates in ascending k across chunks, always in the same thread
  for (int k0 = 0; k0 < n_stft; k0 += kGradChunk) {
    const int kn = n_stft - k0 < kGradChunk ? n_stft - k0 : kGradChunk;
    const bool frame_lanes = g_bin != 1 && g_frame == 1;  // lanes along the contiguous axis of g
    for (int i = threadIdx.x; i < nt * kn; i += kThreads) {
      const int t = frame_lanes ? i % nt : i / kn, kk = frame_lanes ? i / nt : i % kn;
      int first, count;
      float v[kTaps];
      load_bin(p, k0 + kk, first, count, v);
      const float gv = g[t * g_frame + (int64_t)(k0 + kk) * g_bin];
      h[t * (kGradChunk + 1) + kk] = bin_value(z + t * pitch, v, first, count) > 0.f ? gv : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nt * n_mels; i += kThreads) {
      const int t = i / n_mels, m = i - t * n_mels;
      const int kb = max(p.filt_first[m], k0), ke = min(p.filt_first[m] + p.filt_count[m], k0 + kn);
      float acc = w[t * pitch + m];
      for (int k = kb; k < ke; ++k) {
        const int first = __ldg(p.bin_first + k), j = m - first;
        // fb[k][m]; 0 where an interior zero of filter m puts m outside bin k's span
        const float f = j >= 0 && j < __ldg(p.bin_count + k) ? __ldg(p.bin_vals + k * kTaps + j) : 0.f;
        acc = fmaf(f, h[t * (kGradChunk + 1) + (k - k0)], acc);
      }
      w[t * pitch + m] = acc;
    }
    __syncthreads();
  }
  __syncthreads();
  if (threadIdx.x < nt) banded_solve(w + threadIdx.x * pitch, p, n_mels, bw);
  __syncthreads();
  float* dst = grad_mel + (row * frames + t0) * n_mels;
  for (int i = threadIdx.x; i < nt * n_mels; i += kThreads) {
    const int t = i / n_mels, m = i - t * n_mels;
    dst[i] = w[t * pitch + m];
  }
}

bool dims_ok(int64_t n_stft, int64_t n_mels) { return n_stft > 0 && n_mels > 0 && n_stft <= INT32_MAX; }

int check_run_args(const void* plan, const float* mel, const float* out, int64_t rows, int64_t frames, int64_t n_stft,
                   int64_t n_mels) {
  if (rows < 0 || frames < 0 || !dims_ok(n_stft, n_mels)) return B200A_EINVAL;
  if (rows == 0 || frames == 0) return B200A_OK;  // nothing to enqueue (an empty tensor's pointers may be null)
  if (plan == nullptr || mel == nullptr || out == nullptr) return B200A_EINVAL;
  if (n_mels > kMaxMels || n_mels > n_stft) return B200A_EUNSUPPORTED;
  if (rows * ((frames + kTileFrames - 1) / kTileFrames) > INT32_MAX) return B200A_EUNSUPPORTED;  // grid.x
  return B200A_OK;
}

}  // namespace

size_t inverse_mel_plan_bytes_impl(int64_t n_stft, int64_t n_mels) {
  if (!dims_ok(n_stft, n_mels)) return 0;
  return (size_t)plan_words(n_stft, n_mels) * 4;
}

int inverse_mel_plan_impl(const float* fb, int32_t n_stft, int32_t n_mels, int32_t driver, void* plan, size_t plan_bytes,
                          int32_t* bandwidth, int32_t* pivot) {
  if (fb == nullptr || plan == nullptr || bandwidth == nullptr || pivot == nullptr || n_stft <= 0 || n_mels <= 0 ||
      driver < 0 || driver > 3)
    return B200A_EINVAL;
  *bandwidth = -1;
  *pivot = -1;
  if (plan_bytes < inverse_mel_plan_bytes_impl(n_stft, n_mels)) return B200A_EWORKSPACE;
  const int64_t S = n_stft, M = n_mels;
  // nonzero spans, read from fb itself (a state_dict may load any bank)
  std::vector<int32_t> bfirst(S, 0), bcount(S, 0), ffirst(M, 0), fcount(M, 0);
  std::vector<int64_t> flast(M, -1);
  int32_t bw = 0;
  for (int64_t k = 0; k < S; ++k) {
    int64_t lo = -1, hi = -1;
    for (int64_t m = 0; m < M; ++m)
      if (fb[k * M + m] != 0.f) {
        if (lo < 0) lo = m;
        hi = m;
        if (flast[m] < 0) ffirst[m] = (int32_t)k;
        flast[m] = k;
      }
    if (lo >= 0) {
      bfirst[k] = (int32_t)lo;
      bcount[k] = (int32_t)(hi - lo + 1);
      bw = (int32_t)std::max<int64_t>(bw, hi - lo);
    }
  }
  for (int64_t m = 0; m < M; ++m) fcount[m] = flast[m] < 0 ? 0 : (int32_t)(flast[m] - ffirst[m] + 1);
  *bandwidth = bw;
  if (M > S) {
    // overdetermined: gels fails exactly when a bin (a column of fb^T) is empty; a full-rank tall system has a
    // different solution formula that is not implemented
    if (driver == 0)
      for (int64_t k = 0; k < S; ++k)
        if (bcount[k] == 0) {
          *pivot = (int32_t)k;
          return B200A_ESINGULAR;
        }
    return B200A_EUNSUPPORTED;
  }
  if (M > kMaxMels || bw > kBw) return B200A_EUNSUPPORTED;
  // G = fb^T fb within the band, then banded LDL^T, all in double
  std::vector<double> G(M * (kBw + 1), 0.0);  // G[i][i - j] at i * (kBw + 1) + j
  for (int64_t k = 0; k < S; ++k)
    for (int a = 0; a < bcount[k]; ++a)
      for (int b = 0; b <= a; ++b) {
        const int64_t i = bfirst[k] + a, j = bfirst[k] + b;
        G[i * (kBw + 1) + (i - j)] += (double)fb[k * M + i] * (double)fb[k * M + j];
      }
  std::vector<double> L(M * kBw, 0.0), D(M, 0.0);  // L[i][i - 1 - j] at i * kBw + j
  double gmax = 0.0;
  for (int64_t i = 0; i < M; ++i) gmax = std::max(gmax, G[i * (kBw + 1)]);
  for (int64_t i = 0; i < M; ++i) {
    for (int64_t j = std::max<int64_t>(0, i - bw); j < i; ++j) {
      double s = G[i * (kBw + 1) + (i - j)];
      for (int64_t q = std::max<int64_t>(0, i - bw); q < j; ++q) s -= L[i * kBw + (i - 1 - q)] * L[j * kBw + (j - 1 - q)] * D[q];
      L[i * kBw + (i - 1 - j)] = s / D[j];
    }
    double d = G[i * (kBw + 1)];
    for (int64_t q = std::max<int64_t>(0, i - bw); q < i; ++q) d -= L[i * kBw + (i - 1 - q)] * L[i * kBw + (i - 1 - q)] * D[q];
    if (!(d > 64.0 * DBL_EPSILON * (double)M * gmax)) {  // a zero pivot: G is singular (an empty or dependent filter)
      *pivot = (int32_t)i;
      return B200A_ESINGULAR;
    }
    D[i] = d;
  }
  std::memset(plan, 0, plan_bytes < inverse_mel_plan_bytes_impl(S, M) ? plan_bytes : inverse_mel_plan_bytes_impl(S, M));
  uint32_t* base = static_cast<uint32_t*>(plan);
  base[0] = (uint32_t)n_stft, base[1] = (uint32_t)n_mels, base[2] = (uint32_t)bw;
  uint32_t *lsub, *inv_d, *bf, *bc, *bv, *ff, *fc;
  plan_layout(base, S, M, &lsub, &inv_d, &bf, &bc, &bv, &ff, &fc);
  float* lsf = reinterpret_cast<float*>(lsub);
  float* idf = reinterpret_cast<float*>(inv_d);
  float* bvf = reinterpret_cast<float*>(bv);
  for (int64_t i = 0; i < M; ++i) {
    for (int j = 0; j < kBw; ++j) lsf[i * kBw + j] = (float)L[i * kBw + j];
    idf[i] = (float)(1.0 / D[i]);
  }
  std::memcpy(bf, bfirst.data(), S * 4);
  std::memcpy(bc, bcount.data(), S * 4);
  std::memcpy(ff, ffirst.data(), M * 4);
  std::memcpy(fc, fcount.data(), M * 4);
  for (int64_t k = 0; k < S; ++k)
    for (int j = 0; j < bcount[k]; ++j) bvf[k * kTaps + j] = fb[k * M + bfirst[k] + j];
  return B200A_OK;
}

int inverse_mel_run_impl(const void* plan, int32_t n_stft, int32_t n_mels, const float* mel, int64_t rows, int64_t frames,
                         int64_t s_row, int64_t s_mel, int64_t s_frame, float* out, cudaStream_t stream) {
  int rc = check_run_args(plan, mel, out, rows, frames, n_stft, n_mels);
  if (rc != B200A_OK || rows == 0 || frames == 0) return rc;
  const int64_t tiles = (frames + kTileFrames - 1) / kTileFrames;
  const size_t smem = (size_t)kTileFrames * tile_pitch(n_mels) * sizeof(float);
  return launch_kernel(inverse_mel_kernel, rows * tiles, kThreads, smem, stream, plan, mel, frames, tiles, s_row, s_mel,
                       s_frame, out);
}

int inverse_mel_backward_impl(const void* plan, int32_t n_stft, int32_t n_mels, const float* mel, int64_t rows,
                              int64_t frames, int64_t s_row, int64_t s_mel, int64_t s_frame, const float* grad,
                              int64_t g_row, int64_t g_frame, int64_t g_bin, float* grad_mel, cudaStream_t stream) {
  int rc = check_run_args(plan, mel, grad_mel, rows, frames, n_stft, n_mels);
  if (rc == B200A_OK && rows > 0 && frames > 0 && grad == nullptr) rc = B200A_EINVAL;
  if (rc != B200A_OK || rows == 0 || frames == 0) return rc;
  const int64_t tiles = (frames + kTileFrames - 1) / kTileFrames;
  const size_t smem = (size_t)kTileFrames * (2 * tile_pitch(n_mels) + kGradChunk + 1) * sizeof(float);
  return launch_kernel(inverse_mel_backward_kernel, rows * tiles, kThreads, smem, stream, plan, mel, frames, tiles, s_row,
                       s_mel, s_frame, grad, g_row, g_frame, g_bin, grad_mel);
}

}  // namespace b200a
