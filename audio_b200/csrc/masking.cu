// SpecAugment masking (functional/functional.py mask_along_axis_iid / mask_along_axis, transforms FrequencyMasking,
// TimeMasking, SpecAugment): any number of frequency and time masks over rows x freq x time float32 in one pass.
//
// The work is cut into 32 x 32 (freq x time) tiles of one row, dealt round-robin to at most kMaxCtas CTAs of 256
// threads.  Per tile:
//   flags   64 threads evaluate every mask of the row once: thread j < 32 flags freq index f0 + j, thread 32 + j time
//           index t0 + j.  A per-row mask's [start, end) is recomputed from its two draws with the reference's float32
//           arithmetic (__fmul_rn / __fsub_rn, so nothing is contracted into an FMA; truncating conversions), and the
//           index is compared as float32, as the reference compares against a float32 arange.
//   copy    a warp walks 32 elements along the input's unit-stride axis.  When the output's unit-stride axis is the
//           same, each element goes straight to the output; otherwise the tile is staged in shared memory (padded to
//           33 columns, so both walks are free of bank conflicts) and written back along the output's axis.  Masked
//           elements are not read in the forward pass.
// The backward is the same pass on the upstream gradient with fill 0.  When the fill tensor needs a gradient, every
// thread also sums the gradient over its masked elements in double, the CTA folds its threads in a fixed tree into
// one partial per CTA, and a one-CTA kernel folds the partials in a fixed order: no atomics, reruns are bit-identical.
#include <climits>

#include "common.cuh"

namespace b200a {
namespace {

constexpr int kTile = 32;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxCtas = 1024;  // the grid cap (8 resident CTAs on each of 132 SMs), and the backward partial sums

struct MaskArgs {
  int64_t rows1, freq, time;
  int64_t is[4], os[4];
  int64_t tiles_f, tiles_t, tiles;
  const b200a_mask_spec* masks;  // the device copy of the table
  int n_masks;
  int in_fast, out_fast;  // the axis each side walks along its lanes: B200A_MASK_AXIS_FREQ or _TIME
  float fill;
  const float* fill_ptr;
  const float* in;
  float* out;
  double* partials;
};

// Whether index i of `axis` lies in any mask of row r.
__device__ bool masked_index(const MaskArgs& a, int64_t r, int axis, int64_t i) {
  const float fi = (float)i;
  const float size = (float)(axis == B200A_MASK_AXIS_TIME ? a.time : a.freq);
  bool hit = false;
  for (int k = 0; k < a.n_masks; ++k) {
    const b200a_mask_spec& m = a.masks[k];
    if (m.axis != axis) continue;
    int64_t start = m.start, end = m.end;
    if (m.value_draws != nullptr) {
      const float value = __fmul_rn(__ldg(m.value_draws + r), (float)m.mask_param);
      const float lo = __fmul_rn(__ldg(m.start_draws + r), __fsub_rn(size, value));
      start = (int64_t)lo;
      end = start + (int64_t)value;
    }
    hit |= fi >= (float)start && fi < (float)end;
  }
  return hit;
}

template <bool kStage, bool kReduce>
__global__ void __launch_bounds__(kThreads, 8) mask_kernel(const MaskArgs a) {
  __shared__ float tile[kTile][kTile + 1];  // [f][t]
  __shared__ bool flags[2][kTile];          // [B200A_MASK_AXIS_FREQ / _TIME][index in the tile]
  __shared__ double red[kWarps];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float fill = a.fill_ptr != nullptr ? *a.fill_ptr : a.fill;
  double acc = 0.0;

  for (int64_t id = blockIdx.x; id < a.tiles; id += gridDim.x) {
    const int64_t tt = id % a.tiles_t, rest = id / a.tiles_t;
    const int64_t f0 = rest % a.tiles_f * kTile, t0 = tt * kTile, r = rest / a.tiles_f;
    if (tid < 2 * kTile) flags[warp][lane] = masked_index(a, r, warp, (warp ? t0 : f0) + lane);
    __syncthreads();
    const int64_t r0 = r / a.rows1, r1 = r % a.rows1;
    const float* in = a.in + r0 * a.is[0] + r1 * a.is[1] + f0 * a.is[2] + t0 * a.is[3];
    float* out = a.out == nullptr ? nullptr : a.out + r0 * a.os[0] + r1 * a.os[1] + f0 * a.os[2] + t0 * a.os[3];
    const int nf = a.freq - f0 < kTile ? (int)(a.freq - f0) : kTile, nt = a.time - t0 < kTile ? (int)(a.time - t0) : kTile;

#pragma unroll
    for (int k = 0; k < kTile / kWarps; ++k) {
      const int slow = warp + k * kWarps;
      const int f = a.in_fast == B200A_MASK_AXIS_TIME ? slow : lane, t = a.in_fast == B200A_MASK_AXIS_TIME ? lane : slow;
      if (f < nf && t < nt) {
        const bool m = flags[0][f] | flags[1][t];
        float v = fill;
        if (!m || kReduce) {
          const float x = in[f * a.is[2] + t * a.is[3]];
          if (!m) v = x;
          if (kReduce && m) acc += (double)x;
        }
        if (kStage)
          tile[f][t] = v;
        else if (out != nullptr)
          out[f * a.os[2] + t * a.os[3]] = v;
      }
    }
    if (kStage) {
      __syncthreads();
#pragma unroll
      for (int k = 0; k < kTile / kWarps; ++k) {
        const int slow = warp + k * kWarps;
        const int f = a.out_fast == B200A_MASK_AXIS_TIME ? slow : lane;
        const int t = a.out_fast == B200A_MASK_AXIS_TIME ? lane : slow;
        if (f < nf && t < nt) out[f * a.os[2] + t * a.os[3]] = tile[f][t];
      }
    }
    __syncthreads();
  }

  if (kReduce) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
    if (lane == 0) red[warp] = acc;
    __syncthreads();
    if (tid == 0) {
      double s = 0.0;
      for (int w = 0; w < kWarps; ++w) s += red[w];
      a.partials[blockIdx.x] = s;
    }
  }
}

// One CTA: grad_fill = the partials [0, n) summed in a fixed order.
__global__ void __launch_bounds__(kThreads) mask_fold_kernel(const double* partials, int n, float* grad_fill) {
  __shared__ double red[kWarps];
  const int tid = threadIdx.x;
  double acc = 0.0;
  for (int i = tid; i < n; i += kThreads) acc += partials[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((tid & 31) == 0) red[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += red[w];
    *grad_fill = (float)s;
  }
}

// The axis a side walks along its lanes: the one of unit (else smaller) stride among the axes longer than 1.
int fast_axis(const int64_t* s, int64_t freq, int64_t time) {
  const int64_t sf = freq > 1 ? (s[2] < 0 ? -s[2] : s[2]) : INT64_MAX;
  const int64_t st = time > 1 ? (s[3] < 0 ? -s[3] : s[3]) : INT64_MAX;
  return st <= sf ? B200A_MASK_AXIS_TIME : B200A_MASK_AXIS_FREQ;
}

size_t table_bytes(const b200a_mask_desc* d) { return align_up((size_t)d->n_masks * sizeof(b200a_mask_spec), 256); }

bool desc_ok(const b200a_mask_desc* d) {
  return d != nullptr && d->rows0 >= 0 && d->rows1 >= 0 && d->freq >= 0 && d->time >= 0 && d->n_masks >= 0;
}

int validate_mask(const b200a_mask_desc* d, const b200a_mask_spec* masks) {
  if (!desc_ok(d)) return B200A_EINVAL;
  if (masks == nullptr) return d->n_masks == 0 ? B200A_OK : B200A_EINVAL;
  for (int k = 0; k < d->n_masks; ++k) {
    const b200a_mask_spec& m = masks[k];
    if (m.axis != B200A_MASK_AXIS_FREQ && m.axis != B200A_MASK_AXIS_TIME) return B200A_EINVAL;
    if (m.value_draws != nullptr && (m.mask_param < 1 || m.start_draws == nullptr)) return B200A_EINVAL;
  }
  return B200A_OK;
}

// Static shared memory only, so a plain launch (launch_kernel's dynamic shared-memory opt-in would exceed the
// per-CTA limit together with the static tile).
template <bool kReduce>
int launch_mask(const MaskArgs& a, int64_t grid, cudaStream_t stream) {
  if (a.in_fast == a.out_fast)
    mask_kernel<false, kReduce><<<(unsigned)grid, kThreads, 0, stream>>>(a);
  else
    mask_kernel<true, kReduce><<<(unsigned)grid, kThreads, 0, stream>>>(a);
  return launch_status();
}

// Both entry points: out may be null only with grad_fill (the backward's sum alone).
int mask_launch(const b200a_mask_desc* d, const b200a_mask_spec* masks, const float* in, float* out, float fill,
                const float* fill_ptr, float* grad_fill, void* ws, size_t ws_bytes, cudaStream_t stream) {
  if (validate_mask(d, masks) != B200A_OK || ws == nullptr) return B200A_EINVAL;
  if (ws_bytes < mask_workspace_bytes_impl(d)) return B200A_EWORKSPACE;
  const int64_t rows = d->rows0 * d->rows1;
  if (rows == 0 || d->freq == 0 || d->time == 0) {
    if (grad_fill != nullptr && cudaMemsetAsync(grad_fill, 0, sizeof(float), stream) != cudaSuccess) return B200A_ECUDA;
    return B200A_OK;
  }
  if (in == nullptr || (out == nullptr && grad_fill == nullptr)) return B200A_EINVAL;
  if (d->n_masks > 0 &&
      cudaMemcpyAsync(ws, masks, (size_t)d->n_masks * sizeof(b200a_mask_spec), cudaMemcpyHostToDevice, stream) !=
          cudaSuccess)
    return B200A_ECUDA;
  MaskArgs a{};
  a.rows1 = d->rows1;
  a.freq = d->freq;
  a.time = d->time;
  for (int i = 0; i < 4; ++i) {
    a.is[i] = d->in_stride[i];
    a.os[i] = d->out_stride[i];
  }
  a.tiles_f = (d->freq + kTile - 1) / kTile;
  a.tiles_t = (d->time + kTile - 1) / kTile;
  a.tiles = rows * a.tiles_f * a.tiles_t;
  a.masks = static_cast<const b200a_mask_spec*>(ws);
  a.n_masks = d->n_masks;
  a.in_fast = fast_axis(a.is, a.freq, a.time);
  a.out_fast = out != nullptr ? fast_axis(a.os, a.freq, a.time) : a.in_fast;
  a.fill = fill;
  a.fill_ptr = fill_ptr;
  a.in = in;
  a.out = out;
  a.partials = reinterpret_cast<double*>(static_cast<char*>(ws) + table_bytes(d));
  const int64_t grid = a.tiles < kMaxCtas ? a.tiles : kMaxCtas;
  if (grad_fill == nullptr) return launch_mask<false>(a, grid, stream);
  const int rc = launch_mask<true>(a, grid, stream);
  if (rc != B200A_OK) return rc;
  mask_fold_kernel<<<1, kThreads, 0, stream>>>(a.partials, (int)grid, grad_fill);
  return launch_status();
}

}  // namespace

size_t mask_workspace_bytes_impl(const b200a_mask_desc* d) {
  if (!desc_ok(d)) return 0;
  return table_bytes(d) + kMaxCtas * sizeof(double);
}

int mask_run_impl(const b200a_mask_desc* d, const b200a_mask_spec* masks, const float* in, float* out,
                  const float* fill_ptr, void* ws, size_t ws_bytes, cudaStream_t stream) {
  return mask_launch(d, masks, in, out, d == nullptr ? 0.f : d->fill, fill_ptr, nullptr, ws, ws_bytes, stream);
}

int mask_backward_impl(const b200a_mask_desc* d, const b200a_mask_spec* masks, const float* grad_out, float* grad_in,
                       float* grad_fill, void* ws, size_t ws_bytes, cudaStream_t stream) {
  return mask_launch(d, masks, grad_out, grad_in, 0.f, nullptr, grad_fill, ws, ws_bytes, stream);
}

}  // namespace b200a
