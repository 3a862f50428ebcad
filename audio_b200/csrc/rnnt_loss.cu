// rnnt_loss (functional.py:1747-1796, rnnt/cpu/cpu_kernels.h): the RNN-T loss of a joiner output
// logits[B][maxT][maxU][V] (maxU = max target length + 1), float32 or float16, all arithmetic in float32.
//
//   check      one CTA: max / min of both length vectors and a flag for an out-of-range target inside a sequence's
//              length, 20 bytes the caller reads back once per call.
//   rows       per valid (b, t, u) row, one read of the logits with an online max / sum log-sum-exp by a group of G
//              lanes (G sized by V), 16-byte loads between a scalar head and tail; writes the (skip, emit) pair
//              (log-probs, or the raw logits without the fused log-softmax) and, for the gradient, denom.  Padded
//              rows are never read; without the fused log-softmax only the blank and target logits are read.
//   alpha/beta one CTA per (sequence, direction) in one launch, walking the anti-diagonals t + u = n with one CTA
//              barrier per diagonal; the previous diagonal sits in a shared-memory ring and the next diagonal's
//              (skip, emit) values arrive by cp.async while the current one computes.  The beta CTA writes the cost
//              -beta(0, 0).  Without a gradient only the beta CTAs run and nothing is stored.
//   gradient   per row of the joint, clamp(formula) * dy[b] in the logits' dtype, every element written once: padded
//              rows and rows of a sequence with a non-finite cost get zeros without a read.
#include <cuda_fp16.h>

#include <climits>
#include <cmath>

#include "common.cuh"
#include "ptx.cuh"

namespace b200a {
namespace {

constexpr int kRowThreads = 256;
constexpr int kCheckThreads = 1024;
constexpr int kDiagMaxThreads = 1024;

__device__ __forceinline__ float to_f(float x) { return x; }
__device__ __forceinline__ float to_f(__half x) { return __half2float(x); }
template <typename T>
__device__ __forceinline__ T from_f(float x);
template <>
__device__ __forceinline__ float from_f<float>(float x) { return x; }
template <>
__device__ __forceinline__ __half from_f<__half>(float x) { return __float2half_rn(x); }

template <typename T>
constexpr int vec_width() { return 16 / (int)sizeof(T); }

template <typename T, int N>
__device__ __forceinline__ void load_vec(const T* p, float (&x)[N]) {
  const uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
  if constexpr (sizeof(T) == 4) {
    x[0] = __uint_as_float(v.x);
    x[1] = __uint_as_float(v.y);
    x[2] = __uint_as_float(v.z);
    x[3] = __uint_as_float(v.w);
  } else {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h[i]);
      x[2 * i] = f.x;
      x[2 * i + 1] = f.y;
    }
  }
}

template <typename T, int N>
__device__ __forceinline__ void store_vec(T* p, const float (&x)[N]) {
  uint4 v;
  if constexpr (sizeof(T) == 4) {
    v = make_uint4(__float_as_uint(x[0]), __float_as_uint(x[1]), __float_as_uint(x[2]), __float_as_uint(x[3]));
  } else {
    __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(x[2 * i], x[2 * i + 1]);
  }
  *reinterpret_cast<uint4*>(p) = v;
}

// Elements of a row before its first 16-byte boundary (the scalar head); the vector body follows, then a scalar tail.
template <typename T, int VEC>
__device__ __forceinline__ int row_head(const T* row, int V) {
  if constexpr (VEC == 1) return V;
  const int h = (int)(((16u - ((uint32_t)(uintptr_t)row & 15u)) & 15u) / sizeof(T));
  return h < V ? h : V;
}

// The reference's log-sum-exp (rnnt/cpu/math.h), operand order included: lse(-inf, -inf) is NaN.
__device__ __forceinline__ float lse(float x, float y) {
  return y > x ? y + log1pf(expf(x - y)) : x + log1pf(expf(y - x));
}

// Lanes [base, base + G) of the warp: every lane of a group works on the same row, so shuffles stay in the group.
__device__ __forceinline__ unsigned group_mask(int G) {
  return G == 32 ? 0xffffffffu : ((1u << G) - 1u) << ((threadIdx.x & 31) & ~(G - 1));
}

struct RowPos {
  int b, t, u;
};
__device__ __forceinline__ RowPos row_pos(int64_t row, int max_t, int max_u) {
  const int64_t per_b = (int64_t)max_t * max_u;
  const int b = (int)(row / per_b);
  const int r = (int)(row - (int64_t)b * per_b);
  return {b, r / max_u, r % max_u};
}

__global__ void __launch_bounds__(kCheckThreads) rnnt_check_kernel(int batch, int classes, const int32_t* targets,
                                                                  int64_t target_cols, const int32_t* logit_lengths,
                                                                  const int32_t* target_lengths, int32_t* out) {
  __shared__ int s[5];
  if (threadIdx.x == 0) {
    s[0] = INT_MIN;
    s[1] = INT_MAX;
    s[2] = INT_MIN;
    s[3] = INT_MAX;
    s[4] = 0;
  }
  __syncthreads();
  int t_max = INT_MIN, t_min = INT_MAX, u_max = INT_MIN, u_min = INT_MAX, bad = 0;
  for (int b = threadIdx.x; b < batch; b += blockDim.x) {
    const int tl = logit_lengths[b], ul = target_lengths[b];
    t_max = max(t_max, tl);
    t_min = min(t_min, tl);
    u_max = max(u_max, ul);
    u_min = min(u_min, ul);
  }
  const int64_t n = (int64_t)batch * target_cols;
  for (int64_t e = threadIdx.x; e < n; e += blockDim.x) {
    const int b = (int)(e / target_cols);
    const int64_t j = e - (int64_t)b * target_cols;
    if (j < target_lengths[b]) {
      const int v = targets[e];
      bad |= v < 0 || v >= classes;
    }
  }
  atomicMax(&s[0], t_max);
  atomicMin(&s[1], t_min);
  atomicMax(&s[2], u_max);
  atomicMin(&s[3], u_min);
  if (bad) s[4] = 1;
  __syncthreads();
  if (threadIdx.x < 5) out[threadIdx.x] = s[threadIdx.x];
}

// One group of G = 2^g lanes per valid row, grid-strided over all B * maxT * maxU rows.
template <typename T, bool FUSED>
__global__ void __launch_bounds__(kRowThreads) rnnt_rows_kernel(b200a_rnnt_loss_desc d, const T* __restrict__ logits,
                                                                const int32_t* __restrict__ targets,
                                                                const int32_t* __restrict__ logit_lengths,
                                                                const int32_t* __restrict__ target_lengths,
                                                                float2* __restrict__ lp, float* __restrict__ denom,
                                                                int group_log2) {
  constexpr int VEC = vec_width<T>();
  const int G = 1 << group_log2, lane = threadIdx.x & (G - 1);
  const unsigned mask = group_mask(G);
  const int V = d.classes;
  const int64_t rows = (int64_t)d.batch * d.max_t * d.max_u;
  const int64_t stride = ((int64_t)gridDim.x * kRowThreads) >> group_log2;
  for (int64_t row = ((int64_t)blockIdx.x * kRowThreads + threadIdx.x) >> group_log2; row < rows; row += stride) {
    const RowPos p = row_pos(row, d.max_t, d.max_u);
    const int U = target_lengths[p.b] + 1;
    if (p.t >= logit_lengths[p.b] || p.u >= U) continue;
    const T* x = logits + row * V;
    float den = 0.f;
    if constexpr (FUSED) {
      float m = -INFINITY, s = 0.f;
      auto take = [&](float v) {  // one element into the running (max, sum)
        if (v > m) {
          s *= expf(m - v);
          m = v;
        }
        if (m != -INFINITY) s += expf(v - m);
      };
      const int head = row_head<T, VEC>(x, V);
      const int nvec = (V - head) / VEC;
      for (int i = lane; i < head; i += G) take(to_f(x[i]));
#pragma unroll 4
      for (int i = lane; i < nvec; i += G) {
        float v[VEC];
        load_vec<T, VEC>(x + head + i * VEC, v);
        float vm = v[0];
#pragma unroll
        for (int j = 1; j < VEC; ++j) vm = fmaxf(vm, v[j]);
        if (vm > m) {
          s *= expf(m - vm);
          m = vm;
        }
        if (m != -INFINITY) {
#pragma unroll
          for (int j = 0; j < VEC; ++j) s += expf(v[j] - m);
        }
      }
      for (int i = head + nvec * VEC + lane; i < V; i += G) take(to_f(x[i]));
      for (int o = G >> 1; o > 0; o >>= 1) {
        const float m2 = __shfl_xor_sync(mask, m, o), s2 = __shfl_xor_sync(mask, s, o);
        const float mm = fmaxf(m, m2);
        s = (m == -INFINITY ? 0.f : s * expf(m - mm)) + (m2 == -INFINITY ? 0.f : s2 * expf(m2 - mm));
        m = mm;
      }
      den = m + logf(s);
    }
    if (lane == 0) {
      const float skip = to_f(x[d.blank]) - den;
      const float emit = p.u < U - 1 ? to_f(x[targets[(int64_t)p.b * (d.max_u - 1) + p.u]]) - den : 0.f;
      lp[row] = make_float2(skip, emit);
      if (FUSED && denom != nullptr) denom[row] = den;
    }
  }
}

// blockIdx.x = dirs * b + k: k == 0 walks beta (and writes the cost), k == 1 walks alpha.  Shared memory: the ring of
// the previous diagonal's values [2][maxU] floats, then the prefetched (skip, emit) operands [2][maxU] float2.
template <typename T>
__global__ void __launch_bounds__(kDiagMaxThreads) rnnt_alpha_beta_kernel(b200a_rnnt_loss_desc d,
                                                                          const float2* __restrict__ lp,
                                                                          const int32_t* __restrict__ logit_lengths,
                                                                          const int32_t* __restrict__ target_lengths,
                                                                          float* __restrict__ alpha,
                                                                          float* __restrict__ beta, T* __restrict__ costs,
                                                                          int dirs) {
  extern __shared__ float smem[];
  const int max_u = d.max_u;
  float* ring = smem;
  float2* pre = reinterpret_cast<float2*>(smem + 2 * max_u);
  const int b = blockIdx.x / dirs;
  const bool is_alpha = (blockIdx.x % dirs) == 1;
  const int T_b = logit_lengths[b], U = target_lengths[b] + 1;
  const int64_t base = (int64_t)b * d.max_t * max_u;
  const float2* L = lp + base;
  const int last = T_b + U - 2;  // diagonals 0..last
  const bool save = dirs == 2;

  // cell operands of diagonal n into pre[n & 1]: alpha reads skip(t-1, u) and emit(t, u-1), beta the pair at (t, u)
  auto prefetch = [&](int n) {
    float2* slot = pre + (n & 1) * max_u;
    for (int u = threadIdx.x; u < U; u += blockDim.x) {
      const int t = n - u;
      if (t < 0 || t >= T_b) continue;
      const int64_t c = (int64_t)t * max_u + u;
      if (is_alpha) {
        if (t > 0) cp_async4(&slot[u].x, &L[c - max_u].x);
        if (u > 0) cp_async4(&slot[u].y, &L[c - 1].y);
      } else {
        cp_async4(&slot[u].x, &L[c].x);
        cp_async4(&slot[u].y, &L[c].y);
      }
    }
  };

  if (is_alpha) {
    if (threadIdx.x == 0) {
      ring[0] = 0.f;
      alpha[base] = 0.f;
    }
    if (last >= 1) prefetch(1);
    __syncthreads();
    for (int n = 1; n <= last; ++n) {
      cp_async_wait_all();
      if (n < last) prefetch(n + 1);
      const float* prev = ring + ((n - 1) & 1) * max_u;
      float* cur = ring + (n & 1) * max_u;
      const float2* op = pre + (n & 1) * max_u;
      for (int u = threadIdx.x; u < U; u += blockDim.x) {
        const int t = n - u;
        if (t < 0 || t >= T_b) continue;
        float v;
        if (u == 0) {
          v = prev[0] + op[0].x;
        } else if (t == 0) {
          v = prev[u - 1] + op[u].y;
        } else {
          v = lse(prev[u] + op[u].x, prev[u - 1] + op[u].y);
        }
        cur[u] = v;
        alpha[base + (int64_t)t * max_u + u] = v;
      }
      __syncthreads();
    }
    return;
  }

  // beta: diagonal `last` holds only (T-1, U-1)
  const int64_t corner = (int64_t)(T_b - 1) * max_u + (U - 1);
  if (threadIdx.x == 0) {
    const float v = L[corner].x;
    ring[(last & 1) * max_u + U - 1] = v;
    if (save) beta[base + corner] = v;
    if (last == 0) costs[b] = from_f<T>(-v);
  }
  if (last >= 1) prefetch(last - 1);
  __syncthreads();
  for (int n = last - 1; n >= 0; --n) {
    cp_async_wait_all();
    if (n > 0) prefetch(n - 1);
    const float* prev = ring + ((n + 1) & 1) * max_u;
    float* cur = ring + (n & 1) * max_u;
    const float2* op = pre + (n & 1) * max_u;
    for (int u = threadIdx.x; u < U; u += blockDim.x) {
      const int t = n - u;
      if (t < 0 || t >= T_b) continue;
      float v;
      if (u == U - 1) {
        v = prev[u] + op[u].x;
      } else if (t == T_b - 1) {
        v = prev[u + 1] + op[u].y;
      } else {
        v = lse(prev[u] + op[u].x, prev[u + 1] + op[u].y);
      }
      cur[u] = v;
      if (save) beta[base + (int64_t)t * max_u + u] = v;
      if (n == 0) costs[b] = from_f<T>(-v);
    }
    __syncthreads();
  }
}

// The reference's clamp (cpu_kernels.h:339-343): min(g, clamp) then max(., -clamp), by its comparisons
__device__ __forceinline__ float clamp_grad(float g, float clamp) {
  if (clamp > 0.f) {
    g = g > clamp ? clamp : g;
    g = g > -clamp ? g : -clamp;
  }
  return g;
}

// One group per row of the joint.  VEC == 1 when the logits and the gradient are not equally aligned.
template <typename T, int VEC, bool FUSED>
__global__ void __launch_bounds__(kRowThreads) rnnt_grad_kernel(
    b200a_rnnt_loss_desc d, const T* __restrict__ logits, const int32_t* __restrict__ targets,
    const int32_t* __restrict__ logit_lengths, const int32_t* __restrict__ target_lengths,
    const float* __restrict__ denom, const float* __restrict__ alpha, const float* __restrict__ beta,
    const T* __restrict__ grad_costs, int64_t grad_costs_stride, T* __restrict__ grad, int group_log2) {
  const int G = 1 << group_log2, lane = threadIdx.x & (G - 1);
  const int V = d.classes, blank = d.blank;
  const float clamp = d.clamp;
  const int64_t rows = (int64_t)d.batch * d.max_t * d.max_u;
  const int64_t stride = ((int64_t)gridDim.x * kRowThreads) >> group_log2;
  for (int64_t row = ((int64_t)blockIdx.x * kRowThreads + threadIdx.x) >> group_log2; row < rows; row += stride) {
    const RowPos p = row_pos(row, d.max_t, d.max_u);
    const int T_b = logit_lengths[p.b], U = target_lengths[p.b] + 1;
    const T* x = logits + row * V;
    T* out = grad + row * V;
    const int head = row_head<T, VEC>(out, V);
    const int nvec = (V - head) / VEC;
    const int tail = head + nvec * VEC;
    const float cost = p.t < T_b && p.u < U ? -beta[row - ((int64_t)p.t * d.max_u + p.u)] : 0.f;
    if (p.t >= T_b || p.u >= U || !isfinite(cost)) {
      const float z[VEC] = {};
      for (int i = lane; i < head; i += G) out[i] = from_f<T>(0.f);
      if constexpr (VEC > 1)
        for (int i = lane; i < nvec; i += G) store_vec<T, VEC>(out + head + i * VEC, z);
      for (int i = tail + lane; i < V; i += G) out[i] = from_f<T>(0.f);
      continue;
    }
    const float dy = to_f(grad_costs[p.b * grad_costs_stride]);
    const float a = alpha[row], bt = beta[row];
    const bool last_t = p.t == T_b - 1, last_u = p.u == U - 1;
    const float b_next_t = last_t ? 0.f : beta[row + d.max_u];
    const float b_next_u = last_u ? 0.f : beta[row + 1];
    const int tgt = last_u ? -1 : targets[(int64_t)p.b * (d.max_u - 1) + p.u];
    if constexpr (FUSED) {
      const float c = a + cost - denom[row];
      auto value = [&](int k, float xv) {  // cpu_kernels.h:323-345
        const float g = xv + c;
        const float e = expf(g + bt);
        float r = e;
        if (k == blank && last_t && last_u) {
          r = e - expf(g);
        } else if (k == blank && !last_t) {
          r = e - expf(g + b_next_t);
        } else if (k == tgt) {
          r = e - expf(g + b_next_u);
        }
        return clamp_grad(r, clamp) * dy;
      };
      for (int i = lane; i < head; i += G) out[i] = from_f<T>(value(i, to_f(x[i])));
      if constexpr (VEC > 1) {
#pragma unroll 2
        for (int i = lane; i < nvec; i += G) {
          const int k0 = head + i * VEC;
          float v[VEC];
          load_vec<T, VEC>(x + k0, v);
#pragma unroll
          for (int j = 0; j < VEC; ++j) v[j] = value(k0 + j, v[j]);
          store_vec<T, VEC>(out + k0, v);
        }
      }
      for (int i = tail + lane; i < V; i += G) out[i] = from_f<T>(value(i, to_f(x[i])));
    } else {
      // cpu_kernels.h:357-377: -exp(cost + logit + alpha + beta(next)) at the blank and the target, -exp(-inf) elsewhere
      float v_blank = 0.f, v_tgt = 0.f;
      const bool has_blank = (last_t && last_u) || !last_t;
      if (has_blank) v_blank = -expf(cost + to_f(x[blank]) + a + (last_t ? 0.f : b_next_t));
      if (tgt >= 0 && !(tgt == blank && has_blank)) v_tgt = -expf(cost + to_f(x[tgt]) + a + b_next_u);
      v_blank = clamp_grad(v_blank, clamp) * dy;
      v_tgt = clamp_grad(v_tgt, clamp) * dy;
      auto value = [&](int k) { return k == blank && has_blank ? v_blank : k == tgt ? v_tgt : 0.f; };
      for (int i = lane; i < head; i += G) out[i] = from_f<T>(value(i));
      if constexpr (VEC > 1) {
        for (int i = lane; i < nvec; i += G) {
          const int k0 = head + i * VEC;
          float v[VEC];
#pragma unroll
          for (int j = 0; j < VEC; ++j) v[j] = value(k0 + j);
          store_vec<T, VEC>(out + k0, v);
        }
      }
      for (int i = tail + lane; i < V; i += G) out[i] = from_f<T>(value(i));
    }
  }
}

int validate_rnnt(const b200a_rnnt_loss_desc* d) {
  if (d == nullptr || d->batch < 1 || d->max_t < 1 || d->max_u < 1 || d->classes < 1) return B200A_EINVAL;
  if (d->blank < 0 || d->blank >= d->classes) return B200A_EINVAL;
  if ((d->dtype != B200A_DTYPE_F32 && d->dtype != B200A_DTYPE_F16) || (d->fused != 0 && d->fused != 1))
    return B200A_EINVAL;
  if (d->max_u > B200A_RNNT_MAX_U || (int64_t)d->batch * 2 > INT_MAX) return B200A_EUNSUPPORTED;
  return B200A_OK;
}

// lanes per row: enough 16-byte vectors to cover V once, at most a warp
int group_log2_for(const b200a_rnnt_loss_desc& d) {
  const int vec = d.dtype == B200A_DTYPE_F16 ? 8 : 4;
  const int need = (d.classes + vec - 1) / vec;
  int g = 0;
  while ((1 << g) < need && g < 5) ++g;
  return g;
}

int64_t row_grid(const b200a_rnnt_loss_desc& d, int group_log2) {
  const int64_t rows = (int64_t)d.batch * d.max_t * d.max_u;
  const int64_t blocks = ((rows << group_log2) + kRowThreads - 1) / kRowThreads;
  return sm_capped_grid(blocks, 2048 / kRowThreads);
}

template <typename T>
int forward_typed(const b200a_rnnt_loss_desc& d, const void* logits, const int32_t* targets,
                  const int32_t* logit_lengths, const int32_t* target_lengths, void* costs, float* denom, float* alpha,
                  float* beta, float2* lp, cudaStream_t stream) {
  const T* x = static_cast<const T*>(logits);
  int rc;
  if (d.fused) {
    const int g = group_log2_for(d);
    rc = launch_kernel(rnnt_rows_kernel<T, true>, row_grid(d, g), kRowThreads, 0, stream, d, x, targets,
                       logit_lengths, target_lengths, lp, denom, g);
  } else {
    rc = launch_kernel(rnnt_rows_kernel<T, false>, row_grid(d, 0), kRowThreads, 0, stream, d, x, targets,
                       logit_lengths, target_lengths, lp, denom, 0);
  }
  if (rc != B200A_OK) return rc;
  const int dirs = alpha != nullptr ? 2 : 1;
  const int threads = d.max_u >= kDiagMaxThreads ? kDiagMaxThreads : (d.max_u + 31) / 32 * 32;
  const size_t smem = (size_t)d.max_u * (2 * sizeof(float) + 2 * sizeof(float2));
  return launch_kernel(rnnt_alpha_beta_kernel<T>, (int64_t)d.batch * dirs, threads, smem, stream, d,
                       (const float2*)lp, logit_lengths, target_lengths, alpha, beta, static_cast<T*>(costs), dirs);
}

template <typename T, bool FUSED>
int backward_typed(const b200a_rnnt_loss_desc& d, const void* logits, const int32_t* targets,
                   const int32_t* logit_lengths, const int32_t* target_lengths, const float* denom, const float* alpha,
                   const float* beta, const void* grad_costs, int64_t grad_costs_stride, void* grad_logits,
                   cudaStream_t stream) {
  const T* x = static_cast<const T*>(logits);
  const T* dy = static_cast<const T*>(grad_costs);
  T* out = static_cast<T*>(grad_logits);
  const int g = group_log2_for(d);
  const int64_t grid = row_grid(d, g);
  if (((uintptr_t)logits & 15) == ((uintptr_t)grad_logits & 15))
    return launch_kernel(rnnt_grad_kernel<T, vec_width<T>(), FUSED>, grid, kRowThreads, 0, stream, d, x, targets,
                         logit_lengths, target_lengths, denom, alpha, beta, dy, grad_costs_stride, out, g);
  return launch_kernel(rnnt_grad_kernel<T, 1, FUSED>, grid, kRowThreads, 0, stream, d, x, targets, logit_lengths,
                       target_lengths, denom, alpha, beta, dy, grad_costs_stride, out, g);
}

}  // namespace

size_t rnnt_loss_workspace_bytes_impl(const b200a_rnnt_loss_desc* d) {
  if (validate_rnnt(d) != B200A_OK) return 0;
  return sizeof(float2) * (size_t)d->batch * d->max_t * d->max_u;
}

int rnnt_loss_check_impl(int32_t batch, int32_t classes, const int32_t* targets, int64_t target_cols,
                         const int32_t* logit_lengths, const int32_t* target_lengths, int32_t* out,
                         cudaStream_t stream) {
  if (batch < 0 || target_cols < 0 || out == nullptr) return B200A_EINVAL;
  if (batch > 0 && (logit_lengths == nullptr || target_lengths == nullptr)) return B200A_EINVAL;
  if (batch > 0 && target_cols > 0 && targets == nullptr) return B200A_EINVAL;
  rnnt_check_kernel<<<1, kCheckThreads, 0, stream>>>(batch, classes, targets, target_cols, logit_lengths,
                                                     target_lengths, out);
  return launch_status();
}

int rnnt_loss_forward_impl(const b200a_rnnt_loss_desc* d, const void* logits, const int32_t* targets,
                           const int32_t* logit_lengths, const int32_t* target_lengths, void* costs, float* denom,
                           float* alpha, float* beta, void* ws, size_t ws_bytes, cudaStream_t stream) {
  const int rc = validate_rnnt(d);
  if (rc != B200A_OK) return rc;
  if (logits == nullptr || logit_lengths == nullptr || target_lengths == nullptr || costs == nullptr || ws == nullptr)
    return B200A_EINVAL;
  if ((alpha == nullptr) != (beta == nullptr) || (alpha != nullptr && d->fused && denom == nullptr))
    return B200A_EINVAL;
  if (d->max_u > 1 && targets == nullptr) return B200A_EINVAL;
  if (ws_bytes < rnnt_loss_workspace_bytes_impl(d)) return B200A_EWORKSPACE;
  float2* lp = static_cast<float2*>(ws);
  if (d->dtype == B200A_DTYPE_F16)
    return forward_typed<__half>(*d, logits, targets, logit_lengths, target_lengths, costs, denom, alpha, beta, lp,
                                 stream);
  return forward_typed<float>(*d, logits, targets, logit_lengths, target_lengths, costs, denom, alpha, beta, lp, stream);
}

int rnnt_loss_backward_impl(const b200a_rnnt_loss_desc* d, const void* logits, const int32_t* targets,
                            const int32_t* logit_lengths, const int32_t* target_lengths, const float* denom,
                            const float* alpha, const float* beta, const void* grad_costs, int64_t grad_costs_stride,
                            void* grad_logits, cudaStream_t stream) {
  const int rc = validate_rnnt(d);
  if (rc != B200A_OK) return rc;
  if (logits == nullptr || logit_lengths == nullptr || target_lengths == nullptr || alpha == nullptr ||
      beta == nullptr || grad_costs == nullptr || grad_logits == nullptr || grad_costs_stride < 0)
    return B200A_EINVAL;
  if ((d->fused && denom == nullptr) || (d->max_u > 1 && targets == nullptr)) return B200A_EINVAL;
  const bool half = d->dtype == B200A_DTYPE_F16;
  if (d->fused)
    return (half ? backward_typed<__half, true> : backward_typed<float, true>)(
        *d, logits, targets, logit_lengths, target_lengths, denom, alpha, beta, grad_costs, grad_costs_stride,
        grad_logits, stream);
  return (half ? backward_typed<__half, false> : backward_typed<float, false>)(
      *d, logits, targets, logit_lengths, target_lengths, denom, alpha, beta, grad_costs, grad_costs_stride,
      grad_logits, stream);
}

}  // namespace b200a
