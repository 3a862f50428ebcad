// forced_align (functional/_alignment.py, forced_align/cpu/compute.cpp): the CTC Viterbi alignment of targets
// [B][max_l] to log-probs [B][max_t][C] (float32, float16 or float64), bit-identical to the reference CPU per sequence.
//
//   check  one CTA: max / min of both length vectors, the out-of-range / negative / blank flags over each sequence's
//          first L_b targets, the first sequence with T_b < L_b + R_b; R_b goes to the workspace for the walk.
//   walk   one CTA per sequence in one launch, nothing shared between CTAs.  Thread k owns the K contiguous states
//          [kK, kK + K) of the S = 2L + 1 lattice in registers; alpha(t - 1) at the state left of its run comes
//          from lane - 1 by shuffle, or, for lane 0, from a double-buffered per-warp boundary in shared memory: one CTA
//          barrier per frame.  The band [start, end) follows the reference's advance rules; the alphas are in the
//          input dtype with every add rounded to it; the comparisons are the reference's.  The emissions of the next D
//          frames are loaded into registers D frames ahead.  Each frame's 2-bit backpointers (0, 1, 2; 3 for the
//          reference's -1 outside the band) go to the workspace as a state-major bit stream, one coalesced row per
//          frame.  After the walk one warp backtracks 32 frames per memory round-trip (the state falls by at most 2
//          per frame, so the pointers it can need lie in an 80-state window) and writes paths and scores.
#include <cuda_fp16.h>

#include <climits>

#include "common.cuh"

namespace b200a {
namespace {

constexpr int kCheckThreads = 1024;
constexpr int kWalkMaxThreads = 512;
constexpr int kBoundaryWarps = kWalkMaxThreads / 32;
constexpr unsigned kFull = 0xffffffffu;

template <typename T>
struct Acc {
  using type = float;  // float16 alphas are held as float values rounded to half after every add
};
template <>
struct Acc<double> {
  using type = double;
};

__device__ __forceinline__ float to_acc(float x) { return x; }
__device__ __forceinline__ float to_acc(__half x) { return __half2float(x); }
__device__ __forceinline__ double to_acc(double x) { return x; }

// The reference's `result + logProbs[t][label]` in the input dtype (c10::Half adds in float and rounds to half, which
// by the 2p + 2 rule equals a correctly rounded half add).
template <typename T>
__device__ __forceinline__ typename Acc<T>::type add_rn(typename Acc<T>::type x, typename Acc<T>::type y);
template <>
__device__ __forceinline__ float add_rn<float>(float x, float y) { return __fadd_rn(x, y); }
template <>
__device__ __forceinline__ float add_rn<__half>(float x, float y) {
  return __half2float(__float2half_rn(__fadd_rn(x, y)));
}
template <>
__device__ __forceinline__ double add_rn<double>(double x, double y) { return __dadd_rn(x, y); }

template <typename T>
__device__ __forceinline__ T zero_of() { return T(0); }
template <>
__device__ __forceinline__ __half zero_of<__half>() { return __float2half_rn(0.f); }

__device__ __forceinline__ int64_t load_index(const void* p, int64_t i, int is64) {
  return is64 ? static_cast<const int64_t*>(p)[i] : (int64_t) static_cast<const int32_t*>(p)[i];
}
__device__ __forceinline__ void store_index(void* p, int64_t i, int v, int is64) {
  if (is64)
    static_cast<int64_t*>(p)[i] = v;
  else
    static_cast<int32_t*>(p)[i] = v;
}

// out: {max T, min T, max L, min L, out-of-range, negative, blank, first failing b or -1, its T, L, R}
__global__ void __launch_bounds__(kCheckThreads) fa_check_kernel(b200a_forced_align_desc d, const void* targets,
                                                                 const void* in_len, const void* tg_len,
                                                                 long long* out, int32_t* repeats) {
  __shared__ long long s[8];
  if (threadIdx.x == 0) {
    s[0] = LLONG_MIN;
    s[1] = LLONG_MAX;
    s[2] = LLONG_MIN;
    s[3] = LLONG_MAX;
    s[4] = s[5] = s[6] = 0;
    s[7] = LLONG_MAX;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int b = threadIdx.x >> 5; b < d.batch; b += kCheckThreads / 32) {
    const long long T_b = load_index(in_len, b, d.length_dtype), L_b = load_index(tg_len, b, d.length_dtype);
    const int n = (int)(L_b < 0 ? 0 : L_b > d.max_l ? d.max_l : L_b);
    const int64_t row = (int64_t)b * d.max_l;
    int rep = 0, range = 0, neg = 0, blank = 0;
    for (int j = lane; j < n; j += 32) {
      const int64_t v = load_index(targets, row + j, d.target_dtype);
      range |= v >= d.classes;
      neg |= v < 0;
      blank |= v == d.blank;
      if (j >= 1) rep += v == load_index(targets, row + j - 1, d.target_dtype);
    }
    for (int o = 16; o > 0; o >>= 1) rep += __shfl_xor_sync(kFull, rep, o);
    range = __any_sync(kFull, range);
    neg = __any_sync(kFull, neg);
    blank = __any_sync(kFull, blank);
    if (lane == 0) {
      repeats[b] = rep;
      atomicMax(&s[0], T_b);
      atomicMin(&s[1], T_b);
      atomicMax(&s[2], L_b);
      atomicMin(&s[3], L_b);
      if (range) s[4] = 1;
      if (neg) s[5] = 1;
      if (blank) s[6] = 1;
      if (T_b < L_b + rep) atomicMin(&s[7], (long long)b);
    }
  }
  __syncthreads();
  if (threadIdx.x < 7) out[threadIdx.x] = s[threadIdx.x];
  if (threadIdx.x == 0) {
    const long long b = s[7];
    const bool any = b != LLONG_MAX;
    out[7] = any ? b : -1;
    out[8] = any ? load_index(in_len, b, d.length_dtype) : 0;
    out[9] = any ? load_index(tg_len, b, d.length_dtype) : 0;
    out[10] = any ? repeats[b] : 0;
  }
}

template <typename T>
struct WalkArgs {
  b200a_forced_align_desc d;
  const T* lp;
  const void* targets;
  const void* in_len;
  const void* tg_len;
  const int32_t* repeats;
  uint32_t* bp;  // [B][max_t][wpf] words; written and read back by the same CTA, so never loaded through the nc path
  int wpf;
  void* paths;
  T* scores;
};

// Shared memory: the lane-0 boundary [2][warps] and the final pair (alphas), targets[max_l + 1] (blank past L),
// differs-from-previous[max_l + 2] bytes.
template <typename A>
size_t walk_smem(int max_l) {
  return (2 * kBoundaryWarps + 2) * sizeof(A) + 4 * ((size_t)max_l + 1) + (size_t)max_l + 2;
}

template <typename T, int K>
__global__ void __launch_bounds__(kWalkMaxThreads) fa_walk_kernel(WalkArgs<T> p) {
  using A = typename Acc<T>::type;
  // frames of emissions loaded ahead; fp64 with K = 32 has no registers to spare and loads each state's at its use
  constexpr int D = K * sizeof(A) > 128 ? 0 : 2;
  constexpr int DS = D > 0 ? D : 1;
  constexpr int E = K / 2 + 1;                     // emissions per frame and thread: the blank and K / 2 labels
  extern __shared__ __align__(16) unsigned char smem[];
  const b200a_forced_align_desc& d = p.d;
  A* bnd = reinterpret_cast<A*>(smem);
  A* fin = bnd + 2 * kBoundaryWarps;
  int* tgs = reinterpret_cast<int*>(fin + 2);
  unsigned char* nd = reinterpret_cast<unsigned char*>(tgs + d.max_l + 1);

  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int T_b = (int)load_index(p.in_len, b, d.length_dtype);
  const int L = (int)load_index(p.tg_len, b, d.length_dtype);
  const int S = 2 * L + 1, C = d.classes, blank = d.blank;
  const int64_t row0 = (int64_t)b * d.max_t;
  const T* lp = p.lp + row0 * C;
  const A ninf = -INFINITY;

  for (int t = T_b + tid; t < d.max_t; t += blockDim.x) {
    store_index(p.paths, row0 + t, blank, d.target_dtype);
    p.scores[row0 + t] = zero_of<T>();
  }
  if (L == 0) {
    for (int t = tid; t < T_b; t += blockDim.x) {
      store_index(p.paths, row0 + t, blank, d.target_dtype);
      p.scores[row0 + t] = lp[(int64_t)t * C + blank];
    }
    return;
  }
  const int64_t trow = (int64_t)b * d.max_l;
  for (int j = tid; j <= L; j += blockDim.x) {
    tgs[j] = j < L ? (int)load_index(p.targets, trow + j, d.target_dtype) : blank;
    nd[j] = j >= 1 && j < L &&
            load_index(p.targets, trow + j, d.target_dtype) != load_index(p.targets, trow + j - 1, d.target_dtype);
  }
  __syncthreads();

  const int LR = L + p.repeats[b];
  int start = T_b - LR > 0 ? 0 : 1;
  int end = 2;  // S >= 3
  const int i0 = tid * K, j0 = i0 / 2;
  uint32_t skipm = 0;  // bit m: the odd state i0 + 2m + 1 may skip from i0 + 2m - 1
#pragma unroll
  for (int m = 0; m < K / 2; ++m)
    if (j0 + m < L && nd[j0 + m]) skipm |= 1u << m;
  auto fetch = [&](T(&dst)[E], int t) {
    const T* r = lp + (int64_t)t * C;
    dst[0] = r[blank];
#pragma unroll
    for (int m = 1; m < E; ++m) dst[m] = r[tgs[min(j0 + m - 1, L)]];
  };

  A a[K];
  {
    T e0[E];
    fetch(e0, 0);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int i = i0 + k;
      a[k] = i >= start && i < end ? to_acc((k & 1) ? e0[1 + k / 2] : e0[0]) : ninf;
    }
  }
  T e[DS][E];
#pragma unroll
  for (int dd = 0; dd < D; ++dd)
    if (1 + dd < T_b) fetch(e[dd], 1 + dd);
  if (lane == 31) {
    bnd[warp] = a[K - 1];
  }
  __syncthreads();

  uint32_t* bp = p.bp + row0 * p.wpf;
  for (int t = 1; t < T_b; t += DS) {
#pragma unroll
    for (int dd = 0; dd < DS; ++dd) {
      const int tt = t + dd;
      if (tt >= T_b) break;
      const T* lpt = lp + (int64_t)tt * C;  // D == 0: each state's emission is loaded where it is used
      if (T_b - tt <= LR) {
        if ((start & 1) && nd[start / 2 + 1]) ++start;
        ++start;
      }
      if (tt <= LR) {
        if (!(end & 1) && end < 2 * L && nd[end / 2]) ++end;
        ++end;
      }
      // alpha(tt - 1) at i0 - 1, the only state left of the run any state reads: the skip of the odd state i0 + 1
      // comes from i0 - 1, and the even state i0 never skips
      A pm1 = __shfl_up_sync(kFull, a[K - 1], 1);
      if (lane == 0) pm1 = warp > 0 ? bnd[((tt - 1) & 1) * kBoundaryWarps + warp - 1] : ninf;
      uint32_t bits = 0;  // 2 bits per state; with K = 32 each 16-state half is stored as soon as it is done
      uint32_t* row = bp + (int64_t)tt * p.wpf;
#pragma unroll
      for (int k = K - 1; k >= 0; --k) {  // descending: a[k - 1], a[k - 2] still hold frame tt - 1
        const int i = i0 + k;
        const A x0 = a[k];
        const A x1 = k >= 1 ? a[k - 1] : pm1;
        const A x2 = (k & 1) && ((skipm >> (k / 2)) & 1u) ? (k >= 2 ? a[k - 2] : pm1) : ninf;
        A r;
        unsigned c;
        if (x2 > x1 && x2 > x0) {
          r = x2;
          c = 2;
        } else if (x1 > x0 && x1 > x2) {
          r = x1;
          c = 1;
        } else {
          r = x0;
          c = 0;
        }
        const bool in = i >= start && i < end;
        A ev;
        if constexpr (D == 0)
          ev = to_acc(lpt[(k & 1) ? tgs[min(j0 + k / 2, L)] : blank]);
        else
          ev = to_acc((k & 1) ? e[dd][1 + k / 2] : e[dd][0]);
        a[k] = in ? add_rn<T>(r, ev) : ninf;
        bits |= (in ? c : 3u) << (2 * (k & 15));
        if (K > 16 && (k & 15) == 0) {
          row[i0 / 16 + k / 16] = bits;
          bits = 0;
        }
      }
      if (D > 0 && tt + D < T_b) fetch(e[dd], tt + D);
      if constexpr (K <= 16) {
        constexpr int G = 16 / K;  // lanes per 32-bit word
        uint32_t v = (uint32_t)bits << (2 * K * (lane % G));
#pragma unroll
        for (int o = 1; o < G; o <<= 1) v |= __shfl_xor_sync(kFull, v, o);
        if (lane % G == 0) row[i0 / 16] = v;
      }
      if (lane == 31) bnd[(tt & 1) * kBoundaryWarps + warp] = a[K - 1];
      __syncthreads();
    }
  }

#pragma unroll
  for (int k = 0; k < K; ++k) {
    if (i0 + k == S - 1) fin[0] = a[k];
    if (i0 + k == S - 2) fin[1] = a[k];
  }
  __syncthreads();
  if (warp != 0) return;

  // Backtrack: lane j holds frame t - j's pointers for the states [base, base + 80); the chain over the 32 frames is
  // resolved by shuffles.  A -1 pointer (3) raises the state by one; the state never goes above S - 1.
  int s = fin[0] > fin[1] ? S - 1 : S - 2;
  for (int t = T_b - 1; t >= 0;) {
    const int base = (s >= 64 ? s - 64 : 0) & ~15;
    const int tf = t - lane;
    uint32_t w[5];
#pragma unroll
    for (int q = 0; q < 5; ++q) {
      const int wi = base / 16 + q;
      w[q] = tf >= 1 && wi < p.wpf ? bp[(int64_t)tf * p.wpf + wi] : 0u;
    }
    const int n = t + 1 < 32 ? t + 1 : 32;
    int mine = 0, j = 0;
    for (; j < n; ++j) {
      const int rel = s - base;
      if (rel >= 80) break;  // climbed out of the window: reload from here
      if (lane == j) mine = s;
      const int q = rel >> 4;
      const uint32_t ww = q == 0 ? w[0] : q == 1 ? w[1] : q == 2 ? w[2] : q == 3 ? w[3] : w[4];
      const int c = __shfl_sync(kFull, (int)((ww >> ((rel & 15) * 2)) & 3u), j);
      s = min(c == 3 ? s + 1 : s - c, S - 1);
    }
    if (lane < j) {
      const int label = (mine & 1) ? tgs[mine >> 1] : blank;
      store_index(p.paths, row0 + tf, label, d.target_dtype);
      p.scores[row0 + tf] = lp[(int64_t)tf * C + label];
    }
    t -= j;
  }
}

// K: the states per thread, the smallest power of two >= 2 that covers S_max = 2 max_l + 1 with <= 512 threads
int states_per_thread(int max_l) {
  const int64_t S = 2 * (int64_t)max_l + 1;
  int k = 2;
  while ((S + k - 1) / k > kWalkMaxThreads) k *= 2;
  return k;
}
int walk_threads(int max_l, int k) {
  const int64_t need = (2 * (int64_t)max_l + 1 + k - 1) / k;
  return (int)((need + 31) / 32 * 32);
}
int words_per_frame(int max_l) {
  const int k = states_per_thread(max_l);
  return walk_threads(max_l, k) * k / 16;
}

// The check compares the targets with any blank (its range is reported after the targets' own checks, in the
// reference's order); the walk needs it in [0, classes).
int validate_fa(const b200a_forced_align_desc* d, bool walk = true) {
  if (d == nullptr || d->batch < 1 || d->max_t < 1 || d->max_l < 0 || d->classes < 1) return B200A_EINVAL;
  if (walk && (d->blank < 0 || d->blank >= d->classes)) return B200A_EINVAL;
  if (d->dtype != B200A_DTYPE_F32 && d->dtype != B200A_DTYPE_F16 && d->dtype != B200A_DTYPE_F64) return B200A_EINVAL;
  if ((d->target_dtype != 0 && d->target_dtype != 1) || (d->length_dtype != 0 && d->length_dtype != 1))
    return B200A_EINVAL;
  return B200A_OK;
}

size_t repeats_bytes(int batch) { return ((size_t)batch * 4 + 255) / 256 * 256; }

template <typename T, int K>
int launch_walk(const WalkArgs<T>& a, cudaStream_t stream) {
  using A = typename Acc<T>::type;
  return launch_kernel(fa_walk_kernel<T, K>, a.d.batch, walk_threads(a.d.max_l, K), walk_smem<A>(a.d.max_l), stream,
                       a);
}

template <typename T>
int run_typed(const b200a_forced_align_desc& d, const void* log_probs, const void* targets, const void* in_len,
              const void* tg_len, void* paths, void* scores, void* ws, cudaStream_t stream) {
  WalkArgs<T> a{d,
                static_cast<const T*>(log_probs),
                targets,
                in_len,
                tg_len,
                static_cast<const int32_t*>(ws),
                reinterpret_cast<uint32_t*>(static_cast<char*>(ws) + repeats_bytes(d.batch)),
                words_per_frame(d.max_l),
                paths,
                static_cast<T*>(scores)};
  switch (states_per_thread(d.max_l)) {
    case 2: return launch_walk<T, 2>(a, stream);
    case 4: return launch_walk<T, 4>(a, stream);
    case 8: return launch_walk<T, 8>(a, stream);
    case 16: return launch_walk<T, 16>(a, stream);
    default: return launch_walk<T, 32>(a, stream);
  }
}

}  // namespace

size_t forced_align_workspace_bytes_impl(const b200a_forced_align_desc* d) {
  if (validate_fa(d) != B200A_OK || d->max_l > B200A_FORCED_ALIGN_MAX_L) return 0;
  return repeats_bytes(d->batch) + 4 * (size_t)d->batch * d->max_t * words_per_frame(d->max_l);
}

int forced_align_check_impl(const b200a_forced_align_desc* d, const void* targets, const void* input_lengths,
                            const void* target_lengths, int64_t* out, void* ws, size_t ws_bytes, cudaStream_t stream) {
  const int rc = validate_fa(d, false);
  if (rc != B200A_OK) return rc;
  if (input_lengths == nullptr || target_lengths == nullptr || out == nullptr || ws == nullptr ||
      (d->max_l > 0 && targets == nullptr))
    return B200A_EINVAL;
  if (ws_bytes < (size_t)d->batch * 4) return B200A_EWORKSPACE;
  fa_check_kernel<<<1, kCheckThreads, 0, stream>>>(*d, targets, input_lengths, target_lengths,
                                                   reinterpret_cast<long long*>(out), static_cast<int32_t*>(ws));
  return launch_status();
}

int forced_align_run_impl(const b200a_forced_align_desc* d, const void* log_probs, const void* targets,
                          const void* input_lengths, const void* target_lengths, void* paths, void* scores, void* ws,
                          size_t ws_bytes, cudaStream_t stream) {
  const int rc = validate_fa(d);
  if (rc != B200A_OK) return rc;
  if (log_probs == nullptr || input_lengths == nullptr || target_lengths == nullptr || paths == nullptr ||
      scores == nullptr || ws == nullptr || (d->max_l > 0 && targets == nullptr))
    return B200A_EINVAL;
  if (d->max_l > B200A_FORCED_ALIGN_MAX_L) return B200A_EUNSUPPORTED;
  if (ws_bytes < forced_align_workspace_bytes_impl(d)) return B200A_EWORKSPACE;
  if (d->dtype == B200A_DTYPE_F16)
    return run_typed<__half>(*d, log_probs, targets, input_lengths, target_lengths, paths, scores, ws, stream);
  if (d->dtype == B200A_DTYPE_F64)
    return run_typed<double>(*d, log_probs, targets, input_lengths, target_lengths, paths, scores, ws, stream);
  return run_typed<float>(*d, log_probs, targets, input_lengths, target_lengths, paths, scores, ws, stream);
}

}  // namespace b200a
