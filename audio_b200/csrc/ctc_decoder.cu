// cuda_ctc_decoder (models/decoder/_cuda_ctc_decoder.py, cuctc/): CTC prefix beam search over log_prob [B][T][V]
// (float32), blank 0, with the reference's frame skipping, candidate arithmetic, merges and log-sum-exp in its
// operation order.
//
// One CTA per sequence, persistent over its selected frames, in one launch:
//   prologue  the length check (a status word per row), then the selected frames t < T_b with
//             log_prob[b][t][0] < threshold compacted in order into the workspace.
//   step 0    the top `beam` entries of the first selected row, blank included.
//   step s    per beam: K = lse(pb, pnb), the stay entry (blank), the extension by its last token and the extensions by
//             every other token c, whose keys cur[c] + K are monotone in cur[c].  So one block-wide list of the row's
//             top (2 beam + 1) tokens, shared by every beam, holds each beam's best `beam` extensions once the tokens
//             it cannot extend by are struck out (its last token, and the tokens whose extension merges into another
//             beam).  When the best extension left out ties the worst one taken (a rounding tie of cur + K), that beam
//             takes its extensions from an exact in-order pass over the row instead.  Merges (beam A + c == beam B)
//             are found by a 64-bit rolling hash and confirmed by walking both trie chains.  The top `beam` of at most
//             beam (beam + 2) candidates, by (key desc, beam * V + token asc), is a block radix select.
//   histories a trie of (parent, token) nodes in the workspace, one node per surviving extension and step.
//   epilogue  one thread per hypothesis walks the trie into tokens [B][beam][T]; lengths and scores beside them.
// The next selected row is prefetched to L2 while the current one is processed.
#include <cfloat>
#include <climits>

#include "common.cuh"

namespace b200a {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxBeam = B200A_CTC_DECODER_MAX_BEAM;
constexpr int kMaxList = 2 * kMaxBeam + 1;
constexpr uint64_t kHash0 = 0xcbf29ce484222325ull;

// The reference's _logsumexp: max(a, b) + __logf(1 + __expf(-|a - b|)), with the max as `a > b ? a : b` and -|a - b|
// as `(a - b) > 0 ? (b - a) : (a - b)`.  __expf is FMUL by log2(e) then non-ftz MUFU.EX2; __logf is MUFU.LG2 (its
// operand is at least 1, so flushing cannot matter) times ln 2 contracted into the add of the max: written out here so
// the FFMA does not depend on the compiler's contraction choice.
__device__ __forceinline__ float lse(float a, float b) {
  const float m = a > b ? a : b;
  const float d = (a - b) > 0 ? (b - a) : (a - b);
  const float s = __fadd_rn(1.f, __expf(d));
  float l;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(s));
  return __fmaf_rn(l, 0.693147182464599609375f, m);
}

// Total order on float keys: NaN below every number, then the IEEE order (-0 below +0).
__device__ __forceinline__ uint32_t ord_of(float x) {
  if (x != x) return 1u;
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
// A candidate's sort key: the key's order above, the lower index (beam * V + token) first among equal keys.  0 marks
// an empty slot, below every real candidate.
__device__ __forceinline__ uint64_t composite(float key, uint32_t idx) {
  return ((uint64_t)ord_of(key) << 32) | (uint64_t)(0xffffffffu - idx);
}
__device__ __forceinline__ uint32_t index_of(uint64_t c) { return 0xffffffffu - (uint32_t)c; }

__device__ __forceinline__ uint64_t roll(uint64_t h, int token) {
  return (h ^ (uint64_t)(uint32_t)(token + 1)) * 0x100000001b3ull + 0x9e3779b97f4a7c15ull;
}

struct Beam {
  float pb, pnb;
  int clast, len, node, pnode;  // pnode: the parent of node (-1: the root; -2 for the empty prefix)
  uint64_t hash, phash;         // of the prefix and of the prefix without its last token
};

struct Smem {
  Beam st[2][kMaxBeam];
  float K[kMaxBeam], spb[kMaxBeam], spnb[kMaxBeam];
  int mfrom[kMaxBeam], excl_head[kMaxBeam], excl_next[kMaxBeam], exact[kMaxBeam];
  uint64_t list[kMaxList];
  float lval[kMaxList];
  uint64_t gath[kMaxList];
  float gval[kMaxList];
  uint64_t sel[kMaxBeam];
  int hist[256];
  int warp_cnt[kWarps];
  uint64_t prefix;
  int need, ngath, nexact;
};

struct DecodeArgs {
  b200a_ctc_decoder_desc d;
  const float* lp;
  const int32_t* lengths;
  int32_t* frames;  // [B][T] selected frame indices
  int2* nodes;      // [B][T * beam] (parent, token)
  int32_t* tokens;  // [B][beam][T]
  int32_t* lens;    // [B][beam]
  float* scores;    // [B][beam]
  int32_t* status;  // [B]
};

// Block-wide: the key K among n keys get(i) such that fewer than `need` keys are above K and at least `need` are at or
// above it.  Returns K; s.need is left at how many of the keys equal to K belong to the top `need`, and s.hist[digit]
// at how many keys equal K.
template <typename Key, typename Get>
__device__ Key radix_select(Smem& s, int n, int need, Get get, int* n_equal) {
  constexpr int kBits = 8 * sizeof(Key);
  Key prefix = 0, mask = 0;
  if (threadIdx.x == 0) s.need = need;
  for (int shift = kBits - 8; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += kThreads) s.hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kThreads) {
      const Key k = get(i);
      if ((k & mask) == prefix) atomicAdd(&s.hist[(int)((k >> shift) & 255)], 1);
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      const int lane = threadIdx.x;
      const int want = s.need;
      __syncwarp();  // every lane has read s.need before one of them rewrites it below
      int h[8], sum = 0;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        h[q] = s.hist[255 - 8 * lane - q];  // lane 0 holds the highest digits
        sum += h[q];
      }
      int incl = sum;
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      const int above = incl - sum;
      if (above < want && want <= incl) {
        int acc = above;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          if (acc < want && want <= acc + h[q]) {
            s.prefix = (uint64_t)(255 - 8 * lane - q);
            s.need = want - acc;
            s.warp_cnt[0] = h[q];
          }
          acc += h[q];
        }
      }
    }
    __syncthreads();
    prefix |= (Key)s.prefix << shift;
    mask |= (Key)255 << shift;
    __syncthreads();
  }
  *n_equal = s.warp_cnt[0];
  return prefix;
}

// Block-wide, in increasing i over [lo, hi): emit(k, i) for the first `need` i with pred(i), k = 0, 1, ...  Returns
// how many were emitted.
template <typename Pred, typename Emit>
__device__ int ordered_take(Smem& s, int64_t lo, int64_t hi, int need, Pred pred, Emit emit) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int taken = 0;
  for (int64_t base = lo; base < hi && taken < need; base += kThreads) {
    const int64_t i = base + threadIdx.x;
    const bool f = i < hi && pred(i);
    const unsigned m = __ballot_sync(0xffffffffu, f);
    if (lane == 0) s.warp_cnt[warp] = __popc(m);
    __syncthreads();
    int off = taken, total = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      const int c = s.warp_cnt[w];
      if (w < warp) off += c;
      total += c;
    }
    off += __popc(m & ((1u << lane) - 1u));
    if (f && off < need) emit(off, i);
    taken = min(need, taken + total);
    __syncthreads();
  }
  return taken;
}

// The row's top M tokens in [c0, V) by (value desc, token asc) into s.list / s.lval, sorted.
__device__ void row_top(Smem& s, const float* cur, int c0, int V, int M) {
  const int n = V - c0;
  int n_eq;
  const uint32_t thr = radix_select<uint32_t>(s, n, M, [&](int i) { return ord_of(cur[c0 + i]); }, &n_eq);
  const int need_eq = s.need;
  if (threadIdx.x == 0) s.ngath = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const float v = cur[c0 + i];
    const uint32_t o = ord_of(v);
    if (o > thr || (o == thr && n_eq == need_eq)) {
      const int k = atomicAdd(&s.ngath, 1);
      s.gath[k] = composite(v, (uint32_t)(c0 + i));
      s.gval[k] = v;
    }
  }
  __syncthreads();
  if (n_eq != need_eq) {  // more tokens share the boundary value than fit: the lowest ones, in order
    const int base = s.ngath;
    ordered_take(
        s, 0, n, need_eq, [&](int64_t i) { return ord_of(cur[c0 + i]) == thr; },
        [&](int k, int64_t i) {
          const float v = cur[c0 + i];
          s.gath[base + k] = composite(v, (uint32_t)(c0 + i));
          s.gval[base + k] = v;
        });
  }
  for (int i = threadIdx.x; i < M; i += kThreads) {
    const uint64_t k = s.gath[i];
    int r = 0;
    for (int j = 0; j < M; ++j) r += s.gath[j] > k;
    s.list[r] = k;
    s.lval[r] = s.gval[i];
  }
  __syncthreads();
}

__device__ __forceinline__ bool excluded(const Smem& s, const Beam* st, int a, int c) {
  if (c == st[a].clast) return true;
  for (int b = s.excl_head[a]; b >= 0; b = s.excl_next[b])
    if (st[b].clast == c) return true;
  return false;
}

// Whether the prefixes at trie nodes x and y (of equal length) are the same string.
__device__ bool same_prefix(const int2* nodes, int x, int y) {
  while (x != y) {
    if (x < 0 || y < 0) return false;
    const int2 nx = nodes[x], ny = nodes[y];
    if (nx.y != ny.y) return false;
    x = nx.x;
    y = ny.x;
  }
  return true;
}

__global__ void __launch_bounds__(kThreads) ctc_decode_kernel(DecodeArgs p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  uint64_t* cand = reinterpret_cast<uint64_t*>(smem_raw + sizeof(Smem));
  const b200a_ctc_decoder_desc& d = p.d;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int T = d.max_t, V = d.vocab, Bm = d.beam, W = Bm + 2;
  const int T_b = p.lengths[b];
  int32_t* lens = p.lens + (int64_t)b * Bm;
  float* scores = p.scores + (int64_t)b * Bm;
  if (T_b < 0 || T_b > T) {
    if (tid == 0) p.status[b] = 1;
    for (int r = tid; r < Bm; r += kThreads) {
      lens[r] = 0;
      scores[r] = 0.f;
    }
    return;
  }
  if (tid == 0) p.status[b] = 0;
  const float* lp = p.lp + (int64_t)b * T * V;
  int32_t* frames = p.frames + (int64_t)b * T;
  int2* nodes = p.nodes + (int64_t)b * T * Bm;

  const int nsel = ordered_take(
      s, 0, T_b, INT_MAX, [&](int64_t t) { return lp[t * V] < d.threshold; },
      [&](int k, int64_t t) { frames[k] = (int)t; });
  __syncthreads();
  if (nsel == 0) {
    for (int r = tid; r < Bm; r += kThreads) {
      lens[r] = 0;
      scores[r] = 0.f;
    }
    return;
  }
  auto collapse = [&](int step) { return step + 1 < nsel && frames[step + 1] - frames[step] > 1; };
  auto prefetch = [&](int step) {
    if (step >= nsel) return;
    const float* nxt = lp + (int64_t)frames[step] * V;
    for (int i = tid * 32; i < V; i += kThreads * 32) asm volatile("prefetch.global.L2 [%0];" ::"l"(nxt + i));
  };

  // step 0
  {
    const float* cur = lp + (int64_t)frames[0] * V;
    prefetch(1);
    row_top(s, cur, 0, V, Bm);
    const bool col = collapse(0);
    if (tid < Bm) {
      const int c = (int)index_of(s.list[tid]);
      const float key = s.lval[tid];
      Beam& n = s.st[0][tid];
      if (c == 0) {
        n = Beam{key, -FLT_MAX, 0, 0, -1, -2, kHash0, 0};
      } else {
        nodes[tid] = make_int2(-1, c);
        n = Beam{col ? key : -FLT_MAX, col ? -FLT_MAX : key, c, 1, tid, -1, roll(kHash0, c), kHash0};
      }
      scores[tid] = key;
    }
    __syncthreads();
  }

  const int M = min(2 * Bm + 1, V - 1);
  int cb = 0;
  for (int step = 1; step < nsel; ++step) {
    const float* cur = lp + (int64_t)frames[step] * V;
    prefetch(step + 1);
    const Beam* st = s.st[cb];
    if (tid < Bm) {
      const Beam& x = st[tid];
      const float K = lse(x.pb, x.pnb);
      s.K[tid] = K;
      s.spb[tid] = cur[0] + K;
      s.spnb[tid] = x.clast != 0 ? cur[x.clast] + x.pnb : -FLT_MAX;
      s.mfrom[tid] = -1;
      s.excl_head[tid] = -1;
      s.exact[tid] = 0;
    }
    if (M > 0) row_top(s, cur, 1, V, M);  // ends in a barrier
    else __syncthreads();

    // merges: beam A extended by B's last token is B
    for (int q = tid; q < Bm * Bm; q += kThreads) {
      const int a = q / Bm, bb = q - a * Bm;
      const Beam &A = st[a], &B = st[bb];
      if (B.len == A.len + 1 && B.phash == A.hash && same_prefix(nodes, A.node, B.pnode)) s.mfrom[bb] = a;
    }
    __syncthreads();
    if (tid < Bm && s.mfrom[tid] >= 0) {
      const int a = s.mfrom[tid];
      const Beam &A = st[a], &B = st[tid];
      const int c = B.clast;
      const float ext = c == A.clast ? cur[c] + A.pb : cur[c] + s.K[a];
      s.spb[tid] = lse(s.spb[tid], -FLT_MAX);
      s.spnb[tid] = lse(s.spnb[tid], ext);
      s.excl_next[tid] = atomicExch(&s.excl_head[a], tid);
    }
    __syncthreads();

    // candidates of beam a: [0] stay, [1] extension by its last token, [2, 2 + Bm) its best other extensions
    for (int a = warp; a < Bm; a += kWarps) {
      const Beam& A = st[a];
      uint64_t* ca = cand + (int64_t)a * W;
      const float K = s.K[a];
      if (lane == 0) {
        ca[0] = composite(lse(s.spb[a], s.spnb[a]), (uint32_t)(a * V));
        bool clx = A.clast != 0;  // false too when A + clast merges into another beam
        for (int bb = s.excl_head[a]; bb >= 0; bb = s.excl_next[bb]) clx = clx && st[bb].clast != A.clast;
        ca[1] = clx ? composite(lse(-FLT_MAX, cur[A.clast] + A.pb), (uint32_t)(a * V + A.clast)) : 0ull;
      }
      int taken = 0;
      bool has_next = false;
      float last_key = 0.f, next_key = 0.f;
      for (int base = 0; base < M && taken <= Bm; base += 32) {
        const int j = base + lane;
        const int c = j < M ? (int)index_of(s.list[j]) : 0;
        const bool ok = j < M && !excluded(s, st, a, c);
        const unsigned m = __ballot_sync(0xffffffffu, ok);
        const int pos = taken + __popc(m & ((1u << lane) - 1u));
        const float key = ok ? lse(-FLT_MAX, s.lval[j] + K) : 0.f;
        if (ok && pos < Bm) ca[2 + pos] = composite(key, (uint32_t)(a * V + c));
        const unsigned ml = __ballot_sync(0xffffffffu, ok && pos == Bm - 1);
        if (ml) last_key = __shfl_sync(0xffffffffu, key, __ffs(ml) - 1);
        const unsigned mn = __ballot_sync(0xffffffffu, ok && pos == Bm);
        if (mn) {
          next_key = __shfl_sync(0xffffffffu, key, __ffs(mn) - 1);
          has_next = true;
        }
        taken += __popc(m);
      }
      for (int k = min(taken, Bm) + lane; k < Bm; k += 32) ca[2 + k] = 0ull;
      // the best extension left out ties the worst one taken: this beam's come from an exact pass over the row
      if (lane == 0 && has_next && __float_as_uint(next_key) == __float_as_uint(last_key)) s.exact[a] = 1;
    }
    __syncthreads();
    for (int a = 0; a < Bm; ++a) {
      if (!s.exact[a]) continue;  // uniform: read after a barrier
      uint64_t* ca = cand + (int64_t)a * W;
      const float K = s.K[a];
      uint64_t worst = ~0ull;
      for (int k = 0; k < Bm; ++k) worst = min(worst, ca[2 + k]);
      const uint32_t kb = (uint32_t)(worst >> 32);
      __syncthreads();
      if (tid == 0) {  // keep the extensions above the tied key, take the tied ones in token order
        int keep = 0;
        for (int k = 0; k < Bm; ++k)
          if ((uint32_t)(ca[2 + k] >> 32) > kb) ca[2 + keep++] = ca[2 + k];
        s.nexact = keep;
      }
      __syncthreads();
      const int keep = s.nexact;
      ordered_take(
          s, 1, V, Bm - keep,
          [&](int64_t c) { return ord_of(lse(-FLT_MAX, cur[c] + K)) == kb && !excluded(s, st, a, (int)c); },
          [&](int k, int64_t c) { ca[2 + keep + k] = composite(lse(-FLT_MAX, cur[c] + K), (uint32_t)(a * V + c)); });
      __syncthreads();
    }

    // the top Bm candidates
    const int nc = Bm * W;
    int n_eq;
    const uint64_t thr = radix_select<uint64_t>(s, nc, Bm, [&](int i) { return cand[i]; }, &n_eq);
    if (tid == 0) s.ngath = 0;
    __syncthreads();
    for (int i = tid; i < nc; i += kThreads)
      if (cand[i] >= thr) s.sel[atomicAdd(&s.ngath, 1)] = cand[i];
    __syncthreads();
    const bool col = collapse(step);
    Beam* nb = s.st[cb ^ 1];
    if (tid < Bm) {
      const uint64_t k = s.sel[tid];
      int r = 0;
      for (int j = 0; j < Bm; ++j) r += s.sel[j] > k;
      const uint32_t idx = index_of(k);
      const int a = (int)(idx / (uint32_t)V), c = (int)(idx - (uint32_t)a * V);
      const Beam& A = st[a];
      Beam n;
      if (c == 0) {
        n = A;
        n.pb = s.spb[a];
        n.pnb = s.spnb[a];
      } else {
        const int id = step * Bm + r;
        nodes[id] = make_int2(A.node, c);
        n = Beam{-FLT_MAX, c == A.clast ? cur[c] + A.pb : cur[c] + s.K[a], c, A.len + 1, id, A.node,
                 roll(A.hash, c), A.hash};
      }
      const float key = lse(n.pb, n.pnb);
      if (col) {
        n.pb = key;
        n.pnb = -FLT_MAX;
      }
      nb[r] = n;
      scores[r] = key;
    }
    cb ^= 1;
    __syncthreads();
  }

  // hypotheses in the final order: lengths, scores (written with the last step) and tokens from the trie
  if (tid < Bm) {
    const Beam& x = s.st[cb][tid];
    lens[tid] = x.len;
    int32_t* out = p.tokens + ((int64_t)b * Bm + tid) * T;
    int node = x.node;
    for (int k = x.len - 1; k >= 0; --k) {
      const int2 nd = nodes[node];
      out[k] = nd.y;
      node = nd.x;
    }
  }
}

size_t frames_bytes(const b200a_ctc_decoder_desc* d) { return align_up((size_t)d->batch * d->max_t * 4, 256); }

int validate_ctc(const b200a_ctc_decoder_desc* d) {
  if (d == nullptr || d->batch < 1 || d->max_t < 0 || d->vocab < 1 || d->vocab > B200A_CTC_DECODER_MAX_VOCAB ||
      d->beam < 1 || d->beam > kMaxBeam || d->beam > d->vocab || !(d->threshold == d->threshold))
    return B200A_EINVAL;
  return B200A_OK;
}

}  // namespace

size_t ctc_decoder_workspace_bytes_impl(const b200a_ctc_decoder_desc* d) {
  if (validate_ctc(d) != B200A_OK) return 0;
  return frames_bytes(d) + align_up((size_t)d->batch * d->max_t * d->beam * sizeof(int2), 256) + 256;
}

int ctc_decoder_run_impl(const b200a_ctc_decoder_desc* d, const float* log_prob, const int32_t* lengths,
                         int32_t* tokens, int32_t* token_lengths, float* scores, int32_t* status, void* ws,
                         size_t ws_bytes, cudaStream_t stream) {
  if (validate_ctc(d) != B200A_OK) return B200A_EINVAL;
  if (lengths == nullptr || token_lengths == nullptr || scores == nullptr || status == nullptr || ws == nullptr ||
      (d->max_t > 0 && (log_prob == nullptr || tokens == nullptr)))
    return B200A_EINVAL;
  if (ws_bytes < ctc_decoder_workspace_bytes_impl(d)) return B200A_EWORKSPACE;
  char* w = static_cast<char*>(ws);
  DecodeArgs a{*d,
               log_prob,
               lengths,
               reinterpret_cast<int32_t*>(w),
               reinterpret_cast<int2*>(w + frames_bytes(d)),
               tokens,
               token_lengths,
               scores,
               status};
  const size_t smem = sizeof(Smem) + (size_t)d->beam * (d->beam + 2) * sizeof(uint64_t);
  return launch_kernel(ctc_decode_kernel, d->batch, kThreads, smem, stream, a);
}

}  // namespace b200a
