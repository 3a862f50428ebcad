// Polyphase windowed-sinc resampler.
//
// The reference evaluates  y[r][f*new' + j] = sum_i k[j][i] * xpad[r][f*orig' + i]  as a dense
// conv1d with a (new', 1, 2*width+orig') filter and stride orig'
// (src/torchaudio/functional/functional.py:1405-1432).  Almost all of every filter row is
// (numerically) zero: row j only has a contiguous run of ~2*lowpass_width*orig'/min(orig',new')
// taps around the position of output phase j.
//
// Main kernel (resample_mma_kernel): the sum IS a banded matrix product
//     Y[f][j] = sum_i X[f][i] * K[j][i],   X[f][i] = x[f*orig' + i - width]  (a strided view of the signal)
// so a CTA stages the samples of 32 output frames in shared memory with one bulk asynchronous copy
// (double buffered: the next tile lands while this one is multiplied), and its 8 warps run
// mma.sync.m16n8k8 TF32 tiles of 16 frames x 8 phases over just the k-steps where those 8 phases have
// live taps, with error-compensated operands (X_hi*K_hi + X_lo*K_hi + X_hi*K_lo, ~2^-21 relative).
// No padded copy of the input, no (rows, new', frames) intermediate; the output is written already
// interleaved and truncated.  Each input sample is read from HBM once, each output written once.  The plan (per
// phase group its k-steps and hi/lo fragments) and the contraction are the banded product of band_mma.cuh.
//
// Fallback (resample_direct_kernel): one output per thread over the phase's live taps.  It runs when
//   - new' > 1024 (more than kRsMaxTiles groups of 8 phases), or
//   - the two staging buffers of xs_floats floats each (32 orig' + taps + 20 rounded up to a multiple of 4,
//     taps = 2 width + orig'), the barriers and the group table leave less than 1 KiB of kRsSmemBudget
//     (224 KiB) for the fragments, or
//   - `wave` is not 4-byte aligned, which no valid float pointer is.
//
// Adjoint (resample_backward_mma_kernel / resample_backward_direct_kernel): see the section before the host code.
#include <algorithm>

#include "band_mma.cuh"
#include "common.cuh"
#include "ptx.cuh"

namespace b200a {

namespace {

constexpr int kRsMaxWarps = 24;      // warps per CTA are chosen per ratio so the (half, group) items divide evenly
constexpr int kRsFrames = 32;        // frames per CTA tile (two 16-row MMA tiles)
constexpr int kRsMaxTiles = 128;     // groups of 8 phases  (new' <= 1024)
constexpr int kRsSmemBudget = 224 * 1024;

struct RsHeader {
  uint32_t magic;
  int32_t orig_r, new_r, width, taps, max_support, n_tiles, total_steps;
  int32_t reserved[8];
};
static_assert(sizeof(RsHeader) == 64, "header is 64 bytes");

struct RsLayout {
  size_t header, support, tiles, frags, total;
};

inline int rs_tiles(int new_r) { return (new_r + 7) / 8; }

// Warps per CTA of the mma kernels for `items` equal warp items per tile: the count in [8, kRsMaxWarps] that leaves the
// fewest warps idle in the last round (ties go to more warps).
inline int rs_warps(int items) {
  int warps = 8;
  double best_idle = 2.0;
  for (int w = 8; w <= kRsMaxWarps; ++w) {
    const int rounds = (items + w - 1) / w;
    const double idle = 1.0 - (double)items / (double)(rounds * w);
    if (idle <= best_idle + 1e-9) { best_idle = idle; warps = w; }
  }
  return warps;
}

// Shared memory granted to an mma kernel's fragment copy: what smem_fixed leaves of the budget, in whole 512-byte
// k-steps.  The kernel stages the fragments when the plan's step count fits, otherwise it reads them through L1.
inline int rs_frag_smem_bytes(size_t smem_fixed) {
  return (int)(((size_t)kRsSmemBudget - smem_fixed) & ~(size_t)511);
}

inline RsLayout rs_layout(int new_r, int taps) {
  RsLayout l{};
  size_t off = 0;
  l.header = off;
  off = align_up(off + sizeof(RsHeader), 256);
  l.support = off;
  off = align_up(off + sizeof(int2) * (size_t)new_r, 256);
  l.tiles = off;
  off = align_up(off + sizeof(BandTile) * (size_t)rs_tiles(new_r), 256);
  l.frags = off;  // worst case: every group spans every tap
  const size_t nt = rs_tiles(new_r) <= kRsMaxTiles ? rs_tiles(new_r) : 0;
  off = align_up(off + sizeof(float4) * 32 * nt * ((size_t)taps / 8 + 2), 256);
  l.total = off;
  return l;
}

// The tables of a resampler workspace (RsLayout).
template <typename W>
struct RsWs {
  WsPtr<W, RsHeader> header;
  WsPtr<W, int2> support;
  WsPtr<W, BandTile> tiles;
  WsPtr<W, float4> frags;
};

template <typename W>
RsWs<W> rs_ws(int new_r, int taps, W* ws) {
  const RsLayout l = rs_layout(new_r, taps);
  return {ws_at<RsHeader>(ws, l.header), ws_at<int2>(ws, l.support), ws_at<BandTile>(ws, l.tiles),
          ws_at<float4>(ws, l.frags)};
}

// One warp per phase: [first, last] index of taps with |k| > 1e-12 * max|k| of that row.
__global__ void resample_support_kernel(const float* __restrict__ kernel, int new_r, int taps, int orig_r,
                                        int width, RsHeader* hdr, int2* support) {
  const int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    hdr->magic = kWsMagic;
    hdr->orig_r = orig_r;
    hdr->new_r = new_r;
    hdr->width = width;
    hdr->taps = taps;
  }
  if (j >= new_r) return;
  const float* row = kernel + (size_t)j * taps;
  float mx = 0.f;
  for (int i = lane; i < taps; i += 32) mx = fmaxf(mx, fabsf(row[i]));
  mx = warp_max(mx);
  const float thr = mx * 1e-12f;
  int lo = taps, hi = -1;
  for (int i = lane; i < taps; i += 32) {
    if (fabsf(row[i]) > thr) {
      lo = min(lo, i);
      hi = max(hi, i);
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if (lane == 0) {
    if (hi < 0) { lo = 0; hi = -1; }
    support[j] = make_int2(lo, hi - lo + 1);
    atomicMax(&hdr->max_support, hi - lo + 1);
  }
}

// The banded-product plan of a row-major matrix M[rows][k] whose row i is live on k in [range[i].x, range[i].x +
// range[i].y): per group of 8 rows the k-steps covering the union of their ranges, and M split into TF32 hi/lo
// B fragments (B[k][n] = M[n][k]).  The forward plans K[phases][taps] over the supports, the adjoint kt[taps][phases]
// over the tap hulls.
__global__ void resample_plan_kernel(const float* __restrict__ m, const int2* __restrict__ range, int rows, int k,
                                     int n_groups, RsHeader* hdr, BandTile* tiles, float4* frags) {
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int g = 0; g < n_groups; ++g) {
      int lo = k, hi = 0;
      for (int i = 8 * g; i < min(8 * g + 8, rows); ++i) {
        const int2 r = range[i];
        if (r.y > 0) { lo = min(lo, r.x); hi = max(hi, r.x + r.y); }
      }
      const BandTile t = band_tile(g, lo, hi, acc);
      tiles[g] = t;
      acc += t.nsteps;
    }
    hdr->n_tiles = n_groups;
    hdr->total_steps = acc;
  }
  __syncthreads();
  for (int g = 0; g < n_groups; ++g)
    write_band_frags(tiles[g], frags,
                     [&](int n, int kk) { return (n < rows && kk < k) ? m[(size_t)n * k + kk] : 0.f; });
}

struct RsParams {
  const float* wave;
  int64_t rows, length, row_stride;
  float* out;
  int64_t out_row_stride, out_len;
  const RsHeader* hdr;
  const BandTile* tiles;
  const float4* frags;
  int orig_r, new_r, width, taps, n_tiles;
  int64_t frames;           // output frames per row = ceil(out_len / new_r)
  int64_t blocks_per_row;   // ceil(frames / kRsFrames)
  int64_t total_blocks;
  int xs_floats;            // floats per staging buffer
  int frag_smem_bytes;      // shared memory granted to the fragment copy (0: read them from global)
  int row_spread;           // 1, 2 or 4: frame distance of the 8 rows one A-fragment load touches
};

// Fill one staging buffer with the samples frames [f0, f0 + 32) of `row` need:
// xs[q] = x[T0 + q - shift] (zero outside the signal), T0 = f0*orig' - width, shift = (-T0) mod 4 so that
// 16-byte aligned global addresses land on 16-byte aligned shared addresses for the bulk copy.
__device__ __forceinline__ int rs_fill(const RsParams& p, int64_t row, int64_t f0, float* xs, uint64_t* bar, int tid,
                                       int nthreads) {
  const int64_t T0 = f0 * p.orig_r - p.width;
  const float* x = p.wave + row * p.row_stride;
  // word address of sample g is a0 + g (mod 4): the bulk copy needs 16-byte aligned global AND shared
  // addresses, so the tile is shifted by 0..3 floats until the two alignments agree
  const int a0 = (int)((reinterpret_cast<uintptr_t>(x) >> 2) & 3);
  const int shift = (int)((((a0 + T0) % 4) + 4) % 4);  // xs index of sample g: q = g - T0 + shift == a0 + g (mod 4)
  // A group's last 8-tap k-step ends at most 7 taps past its live taps, so the furthest sample a tile reads is
  // xs[shift + 31 orig' + taps + 6]; the + 16 covers that for every orig' >= 1.
  const int64_t span = (int64_t)kRsFrames * p.orig_r + p.taps + 16;
  const int64_t lo = T0 < 0 ? 0 : T0;
  int64_t hi = T0 + span;
  if (hi > p.length) hi = p.length;
  if (hi < lo) hi = lo;
  const int64_t lo_a = lo + ((4 - ((a0 + lo) & 3)) & 3);  // first sample >= lo on a 16-byte boundary
  const int64_t hi_a = hi - ((a0 + hi) & 3);               // last 16-byte boundary <= hi; bulk part [lo_a, hi_a)
  const int q_lo = (int)(lo - T0) + shift, q_hi = (int)(hi - T0) + shift;
  // zeros where the tile sticks out of the signal (only edge tiles), scalar loads for the (< 4 sample)
  // unaligned head and tail of the bulk range
  if (q_lo > 0 && T0 < 0)
    for (int q = tid; q < q_lo; q += nthreads) xs[q] = 0.f;
  if (hi < T0 + span)
    for (int q = q_hi + tid; q < p.xs_floats; q += nthreads) xs[q] = 0.f;
  if (hi_a > lo_a) {
    const int head = (int)(lo_a - lo), tail = (int)(hi - hi_a);
    if (tid < head) xs[q_lo + tid] = x[lo + tid];
    else if (tid >= 32 && tid < 32 + tail) xs[(int)(hi_a - T0) + shift + (tid - 32)] = x[hi_a + (tid - 32)];
  } else {
    for (int q = q_lo + tid; q < q_hi; q += nthreads) xs[q] = x[T0 + q - shift];
  }
  if (tid == 0) {
    if (hi_a > lo_a) {
      const uint32_t bytes = (uint32_t)(hi_a - lo_a) * 4u;
      mbar_expect_tx(bar, bytes);
      bulk_g2s(xs + (lo_a - T0) + shift, x + lo_a, bytes, bar);
    } else {
      mbar_arrive(bar);  // nothing to copy: complete the phase
    }
  }
  return shift;
}

// Frame (0..31 within the tile) of MMA row rho (0..15) of 16-frame half h, for row spread S in {1, 2, 4}:
// rows rho%8 of one load instruction are S frames apart; the remaining frames fill the gaps.
__device__ __forceinline__ int frame_of(int spread, int h, int rho) {
  const int lo = rho & 7, hi = rho >> 3;
  if (spread == 4) return 4 * lo + hi + 2 * h;
  if (spread == 2) return 16 * h + 2 * lo + hi;
  return 16 * h + rho;
}

// m16n8k8 TF32 x 3 (2^-21 relative)
__global__ void __launch_bounds__(kRsMaxWarps * 32, 1) resample_mma_kernel(const RsParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* s_x = reinterpret_cast<float*>(smem_raw);                              // [2][xs_floats]
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(s_x + 2 * (size_t)p.xs_floats);  // [2]
  BandTile* s_tiles = reinterpret_cast<BandTile*>(s_bar + 2);                   // [n_tiles]
  float4* s_frags = reinterpret_cast<float4*>(s_tiles + ((p.n_tiles + 3) & ~3));  // optional

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < p.n_tiles; i += blockDim.x) s_tiles[i] = p.tiles[i];
  const bool frags_in_smem = stage_band_frags(p.frags, p.hdr->total_steps, p.frag_smem_bytes / 512, s_frags);
  if (tid == 0) {
    mbar_init(s_bar + 0, 1);
    mbar_init(s_bar + 1, 1);
  }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();

  int shift[2] = {0, 0};
  int64_t blk = blockIdx.x;
  if (blk < p.total_blocks) {
    const int64_t row = blk / p.blocks_per_row, fb = blk - row * p.blocks_per_row;
    shift[0] = rs_fill(p, row, fb * kRsFrames, s_x, s_bar + 0, tid, blockDim.x);
  }
  __syncthreads();  // the scalar part of the first fill is visible
  const int r = lane >> 2, c = lane & 3;
  const int n_warps = blockDim.x >> 5;
  for (int it = 0; blk < p.total_blocks; blk += gridDim.x, ++it) {
    const int b = it & 1;
    const int64_t nxt = blk + gridDim.x;
    if (nxt < p.total_blocks) {  // stage the next tile into the other buffer (its readers finished last iteration)
      const int64_t nrow = nxt / p.blocks_per_row, nfb = nxt - nrow * p.blocks_per_row;
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      shift[b ^ 1] = rs_fill(p, nrow, nfb * kRsFrames, s_x + (size_t)(b ^ 1) * p.xs_floats, s_bar + (b ^ 1), tid,
                             blockDim.x);
    }
    // the bulk part of this tile has landed; its scalar part was written before the barrier that ended
    // the previous iteration (or the one after the prologue fill)
    mbar_wait(s_bar + b, (it >> 1) & 1);

    const int64_t row = blk / p.blocks_per_row, fb = blk - row * p.blocks_per_row;
    const int64_t f0 = fb * kRsFrames;
    const float* xs = s_x + (size_t)b * p.xs_floats + shift[b];
    float* orow = p.out + row * p.out_row_stride;
    for (int t = warp; t < p.n_tiles; t += n_warps) {  // one phase group, both 16-frame halves
      const BandTile rt = s_tiles[t];
      // A[f][i] = xs[f*orig' + i].  MMA row rho of 16-frame half h is frame_of(S, h, rho): the 8 rows one load
      // instruction touches are S frames apart so that their 4-word windows fall into different banks
      // (S*orig' == 4 (mod 8) words for odd orig').
      int fr[4];              // frames of rows (h=0: r, r+8), (h=1: r, r+8)
      const float* arow[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        fr[q] = frame_of(p.row_spread, q >> 1, r + 8 * (q & 1));
        arow[q] = xs + (size_t)fr[q] * p.orig_r + rt.kstart + c;
      }
      float d[2][3][4];  // both halves share each B fragment load
      band_contract<2, 2>(rt, s_frags, p.frags, frags_in_smem, lane, arow, d);
      // D rows = frames; columns 2c, 2c+1 = phases 8t + 2c (+1): out index = f*new' + phase
      const int j0 = 8 * t + 2 * c;
      const bool pair_ok = j0 + 1 < p.new_r && (p.new_r & 1) == 0 && (p.out_row_stride & 1) == 0;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int half_row = 0; half_row < 2; ++half_row) {
          const float v0 = band_sum(d[h], 2 * half_row), v1 = band_sum(d[h], 2 * half_row + 1);
          const int64_t m = (f0 + fr[2 * h + half_row]) * p.new_r + j0;
          if (pair_ok && m + 1 < p.out_len) {
            *reinterpret_cast<float2*>(orow + m) = make_float2(v0, v1);  // m even, row pitch even: 8-byte aligned
          } else {
            if (j0 < p.new_r && m < p.out_len) orow[m] = v0;
            if (j0 + 1 < p.new_r && m + 1 < p.out_len) orow[m + 1] = v1;
          }
        }
    }
    __syncthreads();  // everyone is done with buffer b before it is refilled
  }
}

// Straightforward one-output-per-thread kernel (any ratio).  Consecutive threads are consecutive
// output samples, i.e. consecutive phases of the same input neighbourhood: input loads hit L1.
__global__ void __launch_bounds__(256)
resample_direct_kernel(const float* __restrict__ wave, int64_t length, int64_t row_stride,
                       const float* __restrict__ kernel, const int2* __restrict__ support, int orig_r,
                       int new_r, int width, int taps, float* __restrict__ out, int64_t out_row_stride,
                       int64_t out_len) {
  const int64_t row = blockIdx.y;
  const float* __restrict__ x = wave + row * row_stride;
  for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < out_len; n += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = n / new_r;
    const int j = (int)(n - f * new_r);
    const int2 sp = support[j];
    const int64_t base = f * orig_r - width + sp.x;  // input index of the first live tap
    const float* __restrict__ k = kernel + (size_t)j * taps + sp.x;
    float acc = 0.f;
    for (int i = 0; i < sp.y; ++i) {
      const int64_t s = base + i;
      const float v = (s >= 0 && s < length) ? x[s] : 0.f;
      acc = fmaf(k[i], v, acc);
    }
    out[row * out_row_stride + n] = acc;
  }
}

// ==== adjoint (waveform gradient) ================================================================
// With G[f][j] = g[f*new' + j] (0 past out_len) the forward's transpose is
//     D = G * K  (frames x taps),   grad_x[s] = sum_f D[f][s + width - f*orig']  over 0 <= s + width - f*orig' < taps,
// with K masked to each phase's live taps (the support the forward uses).  Both kernels below compute every sample of
// [0, length) as a sum over its frames in ascending order; nothing depends on how rows are batched.
//
// Backward workspace: header | support[new'] | tap_range[taps] | kt[taps][new'] | cols[n_cols] | frags.
//   tap_range[i] = (first phase, count) of the hull of the phases whose live taps include tap i;
//   kt[i][j]     = K[j][i] when tap i is live for phase j, else 0 (gaps inside a hull read zeros);
//   cols / frags = the forward's banded-product plan, run on kt and tap_range: per group of 8 taps the 8-phase k-steps
//                  covering the union of its taps' hulls, and the masked taps as TF32 hi/lo B fragments (only for
//                  ratios the mma kernel takes).
constexpr int kRbMaxRows = 512;  // staged frame rows per tile (halo + owned)

// Tile geometry of resample_backward_mma_kernel: a function of the ratio alone, never of the batch.
struct RbConfig {
  bool mma;
  int halo;        // H = ceil(2 width / orig'): frames before the tile whose taps reach its samples
  int rows_tile;   // R: staged frame rows (multiple of 16), R - H of them owned
  int pitch;       // staged row pitch in floats: round8(new') + 4 (== 4 mod 8: conflict-free A-fragment loads)
  int d_pitch;     // D row pitch in floats (== 8 mod 32: conflict-free float2 fragment stores)
  int n_cols;      // groups of 8 taps
  size_t smem_fixed;
};

inline RbConfig rb_config(int orig_r, int new_r, int width) {
  RbConfig c{};
  const int taps = 2 * width + orig_r;
  c.halo = (2 * width + orig_r - 1) / orig_r;
  c.n_cols = (taps + 7) / 8;
  c.pitch = ((new_r + 7) & ~7) + 4;
  c.d_pitch = 8 * c.n_cols + ((8 - (8 * c.n_cols) % 32) + 32) % 32;
  if (rs_tiles(new_r) > kRsMaxTiles) return c;
  auto fixed = [&](int R) {
    return sizeof(float) * ((size_t)2 * R * c.pitch + (size_t)R * c.d_pitch) + sizeof(BandTile) * ((c.n_cols + 3) & ~3);
  };
  // the smallest R that keeps the recomputed halo at <= 1/16 of the rows (and R >= 32) and gives a tile at least 4096
  // owned samples (fewer per-tile barriers for short frames), or the largest that fits
  for (int R = 16; R <= kRbMaxRows; R += 16) {
    if (R <= c.halo) continue;
    if (fixed(R) + 1024 > (size_t)kRsSmemBudget) break;
    c.rows_tile = R;
    if (R >= 32 && R >= 16 * c.halo && (int64_t)(R - c.halo) * orig_r >= 4096) break;
  }
  c.mma = c.rows_tile > 0;
  c.smem_fixed = c.mma ? fixed(c.rows_tile) : 0;
  return c;
}

struct RbLayout {
  size_t header, support, tap_range, kt, cols, frags, total;
};

inline RbLayout rb_layout(int orig_r, int new_r, int width) {
  const int taps = 2 * width + orig_r;
  const RbConfig c = rb_config(orig_r, new_r, width);
  RbLayout l{};
  size_t off = 0;
  l.header = off;
  off = align_up(off + sizeof(RsHeader), 256);
  l.support = off;
  off = align_up(off + sizeof(int2) * (size_t)new_r, 256);
  l.tap_range = off;
  off = align_up(off + sizeof(int2) * (size_t)taps, 256);
  l.kt = off;
  off = align_up(off + sizeof(float) * (size_t)taps * new_r, 256);
  l.cols = off;
  l.frags = off;
  if (c.mma) {
    off = align_up(off + sizeof(BandTile) * (size_t)c.n_cols, 256);
    l.frags = off;  // worst case: every tap group spans every phase group
    off = align_up(off + sizeof(float4) * 32 * (size_t)c.n_cols * rs_tiles(new_r), 256);
  }
  l.total = off;
  return l;
}

// The tables of a resampler adjoint workspace (RbLayout).
template <typename W>
struct RbWs {
  WsPtr<W, RsHeader> header;
  WsPtr<W, int2> support, tap_range;
  WsPtr<W, float> kt;
  WsPtr<W, BandTile> cols;
  WsPtr<W, float4> frags;
};

template <typename W>
RbWs<W> rb_ws(int orig_r, int new_r, int width, W* ws) {
  const RbLayout l = rb_layout(orig_r, new_r, width);
  return {ws_at<RsHeader>(ws, l.header), ws_at<int2>(ws, l.support), ws_at<int2>(ws, l.tap_range),
          ws_at<float>(ws, l.kt),        ws_at<BandTile>(ws, l.cols), ws_at<float4>(ws, l.frags)};
}

// One thread per tap: the hull of the phases for which it is live; and kt, the masked transpose of the kernel.
__global__ void resample_adjoint_table_kernel(const float* __restrict__ kernel, const int2* __restrict__ support,
                                              int new_r, int taps, int2* tap_range, float* kt) {
  const int64_t n = (int64_t)taps * new_r;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(e / new_r), j = (int)(e - (int64_t)i * new_r);
    const int2 sp = support[j];
    kt[e] = (i >= sp.x && i < sp.x + sp.y) ? kernel[(size_t)j * taps + i] : 0.f;
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < taps; i += gridDim.x * blockDim.x) {
    int lo = new_r, hi = -1;
    for (int j = 0; j < new_r; ++j) {
      const int2 sp = support[j];
      if (i >= sp.x && i < sp.x + sp.y) {
        lo = min(lo, j);
        hi = j;
      }
    }
    tap_range[i] = hi < 0 ? make_int2(0, 0) : make_int2(lo, hi - lo + 1);
  }
}

struct RbParams {
  const float* grad;
  int64_t g_row_stride, out_len;
  float* out;
  int64_t length, out_row_stride;
  const RsHeader* hdr;
  const BandTile* cols;
  const float4* frags;
  int orig_r, new_r, width, taps, n_cols;
  int halo, rows_tile, frames_tile, pitch, d_pitch;
  int64_t blocks_per_row, total_blocks;
  int frag_smem_bytes;
};

// Stage the g rows of frames [f0 - H, f0 - H + R) into gs at pitch p.pitch with 4-byte asynchronous copies (the padded
// pitch rules out one 1-D bulk copy; these need no alignment, so every view of g takes the same path).  Zeros for
// frames before the signal, outputs past out_len and the pad columns.
__device__ __forceinline__ void rb_fill(const RbParams& p, int64_t row, int64_t f0, float* gs, int warp, int lane,
                                        int n_warps) {
  const float* g = p.grad + row * p.g_row_stride;
  const int64_t fr0 = f0 - p.halo;
  for (int rho = warp; rho < p.rows_tile; rho += n_warps) {  // one warp per staged row, lanes along its phases
    const int64_t m0 = (fr0 + rho) * p.new_r;
    const int live = fr0 + rho < 0 ? 0 : (int)max((int64_t)0, min((int64_t)p.new_r, p.out_len - m0));
    float* dst = gs + rho * p.pitch;
    for (int j = lane; j < p.pitch; j += 32) {
      if (j < live) cp_async4(dst + j, g + m0 + j);
      else dst[j] = 0.f;
    }
  }
}

// Persistent CTAs over (row, tile of F = R - H frames): D = G * K on mma.sync m16n8k8 TF32 x 3 into shared memory, then
// every owned sample sums its <= H + 1 contributions in ascending frame order.  One warp item = 16 frame rows x one
// group of 8 taps over that group's k-steps; the g tile of the next iteration lands while this one is multiplied.
__global__ void __launch_bounds__(kRsMaxWarps * 32, 1) resample_backward_mma_kernel(const RbParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int stage_floats = p.rows_tile * p.pitch;
  float* s_g = reinterpret_cast<float*>(smem_raw);                                         // [2][R][pitch]
  float* s_d = s_g + 2 * (size_t)stage_floats;                                             // [R][d_pitch]
  BandTile* s_cols = reinterpret_cast<BandTile*>(s_d + (size_t)p.rows_tile * p.d_pitch);  // [n_cols]
  float4* s_frags = reinterpret_cast<float4*>(s_cols + ((p.n_cols + 3) & ~3));           // optional

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < p.n_cols; i += blockDim.x) s_cols[i] = p.cols[i];
  const bool frags_in_smem = stage_band_frags(p.frags, p.hdr->total_steps, p.frag_smem_bytes / 512, s_frags);

  const int n_warps = blockDim.x >> 5;
  int64_t blk = blockIdx.x;
  if (blk < p.total_blocks) {
    const int64_t row = blk / p.blocks_per_row, fb = blk - row * p.blocks_per_row;
    rb_fill(p, row, fb * p.frames_tile, s_g, warp, lane, n_warps);
  }
  cp_async_wait_all();
  __syncthreads();
  const int r = lane >> 2, c = lane & 3;
  const int m_tiles = p.rows_tile >> 4;
  // overlap-add: the owned samples e = (rho - H) orig' + t of a tile, walked with a fixed per-thread stride
  const int e_step_rows = (int)(blockDim.x / p.orig_r), e_step_t = (int)(blockDim.x % p.orig_r);
  const int own = p.frames_tile * p.orig_r;
  const int d_step = p.d_pitch - p.orig_r;  // D address step from frame row rho, tap i to row rho - 1, tap i + orig'
  for (int it = 0; blk < p.total_blocks; blk += gridDim.x, ++it) {
    const int b = it & 1;
    const int64_t nxt = blk + gridDim.x;
    if (nxt < p.total_blocks) {  // the other buffer's readers finished before the barrier that ended the last iteration
      const int64_t nrow = nxt / p.blocks_per_row, nfb = nxt - nrow * p.blocks_per_row;
      rb_fill(p, nrow, nfb * p.frames_tile, s_g + (size_t)(b ^ 1) * stage_floats, warp, lane, n_warps);
    }
    const int64_t row = blk / p.blocks_per_row, fb = blk - row * p.blocks_per_row;
    const int64_t f0 = fb * p.frames_tile;
    const float* gs = s_g + (size_t)b * stage_floats;
    int mt = 0, cg = warp;  // item (mt, cg), advanced by n_warps columns at a time
    while (cg >= p.n_cols) { cg -= p.n_cols; ++mt; }
    for (; mt < m_tiles;) {
      const BandTile ct = s_cols[cg];
      const float* a0 = gs + (size_t)(16 * mt + r) * p.pitch + ct.kstart + c;  // A[f][j] = G[f][j]: rows r and r + 8
      const float* a1 = a0 + 8 * p.pitch;
      float d[1][3][4];
      band_contract<1, 2>(ct, s_frags, p.frags, frags_in_smem, lane, {a0, a1}, d);
      // D rows = frame rows 16 mt + r (+ 8); columns 2c, 2c + 1 = taps 8 cg + 2c (+ 1)
      float* drow = s_d + (size_t)(16 * mt + r) * p.d_pitch + 8 * cg + 2 * c;
      *reinterpret_cast<float2*>(drow) = make_float2(band_sum(d[0], 0), band_sum(d[0], 1));
      *reinterpret_cast<float2*>(drow + 8 * p.d_pitch) = make_float2(band_sum(d[0], 2), band_sum(d[0], 3));
      cg += n_warps;
      while (cg >= p.n_cols) { cg -= p.n_cols; ++mt; }
    }
    __syncthreads();  // the D tile is complete
    // overlap-add: owned sample e (0 <= e < F orig') is s = f0 orig' - width + e, tap t = e mod orig' of frame row
    // rho = H + e / orig'; it sums D[rho - h][t + h orig'] for h = H .. 0 (ascending frames) while t + h orig' < taps
    float* orow = p.out + row * p.out_row_stride;
    const int64_t s_own = f0 * p.orig_r - p.width;
    const int e_lo = s_own < 0 ? (int)min((int64_t)own, -s_own) : 0;
    const int e_hi = (int)min((int64_t)own, p.length - s_own);
    int e = e_lo + tid;
    int rho = p.halo + e / p.orig_r, t = e - (rho - p.halo) * p.orig_r;
    for (; e < e_hi; e += blockDim.x) {
      const float* dp = s_d + ((int64_t)rho * p.d_pitch + t + (int64_t)p.halo * (p.orig_r - p.d_pitch));
      float acc = 0.f;
      for (int h = p.halo, i = t + p.halo * p.orig_r; h >= 0; --h, i -= p.orig_r, dp += d_step)
        if (i < p.taps) acc += *dp;
      orow[s_own + e] = acc;
      rho += e_step_rows;
      t += e_step_t;
      if (t >= p.orig_r) { t -= p.orig_r; ++rho; }
    }
    cp_async_wait_all();  // the next tile has landed ...
    __syncthreads();      // ... for everyone, and the D tile and buffer b are free
  }
}

// One input sample per thread (any ratio): its frames in ascending order, over each frame the live phases of tap
// i = s + width - f orig' from the transposed table.
__global__ void __launch_bounds__(256)
resample_backward_direct_kernel(const float* __restrict__ grad, int64_t rows, int64_t g_row_stride, int64_t out_len,
                                const int2* __restrict__ tap_range, const float* __restrict__ kt, int orig_r, int new_r,
                                int width, int taps, float* __restrict__ out, int64_t length, int64_t out_row_stride) {
  for (int64_t row = blockIdx.y; row < rows; row += gridDim.y) {
    const float* __restrict__ g = grad + row * g_row_stride;
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < length; s += (int64_t)gridDim.x * blockDim.x) {
      const int64_t u = s + width;
      const int64_t f_lo = u - taps + 1 <= 0 ? 0 : (u - taps + orig_r) / orig_r;
      const int64_t f_hi = u / orig_r;
      float acc = 0.f;
      for (int64_t f = f_lo; f <= f_hi; ++f) {
        const int i = (int)(u - f * orig_r);
        const int2 tr = tap_range[i];
        const float* __restrict__ k = kt + (size_t)i * new_r;
        const int64_t base = f * new_r;
        for (int q = 0; q < tr.y; ++q) {
          const int j = tr.x + q;
          if (base + j >= out_len) break;
          acc = fmaf(k[j], g[base + j], acc);
        }
      }
      out[row * out_row_stride + s] = acc;
    }
  }
}

}  // namespace

size_t resample_workspace_bytes_impl(int new_r, int taps) { return rs_layout(new_r, taps).total; }

size_t resample_backward_workspace_bytes_impl(int orig_r, int new_r, int width) {
  return rb_layout(orig_r, new_r, width).total;
}

int resample_backward_prepare_impl(const float* kernel, int orig_r, int new_r, int width, void* ws, size_t ws_bytes,
                                   cudaStream_t stream) {
  if (kernel == nullptr || ws == nullptr || orig_r < 1 || new_r < 1 || width < 0) return B200A_EINVAL;
  const int taps = 2 * width + orig_r;
  if (ws_bytes < resample_backward_workspace_bytes_impl(orig_r, new_r, width)) return B200A_EWORKSPACE;
  const RbConfig c = rb_config(orig_r, new_r, width);
  const RbWs<void> t = rb_ws(orig_r, new_r, width, ws);
  if (cudaMemsetAsync(t.header, 0, sizeof(RsHeader), stream) != cudaSuccess) return B200A_ECUDA;
  resample_support_kernel<<<(new_r + 7) / 8, 256, 0, stream>>>(kernel, new_r, taps, orig_r, width, t.header, t.support);
  const int64_t elems = (int64_t)taps * new_r;
  const unsigned grid = (unsigned)std::min<int64_t>(std::max<int64_t>((elems + 255) / 256, (taps + 255) / 256), 4096);
  resample_adjoint_table_kernel<<<grid, 256, 0, stream>>>(kernel, t.support, new_r, taps, t.tap_range, t.kt);
  if (c.mma)
    resample_plan_kernel<<<1, 256, 0, stream>>>(t.kt, t.tap_range, taps, new_r, c.n_cols, t.header, t.cols, t.frags);
  return launch_status();
}

int resample_backward_impl(const void* ws, int orig_r, int new_r, int width, const float* grad, int64_t rows,
                           int64_t g_row_stride, int64_t out_len, float* grad_wave, int64_t length,
                           int64_t grad_row_stride, cudaStream_t stream) {
  const int taps = 2 * width + orig_r;
  const RbWs<const void> t = rb_ws(orig_r, new_r, width, ws);
  const RbConfig c = rb_config(orig_r, new_r, width);
  if (c.mma) {
    RbParams p{};
    p.grad = grad;
    p.g_row_stride = g_row_stride;
    p.out_len = out_len;
    p.out = grad_wave;
    p.length = length;
    p.out_row_stride = grad_row_stride;
    p.hdr = t.header;
    p.cols = t.cols;
    p.frags = t.frags;
    p.orig_r = orig_r;
    p.new_r = new_r;
    p.width = width;
    p.taps = taps;
    p.n_cols = c.n_cols;
    p.halo = c.halo;
    p.rows_tile = c.rows_tile;
    p.frames_tile = c.rows_tile - c.halo;
    p.pitch = c.pitch;
    p.d_pitch = c.d_pitch;
    const int64_t own_frames = (length - 1 + width) / orig_r + 1;  // frames whose first tap lands on [0, length)
    p.blocks_per_row = (own_frames + p.frames_tile - 1) / p.frames_tile;
    p.total_blocks = rows * p.blocks_per_row;
    p.frag_smem_bytes = rs_frag_smem_bytes(c.smem_fixed);
    const size_t smem = c.smem_fixed + p.frag_smem_bytes;
    const int warps = rs_warps((c.rows_tile / 16) * c.n_cols);  // items: (16-row M tile, tap group)
    return launch_kernel(resample_backward_mma_kernel, persistent_grid(p.total_blocks, 1), warps * 32, smem, stream, p);
  }
  unsigned bx = (unsigned)std::min<int64_t>((length + 255) / 256, 4096);
  dim3 grid(bx, (unsigned)std::min<int64_t>(rows, 65535));
  resample_backward_direct_kernel<<<grid, 256, 0, stream>>>(grad, rows, g_row_stride, out_len, t.tap_range, t.kt, orig_r,
                                                            new_r, width, taps, grad_wave, length, grad_row_stride);
  return launch_status();
}

int resample_prepare_impl(const float* kernel, int orig_r, int new_r, int width, void* ws, size_t ws_bytes,
                          cudaStream_t stream) {
  if (kernel == nullptr || ws == nullptr || orig_r < 1 || new_r < 1 || width < 0) return B200A_EINVAL;
  const int taps = 2 * width + orig_r;
  if (ws_bytes < resample_workspace_bytes_impl(new_r, taps)) return B200A_EWORKSPACE;
  const RsWs<void> t = rs_ws(new_r, taps, ws);
  if (cudaMemsetAsync(t.header, 0, sizeof(RsHeader), stream) != cudaSuccess) return B200A_ECUDA;
  resample_support_kernel<<<(new_r + 7) / 8, 256, 0, stream>>>(kernel, new_r, taps, orig_r, width, t.header, t.support);
  if (rs_tiles(new_r) <= kRsMaxTiles)
    resample_plan_kernel<<<1, 256, 0, stream>>>(kernel, t.support, new_r, taps, rs_tiles(new_r), t.header, t.tiles, t.frags);
  return launch_status();
}

int resample_run_impl(const void* ws, const float* kernel, int orig_r, int new_r, int width, const float* wave,
                      int64_t rows, int64_t length, int64_t row_stride, float* out, int64_t out_row_stride,
                      int64_t out_len, cudaStream_t stream) {
  if (orig_r < 1 || new_r < 1 || width < 0 || rows < 0 || length < 0 || out_len < 0) return B200A_EINVAL;
  if (rows == 0 || out_len == 0) return B200A_OK;  // empty batch: pointers may be null
  if (ws == nullptr || kernel == nullptr || wave == nullptr || out == nullptr) return B200A_EINVAL;
  const int taps = 2 * width + orig_r;
  const RsWs<const void> t = rs_ws(new_r, taps, ws);

  // ---- tensor-pipe path -------------------------------------------------------------------------
  const int n_tiles = rs_tiles(new_r);
  const int xs_floats = (kRsFrames * orig_r + taps + 16 + 4 + 3) & ~3;  // rs_fill's span + its alignment shift
  const size_t smem_fixed = sizeof(float) * 2 * (size_t)xs_floats + 16 + sizeof(BandTile) * ((n_tiles + 3) & ~3);
  const bool aligned = (reinterpret_cast<uintptr_t>(wave) & 3) == 0;  // any float pointer; rows may have any pitch
  if (n_tiles <= kRsMaxTiles && aligned && smem_fixed + 1024 <= (size_t)kRsSmemBudget) {
    RsParams p{};
    p.wave = wave;
    p.rows = rows;
    p.length = length;
    p.row_stride = row_stride;
    p.out = out;
    p.out_row_stride = out_row_stride;
    p.out_len = out_len;
    p.hdr = t.header;
    p.tiles = t.tiles;
    p.frags = t.frags;
    p.orig_r = orig_r;
    p.new_r = new_r;
    p.width = width;
    p.taps = taps;
    p.n_tiles = n_tiles;
    p.frames = (out_len + new_r - 1) / new_r;
    p.blocks_per_row = (p.frames + kRsFrames - 1) / kRsFrames;
    p.total_blocks = rows * p.blocks_per_row;
    p.xs_floats = xs_floats;
    p.frag_smem_bytes = rs_frag_smem_bytes(smem_fixed);
    const size_t smem = smem_fixed + p.frag_smem_bytes;
    // row spread: the candidate with the fewest shared-memory bank conflicts for one A-fragment load
    // (8 rows x 4 consecutive words, rows spread*orig' words apart)
    int best_spread = 1, best_conf = 1 << 30;
    for (int spread = 1; spread <= 4; spread *= 2) {
      int banks[32] = {0};
      int worst = 0;
      for (int rr = 0; rr < 8; ++rr)
        for (int cc = 0; cc < 4; ++cc) {
          const int bnk = (int)(((int64_t)rr * spread * orig_r + cc) & 31);
          if (++banks[bnk] > worst) worst = banks[bnk];
        }
      if (worst < best_conf) { best_conf = worst; best_spread = spread; }
    }
    p.row_spread = best_spread;
    const int warps = rs_warps(n_tiles);  // items: phase groups
    return launch_kernel(resample_mma_kernel, persistent_grid(p.total_blocks, 1), warps * 32, smem, stream, p);
  }

  // ---- direct path --------------------------------------------------------------------------------
  if (rows > 65535) return B200A_EUNSUPPORTED;
  unsigned bx = (unsigned)((out_len + 255) / 256);
  if (bx > 4096) bx = 4096;
  dim3 grid(bx, (unsigned)rows);
  resample_direct_kernel<<<grid, 256, 0, stream>>>(wave, length, row_stride, kernel, t.support, orig_r, new_r, width, taps,
                                                  out, out_row_stride, out_len);
  return launch_status();
}

}  // namespace b200a
