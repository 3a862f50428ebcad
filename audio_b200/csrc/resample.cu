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
// interleaved and truncated.  Each input sample is read from HBM once, each output written once.
//
// Fallback (resample_direct_kernel): one output per thread over the phase's live taps, for ratios whose
// tables or tiles do not fit (new' > 1024, orig' > ~1100) or mis-aligned inputs.
//
// SIMT variant for odd orig' (resample_simt_kernel, opt-in, e.g. 44.1 -> 16 kHz): the pruned FIR is only ~68 flop
// per output sample, so it runs as a register-tiled FP32 product: a thread owns ONE frame of each of two adjacent
// 32-frame half-chunks x a group of 8 phases, lanes are consecutive frames (stride orig' words: conflict-free for odd
// orig'), the 8 taps of a step are one 32-byte broadcast read, and the two frames are a register pair (f32x2.cuh):
//     acc[q] (frame a | frame b) += (x_a[i] | x_b[i]) * tap[q][i]
// Half-chunks stream through a 3-slot ring of bulk asynchronous copies.  Step s pairs half-chunks (s-1, s) and
// handles the phase groups of parity s & 1, so every half-chunk meets both parities (once as the newer, once as
// the older member of a pair) and a slot is free for the next copy as soon as its second step ends.
#include <cstdio>
#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "f32x2.cuh"
#include "ptx.cuh"

namespace b200a {

namespace {

constexpr int kRsMaxWarps = 24;      // warps per CTA are chosen per ratio so the (half, group) items divide evenly
constexpr int kRsFrames = 32;        // frames per CTA tile (two 16-row MMA tiles)
constexpr int kRsMaxTiles = 128;     // groups of 8 phases  (new' <= 1024)
constexpr int kRsSmemBudget = 224 * 1024;

struct RsTile {  // one group of 8 phases
  int kstart;      // first tap of its first k-step (multiple of 8)
  int nsteps;      // 8-tap k-steps covering the union of the group's live taps
  int frag_off;    // first step in the TF32 fragment array
  int frag16_off;  // first 16-tap step in the bf16 fragment array
};

struct RsHeader {
  uint32_t magic;
  int32_t orig_r, new_r, width, taps, max_support, n_tiles, total_steps;
  int32_t simt_tap_floats;  // size of the SIMT tap table (floats)
  int32_t total_steps16;    // 16-tap steps over all groups (bf16 fragments)
  int32_t r3_ok;            // 1: every group of 4 phases spans at most kR3Len taps (resample_r3_kernel applies)
  int32_t reserved[5];
};
static_assert(sizeof(RsHeader) == 64, "header is 64 bytes");

struct RsLayout {
  size_t header, support, tiles, frags, frags16, sgroups, staps, r3base, r3taps, total;
};

constexpr int kR3Len = 44;      // taps per phase quad held in registers (34 live + 3 x 2.76 drift at 441:160, padded)
constexpr int kR3Warps = 8;     // warps per CTA == phase quads per CTA (a multiple of 4: registers are granted per 4 warps)
constexpr int kR3MaxCluster = 8;

struct RsSimtGroup {  // one group of 8 phases for the SIMT kernel
  int base;  // first tap (xp-relative) any phase of the group uses
  int len;   // taps visited (multiple of 8; zero padded)
  int off;   // float offset of the group's [len][8] tap block in the tap table
  int pad;
};

inline int rs_tiles(int new_r) { return (new_r + 7) / 8; }

inline RsLayout rs_layout(int new_r, int taps) {
  RsLayout l{};
  size_t off = 0;
  l.header = off;
  off = align_up(off + sizeof(RsHeader), 256);
  l.support = off;
  off = align_up(off + sizeof(int2) * (size_t)new_r, 256);
  l.tiles = off;
  off = align_up(off + sizeof(RsTile) * (size_t)rs_tiles(new_r), 256);
  l.frags = off;  // worst case: every group spans every tap
  const size_t nt = rs_tiles(new_r) <= kRsMaxTiles ? rs_tiles(new_r) : 0;
  off = align_up(off + sizeof(float4) * 32 * nt * ((size_t)taps / 8 + 2), 256);
  l.frags16 = off;  // bf16 hi / lo fragments of the 16-tap steps (resample_mma_kernel<true>)
  off = align_up(off + sizeof(uint4) * 32 * nt * ((size_t)taps / 16 + 2), 256);
  l.sgroups = off;
  off = align_up(off + sizeof(RsSimtGroup) * (size_t)rs_tiles(new_r), 256);
  l.staps = off;  // worst case: every group spans every tap
  off = align_up(off + sizeof(float) * 8 * (size_t)rs_tiles(new_r) * ((size_t)taps + 8), 256);
  const size_t quads = ((size_t)new_r + 3) / 4;
  l.r3base = off;
  off = align_up(off + sizeof(int) * quads, 256);
  l.r3taps = off;
  off = align_up(off + sizeof(float4) * kR3Len * quads, 256);
  l.total = off;
  return l;
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

// Per group of 8 phases: the k-steps its live taps span, and the taps split into TF32 hi/lo parts in
// mma.m16n8k8 B-fragment order (B[k][n] = K[8 t + n][kstart + k]).
// (x, y) -> packed bf16 pair (x in the low half) and the packed pair of the residuals
__device__ __forceinline__ void rs_split_bf16x2(float x, float y, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(y), "f"(x));
  const float rx = x - __uint_as_float(hi << 16), ry = y - __uint_as_float(hi & 0xffff0000u);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(ry), "f"(rx));
}

__global__ void resample_plan_kernel(const float* __restrict__ kernel, const int2* __restrict__ support, int new_r,
                                     int taps, int n_tiles, RsHeader* hdr, RsTile* tiles, float4* frags, uint4* frags16) {
  if (threadIdx.x == 0) {
    int acc = 0, acc16 = 0;
    for (int t = 0; t < n_tiles; ++t) {
      int lo = taps, hi = 0;
      for (int j = 8 * t; j < min(8 * t + 8, new_r); ++j) {
        const int2 sp = support[j];
        if (sp.y > 0) { lo = min(lo, sp.x); hi = max(hi, sp.x + sp.y); }
      }
      RsTile rt{0, 0, acc, acc16};
      if (hi > lo) {
        rt.kstart = lo & ~7;
        rt.nsteps = (hi - rt.kstart + 7) / 8;
      }
      tiles[t] = rt;
      acc += rt.nsteps;
      acc16 += (rt.nsteps + 1) / 2;
    }
    hdr->n_tiles = n_tiles;
    hdr->total_steps = acc;
    hdr->total_steps16 = acc16;
  }
  __syncthreads();
  for (int t = 0; t < n_tiles; ++t) {
    const RsTile rt = tiles[t];
    for (int i = threadIdx.x; i < rt.nsteps * 32; i += blockDim.x) {
      const int s = i >> 5, lane = i & 31;
      const int j = 8 * t + (lane >> 2);
      const int k0 = rt.kstart + 8 * s + (lane & 3), k1 = k0 + 4;
      const float b0 = (j < new_r && k0 < taps) ? kernel[(size_t)j * taps + k0] : 0.f;
      const float b1 = (j < new_r && k1 < taps) ? kernel[(size_t)j * taps + k1] : 0.f;
      const float b0h = __uint_as_float(__float_as_uint(b0) & 0xffffe000u);
      const float b1h = __uint_as_float(__float_as_uint(b1) & 0xffffe000u);
      frags[(size_t)(rt.frag_off + s) * 32 + lane] = make_float4(b0h, b1h, b0 - b0h, b1 - b1h);
    }
    // 16-tap steps for mma.m16n8k16 bf16: the instruction's k index is a PERMUTATION of the taps chosen so that a
    // thread's A elements (k = 2c, 2c+1, 2c+8, 2c+9) are taps c, c+4, c+8, c+12 of the step -- the same
    // conflict-free shared-memory reads as the 8-tap TF32 steps.  B[k][n] follows the same permutation.
    const int n16 = (rt.nsteps + 1) / 2;
    for (int i = threadIdx.x; i < n16 * 32; i += blockDim.x) {
      const int s = i >> 5, lane = i & 31;
      const int j = 8 * t + (lane >> 2), c = lane & 3;
      float v[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int k = rt.kstart + 16 * s + c + 4 * q;
        v[q] = (j < new_r && k < taps && k < rt.kstart + 8 * rt.nsteps) ? kernel[(size_t)j * taps + k] : 0.f;
      }
      uint4 f;
      rs_split_bf16x2(v[0], v[1], f.x, f.z);  // b0: taps c, c + 4
      rs_split_bf16x2(v[2], v[3], f.y, f.w);  // b1: taps c + 8, c + 12
      frags16[(size_t)(rt.frag16_off + s) * 32 + lane] = f;
    }
  }
}

struct RsParams {
  const float* wave;
  int64_t rows, length, row_stride;
  float* out;
  int64_t out_row_stride, out_len;
  const RsHeader* hdr;
  const RsTile* tiles;
  const float4* frags;
  const uint4* frags16;
  int orig_r, new_r, width, taps, n_tiles;
  int64_t frames;           // output frames per row = ceil(out_len / new_r)
  int64_t blocks_per_row;   // ceil(frames / kRsFrames)
  int64_t total_blocks;
  int xs_floats;            // floats per staging buffer
  int frag_smem_bytes;      // shared memory granted to the fragment copy (0: read them from global)
  int row_spread;           // 1, 2 or 4: frame distance of the 8 rows one A-fragment load touches
  int skip_if_r3_ok;        // launched behind resample_r3_kernel: leave when the header says that kernel did the work
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
  const int64_t span = (int64_t)kRsFrames * p.orig_r + p.taps + 16;  // + the zero-tap tail of the last 16-tap step
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

__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// BF16 == false: m16n8k8 TF32 x 3 (2^-21 relative);  BF16 == true: m16n8k16 bf16 x 3 (2^-16 relative, half the
// tensor-pipe time: the TF32 variant issues three MMAs per tile)
template <bool BF16>
__global__ void __launch_bounds__(kRsMaxWarps * 32, 1) resample_mma_kernel(const RsParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* s_x = reinterpret_cast<float*>(smem_raw);                              // [2][xs_floats]
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(s_x + 2 * (size_t)p.xs_floats);  // [2]
  RsTile* s_tiles = reinterpret_cast<RsTile*>(s_bar + 2);                       // [n_tiles]
  float4* s_frags = reinterpret_cast<float4*>(s_tiles + ((p.n_tiles + 3) & ~3));  // optional

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (p.skip_if_r3_ok && p.hdr->r3_ok != 0) return;
  for (int i = tid; i < p.n_tiles; i += blockDim.x) s_tiles[i] = p.tiles[i];
  const int total_steps = BF16 ? p.hdr->total_steps16 : p.hdr->total_steps;
  const bool frags_in_smem = (size_t)total_steps * 512 <= (size_t)p.frag_smem_bytes;
  if (frags_in_smem) {
    const float4* src = BF16 ? reinterpret_cast<const float4*>(p.frags16) : p.frags;
    for (int i = tid; i < total_steps * 32; i += blockDim.x) s_frags[i] = src[i];
  }
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
      const RsTile rt = s_tiles[t];
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
      // per half: three independent accumulator chains (hi*hi, lo*hi, hi*lo), summed in a fixed order
      float d[2][3][4];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int ch = 0; ch < 3; ++ch)
#pragma unroll
          for (int q = 0; q < 4; ++q) d[h][ch][q] = 0.f;
      auto contract = [&](auto in_smem) {
        if constexpr (BF16) {
          const uint4* frg = (decltype(in_smem)::value ? reinterpret_cast<const uint4*>(s_frags) : p.frags16) +
                             (size_t)rt.frag16_off * 32 + lane;
          const int n16 = (rt.nsteps + 1) >> 1;
#pragma unroll 2
          for (int s = 0; s < n16; ++s) {
            uint4 bf;
            if constexpr (decltype(in_smem)::value) bf = frg[(size_t)s * 32];
            else bf = __ldg(frg + (size_t)s * 32);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              // k = 2c, 2c+1 <-> taps c, c+4;  k = 2c+8, 2c+9 <-> taps c+8, c+12 (see resample_plan_kernel)
              const float* lo_row = arow[2 * h] + 16 * s;
              const float* hi_row = arow[2 * h + 1] + 16 * s;
              uint32_t ah[4], al[4];
              rs_split_bf16x2(lo_row[0], lo_row[4], ah[0], al[0]);
              rs_split_bf16x2(hi_row[0], hi_row[4], ah[1], al[1]);
              rs_split_bf16x2(lo_row[8], lo_row[12], ah[2], al[2]);
              rs_split_bf16x2(hi_row[8], hi_row[12], ah[3], al[3]);
              mma_bf16_16816(d[h][0], ah, bf.x, bf.y);
              mma_bf16_16816(d[h][1], al, bf.x, bf.y);
              mma_bf16_16816(d[h][2], ah, bf.z, bf.w);
            }
          }
        } else {
        const float4* frg = (decltype(in_smem)::value ? s_frags : p.frags) + (size_t)rt.frag_off * 32 + lane;
#pragma unroll 2
        for (int s = 0; s < rt.nsteps; ++s) {
          float4 bf;
          if constexpr (decltype(in_smem)::value) bf = frg[(size_t)s * 32];
          else bf = __ldg(frg + (size_t)s * 32);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float av[4] = {arow[2 * h][8 * s], arow[2 * h + 1][8 * s], arow[2 * h][8 * s + 4],
                                 arow[2 * h + 1][8 * s + 4]};
            uint32_t hi[4], lo[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) split_tf32(av[q], hi[q], lo[q]);
            mma_tf32(d[h][0], hi, __float_as_uint(bf.x), __float_as_uint(bf.y));
            mma_tf32(d[h][1], lo, __float_as_uint(bf.x), __float_as_uint(bf.y));
            mma_tf32(d[h][2], hi, __float_as_uint(bf.z), __float_as_uint(bf.w));
          }
        }
        }
      };
      if (frags_in_smem) contract(std::true_type{});
      else contract(std::false_type{});
      // D rows = frames; columns 2c, 2c+1 = phases 8t + 2c (+1): out index = f*new' + phase
      const int j0 = 8 * t + 2 * c;
      const bool pair_ok = j0 + 1 < p.new_r && (p.new_r & 1) == 0 && (p.out_row_stride & 1) == 0;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int half_row = 0; half_row < 2; ++half_row) {
          const float v0 = d[h][0][2 * half_row] + (d[h][1][2 * half_row] + d[h][2][2 * half_row]);
          const float v1 = d[h][0][2 * half_row + 1] + (d[h][1][2 * half_row + 1] + d[h][2][2 * half_row + 1]);
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

// ---- SIMT kernel tables: per group of 8 phases the union of their live taps, zero padded to a multiple of 8,
// stored tap-major ([i][8 phases]) so one step's taps are one 32-byte broadcast read.
__global__ void resample_simt_plan_kernel(const float* __restrict__ kernel, const int2* __restrict__ support, int new_r,
                                          int taps, int n_groups, RsHeader* hdr, RsSimtGroup* groups, float* table) {
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int g = 0; g < n_groups; ++g) {
      int lo = taps, hi = 0;
      for (int j = 8 * g; j < min(8 * g + 8, new_r); ++j) {
        const int2 sp = support[j];
        if (sp.y > 0) { lo = min(lo, sp.x); hi = max(hi, sp.x + sp.y); }
      }
      RsSimtGroup sg{0, 0, acc, 0};
      if (hi > lo) {
        sg.base = lo;
        sg.len = (hi - lo + 7) & ~7;
      }
      groups[g] = sg;
      acc += sg.len * 8;
    }
    hdr->simt_tap_floats = acc;
  }
  __syncthreads();
  for (int g = 0; g < n_groups; ++g) {
    const RsSimtGroup sg = groups[g];
    for (int e = threadIdx.x; e < sg.len * 8; e += blockDim.x) {
      const int i = e >> 3, q = e & 7, j = 8 * g + q, t = sg.base + i;
      float v = 0.f;
      if (j < new_r && t < taps) {
        const int2 sp = support[j];
        if (t >= sp.x && t < sp.x + sp.y) v = kernel[(size_t)j * taps + t];
      }
      table[sg.off + e] = v;
    }
  }
}

struct RsSimtParams {
  const float* wave;
  int64_t rows, length, row_stride;
  float* out;
  int64_t out_row_stride, out_len;
  const RsHeader* hdr;
  const RsSimtGroup* groups;
  const float* table;
  int orig_r, new_r, width, n_groups;
  int tap_floats;        // shared memory granted to the tap table (floats)
  int64_t frames;        // output frames per row
  int64_t halves;        // 32-frame half-chunks per row
  int64_t total_halves;  // rows * halves
  int slot_floats;       // floats per ring slot
  int out_vec;           // 1: every frame's 8-phase run may be stored as two float4
};

constexpr int kSimtMaxWarps = 12;

// Stage the samples of half-chunk (row, hk) into a ring slot: xs[q] = xp[32 hk orig' + q - shift] with
// xp[m] = x[m - width] (zero outside the signal).  Same alignment rule as rs_fill.
__device__ __forceinline__ int simt_fill(const RsSimtParams& p, int64_t row, int64_t hk, float* xs, uint64_t* bar,
                                         int tid, int nthreads) {
  const int64_t T0 = hk * 32 * p.orig_r - p.width;
  const float* x = p.wave + row * p.row_stride;
  const int a0 = (int)((reinterpret_cast<uintptr_t>(x) >> 2) & 3);
  const int shift = (int)((((a0 + T0) % 4) + 4) % 4);
  const int64_t span = (int64_t)32 * p.orig_r + 2 * p.width;
  const int64_t lo = T0 < 0 ? 0 : T0;
  int64_t hi = T0 + span;
  if (hi > p.length) hi = p.length;
  if (hi < lo) hi = lo;
  const int64_t lo_a = lo + ((4 - ((a0 + lo) & 3)) & 3);
  const int64_t hi_a = hi - ((a0 + hi) & 3);
  const int q_lo = (int)(lo - T0) + shift, q_hi = (int)(hi - T0) + shift;
  if (q_lo > 0 && T0 < 0)
    for (int q = tid; q < q_lo; q += nthreads) xs[q] = 0.f;
  if (hi < T0 + span)
    for (int q = q_hi + tid; q < p.slot_floats; q += nthreads) xs[q] = 0.f;
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
      mbar_arrive(bar);
    }
  }
  return shift;
}
// where sample xp[32 hk orig'] of half-chunk (row, hk) sits in its slot (simt_fill's `shift`)
__device__ __forceinline__ int simt_shift(const RsSimtParams& p, int64_t row, int64_t hk) {
  const int64_t T0 = hk * 32 * p.orig_r - p.width;
  const int a0 = (int)((reinterpret_cast<uintptr_t>(p.wave + row * p.row_stride) >> 2) & 3);
  return (int)((((a0 + T0) % 4) + 4) % 4);
}

__global__ void __launch_bounds__(kSimtMaxWarps * 32, 1) resample_simt_kernel(const RsSimtParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* s_x = reinterpret_cast<float*>(smem_raw);                                   // [3][slot_floats]
  float* s_taps = s_x + 3 * (size_t)p.slot_floats;                                   // [tap_floats]
  RsSimtGroup* s_groups = reinterpret_cast<RsSimtGroup*>(s_taps + ((p.tap_floats + 3) & ~3));  // [n_groups]
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(s_groups + p.n_groups);              // [3]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n_warps = blockDim.x >> 5;
  const int tap_need = p.hdr->simt_tap_floats;
  const bool taps_in_smem = tap_need <= p.tap_floats;
  if (taps_in_smem)
    for (int i = tid; i < tap_need; i += blockDim.x) s_taps[i] = p.table[i];
  for (int i = tid; i < p.n_groups; i += blockDim.x) s_groups[i] = p.groups[i];
  if (tid < 3) mbar_init(s_bar + tid, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();

  // this CTA's contiguous run of half-chunks [h0, h1) in (row, half) order
  const int64_t h0 = p.total_halves * blockIdx.x / gridDim.x, h1 = p.total_halves * (blockIdx.x + 1) / gridDim.x;
  if (h0 >= h1) return;
  uint32_t phase_bits = 0;  // bit i: parity the next wait on slot i expects
  {
    const int64_t row = h0 / p.halves;
    simt_fill(p, row, h0 - row * p.halves, s_x + (size_t)(h0 % 3) * p.slot_floats, s_bar + (h0 % 3), tid, blockDim.x);
  }
  __syncthreads();
  const bool vec_ok = p.out_vec != 0;
  for (int64_t s = h0; s <= h1; ++s) {
    const int slot_hi = (int)(s % 3), slot_lo = (int)((s + 2) % 3), slot_nx = (int)((s + 1) % 3);
    if (s + 1 < h1) {  // the slot of half-chunk s - 2: its last readers left at the barrier that ended step s - 1
      const int64_t nrow = (s + 1) / p.halves;
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      simt_fill(p, nrow, (s + 1) - nrow * p.halves, s_x + (size_t)slot_nx * p.slot_floats, s_bar + slot_nx, tid,
                blockDim.x);
    }
    const bool has_hi = s < h1, has_lo = s > h0;
    if (has_hi) {
      mbar_wait(s_bar + slot_hi, (phase_bits >> slot_hi) & 1u);
      phase_bits ^= 1u << slot_hi;
    }
    // frames of this thread: lane of the older half-chunk (s - 1) and lane of the newer one (s)
    const int64_t hb = has_hi ? s : s - 1, ha = has_lo ? s - 1 : s;  // an absent side mirrors the present one
    const int64_t row_a = ha / p.halves, row_b = hb / p.halves;
    const int64_t fa = (ha - row_a * p.halves) * 32 + lane, fb = (hb - row_b * p.halves) * 32 + lane;
    const float* xa = s_x + (size_t)(has_lo ? slot_lo : slot_hi) * p.slot_floats +
                      simt_shift(p, row_a, ha - row_a * p.halves) + lane * p.orig_r;
    const float* xb = s_x + (size_t)(has_hi ? slot_hi : slot_lo) * p.slot_floats +
                      simt_shift(p, row_b, hb - row_b * p.halves) + lane * p.orig_r;
    const bool st_a = has_lo && fa < p.frames, st_b = has_hi && fb < p.frames;
    float* oa = p.out + row_a * p.out_row_stride + fa * p.new_r;
    float* ob = p.out + row_b * p.out_row_stride + fb * p.new_r;
    const int64_t na = fa * p.new_r, nb = fb * p.new_r;  // output index of phase 0 of the two frames
    for (int g = 2 * warp + (int)(s & 1); g < p.n_groups; g += 2 * n_warps) {
      const RsSimtGroup sg = s_groups[g];
      const float* ta = xa + sg.base;
      const float* tb = xb + sg.base;
      uint64_t acc[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) acc[q] = 0ull;
      auto fir = [&](auto in_smem) {
        const float4* tp = reinterpret_cast<const float4*>((decltype(in_smem)::value ? s_taps : p.table) + sg.off);
        // software pipelined over blocks of 4 taps: the loads of block k + 1 are in flight while block k is multiplied
        float4 tq[2][8];
        float va[2][4], vb[2][4];
        auto load = [&](auto bi, int i4) {
          constexpr int B = decltype(bi)::value;
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            va[B][u] = ta[i4 + u];
            vb[B][u] = tb[i4 + u];
            if constexpr (decltype(in_smem)::value) {
              tq[B][2 * u] = tp[2 * (i4 + u)];
              tq[B][2 * u + 1] = tp[2 * (i4 + u) + 1];
            } else {
              tq[B][2 * u] = __ldg(tp + 2 * (i4 + u));
              tq[B][2 * u + 1] = __ldg(tp + 2 * (i4 + u) + 1);
            }
          }
        };
        auto mac = [&](auto bi) {
          constexpr int B = decltype(bi)::value;
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const uint64_t xx = pk2(va[B][u], vb[B][u]);
            const float4 t0 = tq[B][2 * u], t1 = tq[B][2 * u + 1];
            acc[0] = fma2_raw(xx, pk2(t0.x, t0.x), acc[0]);
            acc[1] = fma2_raw(xx, pk2(t0.y, t0.y), acc[1]);
            acc[2] = fma2_raw(xx, pk2(t0.z, t0.z), acc[2]);
            acc[3] = fma2_raw(xx, pk2(t0.w, t0.w), acc[3]);
            acc[4] = fma2_raw(xx, pk2(t1.x, t1.x), acc[4]);
            acc[5] = fma2_raw(xx, pk2(t1.y, t1.y), acc[5]);
            acc[6] = fma2_raw(xx, pk2(t1.z, t1.z), acc[6]);
            acc[7] = fma2_raw(xx, pk2(t1.w, t1.w), acc[7]);
          }
        };
        using B0 = std::integral_constant<int, 0>;
        using B1 = std::integral_constant<int, 1>;
        if (sg.len > 0) load(B0{}, 0);
#pragma unroll 1
        for (int i8 = 0; i8 < sg.len; i8 += 8) {  // len is a multiple of 8
          load(B1{}, i8 + 4);
          mac(B0{});
          if (i8 + 8 < sg.len) load(B0{}, i8 + 8);
          mac(B1{});
        }
      };
      if (taps_in_smem) fir(std::true_type{});
      else fir(std::false_type{});
      float ya[8], yb[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float2 v = upk2(acc[q]);
        ya[q] = v.x;
        yb[q] = v.y;
      }
      const int j0 = 8 * g;
      const bool full = j0 + 8 <= p.new_r && vec_ok;
      auto store = [&](float* o, int64_t n0, const float (&y)[8]) {
        if (full && n0 + j0 + 8 <= p.out_len) {
          *reinterpret_cast<float4*>(o + j0) = make_float4(y[0], y[1], y[2], y[3]);
          *reinterpret_cast<float4*>(o + j0 + 4) = make_float4(y[4], y[5], y[6], y[7]);
        } else {
#pragma unroll
          for (int q = 0; q < 8; ++q)
            if (j0 + q < p.new_r && n0 + j0 + q < p.out_len) o[j0 + q] = y[q];
        }
      };
      if (st_a) store(oa, na, ya);
      if (st_b) store(ob, nb, yb);
    }
    __syncthreads();  // every reader of slot_lo is done: the next step's copy may overwrite it
  }
}

// ---- cluster kernel tables: per QUAD of 4 phases the first live tap and kR3Len taps x 4 phases (zero padded) -------
__global__ void resample_r3_plan_kernel(const float* __restrict__ kernel, const int2* __restrict__ support, int new_r,
                                        int taps, int n_quads, RsHeader* hdr, int* qbase, float4* qtaps) {
  __shared__ int s_ok;
  if (threadIdx.x == 0) s_ok = 1;
  __syncthreads();
  for (int q = threadIdx.x; q < n_quads; q += blockDim.x) {
    int lo = taps, hi = 0;
    for (int j = 4 * q; j < min(4 * q + 4, new_r); ++j) {
      const int2 sp = support[j];
      if (sp.y > 0) { lo = min(lo, sp.x); hi = max(hi, sp.x + sp.y); }
    }
    if (hi <= lo) lo = hi = 0;
    if (hi - lo > kR3Len) s_ok = 0;
    qbase[q] = lo;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < n_quads * kR3Len; e += blockDim.x) {
    const int q = e / kR3Len, i = e - q * kR3Len, t = qbase[q] + i;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int j = 4 * q + r;
      if (j < new_r && t < taps) {
        const int2 sp = support[j];
        if (t >= sp.x && t < sp.x + sp.y) v[r] = kernel[(size_t)j * taps + t];
      }
    }
    qtaps[e] = make_float4(v[0], v[1], v[2], v[3]);
  }
  if (threadIdx.x == 0) hdr->r3_ok = s_ok;
}

// ================================================================================================
// Cluster kernel (resample_r3_kernel): the taps never leave the register file.
//   A register-tiled FIR is bound by shared-memory wavefronts unless BOTH operands of an FMA are reused from
//   registers.  Here a warp owns ONE quad of 4 output phases for the whole kernel and keeps
//   its 4 x kR3Len taps in 176 registers; lanes are the 32 frames of a tile, so the only shared-memory traffic is one
//   conflict-free 4-byte read per tap position, feeding four FFMA (4 phases) with the sample as the broadcast operand.
//   160 phases = 40 quads need 40 such warps; at ~200 registers per thread an SM holds 8 (registers are granted per 4
//   warps: 10 x 200 does not fit), so a CLUSTER of 5 CTAs covers the phases and shares every staged tile: each CTA
//   fetches a fifth of the tile's samples with ONE bulk copy that is MULTICAST into the same offset of all the CTAs'
//   shared memory (every HBM byte is read once), through a 3-slot ring
//   with cluster-scope full / empty mbarriers.
// ================================================================================================
struct R3Params {
  const float* wave;
  int64_t rows, length, row_stride;
  float* out;
  int64_t out_row_stride, out_len;
  const RsHeader* hdr;
  const int* qbase;
  const float4* qtaps;
  int orig_r, new_r, width, n_quads, csize;
  int64_t frames, tiles_per_row, total_tiles;
  int slot_floats, out_vec;
};

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t rank) {
  uint32_t raddr;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(smem_u32(bar)), "r"(rank));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(raddr) : "memory");
}
// bulk copy global -> the same shared-memory offset of every CTA in `mask`, completing bytes on each one's mbarrier
__device__ __forceinline__ void bulk_g2s_multicast(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "h"(mask)
      : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  for (int spin = 0; spin < (1 << 22); ++spin) {
    uint32_t ok;
    asm volatile(
        "{\n.reg .pred p;\n"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2, %3;\n"
        "selp.u32 %0, 1, 0, p;\n}"
        : "=r"(ok)
        : "r"(addr), "r"(parity), "r"(2000u)
        : "memory");
    if (ok) return;
  }
  __trap();
}

// Stage tile (row, f0) into ring slot `xs` of EVERY CTA of the cluster: local zero fill / unaligned head and tail by all
// threads of each CTA, and this CTA's share of the 16-byte aligned body as one multicast bulk copy.  Returns `shift`.
__device__ __forceinline__ void r3_fill(const R3Params& p, int64_t row, int64_t f0, float* xs, uint64_t* full, uint32_t crank,
                                        int tid, int nthreads) {
  const int64_t T0 = f0 * p.orig_r - p.width;
  const float* x = p.wave + row * p.row_stride;
  const int a0 = (int)((reinterpret_cast<uintptr_t>(x) >> 2) & 3);
  const int shift = (int)((((a0 + T0) % 4) + 4) % 4);
  const int64_t span = (int64_t)32 * p.orig_r + 2 * p.width + 16;  // + the zero-tap tail of a padded quad
  const int64_t lo = T0 < 0 ? 0 : T0;
  int64_t hi = T0 + span;
  if (hi > p.length) hi = p.length;
  if (hi < lo) hi = lo;
  const int64_t lo_a = lo + ((4 - ((a0 + lo) & 3)) & 3);
  const int64_t hi_a = hi - ((a0 + hi) & 3);
  const int q_lo = (int)(lo - T0) + shift, q_hi = (int)(hi - T0) + shift;
  if (q_lo > 0 && T0 < 0)
    for (int q = tid; q < q_lo; q += nthreads) xs[q] = 0.f;
  if (hi < T0 + span)
    for (int q = q_hi + tid; q < p.slot_floats; q += nthreads) xs[q] = 0.f;
  if (hi_a > lo_a) {
    const int head = (int)(lo_a - lo), tail = (int)(hi - hi_a);
    if (tid < head) xs[q_lo + tid] = x[lo + tid];
    else if (tid >= 32 && tid < 32 + tail) xs[(int)(hi_a - T0) + shift + (tid - 32)] = x[hi_a + (tid - 32)];
  } else {
    for (int q = q_lo + tid; q < q_hi; q += nthreads) xs[q] = x[T0 + q - shift];
  }
  if (tid == 0) {
    if (hi_a > lo_a) {
      const int64_t n_al = hi_a - lo_a;                                   // multiple of 4 floats
      const int64_t chunk = ((n_al / 4 + p.csize - 1) / p.csize) * 4;     // floats per CTA, multiple of 4
      mbar_expect_tx(full, (uint32_t)n_al * 4u);                          // the whole body lands in every CTA
      const int64_t c0 = lo_a + (int64_t)crank * chunk;
      int64_t c1 = c0 + chunk;
      if (c1 > hi_a) c1 = hi_a;
      if (c1 > c0)
        bulk_g2s_multicast(xs + (c0 - T0) + shift, x + c0, (uint32_t)(c1 - c0) * 4u, full, (uint16_t)((1u << p.csize) - 1u));
    } else {
      mbar_arrive(full);
    }
  }
}
__device__ __forceinline__ int r3_shift(const R3Params& p, int64_t row, int64_t f0) {
  const int64_t T0 = f0 * p.orig_r - p.width;
  const int a0 = (int)((reinterpret_cast<uintptr_t>(p.wave + row * p.row_stride) >> 2) & 3);
  return (int)((((a0 + T0) % 4) + 4) % 4);
}

__global__ void __maxnreg__(224) resample_r3_kernel(const R3Params p, int require_flag) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* s_x = reinterpret_cast<float*>(smem_raw);                                   // [3][slot_floats]
  uint64_t* s_full = reinterpret_cast<uint64_t*>(s_x + 3 * (size_t)p.slot_floats);   // [3]
  uint64_t* s_empty = s_full + 3;                                                    // [3]
  if (require_flag && p.hdr->r3_ok == 0) return;  // (uniform over the grid) the mma kernel launched next does the work

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t crank = cluster_ctarank();
  const int64_t cid = blockIdx.x / p.csize, n_clusters = gridDim.x / p.csize;
  if (tid < 3) {
    mbar_init(s_full + tid, 1);
    mbar_init(s_empty + tid, p.csize);
  }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  cluster_sync_all();  // every CTA's barriers exist before anyone multicasts into it or arrives on it

  // this warp's quad of phases and its taps (registers for the rest of the kernel)
  const int quad = (int)crank * kR3Warps + warp;
  const bool active = quad < p.n_quads;
  float4 tp[kR3Len];
  int qb = 0;
  if (active) {
    qb = p.qbase[quad];
#pragma unroll
    for (int i = 0; i < kR3Len; ++i) tp[i] = __ldg(p.qtaps + (size_t)quad * kR3Len + i);
  } else {
#pragma unroll
    for (int i = 0; i < kR3Len; ++i) tp[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const int j0 = 4 * quad;

  // tiles of this cluster: T(n) = cid + n * n_clusters
  auto tile_of = [&](int64_t n, int64_t& row, int64_t& f0) {
    const int64_t t = cid + n * n_clusters;
    row = t / p.tiles_per_row;
    f0 = (t - row * p.tiles_per_row) * 32;
    return t < p.total_tiles;
  };
  int64_t row, f0;
  for (int64_t n = 0; n < 2; ++n)  // prologue: two tiles in flight
    if (tile_of(n, row, f0)) r3_fill(p, row, f0, s_x + (size_t)(n % 3) * p.slot_floats, s_full + (n % 3), crank, tid, blockDim.x);
  __syncthreads();
  for (int64_t n = 0; tile_of(n, row, f0); ++n) {
    const int slot = (int)(n % 3);
    {  // stage tile n + 2 into the slot tile n - 1 used: every CTA of the cluster must have released it
      int64_t nrow, nf0;
      if (tile_of(n + 2, nrow, nf0)) {
        const int ns = (int)((n + 2) % 3);
        if (n + 2 >= 3 && tid == 0) mbar_wait_cluster(s_empty + ns, (uint32_t)(((n + 2) / 3 - 1) & 1));
        __syncthreads();  // (the local scalar part may be written now too)
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        r3_fill(p, nrow, nf0, s_x + (size_t)ns * p.slot_floats, s_full + ns, crank, tid, blockDim.x);
      }
    }
    mbar_wait_cluster(s_full + slot, (uint32_t)((n / 3) & 1));
    if (active) {
      const float* xs = s_x + (size_t)slot * p.slot_floats + r3_shift(p, row, f0) + lane * p.orig_r + qb;
      uint64_t a01e = 0ull, a23e = 0ull, a01o = 0ull, a23o = 0ull;
#pragma unroll
      for (int i = 0; i < kR3Len; i += 2) {
        const float x0 = xs[i], x1 = xs[i + 1];
        a01e = fma2_raw(pk2(tp[i].x, tp[i].y), pk2(x0, x0), a01e);
        a23e = fma2_raw(pk2(tp[i].z, tp[i].w), pk2(x0, x0), a23e);
        a01o = fma2_raw(pk2(tp[i + 1].x, tp[i + 1].y), pk2(x1, x1), a01o);
        a23o = fma2_raw(pk2(tp[i + 1].z, tp[i + 1].w), pk2(x1, x1), a23o);
      }
      const float2 y01 = upk2(add2_raw(a01e, a01o)), y23 = upk2(add2_raw(a23e, a23o));
      const int64_t f = f0 + lane;
      if (f < p.frames) {
        const int64_t n0 = f * p.new_r + j0;
        float* o = p.out + row * p.out_row_stride + n0;
        if (p.out_vec && j0 + 4 <= p.new_r && n0 + 4 <= p.out_len) {
          *reinterpret_cast<float4*>(o) = make_float4(y01.x, y01.y, y23.x, y23.y);
        } else {
          const float y[4] = {y01.x, y01.y, y23.x, y23.y};
#pragma unroll
          for (int r = 0; r < 4; ++r)
            if (j0 + r < p.new_r && n0 + r < p.out_len) o[r] = y[r];
        }
      }
    }
    __syncthreads();  // this CTA is done with the slot ...
    if (tid == 0)     // ... tell every CTA of the cluster (they multicast into it)
      for (uint32_t r = 0; r < (uint32_t)p.csize; ++r) mbar_arrive_remote(s_empty + slot, r);
  }
  cluster_sync_all();  // nobody leaves while a peer may still arrive on its barriers
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

}  // namespace

size_t resample_workspace_bytes_impl(int new_r, int taps) { return rs_layout(new_r, taps).total; }

int resample_prepare_impl(const float* kernel, int orig_r, int new_r, int width, void* ws, size_t ws_bytes,
                          cudaStream_t stream) {
  if (kernel == nullptr || ws == nullptr || orig_r < 1 || new_r < 1 || width < 0) return B200A_EINVAL;
  const int taps = 2 * width + orig_r;
  const RsLayout l = rs_layout(new_r, taps);
  if (ws_bytes < l.total) return B200A_EWORKSPACE;
  unsigned char* base = static_cast<unsigned char*>(ws);
  if (cudaMemsetAsync(base + l.header, 0, sizeof(RsHeader), stream) != cudaSuccess) return B200A_ECUDA;
  RsHeader* hdr = reinterpret_cast<RsHeader*>(base + l.header);
  int2* support = reinterpret_cast<int2*>(base + l.support);
  resample_support_kernel<<<(new_r + 7) / 8, 256, 0, stream>>>(kernel, new_r, taps, orig_r, width, hdr, support);
  if (rs_tiles(new_r) <= kRsMaxTiles)
    resample_plan_kernel<<<1, 256, 0, stream>>>(kernel, support, new_r, taps, rs_tiles(new_r), hdr,
                                                reinterpret_cast<RsTile*>(base + l.tiles),
                                                reinterpret_cast<float4*>(base + l.frags),
                                                reinterpret_cast<uint4*>(base + l.frags16));
  resample_r3_plan_kernel<<<1, 256, 0, stream>>>(kernel, support, new_r, taps, (new_r + 3) / 4, hdr,
                                                 reinterpret_cast<int*>(base + l.r3base),
                                                 reinterpret_cast<float4*>(base + l.r3taps));
  resample_simt_plan_kernel<<<1, 256, 0, stream>>>(kernel, support, new_r, taps, rs_tiles(new_r), hdr,
                                                   reinterpret_cast<RsSimtGroup*>(base + l.sgroups),
                                                   reinterpret_cast<float*>(base + l.staps));
  return launch_status();
}

int resample_run_impl(const void* ws, const float* kernel, int orig_r, int new_r, int width, const float* wave,
                      int64_t rows, int64_t length, int64_t row_stride, float* out, int64_t out_row_stride,
                      int64_t out_len, cudaStream_t stream) {
  if (orig_r < 1 || new_r < 1 || width < 0 || rows < 0 || length < 0 || out_len < 0) return B200A_EINVAL;
  if (rows == 0 || out_len == 0) return B200A_OK;  // empty batch: pointers may be null
  if (ws == nullptr || kernel == nullptr || wave == nullptr || out == nullptr) return B200A_EINVAL;
  const int taps = 2 * width + orig_r;
  const RsLayout l = rs_layout(new_r, taps);
  const unsigned char* base = static_cast<const unsigned char*>(ws);

  // B200A_RS=simt|mma|bf16|direct|r3 forces one kernel family (A/B measurements, tests); default: the first that applies
  static const int forced = [] {
    const char* e = std::getenv("B200A_RS");
    if (e == nullptr) return 0;
    return e[0] == 's' ? 1 : (e[0] == 'm' ? 2 : (e[0] == 'd' ? 3 : (e[0] == 'b' ? 4 : (e[0] == 'r' ? 5 : 0))));
  }();
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return B200A_ECUDA;

  // ---- cluster path: taps in registers, tiles multicast to the CTAs that share the phases --------------------------
  bool r3_launched = false;
  {
    const int n_quads = (new_r + 3) / 4;
    const int csize = (n_quads + kR3Warps - 1) / kR3Warps;  // CTAs that share a tile: 5 at 441:160
    const int slot_floats = (32 * orig_r + 2 * width + 16 + 3 + 3 + kR3Len) & ~3;
    const size_t smem = sizeof(float) * 3 * (size_t)slot_floats + 64;
    const bool want = forced == 5;  // experiment kept for A/B timing (cluster-scope barrier per 32-frame tile): opt-in only
    if (want && csize <= kR3MaxCluster && smem <= (size_t)227 * 1024 && (reinterpret_cast<uintptr_t>(wave) & 3) == 0 &&
        length + (int64_t)taps + 64 * (int64_t)orig_r < ((int64_t)1 << 31)) {
      R3Params p{};
      p.wave = wave;
      p.rows = rows;
      p.length = length;
      p.row_stride = row_stride;
      p.out = out;
      p.out_row_stride = out_row_stride;
      p.out_len = out_len;
      p.hdr = reinterpret_cast<const RsHeader*>(base + l.header);
      p.qbase = reinterpret_cast<const int*>(base + l.r3base);
      p.qtaps = reinterpret_cast<const float4*>(base + l.r3taps);
      p.orig_r = orig_r;
      p.new_r = new_r;
      p.width = width;
      p.n_quads = n_quads;
      p.csize = csize;
      p.frames = (out_len + new_r - 1) / new_r;
      p.tiles_per_row = (p.frames + 31) / 32;
      p.total_tiles = rows * p.tiles_per_row;
      p.out_vec = (new_r % 4 == 0 && out_row_stride % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0) ? 1 : 0;
      if (cudaFuncSetAttribute(resample_r3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
        return B200A_ECUDA;
      cudaLaunchConfig_t cfg{};
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = (unsigned)csize;
      attr[0].val.clusterDim.y = 1;
      attr[0].val.clusterDim.z = 1;
      cfg.blockDim = dim3(kR3Warps * 32, 1, 1);
      cfg.dynamicSmemBytes = smem;
      cfg.stream = stream;
      cfg.attrs = attr;
      cfg.numAttrs = 1;
      cfg.gridDim = dim3((unsigned)csize, 1, 1);
      int max_clusters = 0;
      const cudaError_t occ = cudaOccupancyMaxActiveClusters(&max_clusters, resample_r3_kernel, &cfg);
      if (std::getenv("B200A_DEBUG") != nullptr)
        std::fprintf(stderr, "[b200a] r3: csize=%d smem=%zu occupancy query: %s, max_clusters=%d\n", csize, smem,
                     cudaGetErrorString(occ), max_clusters);
      if (occ == cudaSuccess && max_clusters > 0) {
        int64_t n_clusters = p.total_tiles < max_clusters ? p.total_tiles : max_clusters;
        if (n_clusters < 1) n_clusters = 1;
        cfg.gridDim = dim3((unsigned)(n_clusters * csize), 1, 1);
        const int require_flag = forced == 5 ? 0 : 1;
        const cudaError_t le = cudaLaunchKernelEx(&cfg, resample_r3_kernel, p, require_flag);
        if (std::getenv("B200A_DEBUG") != nullptr)
          std::fprintf(stderr, "[b200a] r3: launch %u CTAs: %s\n", cfg.gridDim.x, cudaGetErrorString(le));
        if (le != cudaSuccess) return B200A_ECUDA;
        if (forced == 5) return launch_status();
        r3_launched = true;  // the tensor-pipe kernel below runs only if the plan says the quads did not fit
      } else {
        (void)cudaGetLastError();
      }
    }
    if (forced == 5 && !r3_launched) return B200A_EUNSUPPORTED;
  }

  // ---- packed-FP32 SIMT path: odd orig' (conflict-free frame-per-lane reads) and the 3-slot ring fits -------------
  {
    const int n_groups = rs_tiles(new_r);
    const int slot_floats = (32 * orig_r + 2 * width + 3 + 8 + 3) & ~3;  // span + alignment shift + zero-tap over-read
    const size_t ring_bytes = sizeof(float) * 3 * (size_t)slot_floats;
    const size_t fixed = ring_bytes + sizeof(RsSimtGroup) * (size_t)n_groups + 64;
    const bool want = forced == 1;  // variant kept for A/B timing against the tensor-pipe kernel: opt-in only
    if (want && fixed + 8192 <= (size_t)227 * 1024 && (reinterpret_cast<uintptr_t>(wave) & 3) == 0 &&
        length + (int64_t)taps + 64 * (int64_t)orig_r < ((int64_t)1 << 31)) {
      RsSimtParams p{};
      p.wave = wave;
      p.rows = rows;
      p.length = length;
      p.row_stride = row_stride;
      p.out = out;
      p.out_row_stride = out_row_stride;
      p.out_len = out_len;
      p.hdr = reinterpret_cast<const RsHeader*>(base + l.header);
      p.groups = reinterpret_cast<const RsSimtGroup*>(base + l.sgroups);
      p.table = reinterpret_cast<const float*>(base + l.staps);
      p.orig_r = orig_r;
      p.new_r = new_r;
      p.width = width;
      p.n_groups = n_groups;
      p.frames = (out_len + new_r - 1) / new_r;
      p.halves = (p.frames + 31) / 32;
      p.total_halves = rows * p.halves;
      p.out_vec = (new_r % 4 == 0 && out_row_stride % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0) ? 1 : 0;
      // the tap table gets whatever shared memory is left (the kernel compares the device-side size written by
      // prepare with this room and reads the table through L1 instead when it does not fit)
      const size_t tap_cap = sizeof(float) * 8 * (size_t)n_groups * ((size_t)taps + 8);
      const size_t room = ((size_t)227 * 1024 - fixed) & ~(size_t)15;
      p.tap_floats = (int)((tap_cap < room ? tap_cap : room) / sizeof(float));
      const size_t smem = fixed + sizeof(float) * (size_t)p.tap_floats;
      if (cudaFuncSetAttribute(resample_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
        return B200A_ECUDA;
      int warps = (n_groups + 1) / 2;  // one phase group of the step's parity per warp
      if (warps > kSimtMaxWarps) warps = kSimtMaxWarps;
      if (warps < 4) warps = 4;
      int64_t grid = p.total_halves < sms ? p.total_halves : sms;
      if (grid < 1) grid = 1;
      resample_simt_kernel<<<(unsigned)grid, warps * 32, smem, stream>>>(p);
      return launch_status();
    }
    if (forced == 1) return B200A_EUNSUPPORTED;
  }

  // ---- tensor-pipe path -------------------------------------------------------------------------
  const int n_tiles = rs_tiles(new_r);
  const int xs_floats = (kRsFrames * orig_r + taps + 16 + 4 + 3) & ~3;
  const size_t smem_fixed = sizeof(float) * 2 * (size_t)xs_floats + 16 + sizeof(RsTile) * ((n_tiles + 3) & ~3);
  const bool aligned = (reinterpret_cast<uintptr_t>(wave) & 3) == 0;  // any float pointer; rows may have any pitch
  if (forced != 3 && n_tiles <= kRsMaxTiles && aligned && smem_fixed + 1024 <= (size_t)kRsSmemBudget) {
    RsParams p{};
    p.wave = wave;
    p.rows = rows;
    p.length = length;
    p.row_stride = row_stride;
    p.out = out;
    p.out_row_stride = out_row_stride;
    p.out_len = out_len;
    p.hdr = reinterpret_cast<const RsHeader*>(base + l.header);
    p.tiles = reinterpret_cast<const RsTile*>(base + l.tiles);
    p.frags = reinterpret_cast<const float4*>(base + l.frags);
    p.frags16 = reinterpret_cast<const uint4*>(base + l.frags16);
    p.orig_r = orig_r;
    p.new_r = new_r;
    p.width = width;
    p.taps = taps;
    p.n_tiles = n_tiles;
    p.frames = (out_len + new_r - 1) / new_r;
    p.blocks_per_row = (p.frames + kRsFrames - 1) / kRsFrames;
    p.total_blocks = rows * p.blocks_per_row;
    p.xs_floats = xs_floats;
    // fragments go to shared memory when they fit next to the staging buffers (the kernel compares the
    // device-side step count with the room granted here), otherwise they are read through L1
    p.frag_smem_bytes = (int)(((size_t)kRsSmemBudget - smem_fixed) & ~(size_t)511);  // everything that is left
    const size_t smem = smem_fixed + p.frag_smem_bytes;
    // default: TF32 x 3 (2^-21 relative).  B200A_RS=bf16 selects the bf16 x 3 variant (2^-16 relative, ~30x the rounding
    // error), opt-in for A/B timing
    auto kern = forced == 4 ? resample_mma_kernel<true> : resample_mma_kernel<false>;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
      return B200A_ECUDA;
    int64_t grid = p.total_blocks < sms ? p.total_blocks : sms;
    if (grid < 1) grid = 1;
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
    p.skip_if_r3_ok = r3_launched ? 1 : 0;
    // warps: n_tiles items (phase groups) per tile; prefer the largest count that divides them evenly
    const int items = n_tiles;
    int warps = 8;
    double best_idle = 2.0;
    for (int w = 8; w <= kRsMaxWarps; ++w) {
      const int rounds = (items + w - 1) / w;
      const double idle = 1.0 - (double)items / (double)(rounds * w);
      if (idle <= best_idle + 1e-9) { best_idle = idle; warps = w; }  // ties go to more warps
    }
    kern<<<(unsigned)grid, warps * 32, smem, stream>>>(p);
    return launch_status();
  }

  // ---- direct path --------------------------------------------------------------------------------
  if (rows > 65535) return B200A_EUNSUPPORTED;
  unsigned bx = (unsigned)((out_len + 255) / 256);
  if (bx > 4096) bx = 4096;
  dim3 grid(bx, (unsigned)rows);
  resample_direct_kernel<<<grid, 256, 0, stream>>>(wave, length, row_stride, kernel,
                                                  reinterpret_cast<const int2*>(base + l.support), orig_r, new_r,
                                                  width, taps, out, out_row_stride, out_len);
  return launch_status();
}

}  // namespace b200a
