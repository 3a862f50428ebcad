// Banded TF32 x 3 tensor-core contraction, shared by the mel filterbank (frontend_pow2.cu) and the resampler and its
// adjoint (resample.cu): D[16 rows][8 columns] = A[16][K] * B[K][8] on mma.sync.m16n8k8, visiting only the 8-wide
// k-steps where the group of 8 output columns has live entries, with error-compensated operands
// (A_hi*B_hi + A_lo*B_hi + A_hi*B_lo, ~2^-21 relative).
//
// B is split once, when a plan is prepared: step s of a tile is 32 float4, one per lane,
//   frags[(frag_off + s) * 32 + lane] = (B_hi[k0][n], B_hi[k1][n], B_lo[k0][n], B_lo[k1][n]),
//   n = 8 group + lane / 4,  k0 = kstart + 8 s + lane % 4,  k1 = k0 + 4.
#pragma once
#include <type_traits>

#include "ptx.cuh"

namespace b200a {

struct BandTile {  // one group of 8 output columns
  int group;     // columns [8 group, 8 group + 8)
  int kstart;    // first k of its first k-step (multiple of 8)
  int nsteps;    // 8-wide k-steps covering the union of the group's live ranges
  int frag_off;  // index of its first step in the fragment array
};
static_assert(sizeof(BandTile) == 16, "a tile is one 16-byte vector load");

// The tile of a group whose columns are live on k in [lo, hi) (no k-steps when the range is empty).
__device__ __forceinline__ BandTile band_tile(int group, int lo, int hi, int frag_off) {
  BandTile t{group, 0, 0, frag_off};
  if (hi > lo) {
    t.kstart = lo & ~7;
    t.nsteps = (hi - t.kstart + 7) / 8;
  }
  return t;
}

// Writes tile t's hi/lo B fragments with every thread of the block.  b(n, k) returns B[k][n], or 0 outside the matrix.
template <class B>
__device__ __forceinline__ void write_band_frags(const BandTile t, float4* frags, B b) {
  for (int i = threadIdx.x; i < t.nsteps * 32; i += blockDim.x) {
    const int s = i >> 5, lane = i & 31;
    const int n = 8 * t.group + (lane >> 2);
    const int k0 = t.kstart + 8 * s + (lane & 3);
    uint32_t h0, l0, h1, l1;
    split_tf32(b(n, k0), h0, l0);
    split_tf32(b(n, k0 + 4), h1, l1);
    frags[(size_t)(t.frag_off + s) * 32 + lane] =
        make_float4(__uint_as_float(h0), __uint_as_float(h1), __uint_as_float(l0), __uint_as_float(l1));
  }
}

// Copies the first total_steps fragment steps into shared memory when they fit in room_steps; returns whether it did.
__device__ __forceinline__ bool stage_band_frags(const float4* frags, int total_steps, int room_steps,
                                                 float4* s_frags) {
  const bool in_smem = total_steps <= room_steps;
  if (in_smem)
    for (int i = threadIdx.x; i < total_steps * 32; i += blockDim.x) s_frags[i] = frags[i];
  return in_smem;
}

// Accumulates one warp's D fragments of tile t for MT 16-row M tiles that share each B fragment load, in three
// independent chains per M tile: d[h][0] += A_hi*B_hi, d[h][1] += A_lo*B_hi, d[h][2] += A_hi*B_lo (band_sum adds them).
// a[2 h] and a[2 h + 1] point at this lane's A entries in rows r and r + 8 of M tile h (r = lane / 4) at column
// t.kstart + lane % 4.  The fragments come from s_frags when in_smem, else from g_frags through the read-only cache.
template <int MT, int UNROLL>
__device__ __forceinline__ void band_contract(const BandTile& t, const float4* s_frags, const float4* g_frags,
                                              bool in_smem, int lane, const float* const (&a)[2 * MT],
                                              float (&d)[MT][3][4]) {
#pragma unroll
  for (int h = 0; h < MT; ++h)
#pragma unroll
    for (int ch = 0; ch < 3; ++ch)
#pragma unroll
      for (int q = 0; q < 4; ++q) d[h][ch][q] = 0.f;
  auto run = [&](auto smem) {
    constexpr bool kSmem = decltype(smem)::value;
    const float4* frg = (kSmem ? s_frags : g_frags) + (size_t)t.frag_off * 32 + lane;
#pragma unroll UNROLL
    for (int s = 0; s < t.nsteps; ++s) {
      float4 bf;
      if constexpr (kSmem) bf = frg[(size_t)s * 32];
      else bf = __ldg(frg + (size_t)s * 32);
#pragma unroll
      for (int h = 0; h < MT; ++h) {
        const float av[4] = {a[2 * h][8 * s], a[2 * h + 1][8 * s], a[2 * h][8 * s + 4], a[2 * h + 1][8 * s + 4]};
        uint32_t hi[4], lo[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) split_tf32(av[q], hi[q], lo[q]);
        mma_tf32(d[h][0], hi, __float_as_uint(bf.x), __float_as_uint(bf.y));
        mma_tf32(d[h][1], lo, __float_as_uint(bf.x), __float_as_uint(bf.y));
        mma_tf32(d[h][2], hi, __float_as_uint(bf.z), __float_as_uint(bf.w));
      }
    }
  };
  if (in_smem) run(std::true_type{});
  else run(std::false_type{});
}

// Element q of a D fragment from its three chains, in the fixed order d0 + (d1 + d2).
__device__ __forceinline__ float band_sum(const float (&d)[3][4], int q) { return d[0][q] + (d[1][q] + d[2][q]); }

}  // namespace b200a
