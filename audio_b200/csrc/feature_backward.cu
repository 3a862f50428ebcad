// Input gradients of the feature stages that follow the mel contraction: the MFCC / LFCC adjoint after the mel stage
// (DCT, log or dB map, top_db clamp), AmplitudeToDB, MelScale and SpectralCentroid's ratio.
// Reference: transforms/_transforms.py:701-708 (MFCC), functional.py:356-404 (amplitude_to_DB), :1257-1299
// (spectral_centroid); the gradients are torch's autograd of those op sequences.
//
// The top_db clamp c = maximum(d, thr), thr = amax_g(d) - top_db, is the only cross-row coupling.  torch's rules
// (maximum: the gradient goes to d where d > thr, half of it where d == thr; amax: split evenly over the ties) give
//   g_d[e] = g[e] ([d > thr] + 1/2 [d == thr]) + [d == amax_g] R_g / count_g,   R_g = sum_g g[e] ([d < thr] + 1/2 [d == thr]).
// Three passes, no float atomics, so reruns are bit-identical:
//   1. per tile (tiles never straddle a group): g_d of every element times the map's derivative into the output, the
//      tile's routed sum and tie count into its slot (fixed-order block reduction);
//   2. per group: the slots summed in a fixed order into share_g = R_g / count_g;
//   3. the tiles that hold a tie add share_g times the derivative at the ties.
// Without a clamp (log path, top_db None) only pass 1 runs.
#include "common.cuh"

namespace b200a {

constexpr int kFbThreads = 256;
constexpr int kFbFrames = 64;             // frames per tile of the MFCC adjoint (16 quads of frames)
constexpr int kFbElems = 8 * kFbThreads;  // elements per tile of the AmplitudeToDB adjoint
constexpr float kLn10 = 2.302585092994046f;

struct TileSum {
  float routed;  // sum of the gradient routed to the tile's group threshold
  int ties;      // elements equal to the group maximum
};

struct FeatParams {
  const float* grad;               // MFCC: [rows][T][n_c] at element strides gs_*; AmplitudeToDB: grad[e * gs_flat]
  int64_t gs_row, gs_frame, gs_col, gs_flat;
  const float* dct;                // [n][n_c] (the workspace copy), MFCC only
  int n, n_c;                      // values per unit (n_mels, or 1 for AmplitudeToDB) and DCT coefficients
  int64_t frames;                  // T (MFCC)
  const float* feat;               // the forward's pre-clamp d, or null: recomputed from `mel` (AmplitudeToDB)
  const float* mel;                // m: the recomputed mel stage, or AmplitudeToDB's input
  const float* gmax;               // [groups] the forward's maxima, or null: no clamp
  float top_db, mult, amin, offset;
  int log_path;                    // d = log(m + 1e-6) (MFCC log_mels): no clamp
  int64_t group_units, total_units;  // units (frames / elements) per group and in all
  int64_t tiles_per_group, total_tiles;
  TileSum* tiles;                  // [total_tiles]
  float* share;                    // [groups]
  float* out;                      // g_m, unit-major [total_units][n]
};

struct TileGeom {
  int64_t group, u0;
  int nu;  // units of the tile (may be <= 0 in a short last group)
};

__device__ __forceinline__ TileGeom tile_geom(const FeatParams& p, int64_t tile, int tile_units) {
  TileGeom t;
  t.group = tile / p.tiles_per_group;
  const int64_t g0 = t.group * p.group_units;
  const int64_t g1 = min(g0 + p.group_units, p.total_units);
  t.u0 = g0 + (tile - t.group * p.tiles_per_group) * tile_units;
  t.nu = (int)max((int64_t)0, min((int64_t)tile_units, g1 - t.u0));
  return t;
}

__device__ __forceinline__ float pre_clamp(const FeatParams& p, int64_t e, float m) {
  return p.feat != nullptr ? p.feat[e] : db_value(m, p.mult, p.amin, p.offset);
}

// dL/dm for the d-gradient gd of element e (the tie share is added by pass 3); routed sum and ties into acc.
// torch: log(m + 1e-6) -> gd / (m + 1e-6); mult * log10(clamp(m, min=amin)) -> gd * mult / (ln10 m) where m >= amin, else 0.
__device__ __forceinline__ float element_vjp(const FeatParams& p, int64_t e, float gd, float thr, float gm, TileSum& acc) {
  const float m = p.mel[e];
  if (p.log_path) return gd / (m + 1e-6f);
  float own = gd;
  if (p.gmax != nullptr) {
    const float d = pre_clamp(p, e, m);
    own = d > thr ? gd : (d == thr ? 0.5f * gd : 0.f);
    acc.routed += d < thr ? gd : (d == thr ? 0.5f * gd : 0.f);
    acc.ties += d == gm ? 1 : 0;
  }
  return m >= p.amin ? own * p.mult / (m * kLn10) : 0.f;
}

// Block-wide sum in a fixed order (warp butterflies, then the warps in index order); the result in thread 0.
__device__ __forceinline__ TileSum block_sum(TileSum v) {
  __shared__ float s_f[kFbThreads / 32];
  __shared__ int s_i[kFbThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    v.routed += __shfl_xor_sync(0xffffffffu, v.routed, o);
    v.ties += __shfl_xor_sync(0xffffffffu, v.ties, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();  // the previous call's readers are done
  if (lane == 0) {
    s_f[warp] = v.routed;
    s_i[warp] = v.ties;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    v = TileSum{0.f, 0};
    for (int w = 0; w < kFbThreads / 32; ++w) {
      v.routed += s_f[w];
      v.ties += s_i[w];
    }
  }
  return v;
}

// Pass 1 of the MFCC / LFCC adjoint: a persistent CTA walks tiles of kFbFrames frames.  The DCT [n][n_c] is staged once
// (odd pitch: the lanes of a warp read rows m..m+31 of one column conflict-free), each tile's cepstral gradient as
// [n_c][kFbFrames]; a thread computes g_d for one mel bin of 4 frames (one float4 of gradients per coefficient).
__global__ void __launch_bounds__(kFbThreads) mfcc_vjp_kernel(FeatParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int ldd = p.n_c | 1;
  float* s_dct = reinterpret_cast<float*>(smem_raw);                         // [n][ldd]
  float* s_g = s_dct + (((size_t)p.n * ldd + 3) & ~(size_t)3);               // [n_c][kFbFrames], 16-byte aligned
  __shared__ int64_t s_goff[kFbFrames];
  for (int i = threadIdx.x; i < p.n * p.n_c; i += blockDim.x) {
    const int m = i / p.n_c, j = i - m * p.n_c;
    s_dct[m * ldd + j] = p.dct[i];
  }
  for (int64_t tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileGeom tg = tile_geom(p, tile, kFbFrames);
    __syncthreads();  // the previous tile's gradients are consumed (and s_dct is complete on the first pass)
    if (threadIdx.x < kFbFrames && (int)threadIdx.x < tg.nu) {
      const int64_t u = tg.u0 + threadIdx.x, r = u / p.frames;
      s_goff[threadIdx.x] = r * p.gs_row + (u - r * p.frames) * p.gs_frame;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < p.n_c * kFbFrames; i += blockDim.x) {
      const int j = i / kFbFrames, f = i - j * kFbFrames;
      s_g[i] = f < tg.nu ? p.grad[s_goff[f] + j * p.gs_col] : 0.f;
    }
    __syncthreads();
    const float gm = p.gmax != nullptr ? p.gmax[tg.group] : 0.f;
    const float thr = gm - p.top_db;
    TileSum acc{0.f, 0};
    const int quads = (tg.nu + 3) >> 2;
    for (int w = threadIdx.x; w < p.n * quads; w += blockDim.x) {
      const int fq = w / p.n, m = w - fq * p.n;
      const float* dr = s_dct + m * ldd;
      const float4* gq = reinterpret_cast<const float4*>(s_g) + fq;
      float a[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
      for (int j = 0; j < p.n_c; ++j) {
        const float c = dr[j];
        const float4 v = gq[j * (kFbFrames / 4)];
        a[0] = fmaf(c, v.x, a[0]);
        a[1] = fmaf(c, v.y, a[1]);
        a[2] = fmaf(c, v.z, a[2]);
        a[3] = fmaf(c, v.w, a[3]);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (4 * fq + q < tg.nu) {
          const int64_t e = (tg.u0 + 4 * fq + q) * p.n + m;
          p.out[e] = element_vjp(p, e, a[q], thr, gm, acc);
        }
      }
    }
    if (p.gmax != nullptr) {
      acc = block_sum(acc);
      if (threadIdx.x == 0) p.tiles[tile] = acc;
    }
  }
}

// Pass 1 of the AmplitudeToDB adjoint: tiles of kFbElems contiguous elements, d recomputed from x.
__global__ void __launch_bounds__(kFbThreads) db_vjp_kernel(FeatParams p) {
  for (int64_t tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileGeom tg = tile_geom(p, tile, kFbElems);
    const float gm = p.gmax != nullptr ? p.gmax[tg.group] : 0.f;
    const float thr = gm - p.top_db;
    TileSum acc{0.f, 0};
    for (int i = threadIdx.x; i < tg.nu; i += blockDim.x) {
      const int64_t e = tg.u0 + i;
      p.out[e] = element_vjp(p, e, p.grad[e * p.gs_flat], thr, gm, acc);
    }
    if (p.gmax != nullptr) {
      acc = block_sum(acc);
      if (threadIdx.x == 0) p.tiles[tile] = acc;
    }
  }
}

// Pass 2: one CTA per group sums its tiles' slots in a fixed order; share_g = R_g / count_g.
__global__ void __launch_bounds__(kFbThreads) tie_share_kernel(const TileSum* __restrict__ tiles, int64_t tiles_per_group,
                                                               float* __restrict__ share) {
  const TileSum* t = tiles + (int64_t)blockIdx.x * tiles_per_group;
  TileSum acc{0.f, 0};
  for (int64_t i = threadIdx.x; i < tiles_per_group; i += blockDim.x) {
    acc.routed += t[i].routed;
    acc.ties += t[i].ties;
  }
  acc = block_sum(acc);
  if (threadIdx.x == 0) share[blockIdx.x] = acc.ties > 0 ? acc.routed / (float)acc.ties : 0.f;
}

// Pass 3: the tiles holding a tie add share_g times the derivative at every element equal to the group maximum.
__global__ void __launch_bounds__(kFbThreads) tie_add_kernel(FeatParams p, int tile_units) {
  for (int64_t tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    if (p.tiles[tile].ties == 0) continue;
    const TileGeom tg = tile_geom(p, tile, tile_units);
    const float gm = p.gmax[tg.group], s = p.share[tg.group];
    const int64_t e0 = tg.u0 * p.n, n = (int64_t)tg.nu * p.n;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      const int64_t e = e0 + i;
      const float m = p.mel[e];
      if (pre_clamp(p, e, m) == gm && m >= p.amin) p.out[e] += s * p.mult / (m * kLn10);
    }
  }
}

struct FeatScratch {
  size_t tiles, share, total;
};

static FeatScratch feat_scratch_layout(int64_t groups, int64_t tiles_per_group) {
  FeatScratch s{};
  s.tiles = 0;
  s.share = align_up(sizeof(TileSum) * (size_t)groups * (size_t)tiles_per_group, 256);
  s.total = s.share + align_up(sizeof(float) * (size_t)groups, 256);
  return s;
}

// Shared host part: tiles, scratch pointers, then the three passes.  `pass1` launches pass 1 on `grid` CTAs.
template <typename Pass1>
static int run_feature_vjp(FeatParams& p, int64_t groups, int tile_units, void* scratch, cudaStream_t stream, Pass1 pass1) {
  p.tiles_per_group = (p.group_units + tile_units - 1) / tile_units;
  p.total_tiles = groups * p.tiles_per_group;
  if (p.total_tiles == 0) return B200A_OK;
  if (p.gmax != nullptr) {
    const FeatScratch l = feat_scratch_layout(groups, p.tiles_per_group);
    unsigned char* base = static_cast<unsigned char*>(scratch);
    p.tiles = reinterpret_cast<TileSum*>(base + l.tiles);
    p.share = reinterpret_cast<float*>(base + l.share);
  }
  int rc = pass1(sm_capped_grid(p.total_tiles, 8));
  if (rc != B200A_OK || p.gmax == nullptr) return rc;
  if (groups > 0x7fffffffLL) return B200A_EUNSUPPORTED;
  tie_share_kernel<<<(unsigned)groups, kFbThreads, 0, stream>>>(p.tiles, p.tiles_per_group, p.share);
  rc = launch_status();
  if (rc != B200A_OK) return rc;
  const int64_t grid = sm_capped_grid(p.total_tiles, 8);
  if (grid < 0) return B200A_ECUDA;
  tie_add_kernel<<<(unsigned)grid, kFbThreads, 0, stream>>>(p, tile_units);
  return launch_status();
}

static size_t mfcc_vjp_smem(int n_mels, int n_mfcc) {
  return sizeof(float) * ((((size_t)n_mels * (n_mfcc | 1)) + 3) / 4 * 4 + (size_t)n_mfcc * kFbFrames);
}

size_t mfcc_backward_scratch(int64_t rows, int64_t frames, int64_t rows_per_group) {
  const int64_t groups = (rows + rows_per_group - 1) / rows_per_group;
  const int64_t tpg = (rows_per_group * frames + kFbFrames - 1) / kFbFrames;
  return feat_scratch_layout(groups, tpg).total;
}

int mfcc_backward_impl(const b200a_frontend_desc* d, const void* ws, const float* grad, int64_t gs_row, int64_t gs_frame,
                       int64_t gs_col, const float* feat, const float* mel, const float* group_max, int64_t rows,
                       int64_t frames, int64_t rows_per_group, float top_db, void* scratch, float* grad_mel,
                       cudaStream_t stream) {
  const size_t smem = mfcc_vjp_smem(d->n_mels, d->n_mfcc);
  if (smem > 200 * 1024) return B200A_EUNSUPPORTED;
  const bool clamp = !d->log_mels && group_max != nullptr && top_db >= 0.f;
  FeatParams p{};
  p.grad = grad;
  p.gs_row = gs_row;
  p.gs_frame = gs_frame;
  p.gs_col = gs_col;
  p.dct = frontend_ws(*d, ws).dct;
  p.n = d->n_mels;
  p.n_c = d->n_mfcc;
  p.frames = frames;
  p.feat = feat;
  p.mel = mel;
  p.gmax = clamp ? group_max : nullptr;
  p.top_db = top_db;
  p.mult = d->db_multiplier;
  p.amin = d->db_amin;
  p.offset = d->db_offset;
  p.log_path = d->log_mels ? 1 : 0;
  p.total_units = rows * frames;
  p.group_units = clamp ? rows_per_group * frames : p.total_units;
  p.out = grad_mel;
  const int64_t groups = clamp ? (rows + rows_per_group - 1) / rows_per_group : 1;
  return run_feature_vjp(p, groups, kFbFrames, scratch, stream, [&](int64_t grid) {
    // the kernel also has static shared memory (the frame offsets, the block reduction), so its dynamic limit is raised
    // to what this call needs rather than to kSmemLimit (launch_kernel), which together would exceed the per-CTA maximum
    if (grid < 0 || cudaFuncSetAttribute(mfcc_vjp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
      return (int)B200A_ECUDA;
    mfcc_vjp_kernel<<<(unsigned)grid, kFbThreads, smem, stream>>>(p);
    return launch_status();
  });
}

size_t amplitude_to_db_backward_scratch(int64_t groups, int64_t group_elems) {
  return feat_scratch_layout(groups, (group_elems + kFbElems - 1) / kFbElems).total;
}

int amplitude_to_db_backward_impl(const float* x, const float* grad, int64_t g_stride, int64_t groups, int64_t group_elems,
                                  float mult, float amin, float offset, float top_db, const float* group_max, void* scratch,
                                  float* grad_x, cudaStream_t stream) {
  const bool clamp = group_max != nullptr && top_db >= 0.f;
  FeatParams p{};
  p.grad = grad;
  p.gs_flat = g_stride;
  p.n = 1;
  p.mel = x;
  p.gmax = clamp ? group_max : nullptr;
  p.top_db = top_db;
  p.mult = mult;
  p.amin = amin;
  p.offset = offset;
  p.total_units = groups * group_elems;
  p.group_units = clamp ? group_elems : p.total_units;
  p.out = grad_x;
  return run_feature_vjp(p, clamp ? groups : 1, kFbElems, scratch, stream, [&](int64_t grid) {
    if (grid < 0) return (int)B200A_ECUDA;
    db_vjp_kernel<<<(unsigned)grid, kFbThreads, 0, stream>>>(p);
    return launch_status();
  });
}

// MelScale adjoint, the transpose of apply_fbank_kernel: grad_spec[r][t][k] = sum_m fb[k][m] g[r][m][t].  Lanes run
// along the frames (g's logical (.., n_filters, T) layout), warps along the bins.
__global__ void __launch_bounds__(256)
apply_fbank_backward_kernel(const float* __restrict__ g, int64_t gs_row, int64_t gs_filter, int64_t gs_frame, int64_t frames,
                            const float* __restrict__ fb, int64_t n_bins, int n_filters, float* __restrict__ out) {
  const int64_t row = blockIdx.y;
  const int64_t t = (int64_t)blockIdx.x * 32 + (threadIdx.x & 31);
  if (t >= frames) return;
  const float* gr = g + row * gs_row + t * gs_frame;
  for (int64_t k = threadIdx.x >> 5; k < n_bins; k += blockDim.x >> 5) {
    const float* fk = fb + k * n_filters;
    float acc = 0.f;
    for (int m = 0; m < n_filters; ++m) acc = fmaf(fk[m], gr[m * gs_filter], acc);
    out[(row * frames + t) * n_bins + k] = acc;
  }
}

int apply_fbank_backward_impl(const float* grad, int64_t rows, int64_t n_filters, int64_t frames, int64_t gs_row,
                              int64_t gs_filter, int64_t gs_frame, const float* fb, int64_t n_bins, float* grad_spec,
                              cudaStream_t stream) {
  if (rows > 65535) return B200A_EUNSUPPORTED;
  dim3 grid((unsigned)((frames + 31) / 32), (unsigned)rows);
  apply_fbank_backward_kernel<<<grid, 256, 0, stream>>>(grad, gs_row, gs_filter, gs_frame, frames, fb, n_bins,
                                                        (int)n_filters, grad_spec);
  return launch_status();
}

// SpectralCentroid's ratio y = N / D per frame: (g_N, g_D) = (g / D, -g N / D^2), as torch's div backward.
__global__ void __launch_bounds__(256) ratio_backward_kernel(const float2* __restrict__ pairs, const float* __restrict__ g,
                                                             int64_t gs_row, int64_t gs_frame, int64_t frames, int64_t n,
                                                             float2* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t r = i / frames, t = i - r * frames;
  const float gv = g[r * gs_row + t * gs_frame];
  const float2 v = pairs[i];
  out[i] = make_float2(gv / v.y, -gv * v.x / (v.y * v.y));
}

int ratio_backward_impl(const float* pairs, const float* grad, int64_t rows, int64_t frames, int64_t gs_row,
                        int64_t gs_frame, float* grad_pairs, cudaStream_t stream) {
  const int64_t n = rows * frames;
  if ((n + 255) / 256 > 0x7fffffffLL) return B200A_EUNSUPPORTED;
  ratio_backward_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float2*>(pairs), grad, gs_row,
                                                                         gs_frame, frames, n,
                                                                         reinterpret_cast<float2*>(grad_pairs));
  return launch_status();
}

}  // namespace b200a
