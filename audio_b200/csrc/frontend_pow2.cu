// Register-FFT fast path of the fused front end (n_fft = 256 / 512 / 1024 / 2048, one-sided, real output stages).
//
// A group of G = n_fft/32 lanes transforms one PAIR of consecutive frames (a, b); a warp holds 32/G
// such groups (1, 2 or 4 pairs = 2, 4 or 8 consecutive frames of one utterance = one "unit"):
//   input   the unit's n_fft + (frames-1)*hop contiguous samples are staged into shared memory by ONE
//           bulk asynchronous copy (cp.async.bulk + mbarrier, the TMA engine's 1-D mode), issued a
//           unit ahead so its latency hides behind the previous unit's arithmetic
//   z[n] = w[n] * (a[n] + i b[n]),  n = g + G j          -- 32 complex values per lane
//   pass 1  32-point DFT over j in registers (radix-2 DIT, compile-time twiddles, FMA-form butterflies)
//   twiddle W_nfft^(g * k2) from a shared 32 x G table, transpose through a padded per-warp shared tile
//   pass 2  32/G DFTs of G points over the former lane index, in registers  -> Z[l + G q + 32 k1]
//   un-pack the two real spectra with one shuffle per needed value:  A = (Z[k] + conj Z[N-k]) / 2,
//                                                                    B = (Z[k] - conj Z[N-k]) / 2i
//   every lane ends with bins k = l + G m (m < 16) of its two frames; |.|^p -> global (Spectrogram: 16
//   independent warps per CTA), or -> shared memory for the mel contraction.
//   mel     (any filterbank up to 512 filters) the power tile times the filterbank on the tensor cores:
//           mma.sync m16n8k8 TF32 with error-compensated operands (P_hi*F_hi + P_lo*F_hi + P_hi*F_lo,
//           ~2^-21 relative), visiting only the k-steps where a group of 8 filters is non-zero.
//           (-> dB / log) -> global.  n_fft <= 1024: 16 uniform warps at 128 registers, each transforms a unit,
//           publishes its rows between two CTA barriers and contracts its share of the (16-frame tile, filter group)
//           items.  n_fft = 2048: 8 transform and 4 contraction warps meeting at mbarriers.
// Nothing but the waveform is read from HBM and nothing but the final features is written.
//
// Reference semantics: src/torchaudio/functional/functional.py:54-145 and
// transforms/_transforms.py:403-415, :701-705 (see frontend_generic.cu for the any-size path).
#include <type_traits>
#include <utility>

#include "band_mma.cuh"
#include "common.cuh"
#include "f32x2.cuh"
#include "ptx.cuh"

namespace b200a {

namespace {

constexpr int kWarps = 8;     // transform warps per CTA (n_fft = 2048 kernels)
constexpr int kMelWarps = 4;  // contraction warps per CTA (n_fft = 2048 mel kernel)
constexpr int kUniWarps = 16;  // warps per CTA of the 256 / 512 / 1024-point mel kernel, each transforms and contracts
constexpr int kMaxItems = 64;  // filter groups (of 8) per contraction
constexpr int kMaxItemsPerWarp = 32;
constexpr int kMaxMTiles = 8;  // 16-frame MMA tiles per iteration of the 16-warp mel kernel (n_fft = 256: 128 frames)
constexpr int kFragSmemSteps = 112;  // filterbank fragments kept in shared memory (x 512 B)
constexpr int kMaxSlots = 128;

// Geometry of one transform size: G lanes per frame pair.
template <int G>
struct Geo {
  static constexpr int kNfft = 32 * G;
  static constexpr int kBins = kNfft / 2 + 1;
  static constexpr int kGroups = 32 / G;        // frame pairs per warp
  static constexpr int kFrames = 2 * kGroups;   // frames per warp and iteration ("unit")
  static constexpr int kRowLd = G + 1;          // pitch of one transpose row (bank-conflict free)
  static constexpr int kRegion = 32 * (G + 1) + (G == 8 ? 8 : 0);  // float2 per lane group (skewed for G = 8)
  static constexpr int kTileF2 = kGroups * kRegion;                // float2 per warp
  // the mel kernel transposes real and imaginary parts in two float passes: kRegionF floats per lane group, skewed by
  // G floats so that the 32 / G groups of a warp hit disjoint banks
  static constexpr int kRegionF = 32 * (G + 1) + (G < 32 ? G : 0);
  // floats per warp in the mel kernel: the split transpose, or the staged span of a unit (n_fft + (kFrames-1) hop:
  // hop <= 512 / 330 / 173 at n_fft = 1024 / 512 / 256), whichever is larger; sized to the shared-memory budget
  static constexpr int kMelRegion = G == 32 ? 1536 : (G == 16 ? 1504 : 1472);
  // filterbank fragment steps the mel kernel keeps in shared memory (n_fft = 1024, 80 mels: 91)
  static constexpr int kMelFragSteps = G == 32 ? 100 : kFragSmemSteps;
  static constexpr int kSlots = kUniWarps * kFrames;               // frames finished per mel CTA iteration
  static constexpr int kMTiles = kSlots / 16;                      // 16-frame MMA tiles per iteration
  // floats per power row: every k-step of 8 bins, and == 4 (mod 8) so the A-fragment loads are bank-conflict free
  static constexpr int kPitch = (kBins + 7) / 8 * 8 + 4;
  static constexpr int kLogG = G == 32 ? 5 : (G == 16 ? 4 : 3);
  static_assert(kMelRegion >= kGroups * kRegionF && kMelRegion % 4 == 0, "mel warp region");
};

// The mel contraction D[16 frames][n_mels] = P[16][bins] * F[bins][n_mels] is cut into ITEMS =
// groups of 8 filters with the k-steps where the group is non-zero (band_mma.cuh's tiles), spread over the
// contraction warps by descending size.
struct MelPlan {  // built on the device by prepare_mma_kernel
  int n_tiles, n_items, total_steps, n_work;
  // n_fft = 2048 kernel: the filter groups of each of its kMelWarps contraction warps
  int warp_cnt[kMelWarps];
  int warp_items[kMelWarps][kMaxItemsPerWarp];
  // 16-warp mel kernel: warp w contracts work[work_begin[w] .. work_begin[w + 1]), entries (16-frame tile << 8) | group
  int work_begin[kUniWarps + 4];
  unsigned short work[kMaxMTiles * kMaxItems];
  BandTile items[kMaxItems];
};

struct Pow2Extra {  // tables appended to the generic workspace
  size_t tw2d, tw_eo, plan, frags, total;
};

inline int mel_tiles(int n_mels) { return (n_mels + 7) / 8; }

inline Pow2Extra pow2_layout(const b200a_frontend_desc& d, size_t base) {
  Pow2Extra e{};
  const size_t n_bins = d.n_fft / 2 + 1;
  const size_t nt = d.n_mels > 0 ? mel_tiles(d.n_mels) : 0;
  size_t off = base;
  e.tw2d = off;
  off = align_up(off + sizeof(float2) * 32 * 32, 256);
  e.tw_eo = off;
  off = align_up(off + sizeof(float2) * 17 * 32, 256);
  e.plan = off;
  off = align_up(off + sizeof(MelPlan), 256);
  e.frags = off;  // worst case: every tile spans every bin
  off = align_up(off + sizeof(float4) * 32 * nt * ((n_bins + 7) / 8 + 1), 256);
  e.total = off;
  return e;
}

// The register-FFT tables of a front-end workspace (Pow2Extra), after its front-end tables.
template <typename W>
struct Pow2Ws {
  WsPtr<W, float2> tw2d, tw_eo;
  WsPtr<W, MelPlan> plan;
  WsPtr<W, float4> frags;
};

template <typename W>
Pow2Ws<W> pow2_ws(const b200a_frontend_desc& d, W* ws) {
  const Pow2Extra e = pow2_layout(d, ws_layout(d).total);
  return {ws_at<float2>(ws, e.tw2d), ws_at<float2>(ws, e.tw_eo), ws_at<MelPlan>(ws, e.plan), ws_at<float4>(ws, e.frags)};
}

bool pow2_applicable(const b200a_frontend_desc& d) {
  return (d.n_fft == 2048 || d.n_fft == 1024 || d.n_fft == 512 || d.n_fft == 256) && d.onesided != 0;
}

// ---- compile-time helpers -----------------------------------------------------------------
template <int... Is, typename F>
__device__ __forceinline__ void static_for_impl(std::integer_sequence<int, Is...>, F&& f) {
  (f(std::integral_constant<int, Is>{}), ...);
}
template <int N, typename F>
__device__ __forceinline__ void static_for(F&& f) {
  static_for_impl(std::make_integer_sequence<int, N>{}, static_cast<F&&>(f));
}

__host__ __device__ constexpr int brev5(int v) {
  return ((v & 1) << 4) | ((v & 2) << 2) | (v & 4) | ((v & 8) >> 2) | ((v & 16) >> 4);
}
template <int LOG>
__host__ __device__ constexpr int brev(int v) {  // bit reversal of a LOG-bit index
  return brev5(v) >> (5 - LOG);
}

// cos / sin of 2 pi k / 32, k = 0..16
__device__ constexpr float kCos32[17] = {1.f, 0.98078528040323043f, 0.92387953251128674f, 0.83146961230254524f,
                                         0.70710678118654757f, 0.55557023301960229f, 0.38268343236508984f,
                                         0.19509032201612833f, 0.f, -0.19509032201612819f, -0.38268343236508973f,
                                         -0.55557023301960196f, -0.70710678118654746f, -0.83146961230254535f,
                                         -0.92387953251128674f, -0.98078528040323043f, -1.f};
__device__ constexpr float kSin32[17] = {0.f, 0.19509032201612825f, 0.38268343236508978f, 0.55557023301960218f,
                                         0.70710678118654746f, 0.83146961230254524f, 0.92387953251128674f,
                                         0.98078528040323043f, 1.f, 0.98078528040323043f, 0.92387953251128674f,
                                         0.83146961230254546f, 0.70710678118654757f, 0.55557023301960218f,
                                         0.38268343236508989f, 0.19509032201612861f, 0.f};

// DIT butterfly (a, b) -> (a + W b, a - W b), W = exp(-2 pi i E / 32), E in [0, 16), on packed FP32 pairs
// (f32x2.cuh).
template <int E>
__device__ __forceinline__ void bfly(float2& a, float2& b) {
  if constexpr (E == 0) {
    const float2 t = b;
    b = sub2(a, t);
    a = add2(a, t);
  } else if constexpr (E == 8) {  // W = -i : W b = (b.y, -b.x) = -i b
    const float2 t = b;
    b = add_i(a, t);
    a = sub_i(a, t);
  } else if constexpr (E == 4) {  // W = (1 - i)/sqrt2 : W b = c (b - i b)
    constexpr float c = 0.70710678118654752f;
    const float2 t = sub_i(b, b);  // (b.x + b.y, b.y - b.x)
    b = fmas2(-c, t, a);
    a = fmas2(c, t, a);
  } else if constexpr (E == 12) {  // W = (-1 - i)/sqrt2 : W b = -c (b + i b)
    constexpr float c = 0.70710678118654752f;
    const float2 u = add_i(b, b);  // (b.x - b.y, b.y + b.x)
    b = fmas2(c, u, a);
    a = fmas2(-c, u, a);
  } else {
    constexpr float wr = kCos32[E], wi = -kSin32[E];
    const float2 p = cfma2(wr, wi, b, a);               // a + W b
    b = fma2(make_float2(2.f, 2.f), a, make_float2(-p.x, -p.y));  // 2 a - p = a - W b
    a = p;
  }
}

// In-register LEN-point DFT on a[OFF .. OFF+LEN).  Input a[OFF + brev<log2 LEN>(j)] = x[j]; output
// a[OFF + k] = X[k] (natural order).
template <int LEN, int OFF, int S0 = 0, int S1 = 5>
__device__ __forceinline__ void fft_regs(float2 (&a)[32]) {
  constexpr int kStages = LEN == 32 ? 5 : (LEN == 16 ? 4 : 3);
  constexpr int kFirst = S0, kLast = S1 < kStages ? S1 : kStages;  // stages [kFirst, kLast)
  static_for<kLast - kFirst>([&](auto si) {
    constexpr int len = 2 << (decltype(si)::value + kFirst);  // 2, 4, ..., LEN
    constexpr int half = len / 2;
    static_for<LEN / 2>([&](auto bi) {
      constexpr int b = decltype(bi)::value;
      constexpr int i = (b / half) * len, j = b % half;
      bfly<j*(32 / len)>(a[OFF + i + j], a[OFF + i + j + half]);
    });
  });
}

struct Pow2Params {
  const float* wave;
  int64_t length, row_stride, frames, units_per_row, total_units;
  float* out;
  float* group_max;
  int64_t rows_per_group;
  const float* window;   // [n_fft] centre padded
  const float2* tw2d;    // [32][G]  W_nfft^(k2 * g) at [k2][g]
  const MelPlan* plan;
  const float4* frags;   // [steps][32] (b0_hi, b1_hi, b0_lo, b1_lo) in mma B-fragment order
  const WsHeader* hdr;
  int hop, pad, center, pad_mode, n_mels;
  int stage, log_mels, bulk_ok, stage_ok;
  // output row geometry: value m of frame t goes to out[(row * frames + t) * out_width + out_col0 + m]
  int out_width, out_col0, out_vec;  // out_vec: floats every row start is aligned to (1, 2 or 4)
  // Kaldi framing / per-frame conditioning (compliance/kaldi.py:44-83, :153-216); kaldi == 0: torch.stft framing
  int kaldi, k_off, k_win, k_dc, k_energy_mode, k_energy_col, k_log;
  int k_prelog;  // the gradient's recompute: the energy column receives E itself, not its floored log
  float k_preemph, k_energy_floor;
  float power, db_mult, db_amin, db_offset;
  // iSTFT adjoint (kIstftGrad): frames [env_t_lo, env_t_hi] have the full window envelope at every sample
  int64_t env_t_lo, env_t_hi;
};

// samples before t * hop where frame t starts: n_fft/2 (torch.stft center), 0, or Kaldi's win/2 - shift/2
__device__ __forceinline__ int frame_lead(const Pow2Params& p, int n_fft) {
  return p.kaldi ? p.k_off : (p.center ? n_fft / 2 : 0);
}

constexpr int kComplexOut = 3;  // POWER_MODE of the complex (power = None) Spectrogram kernel
constexpr int kSpectra = 4;     // POWER_MODE of the gradient kernel: transform_unit returns the two complex spectra
// POWER_MODE of the iSTFT adjoint (b200a_istft_backward): the COMPLEX Spectrogram kernel over the upstream gradient g,
// staged as g / env (env: the overlap-added squared window), with c_k / (N scale) in place of scale
constexpr int kIstftGrad = 5;

template <int POWER_MODE>  // 2: |.|^2, 0: general exponent (1 handled inside)
__device__ __forceinline__ float pow_of(float re, float im, float power) {
  if constexpr (POWER_MODE == 2) return fmaf(re, re, im * im);
  const float mag = hypotf(re, im);
  return power == 1.f ? mag : powf(mag, power);
}

// Running maximum of the dB features per top_db group, flushed with as few atomics as possible.
struct GroupMax {
  float* dst;
  int64_t group;
  float value;
  // Warp-collective (all 32 lanes call it together; `dst` is warp-uniform).
  __device__ __forceinline__ void flush() {
    if (dst == nullptr) return;
    const int64_t g0 = __shfl_sync(0xffffffffu, group, 0);
    if (__all_sync(0xffffffffu, group == g0)) {
      const float mx = warp_max(value);
      if ((threadIdx.x & 31) == 0 && g0 >= 0 && mx > -CUDART_INF_F) atomic_max_f32(dst + g0, mx);
    } else if (group >= 0 && value > -CUDART_INF_F) {
      atomic_max_f32(dst + group, value);
    }
    value = -CUDART_INF_F;
  }
  // Must be called by all 32 lanes together; `valid == false` lanes contribute nothing.
  __device__ __forceinline__ void add(int64_t g, float v, bool valid) {
    if (dst == nullptr) return;
    if (!valid) {
      g = group;
      v = -CUDART_INF_F;
    }
    // warp-collective flush only when ANY lane changes group (keeps the shuffles converged)
    if (__any_sync(0xffffffffu, g != group && group >= 0)) flush();
    group = g;
    value = fmaxf(value, v);
  }
};

template <int N>
__device__ __forceinline__ void reg_alloc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void reg_dealloc() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

// Per-warp walker over this warp's units: (row, unit-in-row) of the current and the next unit,
// advanced without divisions.
struct UnitCursor {
  int64_t u, stride, step_rows, step_units, upr;
  int64_t row, ub, nrow, nub;
  __device__ __forceinline__ void init(int64_t first, int64_t stride_, int64_t units_per_row) {
    u = first;
    stride = stride_;
    upr = units_per_row;
    step_rows = stride / upr;
    step_units = stride - step_rows * upr;
    row = first / upr;
    ub = first - row * upr;
    nrow = row + step_rows;
    nub = ub + step_units;
    if (nub >= upr) { nub -= upr; ++nrow; }
  }
  __device__ __forceinline__ void advance() {
    u += stride;
    row = nrow;
    ub = nub;
    nrow += step_rows;
    nub += step_units;
    if (nub >= upr) { nub -= upr; ++nrow; }
  }
};

// a unit can be staged by one bulk copy iff all its frames exist and lie inside the row un-padded (ADJ: and have the
// full window envelope, so that the staged samples need no division)
template <int G, bool ADJ = false>
__device__ __forceinline__ bool bulk_eligible(const Pow2Params& p, int half, int64_t u, int64_t ub) {
  using Ge = Geo<G>;
  if (!p.bulk_ok || u >= p.total_units) return false;
  const int64_t t0 = ub * Ge::kFrames;
  if constexpr (ADJ)
    if (t0 < p.env_t_lo || t0 + Ge::kFrames - 1 > p.env_t_hi) return false;
  const int64_t s0 = t0 * p.hop - half - p.pad;
  return t0 + Ge::kFrames <= p.frames && s0 >= 0 && s0 + (int64_t)(Ge::kFrames - 1) * p.hop + Ge::kNfft <= p.length;
}
template <int G>
__device__ __forceinline__ void issue_bulk(const Pow2Params& p, int half, int64_t row, int64_t ub, void* dst,
                                           uint64_t* bar) {
  using Ge = Geo<G>;
  const float* src = p.wave + row * p.row_stride + (ub * Ge::kFrames * p.hop - half - p.pad);
  const uint32_t bytes = (uint32_t)(Ge::kNfft + (Ge::kFrames - 1) * p.hop) * 4u;
  mbar_expect_tx(bar, bytes);
  bulk_g2s(dst, src, bytes, bar);
}

// The (32 G)-point complex FFT of one lane group, in place, as fft_pass1 then fft_pass2: lane l holds x[l + G j] in
// a[brev5(j)] and ends with X[(l + G q) + 32 k1] in a[q*G + k1].  Between the two calls the group's region is free:
// a forward kernel stages its next input into it there.
//
// fft_pass1: a 32-point DFT over j in registers, the twiddle W^(l * k2) from s_tw ([32][G]), and a transpose through
// the group's region, after which lane l owns k2 = l + G q.  SPLIT: transpose the real parts, then the imaginary parts,
// through kRegionF floats (half the shared memory of the float2 transpose, kRegion float2).  kTwAhead: how many
// twiddle loads are in flight; they are issued before the last butterfly stage, and every multiply issues the load
// kTwAhead positions ahead of it, so no multiply waits for its own load.  0 loads each twiddle at its multiply.
template <int G, bool SPLIT, int kTwAhead>
__device__ __forceinline__ void fft_pass1(float2 (&a)[32], const float2* s_tw, float* region, int l) {
  using Ge = Geo<G>;
  fft_regs<32, 0, 0, 4>(a);
  float2 tw[32];
  static_for<kTwAhead>([&](auto ki) {
    constexpr int k2 = decltype(ki)::value + 1;
    tw[k2] = s_tw[k2 * G + l];
  });
  fft_regs<32, 0, 4, 5>(a);  // a[k2] = Y[l][k2]
  // slot q*G + brev(g) <- element (g, l + G q)
  if constexpr (SPLIT) {
    region[l] = a[0].x;
    static_for<31>([&](auto ki) {
      constexpr int k2 = decltype(ki)::value + 1;
      if constexpr (k2 + kTwAhead < 32) tw[k2 + kTwAhead] = s_tw[(k2 + kTwAhead) * G + l];
      a[k2] = cmul2(a[k2], tw[k2]);
      region[k2 * Ge::kRowLd + l] = a[k2].x;
    });
    __syncwarp();
    float re[32];
    static_for<32>([&](auto si) {
      constexpr int s = decltype(si)::value;
      re[s] = region[(l + G * (s / G)) * Ge::kRowLd + s % G];
    });
    __syncwarp();
    static_for<32>([&](auto ki) {
      constexpr int k2 = decltype(ki)::value;
      region[k2 * Ge::kRowLd + l] = a[k2].y;
    });
    __syncwarp();
    static_for<32>([&](auto si) {
      constexpr int s = decltype(si)::value;
      constexpr int q = s / G, g = s % G;
      a[q * G + brev<Ge::kLogG>(g)] = make_float2(re[s], region[(l + G * q) * Ge::kRowLd + g]);
    });
  } else {
    float2* tile = reinterpret_cast<float2*>(region);
    tile[l] = a[0];
    static_for<31>([&](auto ki) {
      constexpr int k2 = decltype(ki)::value + 1;
      if constexpr (k2 + kTwAhead < 32) tw[k2 + kTwAhead] = s_tw[(k2 + kTwAhead) * G + l];
      tile[k2 * Ge::kRowLd + l] = cmul2(a[k2], tw[k2]);
    });
    __syncwarp();
    static_for<32>([&](auto si) {
      constexpr int s = decltype(si)::value;
      constexpr int q = s / G, g = s % G;
      a[q * G + brev<Ge::kLogG>(g)] = tile[(l + G * q) * Ge::kRowLd + g];
    });
  }
  __syncwarp();
}

// fft_pass2: 32/G G-point DFTs over the former lane index, in registers.
template <int G>
__device__ __forceinline__ void fft_pass2(float2 (&a)[32]) {
  static_for<Geo<G>::kGroups>([&](auto qi) { fft_regs<G, decltype(qi)::value * G>(a); });
}

// The frames an inverse transform rebuilt: a[(m % NG)*G + m/NG] = FFT(conj Z)[l + G m] = N (a[n] - i b[n]) with
// Z = A + i B.  Stores sample n = l + G m of frame a (Re) and frame b (-Im) times w_mul * s_win[n] from frame_a, frame
// a's row of the frame buffer offset by l; a frame marked bad gets NaN instead.
template <int G>
__device__ __forceinline__ void store_frame_pair(const float2 (&a)[32], float* frame_a, const float* s_win, float w_mul,
                                                 int l, bool has_a, bool has_b, bool bad_a, bool bad_b) {
  constexpr int N = Geo<G>::kNfft, NG = Geo<G>::kGroups;
  static_for<32>([&](auto mi) {
    constexpr int m = decltype(mi)::value;
    constexpr int slot = (m % NG) * G + m / NG;
    const float w = w_mul * s_win[l + G * m];
    if (has_a) frame_a[G * m] = bad_a ? CUDART_NAN_F : a[slot].x * w;
    if (has_b) frame_a[N + G * m] = bad_b ? CUDART_NAN_F : -a[slot].y * w;
  });
}

// The inter-pass twiddles [32][G] and the window times gain [32 G] into shared memory.
template <int G>
__device__ __forceinline__ void load_fft_tables(const float2* tw2d, const float* window, float gain, float2* s_tw,
                                                float* s_win) {
  for (int i = threadIdx.x; i < 32 * G; i += blockDim.x) {
    s_tw[i] = tw2d[i];
    s_win[i] = window[i] * gain;
  }
}

// One warp, one unit (32/G frame pairs): samples -> windowed complex signals -> n_fft-point FFTs -> the
// power spectra.  On return lane (group gi, l) holds bins k = l + G m in pa[m] / pb[m] (m < 16) of frames
// t0 + 2 gi and t0 + 2 gi + 1, and lanes with l == 0 bin n_fft/2 in [16].
// The staging buffer is the warp's transpose tile itself: the NEXT unit's bulk copy is issued only after
// fft_pass1 has read the tile back.  s_win: the window x 1/2 (un-packing) x the normalisation scale, [n_fft].
// SPLIT: the transpose of fft_pass1, through kRegionF floats per lane group.
// POWER_MODE == kSpectra: PT = float2, pa / pb receive the complex bins themselves (bin N/2 with a zero imaginary part).
template <int POWER_MODE, int G, int HG, bool KALDI, bool SPLIT, typename PT>
__device__ __forceinline__ void transform_unit(const Pow2Params& p, const float* s_win, const float2* s_tw,
                                               float2* tile, uint64_t* bar, uint32_t& parity, bool& staged,
                                               const UnitCursor& cur, int half, int lane, PT (&pa)[17],
                                               PT (&pb)[17]) {
  using Ge = Geo<G>;
  constexpr bool ADJ = POWER_MODE == kIstftGrad;
  float* stage = reinterpret_cast<float*>(tile);
  const int gi = lane / G, l = lane % G;
  const int64_t row = cur.row, t0 = cur.ub * Ge::kFrames;
  const int64_t ta = t0 + 2 * gi, tb = ta + 1;
  const bool has_a = ta < p.frames, has_b = tb < p.frames;
  const float* __restrict__ x = p.wave + row * p.row_stride;
  const int64_t s0 = t0 * p.hop - half - p.pad;  // first raw sample of the unit
  const int64_t sa = s0 + (int64_t)2 * gi * p.hop, sb = sa + p.hop;
  const bool next_staged = bulk_eligible<G, ADJ>(p, half, cur.u + cur.stride, cur.nub);
  // every frame of the unit inside the signal: plain loads; otherwise the padding-aware gather
  const int64_t last = p.frames - t0 < Ge::kFrames ? p.frames - t0 : Ge::kFrames;  // frames present
  const bool interior = s0 >= 0 && s0 + (last - 1) * p.hop + Ge::kNfft <= p.length;
  // ADJ: a unit that is gathered (a sample short of the full window envelope, or outside g) divides by env in the
  // gather and takes the plain window table; every other unit takes the table with 1/env folded in (s_win + n_fft)
  bool env_edge = false;
  if constexpr (ADJ) env_edge = t0 < p.env_t_lo || t0 + last - 1 > p.env_t_hi;
  const float* win = ADJ && interior && !env_edge ? s_win + Ge::kNfft : s_win;

  float2 a[32];
  float* grp_f = stage + gi * (SPLIT ? Ge::kRegionF : 2 * Ge::kRegion);  // the lane group's region as floats
  bool from_stage = staged;
  if (staged) {
    mbar_wait(bar, parity);
    parity ^= 1;
  } else if ((!interior || KALDI || env_edge) && p.stage_ok) {
    // edge unit (padding / reflection / ragged end): the lanes gather the unit's whole span into the (idle)
    // staging buffer with 4-byte asynchronous copies -- every sample once, all copies in flight together --
    // and the unit then takes the same register-load path as a bulk-staged one
    const int span = Ge::kNfft + (Ge::kFrames - 1) * p.hop;
    // 32-bit index arithmetic (the launch guarantees length + 2 pad + n_fft < 2^31): j indexes the constant
    // pre-padded signal of `ext` samples, exactly as source_index() does in 64 bits
    const int len = (int)p.length, ext = len + 2 * p.pad, j0 = (int)(t0 * p.hop) - half, mode = p.pad_mode;
    if constexpr (ADJ) {  // constant padding, half = 0: sample n of the span is output sample s = j0 + n of the iSTFT
#pragma unroll 4
      for (int n = lane; n < span; n += 32) {
        const int src = j0 + n - p.pad;
        float v = 0.f;
        if ((unsigned)src < (unsigned)len) {
          const float env = istft_envelope(p.window, Ge::kNfft, p.hop, p.frames, j0 + n);
          v = env > 0.f ? __fdividef(__ldg(x + src), env) : 0.f;  // no IEEE-division slow path: 2 ulp
        }
        stage[n] = v;
      }
    } else {
#pragma unroll 4
    for (int n = lane; n < span; n += 32) {
      int j = j0 + n;
      if ((unsigned)j >= (unsigned)ext) {
        if (mode == B200A_PAD_REFLECT)
          j = j < 0 ? -j : 2 * (ext - 1) - j;
        else if (mode == B200A_PAD_REPLICATE)
          j = j < 0 ? 0 : ext - 1;
        else if (mode == kPadSymmetric)
          j = j < 0 ? -1 - j : 2 * ext - 1 - j;
        else if (mode == B200A_PAD_CIRCULAR) {
          j %= ext;
          if (j < 0) j += ext;
        } else
          j = -1;
      }
      const int src = j - p.pad;
      if (j >= 0 && (unsigned)src < (unsigned)len)
        cp_async4(stage + n, x + src);
      else
        stage[n] = 0.f;
    }
    cp_async_wait_all();
    }
    __syncwarp();
    from_stage = true;
  }
  if (KALDI && from_stage) {
    // Kaldi conditioning of the two staged frames (sample n = l + G j, n < win): DC removal, [raw log energy],
    // pre-emphasis s[n] - c s[max(n - 1, 0)], window (zero beyond win), [log energy after the window]
    const float* fa = stage + 2 * gi * p.hop;
    const float* fb = fa + p.hop;
    const int win = p.k_win;
    // the gradient kernel (kSpectra) forms no energy: its adjoint runs in kaldi_cond_vjp_kernel
    const int energy_mode = POWER_MODE == kSpectra ? 0 : p.k_energy_mode;
    float ma = 0.f, mb = 0.f;
    if (p.k_dc) {
#pragma unroll 4
      for (int n = l; n < win; n += G) {
        ma += fa[n];
        mb += fb[n];
      }
#pragma unroll
      for (int o = G / 2; o > 0; o >>= 1) {
        ma += __shfl_xor_sync(0xffffffffu, ma, o);
        mb += __shfl_xor_sync(0xffffffffu, mb, o);
      }
      ma /= (float)win;
      mb /= (float)win;
    }
    float ea = 0.f, eb = 0.f;
    if (energy_mode == 1) {
#pragma unroll 4
      for (int n = l; n < win; n += G) {
        const float da = fa[n] - ma, db = fb[n] - mb;
        ea = fmaf(da, da, ea);
        eb = fmaf(db, db, eb);
      }
    }
    const float c = p.k_preemph;
    static_for<32>([&](auto ji) {
      constexpr int j = decltype(ji)::value;
      const int n = l + G * j;
      float va = 0.f, vb = 0.f;
      if (n < win) {
        const int np = n > 0 ? n - 1 : 0;
        const float w = s_win[n];
        va = ((fa[n] - ma) - c * (fa[np] - ma)) * w;
        vb = ((fb[n] - mb) - c * (fb[np] - mb)) * w;
      }
      a[brev5(j)] = make_float2(va, vb);
      if (energy_mode == 2) {  // s_win carries the un-packing's 1/2
        ea = fmaf(2.f * va, 2.f * va, ea);
        eb = fmaf(2.f * vb, 2.f * vb, eb);
      }
    });
    if (energy_mode != 0) {
#pragma unroll
      for (int o = G / 2; o > 0; o >>= 1) {
        ea += __shfl_xor_sync(0xffffffffu, ea, o);
        eb += __shfl_xor_sync(0xffffffffu, eb, o);
      }
      if (l == 0) {
        const float fl = p.k_energy_floor > 0.f ? logf(p.k_energy_floor) : -CUDART_INF_F;
        float* e_out = p.out + (row * p.frames + ta) * p.out_width + p.k_energy_col;
        if (has_a) e_out[0] = p.k_prelog ? ea : fmaxf(logf(fmaxf(ea, kKaldiEps)), fl);
        if (has_b) e_out[p.out_width] = p.k_prelog ? eb : fmaxf(logf(fmaxf(eb, kKaldiEps)), fl);
      }
    }
    __syncwarp();  // every lane has consumed the staging buffer
  } else if (from_stage) {
    if constexpr (HG >= 0) {  // G == 32: frame b is frame a shifted by HG lane-rows
      constexpr int kV = 32 + (HG >= 0 ? HG : 0);
      float v[kV];
      static_for<kV>([&](auto ji) {
        constexpr int j = decltype(ji)::value;
        v[j] = stage[lane + 32 * j];
      });
      static_for<32>([&](auto ji) {
        constexpr int j = decltype(ji)::value;
        const float w = win[lane + 32 * j];
        a[brev5(j)] = make_float2(v[j] * w, v[j + (HG >= 0 ? HG : 0)] * w);
      });
    } else {
      const float* pa_ptr = stage + 2 * gi * p.hop + l;
      const float* pb_ptr = pa_ptr + p.hop;
      static_for<32>([&](auto ji) {
        constexpr int j = decltype(ji)::value;
        a[brev5(j)] = scale2(win[l + G * j], make_float2(pa_ptr[G * j], pb_ptr[G * j]));
      });
    }
    __syncwarp();  // every lane has consumed the staging buffer
  } else if (interior) {
    static_for<32>([&](auto ji) {
      constexpr int j = decltype(ji)::value;
      const float va = has_a ? __ldg(x + sa + l + G * j) : 0.f;
      const float vb = has_b ? __ldg(x + sb + l + G * j) : 0.f;
      a[brev5(j)] = scale2(win[l + G * j], make_float2(va, vb));
    });
  } else if constexpr (!ADJ) {  // (the adjoint launches only with stage_ok)
    // edge unit whose span does not fit the staging buffer: gather frame a, then frame b, through the group's region
    // (n_fft floats) with a rolled loop so the index arithmetic is not replicated 64 times in the instruction stream
#pragma unroll
    for (int f = 0; f < 2; ++f) {
      const int64_t t = ta + f;
#pragma unroll 1
      for (int j = 0; j < 32; ++j) {
        const int n = l + G * j;
        const int64_t i = t < p.frames ? source_index(t * p.hop + n, p.length, p.pad, half, p.pad_mode) : -1;
        grp_f[n] = i >= 0 ? __ldg(x + i) : 0.f;
      }
      __syncwarp();
      static_for<32>([&](auto ji) {
        constexpr int j = decltype(ji)::value;
        const float v = __fmul_rn(s_win[l + G * j], grp_f[l + G * j]);  // the product scale2 forms
        if (f == 0) a[brev5(j)].x = v;
        else a[brev5(j)].y = v;
      });
      __syncwarp();
    }
  }

  // the float2 transpose's region is grp_f, addressed from the tile: through grp_f, ptxas spills 8 B instead of 4 B in
  // the n_fft = 1024 general-power Spectrogram kernel
  fft_pass1<G, SPLIT, 8>(a, s_tw, SPLIT ? grp_f : reinterpret_cast<float*>(tile + gi * Ge::kRegion), l);
  staged = next_staged;  // the tile is free until the next unit's transpose: stage into it
  if (staged && lane == 0) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic reads above -> async write
    issue_bulk<G>(p, half, cur.nrow, cur.nub, stage, bar);
  }
  fft_pass2<G>(a);
  // a[q*G + k1] = Z[(l + G q) + 32 k1]; bin k = l + G m with m = q + (32/G) k1  <->  slot (m % NG)*G + m / NG

  // ---- un-pack the two spectra: need Z[N - k] for k = l + G m, m = 0..15 (+ bin N/2 on l == 0) ----
  constexpr int NG = Ge::kGroups;
  const int src = (lane & ~(G - 1)) | ((G - l) & (G - 1));
  static_for<16>([&](auto mi) {
    constexpr int m = decltype(mi)::value;
    constexpr int slot = (m % NG) * G + m / NG;
    // l >= 1: N - k = (G - l) + G (31 - m): on lane `src`, slot of m' = 31 - m
    constexpr int mm = 31 - m, mslot = (mm % NG) * G + mm / NG;
    float mr = __shfl_sync(0xffffffffu, a[mslot].x, src);
    float mi_ = __shfl_sync(0xffffffffu, a[mslot].y, src);
    if (l == 0) {  // l == 0: N - k = G (32 - m): own slot of m' = 32 - m (slot 0 for m = 0)
      constexpr int m0 = (32 - m) & 31, slot0 = (m0 % NG) * G + m0 / NG;
      mr = a[slot0].x;
      mi_ = a[slot0].y;
    }
    // A = Z[k] + conj Z[N-k] = (sx.x, sy.x),  B = (Z[k] - conj Z[N-k]) / i = (sy.y, -sx.y): two packed adds
    const float zr = a[slot].x, zi = a[slot].y;
    const float2 sx = add2(make_float2(zr, zr), make_float2(mr, -mr));    // (zr + mr, zr - mr)
    const float2 sy = add2(make_float2(zi, zi), make_float2(-mi_, mi_));  // (zi - mi, zi + mi)
    if constexpr (POWER_MODE == kComplexOut) {  // power = None: the two spectra go straight to out[row][t][bin] (complex64)
      float2* oc = reinterpret_cast<float2*>(p.out) + (row * p.frames + ta) * Ge::kBins + l + G * m;
      if (has_a) oc[0] = make_float2(sx.x, sy.x);
      if (has_b) oc[Ge::kBins] = make_float2(sy.y, -sx.y);
    } else if constexpr (ADJ) {  // c_k = 2 at bins 1 .. N/2 - 1 (the window table carries the 1/2 of c_0 = 1)
      const float c = m == 0 && l == 0 ? 1.f : 2.f;
      float2* oc = reinterpret_cast<float2*>(p.out) + (row * p.frames + ta) * Ge::kBins + l + G * m;
      if (has_a) oc[0] = make_float2(c * sx.x, c * sy.x);
      if (has_b) oc[Ge::kBins] = make_float2(c * sy.y, -c * sx.y);
    } else if constexpr (POWER_MODE == kSpectra) {
      pa[m] = make_float2(sx.x, sy.x);
      pb[m] = make_float2(sy.y, -sx.y);
    } else if constexpr (POWER_MODE == 2) {  // (|A|^2, |B|^2) as one packed multiply + one packed FMA
      const float2 pw = fma2(sx, sx, mul2(sy, sy));
      pa[m] = pw.x;
      pb[m] = pw.y;
    } else {
      pa[m] = pow_of<POWER_MODE>(sx.x, sy.x, p.power);
      pb[m] = pow_of<POWER_MODE>(sy.y, sx.y, p.power);
    }
  });
  // bin N/2 (l == 0, m = 16) is its own mirror: A = Re, B = Im  (x2 because wreg carries the 1/2)
  constexpr int slot16 = (16 % NG) * G + 16 / NG;
  if constexpr (POWER_MODE == kComplexOut || ADJ) {  // ADJ: c_{N/2} = 1
    if (l == 0) {
      float2* oc = reinterpret_cast<float2*>(p.out) + (row * p.frames + ta) * Ge::kBins + Ge::kNfft / 2;
      if (has_a) oc[0] = make_float2(2.f * a[slot16].x, 0.f);
      if (has_b) oc[Ge::kBins] = make_float2(2.f * a[slot16].y, 0.f);
    }
  } else if constexpr (POWER_MODE == kSpectra) {
    pa[16] = make_float2(2.f * a[slot16].x, 0.f);
    pb[16] = make_float2(2.f * a[slot16].y, 0.f);
  } else {
    pa[16] = pow_of<POWER_MODE>(2.f * a[slot16].x, 0.f, p.power);
    pb[16] = pow_of<POWER_MODE>(2.f * a[slot16].y, 0.f, p.power);
  }
}

// ------------------------------------------------------------------------------------------------
// Spectrogram kernel: NW independent warps, power spectra straight to global memory.
// ------------------------------------------------------------------------------------------------
template <int POWER_MODE, int G, int HG, int NW, bool KALDI>
__global__ void __launch_bounds__(NW * 32, 1) stft_pow2_power_kernel(const Pow2Params p) {
  using Ge = Geo<G>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float2* s_tw = reinterpret_cast<float2*>(smem_raw);                                    // [32][G]
  constexpr bool ADJ = POWER_MODE == kIstftGrad;
  float* s_win = reinterpret_cast<float*>(s_tw + 32 * 32);                               // [n_fft] (ADJ: [2][n_fft])
  float2* s_tile_all = reinterpret_cast<float2*>(s_win + (ADJ ? 2 : 1) * Ge::kNfft);     // [NW][kTileF2] (also staging)
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(s_tile_all + NW * Ge::kTileF2);          // [NW]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // the tables of load_fft_tables, written out: through the helper the n_fft = 1024 general-power variant spills more
  for (int i = tid; i < 32 * G; i += blockDim.x) s_tw[i] = p.tw2d[i];
  if constexpr (ADJ) {
    // the window x 1/2 / (N scale), and the same over the full envelope at sample i (period hop), 0 where that is 0
    const float hs = 0.5f / ((float)Ge::kNfft * p.hdr->scale);
    for (int i = tid; i < Ge::kNfft; i += blockDim.x) {
      const float w = p.window[i] * hs;
      const int r = i % p.hop;
      const float env = istft_envelope(p.window, Ge::kNfft, p.hop, p.frames, r + (Ge::kNfft - 1 - r) / p.hop * p.hop);
      s_win[i] = w;
      s_win[Ge::kNfft + i] = env > 0.f ? __fdividef(w, env) : 0.f;
    }
  } else {
    const float hs = 0.5f * p.hdr->scale;  // the window x 1/2 (un-packing) x scale
    for (int i = tid; i < Ge::kNfft; i += blockDim.x) s_win[i] = p.window[i] * hs;
  }
  if (tid < NW) mbar_init(s_bar + tid, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();

  float2* tile = s_tile_all + warp * Ge::kTileF2;
  float* stage = reinterpret_cast<float*>(tile);
  uint64_t* bar = s_bar + warp;
  const int half = frame_lead(p, Ge::kNfft);
  const int gi = lane / G, l = lane % G;
  uint32_t parity = 0;
  bool staged = false;
  UnitCursor cur;
  cur.init((int64_t)blockIdx.x * NW + warp, (int64_t)gridDim.x * NW, p.units_per_row);
  if (bulk_eligible<G, ADJ>(p, half, cur.u, cur.ub)) {
    if (lane == 0) issue_bulk<G>(p, half, cur.row, cur.ub, stage, bar);
    staged = true;
  }
  for (; cur.u < p.total_units; cur.advance()) {
    float pa[17], pb[17];
    transform_unit<POWER_MODE, G, HG, KALDI, false>(p, s_win, s_tw, tile, bar, parity, staged, cur, half, lane, pa, pb);
    if constexpr (POWER_MODE == kComplexOut || ADJ) continue;  // transform_unit has written the complex spectra
    const int64_t ta = cur.ub * Ge::kFrames + 2 * gi;
    const bool has_a = ta < p.frames, has_b = ta + 1 < p.frames;
    float* oa = p.out + (cur.row * p.frames + ta) * p.out_width + p.out_col0;
    float* ob = oa + p.out_width;
    if (KALDI && p.k_log) {  // Kaldi spectrogram: log(max(|X|^2, eps)), kaldi.py:310
#pragma unroll
      for (int m = 0; m < 17; ++m) {
        pa[m] = logf(fmaxf(pa[m], kKaldiEps));
        pb[m] = logf(fmaxf(pb[m], kKaldiEps));
      }
    }
    const int skip = KALDI ? p.k_energy_col - p.out_col0 : -1;  // the bin whose column holds the frame's log energy
#pragma unroll
    for (int m = 0; m < 16; ++m) {
      if (l + G * m == skip) continue;
      if (has_a) oa[l + G * m] = pa[m];
      if (has_b) ob[l + G * m] = pb[m];
    }
    if (l == 0 && Ge::kNfft / 2 != skip) {
      if (has_a) oa[Ge::kNfft / 2] = pa[16];
      if (has_b) ob[Ge::kNfft / 2] = pb[16];
    }
  }
}

// One filter group of a 16-frame power tile: D[16 x 8] = P[16 x bins] * F[bins x 8] on the tensor pipe, (dB / log),
// store.  pw: the tile's 16 power rows (pitch PITCH); o_lo / o_hi, g_lo / g_hi: output offset (or -1) and top_db
// group of rows r and r + 8 (r = lane / 4).
template <int PITCH>
__device__ __forceinline__ void contract_item(const Pow2Params& p, const BandTile& mi, const float4* s_frags,
                                              bool frags_in_smem, int lane, const float* pw, int64_t o_lo,
                                              int64_t o_hi, int64_t g_lo, int64_t g_hi, GroupMax& gmax) {
  const int r = lane >> 2, c = lane & 3;
  const float* a_lo_row = pw + (size_t)r * PITCH + mi.kstart + c;
  const float* a_hi_row = a_lo_row + 8 * PITCH;
  float acc[1][3][4];
  band_contract<1, 4>(mi, s_frags, p.frags, frags_in_smem, lane, {a_lo_row, a_hi_row}, acc);
  float d[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) d[q] = band_sum(acc[0], q);
  const int n0 = 8 * mi.group + 2 * c;
  const bool n0_ok = n0 < p.n_mels, n1_ok = n0 + 1 < p.n_mels;
  if (p.k_log) {  // Kaldi fbank: log(max(mel, FLT_EPSILON)), kaldi.py:629-631
#pragma unroll
    for (int q = 0; q < 4; ++q) d[q] = logf(fmaxf(d[q], kKaldiEps));
  }
  if (p.stage == B200A_STAGE_FEAT) {
#pragma unroll
    for (int q = 0; q < 4; ++q)
      d[q] = p.log_mels ? logf(d[q] + 1e-6f) : p.db_mult * log10f(fmaxf(d[q], p.db_amin)) - p.db_offset;
    const float m_lo = fmaxf(n0_ok ? d[0] : -CUDART_INF_F, n1_ok ? d[1] : -CUDART_INF_F);
    const float m_hi = fmaxf(n0_ok ? d[2] : -CUDART_INF_F, n1_ok ? d[3] : -CUDART_INF_F);
    gmax.add(g_lo, m_lo, o_lo >= 0);
    gmax.add(g_hi, m_hi, o_hi >= 0);
  }
  const bool vec = n1_ok && p.out_vec >= 2;  // 8-byte aligned pair
  if (o_lo >= 0) {
    if (vec) *reinterpret_cast<float2*>(p.out + o_lo + n0) = make_float2(d[0], d[1]);
    else {
      if (n0_ok) p.out[o_lo + n0] = d[0];
      if (n1_ok) p.out[o_lo + n0 + 1] = d[1];
    }
  }
  if (o_hi >= 0) {
    if (vec) *reinterpret_cast<float2*>(p.out + o_hi + n0) = make_float2(d[2], d[3]);
    else {
      if (n0_ok) p.out[o_hi + n0] = d[2];
      if (n1_ok) p.out[o_hi + n0 + 1] = d[3];
    }
  }
}

// The n_fft = 2048 contraction warp mw's share of a 16-frame power tile: its filter groups, one after the other.
template <int PITCH>
__device__ __forceinline__ void contract_tile(const Pow2Params& p, const MelPlan* s_plan, const float4* s_frags,
                                              bool frags_in_smem, int mw, int lane, const float* pw,
                                              const int64_t* slot, const int64_t* grp, GroupMax& gmax) {
  const int r = lane >> 2;
  const int cnt = s_plan->warp_cnt[mw];
  const int64_t o_lo = slot[r], o_hi = slot[r + 8];
  const int64_t g_lo = grp[r], g_hi = grp[r + 8];
  for (int ii = 0; ii < cnt; ++ii)
    contract_item<PITCH>(p, s_plan->items[s_plan->warp_items[mw][ii]], s_frags, frags_in_smem, lane, pw, o_lo, o_hi,
                         g_lo, g_hi, gmax);
}

// The mel kernels' tables: copies the MelPlan into shared memory, stages the filterbank fragments when the plan has at
// most max_steps k-steps (returns whether it did), and zeroes columns [bins, pitch) of the `slots` power rows, which the
// last k-step reads.
__device__ __forceinline__ bool load_mel_plan(const Pow2Params& p, MelPlan* s_plan, float4* s_frags, int max_steps,
                                              float* s_pow, int slots, int pitch, int bins) {
  const int tid = threadIdx.x;
  const int* src = reinterpret_cast<const int*>(p.plan);
  int* dst = reinterpret_cast<int*>(s_plan);
  for (int i = tid; i < (int)(sizeof(MelPlan) / sizeof(int)); i += blockDim.x) dst[i] = src[i];
  const bool frags_in_smem = stage_band_frags(p.frags, p.plan->total_steps, max_steps, s_frags);
  for (int i = tid; i < slots * (pitch - bins); i += blockDim.x) {
    const int r = i / (pitch - bins), c = i - r * (pitch - bins);
    s_pow[r * pitch + bins + c] = 0.f;
  }
  return frags_in_smem;
}

// ------------------------------------------------------------------------------------------------
// Mel / MFCC-feature kernel (n_fft = 256 / 512 / 1024): 16 uniform warps.  Every iteration each warp transforms
// one unit, waits at a CTA barrier until the previous contraction has read the (single) power tile, publishes
// its power rows, waits at a second barrier and then contracts its share of the tile's (16-frame MMA tile,
// filter group) items on the tensor pipe and stores the features.  The transform is latency bound, so the warps
// are not specialised: all 16 run the FFT at 128 registers, which is what hides its stalls.
// ------------------------------------------------------------------------------------------------
constexpr int kFftRegs = 200, kMelRegs = 96;  // n_fft = 2048: 256*200 + 128*96 = 63488 <= 64512 = 384 * 168

// shared memory of the 16-warp mel kernel, in the order of the carve-up in mel_body
template <int G>
constexpr size_t mel_smem_bytes() {
  using Ge = Geo<G>;
  return sizeof(float2) * 32 * G + sizeof(float) * Ge::kNfft + sizeof(float) * kUniWarps * Ge::kMelRegion +
         sizeof(float) * Ge::kSlots * Ge::kPitch + sizeof(int64_t) * 2 * Ge::kSlots + sizeof(uint64_t) * kUniWarps +
         sizeof(MelPlan) + sizeof(float4) * 32 * Ge::kMelFragSteps;
}

template <int POWER_MODE, int G, int HG, bool KALDI>
__device__ __forceinline__ void mel_body(const Pow2Params& p, unsigned char* smem_raw) {
  using Ge = Geo<G>;
  constexpr int kSlots = Ge::kSlots, kPitch = Ge::kPitch;
  float2* s_tw = reinterpret_cast<float2*>(smem_raw);                              // [32][G]
  float* s_win = reinterpret_cast<float*>(s_tw + 32 * G);                          // [n_fft]
  float* s_region_all = s_win + Ge::kNfft;                                         // [kUniWarps][kMelRegion]
  float* s_pow = s_region_all + kUniWarps * Ge::kMelRegion;                        // [kSlots][kPitch]
  int64_t* s_slot = reinterpret_cast<int64_t*>(s_pow + kSlots * kPitch);           // [kSlots] out offsets
  int64_t* s_grp = s_slot + kSlots;                                                // [kSlots] top_db group
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(s_grp + kSlots);                   // [kUniWarps] staging
  MelPlan* s_plan = reinterpret_cast<MelPlan*>(s_bar + kUniWarps);
  float4* s_frags = reinterpret_cast<float4*>(s_plan + 1);                         // [<= kMelFragSteps][32]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  load_fft_tables<G>(p.tw2d, p.window, 0.5f * p.hdr->scale, s_tw, s_win);  // the window x 1/2 (un-packing) x scale
  const bool frags_in_smem = load_mel_plan(p, s_plan, s_frags, Ge::kMelFragSteps, s_pow, kSlots, kPitch, Ge::kBins);
  if (tid < kUniWarps) mbar_init(s_bar + tid, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();

  const int64_t stride = (int64_t)gridDim.x * kUniWarps;
  const int64_t u0 = (int64_t)blockIdx.x * kUniWarps;
  const int width = p.out_width;
  float2* tile = reinterpret_cast<float2*>(s_region_all + warp * Ge::kMelRegion);
  float* stage = reinterpret_cast<float*>(tile);
  uint64_t* bar = s_bar + warp;
  const int half = frame_lead(p, Ge::kNfft);
  const int gi = lane / G, l = lane % G;
  const int work_begin = s_plan->work_begin[warp], work_end = s_plan->work_begin[warp + 1];
  GroupMax gmax{p.stage == B200A_STAGE_FEAT ? p.group_max : nullptr, -1, -CUDART_INF_F};
  uint32_t parity = 0;
  bool staged = false;
  UnitCursor cur;
  cur.init(u0 + warp, stride, p.units_per_row);
  if (bulk_eligible<G>(p, half, cur.u, cur.ub)) {
    if (lane == 0) issue_bulk<G>(p, half, cur.row, cur.ub, stage, bar);
    staged = true;
  }
  for (int64_t base = u0; base < p.total_units; base += stride, cur.advance()) {
    const bool valid = cur.u < p.total_units;
    float pa[17], pb[17];
    if (valid)
      transform_unit<POWER_MODE, G, HG, KALDI, true>(p, s_win, s_tw, tile, bar, parity, staged, cur, half, lane, pa, pb);
    __syncthreads();  // the previous iteration's contraction has read the power tile and the slot table
    const int slot_a = Ge::kFrames * warp + 2 * gi;
    float* prow_a = s_pow + (size_t)slot_a * kPitch;
    float* prow_b = prow_a + kPitch;
    if (valid) {
#pragma unroll
      for (int m = 0; m < 16; ++m) {
        prow_a[l + G * m] = pa[m];
        prow_b[l + G * m] = pb[m];
      }
      if (l == 0) {
        prow_a[Ge::kNfft / 2] = pa[16];
        prow_b[Ge::kNfft / 2] = pb[16];
      }
    }
    if (l == 0) {
      const int64_t ta = cur.ub * Ge::kFrames + 2 * gi;
      const int64_t oa = (cur.row * p.frames + ta) * (int64_t)width + p.out_col0;
      s_slot[slot_a] = (valid && ta < p.frames) ? oa : -1;
      s_slot[slot_a + 1] = (valid && ta + 1 < p.frames) ? oa + width : -1;
      const int64_t g = cur.row / p.rows_per_group;
      s_grp[slot_a] = g;
      s_grp[slot_a + 1] = g;
    }
    __syncthreads();  // every power row of this iteration is in place
#pragma unroll 1
    for (int i = work_begin; i < work_end; ++i) {
      const int w = s_plan->work[i], mt = w >> 8;
      const int64_t* slot = s_slot + 16 * mt;
      const int64_t* grp = s_grp + 16 * mt;
      const int r = lane >> 2;
      contract_item<kPitch>(p, s_plan->items[w & 255], s_frags, frags_in_smem, lane, s_pow + (size_t)16 * mt * kPitch,
                            slot[r], slot[r + 8], grp[r], grp[r + 8], gmax);
    }
  }
  gmax.flush();
}

// ================================================================================================
// n_fft = 2048: one real frame per 1024-point complex FFT ("even/odd packing").
//   z[m] = w[2m] x[2m] + i w[2m+1] x[2m+1],  Z = FFT_1024(z);  with E = (Z[k] + conj Z[1024-k]) / 2 and
//   O = (Z[k] - conj Z[1024-k]) / 2i:   X[k] = E + W_2048^k O,   X[1024-k] = conj(E - W_2048^k O),
// so each lane turns its 16 (Z[k], Z[1024-k]) pairs into 32 power bins.  The same 32 x 32 register FFT,
// tile transposes, bulk staging and tensor-pipe contraction as above; a warp handles 2 frames per iteration
// one after the other, and the (16 x 1025) power tile is single buffered.
// ================================================================================================
constexpr int kEoN = 2048, kEoBins = 1025, kEoPitch = 1060, kEoSlots = 16;
constexpr int kEoFragSteps = 136;  // fragments kept in shared memory when the plan has at most this many steps

__device__ __forceinline__ bool eo_frame_bulk_ok(const Pow2Params& p, int half, int64_t t) {
  const int64_t sa = t * p.hop - half - p.pad;
  return p.bulk_ok && t < p.frames && sa >= 0 && sa + kEoN <= p.length;
}

// One warp, one frame of 2048 samples.  On return lane l holds bins l + 32 k1 in plo[k1], bins
// 1024 - l - 32 k1 in phi[k1] (k1 < 16), and lane 0 bin 512 in pmid.
template <int POWER_MODE>
__device__ __forceinline__ void transform_frame_eo(const Pow2Params& p, const float2* s_win, const float2* s_tw,
                                                   const float2* s_tw2, float2* tile, uint64_t* bar, uint32_t& parity,
                                                   bool& staged, int64_t row, int64_t t, bool next_ok, int64_t next_row,
                                                   int64_t next_t, int half, int lane, float (&plo)[16],
                                                   float (&phi)[16], float& pmid) {
  const float* __restrict__ x = p.wave + row * p.row_stride;
  const int64_t sa = t * p.hop - half - p.pad;
  float* stage = reinterpret_cast<float*>(tile);
  float2 a[32];
  if (staged) {
    mbar_wait(bar, parity);
    parity ^= 1;
    const float2* st2 = reinterpret_cast<const float2*>(stage);
    static_for<32>([&](auto ji) {
      constexpr int j = decltype(ji)::value;
      const float2 v = st2[lane + 32 * j], w = s_win[lane + 32 * j];
      a[brev5(j)] = make_float2(v.x * w.x, v.y * w.y);
    });
    __syncwarp();
  } else if (sa >= 0 && sa + kEoN <= p.length) {
    static_for<32>([&](auto ji) {
      constexpr int j = decltype(ji)::value;
      const float2 w = s_win[lane + 32 * j];
      const float ve = __ldg(x + sa + 2 * (lane + 32 * j)), vo = __ldg(x + sa + 2 * (lane + 32 * j) + 1);
      a[brev5(j)] = make_float2(ve * w.x, vo * w.y);
    });
  } else {
#pragma unroll 1
    for (int j = 0; j < 32; ++j) {
      const int m = lane + 32 * j;
      const int64_t ie = source_index(t * p.hop + 2 * m, p.length, p.pad, half, p.pad_mode);
      const int64_t io = source_index(t * p.hop + 2 * m + 1, p.length, p.pad, half, p.pad_mode);
      tile[m] = make_float2(ie >= 0 ? __ldg(x + ie) : 0.f, io >= 0 ? __ldg(x + io) : 0.f);
    }
    __syncwarp();
    static_for<32>([&](auto ji) {
      constexpr int j = decltype(ji)::value;
      const float2 v = tile[lane + 32 * j], w = s_win[lane + 32 * j];
      a[brev5(j)] = make_float2(v.x * w.x, v.y * w.y);
    });
    __syncwarp();
  }

  fft_pass1<32, false, 0>(a, s_tw, stage, lane);
  staged = next_ok && eo_frame_bulk_ok(p, half, next_t);
  if (staged && lane == 0) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    const float* src = p.wave + next_row * p.row_stride + (next_t * p.hop - half - p.pad);
    mbar_expect_tx(bar, kEoN * 4u);
    bulk_g2s(stage, src, kEoN * 4u, bar);
  }
  fft_pass2<32>(a);  // a[k1] = Z[lane + 32 k1]

  const int src_lane = (32 - lane) & 31;
  static_for<16>([&](auto ki) {
    constexpr int k1 = decltype(ki)::value;
    float mr = __shfl_sync(0xffffffffu, a[31 - k1].x, src_lane);
    float mi = __shfl_sync(0xffffffffu, a[31 - k1].y, src_lane);
    if (lane == 0) {
      mr = a[(32 - k1) & 31].x;
      mi = a[(32 - k1) & 31].y;
    }
    const float zr = a[k1].x, zi = a[k1].y;
    const float er = zr + mr, ei = zi - mi;   // E (x 2, the 1/2 rides on the window)
    const float orr = zi + mi, oi = mr - zr;  // O
    const float2 w = s_tw2[k1 * 32 + lane];   // W_2048^(lane + 32 k1)
    const float tr = fmaf(orr, w.x, -oi * w.y), ti = fmaf(orr, w.y, oi * w.x);
    plo[k1] = pow_of<POWER_MODE>(er + tr, ei + ti, p.power);
    phi[k1] = pow_of<POWER_MODE>(er - tr, ei - ti, p.power);
  });
  // bin 512 = lane 0, slot 16: E = 2 Re Z, O = 2 Im Z, W^512 = -i  ->  X = E - i O
  pmid = pow_of<POWER_MODE>(2.f * a[16].x, -2.f * a[16].y, p.power);
}

__device__ __forceinline__ void eo_store_row(float* row, int lane, const float (&plo)[16], const float (&phi)[16],
                                             float pmid) {
#pragma unroll
  for (int k1 = 0; k1 < 16; ++k1) {
    row[lane + 32 * k1] = plo[k1];
    row[1024 - lane - 32 * k1] = phi[k1];
  }
  if (lane == 0) row[512] = pmid;
}

__device__ __forceinline__ void eo_load_tables(const Pow2Params& p, const float2* tw_eo, float2* s_win, float2* s_tw,
                                               float2* s_tw2, int tid, int nthreads) {
  const float hs = 0.5f * p.hdr->scale;
  for (int i = tid; i < 1024; i += nthreads) {
    s_tw[i] = p.tw2d[i];
    s_win[i] = make_float2(p.window[2 * i] * hs, p.window[2 * i + 1] * hs);
  }
  for (int i = tid; i < 17 * 32; i += nthreads) s_tw2[i] = tw_eo[i];
}

struct EoNext {  // the frame that follows (row, t) in this warp's walk
  bool ok;
  int64_t row, t;
};
__device__ __forceinline__ EoNext eo_next_frame(const Pow2Params& p, const UnitCursor& cur, int f) {
  if (f == 0) return EoNext{true, cur.row, 2 * cur.ub + 1};
  return EoNext{cur.u + cur.stride < p.total_units, cur.nrow, 2 * cur.nub};
}

template <int POWER_MODE>
__global__ void __launch_bounds__(kWarps * 32, 1) stft2048_power_kernel(const Pow2Params p, const float2* tw_eo) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float2* s_tw = reinterpret_cast<float2*>(smem_raw);   // [32][32]
  float2* s_win = s_tw + 1024;                          // [1024] (w[2m], w[2m+1]) x scale
  float2* s_tw2 = s_win + 1024;                         // [17][32] W_2048^(l + 32 k1)
  float2* s_tile_all = s_tw2 + 17 * 32;                 // [kWarps][32 * 33]
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(s_tile_all + kWarps * 32 * 33);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  eo_load_tables(p, tw_eo, s_win, s_tw, s_tw2, tid, blockDim.x);
  if (tid < kWarps) mbar_init(s_bar + tid, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  float2* tile = s_tile_all + warp * 32 * 33;
  uint64_t* bar = s_bar + warp;
  const int half = p.center ? kEoN / 2 : 0;
  uint32_t parity = 0;
  bool staged = false;
  UnitCursor cur;
  cur.init((int64_t)blockIdx.x * kWarps + warp, (int64_t)gridDim.x * kWarps, p.units_per_row);
  if (cur.u < p.total_units && eo_frame_bulk_ok(p, half, 2 * cur.ub)) {
    if (lane == 0) {
      mbar_expect_tx(bar, kEoN * 4u);
      bulk_g2s(tile, p.wave + cur.row * p.row_stride + (2 * cur.ub * p.hop - half - p.pad), kEoN * 4u, bar);
    }
    staged = true;
  }
  for (; cur.u < p.total_units; cur.advance()) {
#pragma unroll 1
    for (int f = 0; f < 2; ++f) {
      const int64_t t = 2 * cur.ub + f;
      if (t >= p.frames) { staged = false; break; }  // (never staged: eo_frame_bulk_ok checks t < frames)
      const EoNext nx = eo_next_frame(p, cur, f);
      float plo[16], phi[16], pmid;
      transform_frame_eo<POWER_MODE>(p, s_win, s_tw, s_tw2, tile, bar, parity, staged, cur.row, t, nx.ok, nx.row, nx.t,
                                     half, lane, plo, phi, pmid);
      eo_store_row(p.out + (cur.row * p.frames + t) * kEoBins, lane, plo, phi, pmid);
    }
  }
}

template <int POWER_MODE>
__global__ void __launch_bounds__((kWarps + kMelWarps) * 32, 1) stft2048_mel_kernel(const Pow2Params p,
                                                                                     const float2* tw_eo) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float2* s_tw = reinterpret_cast<float2*>(smem_raw);
  float2* s_win = s_tw + 1024;
  float2* s_tw2 = s_win + 1024;
  float2* s_tile_all = s_tw2 + 17 * 32;
  float* s_pow = reinterpret_cast<float*>(s_tile_all + kWarps * 32 * 33);  // [kEoSlots][kEoPitch]
  int64_t* s_slot = reinterpret_cast<int64_t*>(s_pow + kEoSlots * kEoPitch);
  int64_t* s_grp = s_slot + kEoSlots;
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(s_grp + kEoSlots);  // [kWarps] staging, full, empty
  uint64_t* s_full = s_bar + kWarps;
  uint64_t* s_empty = s_full + 1;
  MelPlan* s_plan = reinterpret_cast<MelPlan*>(s_empty + 1);
  float4* s_frags = reinterpret_cast<float4*>(s_plan + 1);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  eo_load_tables(p, tw_eo, s_win, s_tw, s_tw2, tid, blockDim.x);
  const bool frags_in_smem = load_mel_plan(p, s_plan, s_frags, kEoFragSteps, s_pow, kEoSlots, kEoPitch, kEoBins);
  if (tid < kWarps) mbar_init(s_bar + tid, 1);
  if (tid == 0) {
    mbar_init(s_full, kWarps);
    mbar_init(s_empty, kMelWarps);
  }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();

  const int64_t stride = (int64_t)gridDim.x * kWarps;
  const int64_t u0 = (int64_t)blockIdx.x * kWarps;
  if (warp < kWarps) {
    reg_alloc<kFftRegs>();
    float2* tile = s_tile_all + warp * 32 * 33;
    uint64_t* bar = s_bar + warp;
    const int half = p.center ? kEoN / 2 : 0;
    uint32_t parity = 0;
    bool staged = false;
    UnitCursor cur;
    cur.init(u0 + warp, stride, p.units_per_row);
    if (cur.u < p.total_units && eo_frame_bulk_ok(p, half, 2 * cur.ub)) {
      if (lane == 0) {
        mbar_expect_tx(bar, kEoN * 4u);
        bulk_g2s(tile, p.wave + cur.row * p.row_stride + (2 * cur.ub * p.hop - half - p.pad), kEoN * 4u, bar);
      }
      staged = true;
    }
    int it = 0;
    for (int64_t base = u0; base < p.total_units; base += stride, ++it, cur.advance()) {
      const bool valid = cur.u < p.total_units;
#pragma unroll 1
      for (int f = 0; f < 2; ++f) {
        const int64_t t = 2 * cur.ub + f;
        const bool live = valid && t < p.frames;
        float plo[16], phi[16], pmid = 0.f;
        if (live) {
          const EoNext nx = eo_next_frame(p, cur, f);
          transform_frame_eo<POWER_MODE>(p, s_win, s_tw, s_tw2, tile, bar, parity, staged, cur.row, t, nx.ok, nx.row,
                                         nx.t, half, lane, plo, phi, pmid);
        } else {
          staged = false;
        }
        if (f == 0 && it >= 1) mbar_wait(s_empty, (it - 1) & 1);  // the contraction warps have drained the tile
        if (live) eo_store_row(s_pow + (size_t)(2 * warp + f) * kEoPitch, lane, plo, phi, pmid);
        if (lane == 0) {
          s_slot[2 * warp + f] = live ? (cur.row * p.frames + t) * (int64_t)p.n_mels : -1;
          s_grp[2 * warp + f] = cur.row / p.rows_per_group;
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(s_full);
    }
  } else {
    reg_dealloc<kMelRegs>();
    const int mw = warp - kWarps;
    GroupMax gmax{p.stage == B200A_STAGE_FEAT ? p.group_max : nullptr, -1, -CUDART_INF_F};
    int it = 0;
    for (int64_t base = u0; base < p.total_units; base += stride, ++it) {
      mbar_wait(s_full, it & 1);
      contract_tile<kEoPitch>(p, s_plan, s_frags, frags_in_smem, mw, lane, s_pow, s_slot, s_grp, gmax);
      __syncwarp();
      if (lane == 0) mbar_arrive(s_empty);
    }
    gmax.flush();
  }
}

__global__ void prepare_tw_eo_kernel(float2* tw_eo) {  // [17][32]: W_2048^(l + 32 k1)
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 17 * 32) {
    const int k1 = i >> 5, l = i & 31;
    double s, c;
    sincospi(-2.0 * (double)(l + 32 * k1) / 2048.0, &s, &c);
    tw_eo[i] = make_float2((float)c, (float)s);
  }
}

// The mel / MFCC-feature kernel: 16 warps at 128 registers, each transforming and contracting (mel_body).
template <int POWER_MODE, int G, int HG, bool KALDI>
__global__ void __launch_bounds__(kUniWarps * 32, 1) stft_pow2_mel_kernel(const Pow2Params p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  mel_body<POWER_MODE, G, HG, KALDI>(p, smem_raw);
}

// ================================================================================================
// Inverse STFT frames on the register FFT (n_fft = 256 / 512 / 1024): the first half of b200a_istft_run.
// A lane group rebuilds the PAIR of frames (a, b) from their two Hermitian spectra with ONE complex transform:
//   Z[k] = A[k] + i B[k] (k <= N/2),  Z[N-k] = conj(A[k]) + i conj(B[k]);  z = IFFT(Z) = a + i b
// computed as conj(FFT(conj Z)) / N with the forward passes (32-point register DFT, twiddle, transpose through the
// padded tile, then fft_pass2).  Pass 1 is fft_pass1<G, false, 0> written out: through fft_pass1 the n_fft = 1024
// kernel took 1.92 ms instead of 1.61 ms for a 256 x 160000-sample inverse (H100 80GB HBM3, 400 W limit).  Lane l
// loads bins n = l + G j and ends with time samples n = l + G m, which store_frame_pair multiplies by
// window / (N * forward normalisation) and stores to the frame buffer.
// C2R semantics: the imaginary parts of bins 0 and N/2 are ignored.
// ================================================================================================
struct IstftPow2Params {
  const float2* spec;  // logical [rows][bins][frames], element strides below
  int64_t stride_row, stride_bin, stride_frame;
  int64_t frames, units_per_row, total_units;
  float* frame_buf;  // [rows][frames][n_fft]
  const float* window;
  const float2* tw2d;
  const WsHeader* hdr;
};

constexpr int kIsWarps = 16;

template <int G>
constexpr size_t istft_smem() {  // twiddles, window, transpose tiles
  return sizeof(float2) * (32 * G + kIsWarps * Geo<G>::kTileF2) + sizeof(float) * Geo<G>::kNfft;
}

template <int G>
__global__ void __launch_bounds__(kIsWarps * 32, 1) istft_pow2_kernel(const IstftPow2Params p) {
  using Ge = Geo<G>;
  constexpr int N = Ge::kNfft;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float2* s_tw = reinterpret_cast<float2*>(smem_raw);  // [32][G]
  float* s_win = reinterpret_cast<float*>(s_tw + 32 * G);  // [N] window / (N * forward normalisation)
  float2* s_tile_all = reinterpret_cast<float2*>(s_win + N);  // [kIsWarps][kTileF2]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  load_fft_tables<G>(p.tw2d, p.window, 1.f / ((float)N * p.hdr->scale), s_tw, s_win);
  __syncthreads();
  float2* grp_tile = s_tile_all + warp * Ge::kTileF2 + (lane / G) * Ge::kRegion;
  const int gi = lane / G, l = lane % G;
  UnitCursor cur;
  cur.init((int64_t)blockIdx.x * kIsWarps + warp, (int64_t)gridDim.x * kIsWarps, p.units_per_row);
  for (; cur.u < p.total_units; cur.advance()) {
    const int64_t ta = cur.ub * Ge::kFrames + 2 * gi, tb = ta + 1;
    const bool has_a = ta < p.frames, has_b = tb < p.frames;
    const float2* __restrict__ sp = p.spec + cur.row * p.stride_row;
    float2 a[32];
    static_for<32>([&](auto ji) {
      constexpr int j = decltype(ji)::value;
      const int n = l + G * j;
      const int kk = n <= N / 2 ? n : N - n;
      float2 za = make_float2(0.f, 0.f), zb = za;
      if (has_a) za = __ldg(sp + kk * p.stride_bin + ta * p.stride_frame);
      if (has_b) zb = __ldg(sp + kk * p.stride_bin + tb * p.stride_frame);
      if (kk == 0 || kk == N / 2) za.y = zb.y = 0.f;
      if (n > N / 2) {
        za.y = -za.y;
        zb.y = -zb.y;
      }
      a[brev5(j)] = make_float2(za.x - zb.y, -(za.y + zb.x));  // conj(Z[n])
    });
    fft_regs<32, 0>(a);
    grp_tile[l] = a[0];
    static_for<31>([&](auto ki) {
      constexpr int k2 = decltype(ki)::value + 1;
      const float2 w = s_tw[k2 * G + l];
      const float2 v = a[k2];
      grp_tile[k2 * Ge::kRowLd + l] = cmul2(v, w);
    });
    __syncwarp();
    static_for<32>([&](auto si) {
      constexpr int s = decltype(si)::value;
      constexpr int q = s / G, g = s % G;
      a[q * G + brev<Ge::kLogG>(g)] = grp_tile[(l + G * q) * Ge::kRowLd + g];
    });
    __syncwarp();
    fft_pass2<G>(a);
    store_frame_pair<G>(a, p.frame_buf + (cur.row * p.frames + ta) * N + l, s_win, 1.f, l, has_a, has_b, false, false);
  }
}

// ================================================================================================
// Waveform gradient on the register FFT (n_fft = 256 / 512 / 1024), the first half of b200a_frontend_backward.
// Per unit a warp recomputes the forward transform from the waveform (transform_unit, the spectra kept complex), forms
// the per-bin gradient G (upstream value, or p |X|^(p-2) X s with s = g or sum_m fb[k][m] g_m) and its Hermitian part
// H_k = (G_k + conj G_{N-k}) / 2 in registers, fetches the mirrored half of H with one shuffle per value as the forward
// un-packing does, and runs the inverse transform of istft_pow2_kernel.  The frame gradients scale * w * N * irfft(H) go
// to frame_buf; X never leaves the registers.  Units are loaded without the bulk prefetch, so the transpose tile is
// free for the inverse passes.  A frame with a NaN bin gets NaN everywhere (torch's p < 1 gradient at X = 0).
// ================================================================================================
constexpr int kBwWarps = 16;

struct BwdParams {
  Pow2Params f;      // the forward geometry (bulk_ok = 0)
  const float* grad;  // upstream gradient, element strides (complex elements for COMPLEX)
  int64_t gs_row, gs_frame, gs_col;
  float* frame_buf;  // [rows][frames][n_fft]
  const float* fb;   // [n_bins][n_mels]
  const int2* bands;  // [n_mels]
};

template <int G>
constexpr size_t bwd_smem_fixed() {  // twiddles, window, transpose tiles, per-bin filter ranges
  return sizeof(float2) * (32 * G + kBwWarps * Geo<G>::kTileF2) + sizeof(float) * Geo<G>::kNfft + sizeof(int2) * Geo<G>::kBins;
}

// KALDI: the Kaldi variant (b200a_kaldi_backward): X is recomputed with transform_unit's Kaldi load stage (framing with
// mirrored edges, DC removal, pre-emphasis, window), and `grad` holds dL/dv of the spectral values after the log adjoint.
template <int G, int STAGE, bool KALDI>
__global__ void __launch_bounds__(kBwWarps * 32, 1) stft_pow2_backward_kernel(const BwdParams bp) {
  using Ge = Geo<G>;
  constexpr int N = Ge::kNfft;
  const Pow2Params& p = bp.f;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float2* s_tw = reinterpret_cast<float2*>(smem_raw);                    // [32][G]
  float2* s_tile_all = s_tw + 32 * G;                                     // [kBwWarps][kTileF2]
  float* s_win = reinterpret_cast<float*>(s_tile_all + kBwWarps * Ge::kTileF2);  // [N] window x 1/2 x scale
  int2* s_range = reinterpret_cast<int2*>(s_win + N);                     // [bins] MEL: filters non-zero at the bin
  float* s_g_all = reinterpret_cast<float*>(s_range + Ge::kBins);        // [kBwWarps][kFrames][n_mels] MEL

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  load_fft_tables<G>(p.tw2d, p.window, 0.5f * p.hdr->scale, s_tw, s_win);
  const int n_mels = p.n_mels;
  if constexpr (STAGE == B200A_STAGE_MEL)
    for (int k = tid; k < Ge::kBins; k += blockDim.x) s_range[k] = filter_range(bp.bands, n_mels, k);
  __syncthreads();

  float2* tile = s_tile_all + warp * Ge::kTileF2;
  float* region = reinterpret_cast<float*>(tile) + (lane / G) * 2 * Ge::kRegion;
  float* s_g = s_g_all + (size_t)warp * Ge::kFrames * n_mels;
  const int half = frame_lead(p, N);
  const int gi = lane / G, l = lane % G;
  const unsigned gmask = G == 32 ? 0xffffffffu : ((1u << G) - 1u) << (gi * G);
  uint32_t parity = 0;
  bool staged = false;
  UnitCursor cur;
  cur.init((int64_t)blockIdx.x * kBwWarps + warp, (int64_t)gridDim.x * kBwWarps, p.units_per_row);
  for (; cur.u < p.total_units; cur.advance()) {
    float2 xa[17], xb[17];
    transform_unit<kSpectra, G, -1, KALDI, false>(p, s_win, s_tw, tile, nullptr, parity, staged, cur, half, lane, xa, xb);
    const int64_t t0 = cur.ub * Ge::kFrames, ta = t0 + 2 * gi, tb = ta + 1;
    const bool has_a = ta < p.frames, has_b = tb < p.frames;
    const float* ga = bp.grad + (cur.row * bp.gs_row + ta * bp.gs_frame) * (STAGE == B200A_STAGE_COMPLEX ? 2 : 1);
    const float* gb = ga + bp.gs_frame * (STAGE == B200A_STAGE_COMPLEX ? 2 : 1);
    if constexpr (STAGE == B200A_STAGE_MEL) {  // the unit's upstream rows, [kFrames][n_mels]
      for (int i = lane; i < Ge::kFrames * n_mels; i += 32) {
        const int f = i / n_mels, m = i - f * n_mels;
        s_g[i] = t0 + f < p.frames ? bp.grad[cur.row * bp.gs_row + (t0 + f) * bp.gs_frame + m * bp.gs_col] : 0.f;
      }
      __syncwarp();
    }
    // ---- G -> H for bins k = l + G m (m < 16) and, on l == 0, k = N/2 (m = 16) ----
    bool nan_a = false, nan_b = false;
    static_for<17>([&](auto mi) {
      constexpr int m = decltype(mi)::value;
      const int k = m < 16 ? l + G * m : N / 2;
      float2 da = make_float2(0.f, 0.f), db = da;
      if (m < 16 || l == 0) {
        if constexpr (STAGE == B200A_STAGE_COMPLEX) {
          if (has_a) da = reinterpret_cast<const float2*>(ga)[k * bp.gs_col];
          if (has_b) db = reinterpret_cast<const float2*>(gb)[k * bp.gs_col];
        } else {
          float sa = 0.f, sb = 0.f;
          if constexpr (STAGE == B200A_STAGE_MEL) {
            const int2 r = s_range[k];
            const float* ra = s_g + 2 * gi * n_mels;
            for (int q = r.x; q < r.y; ++q) {
              const float w = __ldg(bp.fb + (size_t)k * n_mels + q);
              sa = fmaf(w, ra[q], sa);
              sb = fmaf(w, ra[n_mels + q], sb);
            }
          } else {
            if (has_a) sa = ga[k * bp.gs_col];
            if (has_b) sb = gb[k * bp.gs_col];
          }
          if (has_a) da = power_vjp(xa[m].x, xa[m].y, p.power, sa);
          if (has_b) db = power_vjp(xb[m].x, xb[m].y, p.power, sb);
        }
      }
      // H = G / 2 inside, Re G at bins 0 and N/2 (the scale is applied with the window at the end)
      const bool edge = k == 0 || m == 16;
      xa[m] = edge ? make_float2(da.x, 0.f) : make_float2(0.5f * da.x, 0.5f * da.y);
      xb[m] = edge ? make_float2(db.x, 0.f) : make_float2(0.5f * db.x, 0.5f * db.y);
      nan_a |= isnan(xa[m].x) || isnan(xa[m].y);
      nan_b |= isnan(xb[m].x) || isnan(xb[m].y);
    });
    const bool bad_a = (__ballot_sync(0xffffffffu, nan_a) & gmask) != 0;
    const bool bad_b = (__ballot_sync(0xffffffffu, nan_b) & gmask) != 0;
    if (bad_a || bad_b) {  // keep the frame it shares the complex transform with clean
      static_for<17>([&](auto mi) {
        constexpr int m = decltype(mi)::value;
        if (bad_a) xa[m] = make_float2(0.f, 0.f);
        if (bad_b) xb[m] = make_float2(0.f, 0.f);
      });
    }
    // ---- conj(Z[n]), Z = Ha + i Hb, n = l + G j: j < 16 own bins, j >= 16 the conjugate of bin N - n ----
    float2 a[32];
    const int src = (lane & ~(G - 1)) | ((G - l) & (G - 1));
    static_for<32>([&](auto ji) {
      constexpr int j = decltype(ji)::value;
      float2 ha, hb;
      if constexpr (j < 16) {
        ha = xa[j];
        hb = xb[j];
      } else {
        // l >= 1: N - n = (G - l) + G (31 - j) on lane src;  l == 0: N - n = G (32 - j), own bin m = 32 - j
        constexpr int mm = 31 - j, m0 = 32 - j;
        float4 v = make_float4(__shfl_sync(0xffffffffu, xa[mm].x, src), __shfl_sync(0xffffffffu, xa[mm].y, src),
                               __shfl_sync(0xffffffffu, xb[mm].x, src), __shfl_sync(0xffffffffu, xb[mm].y, src));
        if (l == 0) v = make_float4(xa[m0].x, xa[m0].y, xb[m0].x, xb[m0].y);
        ha = make_float2(v.x, -v.y);
        hb = make_float2(v.z, -v.w);
        if (j == 16 && l == 0) {  // bin N/2 itself (real)
          ha = xa[16];
          hb = xb[16];
        }
      }
      a[brev5(j)] = make_float2(ha.x - hb.y, -(ha.y + hb.x));
    });
    // ---- the inverse transform, as in istft_pow2_kernel: dframe = scale * w * N * irfft(H) (2 s_win = window x scale) ----
    fft_pass1<G, false, 0>(a, s_tw, region, l);
    fft_pass2<G>(a);
    store_frame_pair<G>(a, bp.frame_buf + (cur.row * p.frames + ta) * N + l, s_win, 2.f, l, has_a, has_b, bad_a, bad_b);
  }
}

// ---- table preparation ------------------------------------------------------------------------
__global__ void prepare_tw2d_kernel(float2* tw2d, int G) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // i = k2 * G + g
  if (i < 32 * G) {
    const int k2 = i / G, g = i - k2 * G;
    double s, c;
    sincospi(-2.0 * (double)(k2 * g) / (double)(32 * G), &s, &c);
    tw2d[i] = make_float2((float)c, (float)s);
  }
}

// Builds the mel contraction plan: per group of 8 filters the 8-bin k-steps its non-zero bins span,
// groups spread over the contraction warps by descending size; and the filterbank values split
// into TF32 hi/lo parts in mma.m16n8k8 B-fragment order.  n_mtiles > 0: also the 16-warp kernel's work lists,
// every (16-frame tile, group) pair of an iteration spread over the kUniWarps warps the same way.
__global__ void prepare_mma_kernel(const float* __restrict__ fb, const int2* __restrict__ bands, int n_bins, int n_mels,
                                   int n_tiles, int n_mtiles, MelPlan* plan, float4* frags) {
  __shared__ BandTile tiles[kMaxItems];
  __shared__ int order[kMaxItems];
  __shared__ unsigned char owner[kMaxMTiles * kMaxItems];
  if (threadIdx.x == 0) {
    int total = 0;
    for (int t = 0; t < n_tiles; ++t) {
      int lo = n_bins, hi = 0;
      for (int m = 8 * t; m < min(8 * t + 8, n_mels); ++m) {
        const int2 b = bands[m];
        if (b.y > b.x) { lo = min(lo, b.x); hi = max(hi, b.y); }
      }
      tiles[t] = band_tile(t, lo, hi, total);
      plan->items[t] = tiles[t];
      total += tiles[t].nsteps;
    }
    plan->n_tiles = n_tiles;
    plan->n_items = n_tiles;
    plan->total_steps = total;
    plan->n_work = n_mtiles * n_tiles;
    // longest-processing-time-first assignment of the groups to the contraction warps whose lists have room (a skewed
    // bank, a few full-band groups and many empty ones, would otherwise pile more than kMaxItemsPerWarp on one warp)
    int load[kUniWarps], cnt[kUniWarps];
    bool used[kMaxItems];
    for (int w = 0; w < kMelWarps; ++w) { load[w] = 0; plan->warp_cnt[w] = 0; }
    for (int i = 0; i < n_tiles; ++i) used[i] = false;
    for (int k = 0; k < n_tiles; ++k) {
      int best = -1;
      for (int i = 0; i < n_tiles; ++i)
        if (!used[i] && (best < 0 || tiles[i].nsteps > tiles[best].nsteps)) best = i;
      used[best] = true;
      order[k] = best;
      int w = -1;
      for (int q = 0; q < kMelWarps; ++q)
        if (plan->warp_cnt[q] < kMaxItemsPerWarp &&
            (w < 0 || load[q] < load[w] || (load[q] == load[w] && plan->warp_cnt[q] < plan->warp_cnt[w])))
          w = q;
      plan->warp_items[w][plan->warp_cnt[w]++] = best;
      load[w] += tiles[best].nsteps + 2;  // + epilogue cost
    }
    // the same for the (tile, group) pairs over the 16 uniform warps, then listed warp by warp
    for (int w = 0; w < kUniWarps; ++w) { load[w] = 0; cnt[w] = 0; }
    for (int k = 0; k < n_tiles; ++k)
      for (int mt = 0; mt < n_mtiles; ++mt) {
        int w = 0;
        for (int q = 1; q < kUniWarps; ++q)
          if (load[q] < load[w] || (load[q] == load[w] && cnt[q] < cnt[w])) w = q;
        owner[k * n_mtiles + mt] = (unsigned char)w;
        ++cnt[w];
        load[w] += tiles[order[k]].nsteps + 2;
      }
    int begin = 0;
    for (int w = 0; w < kUniWarps; ++w) {
      plan->work_begin[w] = begin;
      begin += cnt[w];
      cnt[w] = plan->work_begin[w];  // fill cursor
    }
    for (int w = kUniWarps; w < kUniWarps + 4; ++w) plan->work_begin[w] = begin;
    for (int k = 0; k < n_tiles; ++k)
      for (int mt = 0; mt < n_mtiles; ++mt)
        plan->work[cnt[owner[k * n_mtiles + mt]]++] = (unsigned short)((mt << 8) | order[k]);
  }
  __syncthreads();
  for (int t = 0; t < n_tiles; ++t)
    write_band_frags(tiles[t], frags,
                     [&](int n, int k) { return (n < n_mels && k < n_bins) ? fb[(size_t)k * n_mels + n] : 0.f; });
}

// prepare_mma_kernel gives a group only to a warp with fewer than kMaxItemsPerWarp groups; while groups remain, the
// warps hold fewer than kMaxItems <= kMelWarps * kMaxItemsPerWarp of them, so one such warp always exists.  (The 16-warp
// kernel's work list is one array of kMaxMTiles * kMaxItems entries, cut into per-warp ranges: no per-warp cap.)
static_assert(kMaxItemsPerWarp * kMelWarps >= kMaxItems,
              "every filter group must find a place in a contraction warp's list");

}  // namespace

// The register FFT's lanes per frame pair G (n_fft = 2048 runs on the 1024-point complex core) and frames per unit,
// Geo<G>::kFrames.
static int fft_g(int n_fft) { return n_fft == 2048 ? 32 : n_fft / 32; }
static int unit_frames(int n_fft) { return 2 * (32 / fft_g(n_fft)); }

// f(std::integral_constant<int, G>{}) with the G of n_fft
template <typename F>
static auto with_g(int n_fft, F&& f) {
  switch (fft_g(n_fft)) {
    case 8: return f(std::integral_constant<int, 8>{});
    case 16: return f(std::integral_constant<int, 16>{});
    default: return f(std::integral_constant<int, 32>{});
  }
}

// The bulk copies stage 16-byte aligned spans of whole 16-byte words: the source, its row stride, the hop and the lead
// (samples a row's first frame starts before sample 0; every unit starts at a multiple of frames-per-unit * hop minus
// the lead) are multiples of 4 floats.
static bool bulk_aligned(int hop, int64_t lead, int64_t row_stride, const float* src) {
  return hop % 4 == 0 && lead % 4 == 0 && row_stride % 4 == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0;
}

size_t pow2_workspace_extra(const b200a_frontend_desc* d) {
  if (!pow2_applicable(*d)) return 0;
  const size_t base = ws_layout(*d).total;
  return pow2_layout(*d, base).total - base;
}

int pow2_prepare(const b200a_frontend_desc* d, void* ws, size_t ws_bytes, cudaStream_t stream) {
  if (!pow2_applicable(*d)) return B200A_OK;
  if (ws_bytes < b200a_frontend_workspace_bytes(d)) return B200A_EWORKSPACE;
  const FrontendWs<void> t = frontend_ws(*d, ws);
  const Pow2Ws<void> x = pow2_ws(*d, ws);
  const int G = fft_g(d->n_fft);
  prepare_tw2d_kernel<<<(32 * G + 255) / 256, 256, 0, stream>>>(x.tw2d, G);
  if (d->n_fft == 2048) prepare_tw_eo_kernel<<<3, 256, 0, stream>>>(x.tw_eo);
  if (d->n_mels > 0 && mel_tiles(d->n_mels) <= kMaxItems) {
    const int n_mtiles = d->n_fft == 2048 ? 0 : kUniWarps * unit_frames(d->n_fft) / 16;  // Geo<G>::kMTiles
    prepare_mma_kernel<<<1, 256, 0, stream>>>(t.fb, t.bands, d->n_fft / 2 + 1, d->n_mels, mel_tiles(d->n_mels), n_mtiles,
                                              x.plan, x.frags);
  }
  return launch_status();
}

template <int POWER_MODE, int G, int HG>
static int launch_power(const Pow2Params& p, cudaStream_t stream) {
  using Ge = Geo<G>;
  // the transform is latency bound: as many warps as shared memory (one tile each, also the staging buffer) and the
  // register file (at 16 warps, 128 registers a thread) allow
  constexpr int NW = 16;
  const size_t smem = sizeof(float2) * (32 * 32 + NW * Ge::kTileF2) +
                      sizeof(float) * Ge::kNfft * (POWER_MODE == kIstftGrad ? 2 : 1) + sizeof(uint64_t) * NW;
  auto kern = stft_pow2_power_kernel<POWER_MODE, G, HG, NW, false>;
  if constexpr (POWER_MODE != kComplexOut && POWER_MODE != kIstftGrad)
    if (p.kaldi) kern = stft_pow2_power_kernel<POWER_MODE, G, -1, NW, true>;
  return launch_kernel(kern, persistent_grid(p.total_units, NW), NW * 32, smem, stream, p);
}

template <int POWER_MODE, int G, int HG>
static int launch_mel(const Pow2Params& p, cudaStream_t stream) {
  using Ge = Geo<G>;
  static_assert(sizeof(MelPlan) % 16 == 0, "fragment array must stay 16-byte aligned");
  static_assert(Ge::kSlots <= kMaxSlots && Ge::kMTiles <= kMaxMTiles, "slot tables");
  static_assert((Ge::kSlots * Ge::kPitch) % 4 == 0, "slot tables and plan stay 16-byte aligned");
  constexpr size_t smem = mel_smem_bytes<G>();
  static_assert(smem <= kSmemLimit, "16-warp mel kernel exceeds the shared-memory budget");
  auto kern = p.kaldi ? stft_pow2_mel_kernel<POWER_MODE, G, -1, true> : stft_pow2_mel_kernel<POWER_MODE, G, HG, false>;
  return launch_kernel(kern, persistent_grid(p.total_units, kUniWarps), kUniWarps * 32, smem, stream, p);
}

template <int POWER_MODE, int G>
static int launch_g(const Pow2Params& p, bool mel, cudaStream_t stream) {
  if constexpr (POWER_MODE == kComplexOut || POWER_MODE == kIstftGrad) {  // complex spectra: only the Spectrogram kernel
    if constexpr (G == 32)
      if (p.bulk_ok && p.hop == 256) return launch_power<POWER_MODE, 32, 8>(p, stream);
    return launch_power<POWER_MODE, G, -1>(p, stream);
  } else {
    if constexpr (G == 32) {
      if (p.bulk_ok && p.hop == 256 && !p.kaldi)  // frame b = frame a shifted by 8 lane-rows: shared register loads
        return mel ? launch_mel<POWER_MODE, 32, 8>(p, stream) : launch_power<POWER_MODE, 32, 8>(p, stream);
    }
    return mel ? launch_mel<POWER_MODE, G, -1>(p, stream) : launch_power<POWER_MODE, G, -1>(p, stream);
  }
}

template <int POWER_MODE>
static int launch_eo(const Pow2Params& p, const float2* tw_eo, bool mel, cudaStream_t stream) {
  const int64_t grid = persistent_grid(p.total_units, kWarps);
  const size_t tables = sizeof(float2) * (1024 + 1024 + 17 * 32 + kWarps * 32 * 33);
  if (!mel)
    return launch_kernel(stft2048_power_kernel<POWER_MODE>, grid, kWarps * 32, tables + sizeof(uint64_t) * kWarps, stream,
                         p, tw_eo);
  const size_t smem = tables + sizeof(float) * kEoSlots * kEoPitch + sizeof(int64_t) * 2 * kEoSlots +
                      sizeof(uint64_t) * (kWarps + 2) + sizeof(MelPlan) + sizeof(float4) * 32 * kEoFragSteps;
  if (smem > kSmemLimit) return kPathDeclined;
  return launch_kernel(stft2048_mel_kernel<POWER_MODE>, grid, (kWarps + kMelWarps) * 32, smem, stream, p, tw_eo);
}

// floats of a warp's staging region: the mel kernel's region, or the float2 transpose tile of the Spectrogram and
// gradient kernels
static int stage_floats(int n_fft, bool mel) {
  return with_g(n_fft, [&](auto g) {
    using Ge = Geo<decltype(g)::value>;
    return mel ? Ge::kMelRegion : 2 * Ge::kTileF2;
  });
}

// The Pow2Params fields the forward and the gradient kernels fill alike: the waveform and its framing, the window,
// twiddle and header tables of the workspace, and stage_ok: an edge unit's span fits the warp's staging region of
// `staging` floats, and its gather can index with 32 bits.
static Pow2Params pow2_geometry(const b200a_frontend_desc& d, const void* ws, const float* wave, int64_t rows,
                                int64_t length, int64_t row_stride, int64_t frames, int staging) {
  const FrontendWs<const void> t = frontend_ws(d, ws);
  const int frames_per_unit = unit_frames(d.n_fft);
  Pow2Params p{};
  p.wave = wave;
  p.length = length;
  p.row_stride = row_stride;
  p.frames = frames;
  p.units_per_row = (frames + frames_per_unit - 1) / frames_per_unit;
  p.total_units = rows * p.units_per_row;
  p.window = t.window;
  p.tw2d = pow2_ws(d, ws).tw2d;
  p.hdr = t.header;
  p.hop = d.hop;
  p.pad = d.pad;
  p.center = d.center;
  p.pad_mode = d.pad_mode;
  p.power = d.power;
  p.stage_ok = d.n_fft + (frames_per_unit - 1) * (int64_t)d.hop <= staging &&
               length + 2 * (int64_t)d.pad + d.n_fft < (int64_t)1 << 31;
  return p;
}

int frontend_run_pow2(const b200a_frontend_desc* d, const void* ws, int stage, const float* wave, int64_t rows,
                      int64_t length, int64_t row_stride, int64_t frames, float* out, float* group_max,
                      int64_t rows_per_group, cudaStream_t stream, const b200a_kaldi_desc* kd, bool kaldi_prelog) {
  if (!pow2_applicable(*d)) return kPathDeclined;
  if (stage == B200A_STAGE_COMPLEX && (d->n_fft > 1024 || kd != nullptr)) return kPathDeclined;
  // Kaldi features with a 256 / 512 / 1024-point FFT; every other size takes the generic kernel
  if (kd != nullptr && d->n_fft > 1024) return kPathDeclined;
  if (stage >= B200A_STAGE_MEL && mel_tiles(d->n_mels) > kMaxItems) return kPathDeclined;  // > 512 filters
  const Pow2Ws<const void> x = pow2_ws(*d, ws);
  const bool eo = d->n_fft == 2048;
  const bool mel = stage >= B200A_STAGE_MEL;
  const int staging = stage_floats(d->n_fft, mel);
  Pow2Params p = pow2_geometry(*d, ws, wave, rows, length, row_stride, frames, staging);
  p.out = out;
  p.group_max = group_max;
  p.rows_per_group = rows_per_group;
  p.plan = x.plan;
  p.frags = x.frags;
  p.n_mels = d->n_mels;
  p.stage = stage;
  p.log_mels = d->log_mels;
  p.db_mult = d->db_multiplier;
  p.db_amin = d->db_amin;
  p.db_offset = d->db_offset;
  p.out_width = stage >= B200A_STAGE_MEL ? d->n_mels : d->n_fft / 2 + 1;
  p.k_energy_col = -1;
  int64_t lead = (d->center ? d->n_fft / 2 : 0) + d->pad;
  if (kd != nullptr) {
    fill_kaldi(p, *kd, true);
    p.k_off = kaldi_lead(*kd);
    p.k_energy_mode = kd->energy_col >= 0 ? kd->energy_mode : 0;
    p.k_log = kaldi_prelog ? 0 : kd->use_log;
    p.k_prelog = kaldi_prelog;
    p.pad_mode = kPadSymmetric;  // only reached when snip_edges == 0 (frames never leave the signal otherwise)
    lead = p.k_off;
    if (!p.stage_ok) return kPathDeclined;  // the conditioning reads the staged span
  }
  // the unit's span must also fit the staging buffer (the warp's mel region, or the Spectrogram kernel's float2
  // transpose tile); the n_fft = 2048 kernels stage into tables of their own
  p.bulk_ok = bulk_aligned(d->hop, lead, row_stride, wave) &&
              (eo || d->n_fft + (unit_frames(d->n_fft) - 1) * (int64_t)d->hop <= staging);
  p.out_vec = (p.out_width % 4 == 0 && p.out_col0 % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0)   ? 4
              : (p.out_width % 2 == 0 && p.out_col0 % 2 == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0) ? 2
                                                                                                              : 1;
  if (eo) return d->power == 2.f ? launch_eo<2>(p, x.tw_eo, mel, stream) : launch_eo<0>(p, x.tw_eo, mel, stream);
  return with_g(d->n_fft, [&](auto g) {
    constexpr int G = decltype(g)::value;
    if (stage == B200A_STAGE_COMPLEX) return launch_g<kComplexOut, G>(p, false, stream);
    return d->power == 2.f ? launch_g<2, G>(p, mel, stream) : launch_g<0, G>(p, mel, stream);
  });
}

// First half of b200a_istft_run for n_fft = 256 / 512 / 1024: windowed time frames into frame_buf.
int istft_frames_pow2(const b200a_frontend_desc* d, const void* ws, const float* spec, int64_t rows, int64_t frames,
                      int64_t stride_row, int64_t stride_bin, int64_t stride_frame, float* frame_buf, cudaStream_t stream) {
  if (!pow2_applicable(*d) || d->n_fft > 1024) return kPathDeclined;
  const Pow2Params g = pow2_geometry(*d, ws, nullptr, rows, 0, 0, frames, 0);  // the unit grid and the FFT tables
  IstftPow2Params p{};
  p.spec = reinterpret_cast<const float2*>(spec);
  p.stride_row = stride_row;
  p.stride_bin = stride_bin;
  p.stride_frame = stride_frame;
  p.frames = frames;
  p.units_per_row = g.units_per_row;
  p.total_units = g.total_units;
  p.frame_buf = frame_buf;
  p.window = g.window;
  p.tw2d = g.tw2d;
  p.hdr = g.hdr;
  const int64_t grid = persistent_grid(p.total_units, kIsWarps);
  return with_g(d->n_fft, [&](auto g) {
    constexpr int G = decltype(g)::value;
    return launch_kernel(istft_pow2_kernel<G>, grid, kIsWarps * 32, istft_smem<G>(), stream, p);
  });
}

// Shared memory of the fused gradient kernel, 0 when the descriptor / stage does not take it.
static size_t backward_smem(const b200a_frontend_desc* d, int stage) {
  if (!pow2_applicable(*d) || d->n_fft > 1024) return 0;
  if (stage != B200A_STAGE_COMPLEX && stage != B200A_STAGE_POWER && stage != B200A_STAGE_MEL) return 0;
  const size_t fixed = with_g(d->n_fft, [](auto g) { return bwd_smem_fixed<decltype(g)::value>(); });
  const size_t g_rows = stage == B200A_STAGE_MEL ? sizeof(float) * kBwWarps * unit_frames(d->n_fft) * (size_t)d->n_mels : 0;
  return fixed + g_rows <= (size_t)kSmemLimit ? fixed + g_rows : 0;
}

bool backward_fused_applicable(const b200a_frontend_desc* d, int stage) { return backward_smem(d, stage) != 0; }

// The Kaldi gradient takes the fused kernel when the padded size is 256 / 512 / 1024, the staged g rows fit shared
// memory (backward_smem) and a unit's span fits the transpose tile the Kaldi load stage conditions in -- all decided by
// the descriptors and the signal length, never by the batch.
bool kaldi_backward_fused_applicable(const b200a_frontend_desc* d, const b200a_kaldi_desc* kd, int stage, int64_t length) {
  if (backward_smem(d, stage) == 0) return false;
  const int64_t span = d->n_fft + (unit_frames(d->n_fft) - 1) * (int64_t)kd->window_shift;
  return span <= stage_floats(d->n_fft, false) && length + d->n_fft < (int64_t)1 << 31;
}

// First half of b200a_frontend_backward and b200a_kaldi_backward for n_fft = 256 / 512 / 1024: frame gradients
// w * N * irfft(H) into frame_buf.  With kd, `grad` is the log adjoint's dL/dv (value k or filter m of frame t at
// grad[row gs_row + t gs_frame + (k | m) gs_col]).
int frontend_backward_pow2(const b200a_frontend_desc* d, const void* ws, int stage, const float* wave, int64_t rows,
                           int64_t length, int64_t row_stride, int64_t frames, const float* grad, int64_t gs_row,
                           int64_t gs_frame, int64_t gs_col, float* frame_buf, cudaStream_t stream,
                           const b200a_kaldi_desc* kd) {
  if (kd != nullptr ? !kaldi_backward_fused_applicable(d, kd, stage, length) : !backward_fused_applicable(d, stage))
    return B200A_EUNSUPPORTED;
  const size_t smem = backward_smem(d, stage);
  BwdParams bp{};
  // edge units gather their span into the Spectrogram kernel's float2 transpose tile; bulk_ok stays 0: the tile doubles
  // as the inverse transform's, so nothing is staged into it ahead
  bp.f = pow2_geometry(*d, ws, wave, rows, length, row_stride, frames, stage_floats(d->n_fft, false));
  bp.f.n_mels = stage == B200A_STAGE_MEL ? d->n_mels : 0;
  bp.f.stage = stage;
  if (kd != nullptr) {
    // k_energy_mode stays 0: the energy's adjoint is kaldi_cond_vjp_kernel's; nothing is written to an output row
    fill_kaldi(bp.f, *kd, false);
    bp.f.k_off = kaldi_lead(*kd);
    bp.f.pad_mode = kPadSymmetric;
  }
  bp.grad = grad;
  bp.gs_row = gs_row;
  bp.gs_frame = gs_frame;
  bp.gs_col = gs_col;
  bp.frame_buf = frame_buf;
  const FrontendWs<const void> t = frontend_ws(*d, ws);
  bp.fb = t.fb;
  bp.bands = t.bands;
  const int64_t grid = persistent_grid(bp.f.total_units, kBwWarps);
  if (kd == nullptr)
    return with_g(d->n_fft, [&](auto g) {
      constexpr int G = decltype(g)::value;
      auto kern = stage == B200A_STAGE_COMPLEX ? stft_pow2_backward_kernel<G, B200A_STAGE_COMPLEX, false>
                  : stage == B200A_STAGE_POWER ? stft_pow2_backward_kernel<G, B200A_STAGE_POWER, false>
                                               : stft_pow2_backward_kernel<G, B200A_STAGE_MEL, false>;
      return launch_kernel(kern, grid, kBwWarps * 32, smem, stream, bp);
    });
  return with_g(d->n_fft, [&](auto g) {  // the Kaldi stages are POWER and MEL
    constexpr int G = decltype(g)::value;
    auto kern = stage == B200A_STAGE_POWER ? stft_pow2_backward_kernel<G, B200A_STAGE_POWER, true>
                                           : stft_pow2_backward_kernel<G, B200A_STAGE_MEL, true>;
    return launch_kernel(kern, grid, kBwWarps * 32, smem, stream, bp);
  });
}

// The iSTFT adjoint runs on the register FFT when n_fft is 256 / 512 / 1024 (one-sided), an edge unit's span fits the
// Spectrogram kernel's staging tile (hop <= ~n_fft) and the frames' samples index with 32 bits.
bool istft_backward_fused_applicable(const b200a_frontend_desc* d, int64_t frames) {
  if (!pow2_applicable(*d) || d->n_fft > 1024) return false;
  const int64_t span = d->n_fft + (unit_frames(d->n_fft) - 1) * (int64_t)d->hop;
  return span <= stage_floats(d->n_fft, false) && d->n_fft + (int64_t)d->hop * (frames - 1) + 2 * d->n_fft < (int64_t)1 << 31;
}

// b200a_istft_backward for n_fft = 256 / 512 / 1024: the COMPLEX Spectrogram kernel in its kIstftGrad variant over g,
// framed with a lead of `start` samples and constant padding, straight into grad_spec.
int istft_backward_pow2(const b200a_frontend_desc* d, const void* ws, const float* grad, int64_t rows, int64_t g_row_stride,
                        int64_t start, int64_t g_len, int64_t frames, float* grad_spec, cudaStream_t stream) {
  if (!istft_backward_fused_applicable(d, frames)) return kPathDeclined;
  // samples at or past expected = n_fft + hop (frames - 1) get no gradient: clamp so that every index fits 32 bits
  const int64_t expected = d->n_fft + (int64_t)d->hop * (frames - 1);
  const int64_t lead = start < expected ? start : expected;
  const int64_t len = g_len < expected - lead ? g_len : expected - lead;
  Pow2Params p = pow2_geometry(*d, ws, grad, rows, len, g_row_stride, frames, stage_floats(d->n_fft, false));
  p.center = 0;
  p.pad = (int)lead;
  p.pad_mode = B200A_PAD_CONSTANT;
  p.stage_ok = 1;
  p.out = grad_spec;
  p.bulk_ok = bulk_aligned(d->hop, lead, g_row_stride, grad);  // the span fits the tile: istft_backward_fused_applicable
  const int64_t cover = (d->n_fft + d->hop - 1) / d->hop;  // frames overlapping one sample, at most
  p.env_t_lo = cover - 1;
  p.env_t_hi = frames - cover;
  return with_g(d->n_fft, [&](auto g) { return launch_g<kIstftGrad, decltype(g)::value>(p, false, stream); });
}

}  // namespace b200a
