// Shared declarations for libb200audio (sm_90a).  No torch headers anywhere in csrc/.
#pragma once
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>
#include <type_traits>

#include "../../include/b200audio.h"

namespace b200a {

constexpr uint32_t kWsMagic = 0xB200A0D1u;
constexpr int kMaxStages = 16;
constexpr int kMaxFft = 8192;
constexpr float kKaldiEps = 1.1920928955078125e-07f;  // numeric_limits<float>::epsilon(), kaldi.py:21-22
constexpr int kPadSymmetric = 4;  // internal pad mode: x[-1-j] = x[j], x[L+j] = x[L-1-j] (Kaldi snip_edges = false)

// Device-side header at the start of a front-end workspace.
struct WsHeader {
  uint32_t magic;
  int32_t n_fft;
  int32_t n_bins;
  int32_t n_mels;
  int32_t n_mfcc;
  float scale;  // frame_length / window normalisation folded into one factor
  int32_t reserved[10];
};
static_assert(sizeof(WsHeader) == 64, "header is 64 bytes");

// Byte offsets of the tables inside a front-end workspace (host + device agree via this struct).
struct WsLayout {
  size_t header, window, twiddle, bands, fb, dct, total;
};

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

inline WsLayout ws_layout(const b200a_frontend_desc& d) {
  WsLayout l{};
  const size_t n_bins = d.onesided ? d.n_fft / 2 + 1 : d.n_fft;
  size_t off = 0;
  l.header = off;
  off = align_up(off + sizeof(WsHeader), 256);
  l.window = off;
  off = align_up(off + sizeof(float) * d.n_fft, 256);
  l.twiddle = off;
  off = align_up(off + sizeof(float2) * d.n_fft, 256);
  l.bands = off;
  off = align_up(off + sizeof(int2) * (d.n_mels > 0 ? d.n_mels : 1), 256);
  l.fb = off;
  off = align_up(off + sizeof(float) * n_bins * (d.n_mels > 0 ? d.n_mels : 0), 256);
  l.dct = off;
  off = align_up(off + sizeof(float) * (size_t)(d.n_mels > 0 ? d.n_mels : 0) * (d.n_mfcc > 0 ? d.n_mfcc : 0), 256);
  l.total = off;
  return l;
}

// A T* into a workspace, const when the workspace pointer W* is: prepare functions write their tables through a view
// made from `void*`, launchers read them through one made from `const void*`.
template <typename W, typename T>
using WsPtr = std::conditional_t<std::is_const<W>::value, const T, T>*;

template <typename T, typename W>
WsPtr<W, T> ws_at(W* ws, size_t off) {
  return reinterpret_cast<WsPtr<W, T>>(static_cast<WsPtr<W, unsigned char>>(ws) + off);
}

// The tables of a front-end workspace (WsLayout).
template <typename W>
struct FrontendWs {
  WsPtr<W, WsHeader> header;
  WsPtr<W, float> window;
  WsPtr<W, float2> twiddle;
  WsPtr<W, int2> bands;
  WsPtr<W, float> fb, dct;
};

template <typename W>
FrontendWs<W> frontend_ws(const b200a_frontend_desc& d, W* ws) {
  const WsLayout l = ws_layout(d);
  return {ws_at<WsHeader>(ws, l.header), ws_at<float>(ws, l.window), ws_at<float2>(ws, l.twiddle),
          ws_at<int2>(ws, l.bands),      ws_at<float>(ws, l.fb),     ws_at<float>(ws, l.dct)};
}

// Samples Kaldi frame t starts before t * window_shift: 0 with snip_edges, else win/2 - shift/2 (kaldi.py:_get_strided)
inline int kaldi_lead(const b200a_kaldi_desc& kd) { return kd.snip_edges ? 0 : kd.window_size / 2 - kd.window_shift / 2; }

// The Kaldi fields GenericParams and Pow2Params share; output = false (the gradient writes no feature rows) skips the
// energy column and output row geometry.  Energy mode, k_log / k_prelog, pad mode and lead (k_snip / k_off): the caller's.
template <typename Params>
void fill_kaldi(Params& p, const b200a_kaldi_desc& kd, bool output) {
  p.kaldi = 1;
  p.k_win = kd.window_size;
  p.k_dc = kd.remove_dc_offset;
  p.k_preemph = kd.preemphasis;
  if (!output) return;
  p.k_energy_floor = kd.energy_floor;
  p.k_energy_col = kd.energy_col;
  p.out_width = kd.out_width;
  p.out_col0 = kd.out_col0;
}

constexpr int kSmemLimit = 227 * 1024;  // dynamic shared memory per CTA on sm_90

// Returned by a register-FFT entry point whose path does not take the call: its dispatcher runs the shared-memory
// Stockham path instead.  Never leaves the library (every public status is <= 0).
constexpr int kPathDeclined = 1;

// min(blocks, per_sm * SMs of the current device), the grid of a kernel that grid-strides over `blocks` CTAs' worth of
// work; -1 if the SM count cannot be read
inline int64_t sm_capped_grid(int64_t blocks, int per_sm) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      sms <= 0)
    return -1;
  return blocks < (int64_t)per_sm * sms ? blocks : (int64_t)per_sm * sms;
}

// persistent: one resident CTA per SM, units dealt round-robin (every CTA gets the same count +-1); -1 when the SM
// count cannot be read
inline int64_t persistent_grid(int64_t total_units, int warps) {
  const int64_t grid = sm_capped_grid((total_units + warps - 1) / warps, 1);
  return grid == 0 ? 1 : grid;
}

inline int launch_status() { return cudaGetLastError() == cudaSuccess ? B200A_OK : B200A_ECUDA; }

// Raises the kernel's dynamic shared-memory limit to kSmemLimit and launches it on `grid` CTAs (grid < 0: the
// sm_capped_grid error).  The limit is a cap, not a carve-out: the launch still reserves only `smem`.
template <typename Kernel, typename... Args>
int launch_kernel(Kernel kern, int64_t grid, int threads, size_t smem, cudaStream_t stream, const Args&... args) {
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit) != cudaSuccess || grid < 0)
    return B200A_ECUDA;
  kern<<<(unsigned)grid, threads, smem, stream>>>(args...);
  return launch_status();
}

// ---- host functions shared across csrc/ -----------------------------------------------------
// frontend_generic.cu
int validate_desc(const b200a_frontend_desc* d);
int frontend_prepare_impl(const b200a_frontend_desc* d, const float* window, const float* fb, const float* dct, void* ws,
                          size_t ws_bytes, cudaStream_t stream);
// The forward front end: the register-FFT kernels when they take the call, the Stockham kernel otherwise.  kd: Kaldi
// framing and conditioning, or null.  kaldi_prelog: the Kaldi gradient's recompute -- the values before the log and
// the frame energy E in place of its floored log, from the same kernel (so bit-identical to what the forward logged).
// The COMPLEX stage with kd writes the conditioned spectrum only (no energy column).
int frontend_run_impl(const b200a_frontend_desc* d, const void* ws, int stage, const float* wave, int64_t rows,
                      int64_t length, int64_t row_stride, int64_t frames, float* out, float* group_max,
                      int64_t rows_per_group, cudaStream_t stream, const b200a_kaldi_desc* kd, bool kaldi_prelog = false);
int istft_run_impl(const b200a_frontend_desc* d, const void* ws, const float* spec, int64_t rows, int64_t frames,
                   int64_t stride_row, int64_t stride_bin, int64_t stride_frame, float* frame_buf, float* out,
                   int64_t out_row_stride, int64_t start, int64_t out_len, cudaStream_t stream);
size_t frontend_backward_scratch(const b200a_frontend_desc* d, int stage, int64_t rows, int64_t frames);
int frontend_backward_impl(const b200a_frontend_desc* d, const void* ws, int stage, const float* wave, int64_t rows,
                           int64_t length, int64_t row_stride, int64_t frames, const float* grad, int64_t gs_row,
                           int64_t gs_frame, int64_t gs_col, void* scratch, float* grad_wave, int64_t grad_row_stride,
                           cudaStream_t stream);
// inverse_mel.cu
size_t inverse_mel_plan_bytes_impl(int64_t n_stft, int64_t n_mels);
int inverse_mel_plan_impl(const float* fb, int32_t n_stft, int32_t n_mels, int32_t driver, void* plan, size_t plan_bytes,
                          int32_t* bandwidth, int32_t* pivot);
int inverse_mel_run_impl(const void* plan, int32_t n_stft, int32_t n_mels, const float* mel, int64_t rows, int64_t frames,
                         int64_t s_row, int64_t s_mel, int64_t s_frame, float* out, cudaStream_t stream);
int inverse_mel_backward_impl(const void* plan, int32_t n_stft, int32_t n_mels, const float* mel, int64_t rows,
                              int64_t frames, int64_t s_row, int64_t s_mel, int64_t s_frame, const float* grad,
                              int64_t g_row, int64_t g_frame, int64_t g_bin, float* grad_mel, cudaStream_t stream);
// lfilter.cu
size_t lfilter_workspace_bytes_impl(int64_t rows, int64_t length, int n_order, int n_filters, bool backward);
int lfilter_run_impl(const float* a, const float* b, int n_filters, int n_order, const float* x, int64_t batch,
                     int64_t length, int64_t s_batch, int64_t s_filter, bool clamp, bool reverse, float* y,
                     float* y_raw, void* ws, size_t ws_bytes, cudaStream_t stream);
int lfilter_backward_impl(const float* a, const float* b, int n_filters, int n_order, const float* x, int64_t batch,
                          int64_t length, int64_t s_batch, int64_t s_filter, const float* y_raw, const float* grad,
                          bool clamp, bool reverse, float* grad_x, float* grad_a, float* grad_b, void* ws,
                          size_t ws_bytes, cudaStream_t stream);
// convolve.cu
size_t fftconvolve_workspace_bytes_impl(const b200a_fftconvolve_desc* d, bool backward);
int fftconvolve_run_impl(const b200a_fftconvolve_desc* d, const float* x, const float* y, float* out, void* ws,
                         size_t ws_bytes, cudaStream_t stream);
int fftconvolve_backward_impl(const b200a_fftconvolve_desc* d, const float* x, const float* y, const float* grad,
                              float* grad_x, float* grad_y, void* ws, size_t ws_bytes, cudaStream_t stream);
// convolve_direct.cu
size_t convolve_workspace_bytes_impl(const b200a_convolve_desc* d, bool backward);
int convolve_run_impl(const b200a_convolve_desc* d, const float* x, const float* y, float* out, void* ws,
                      size_t ws_bytes, cudaStream_t stream);
int convolve_backward_impl(const b200a_convolve_desc* d, const float* x, const float* y, const float* grad,
                           float* grad_x, float* grad_y, void* ws, size_t ws_bytes, cudaStream_t stream);
// vad.cu
size_t vad_workspace_bytes_impl(const b200a_vad_desc* d, int64_t chunk);
int vad_walk_impl(const b200a_vad_desc* d, int64_t chunk, int64_t frame0, int64_t frames, const float* spectrum,
                  const float* cepstrum_window, float* rows, void* ws, size_t ws_bytes, cudaStream_t stream);
int vad_trigger_impl(const b200a_vad_desc* d, int64_t chunk, int64_t frame0, int64_t frames, const float* power,
                     float* measures, void* ws, size_t ws_bytes, cudaStream_t stream);
// rnnt_loss.cu
size_t rnnt_loss_workspace_bytes_impl(const b200a_rnnt_loss_desc* d);
int rnnt_loss_check_impl(int32_t batch, int32_t classes, const int32_t* targets, int64_t target_cols,
                         const int32_t* logit_lengths, const int32_t* target_lengths, int32_t* out,
                         cudaStream_t stream);
int rnnt_loss_forward_impl(const b200a_rnnt_loss_desc* d, const void* logits, const int32_t* targets,
                           const int32_t* logit_lengths, const int32_t* target_lengths, void* costs, float* denom,
                           float* alpha, float* beta, void* ws, size_t ws_bytes, cudaStream_t stream);
int rnnt_loss_backward_impl(const b200a_rnnt_loss_desc* d, const void* logits, const int32_t* targets,
                            const int32_t* logit_lengths, const int32_t* target_lengths, const float* denom,
                            const float* alpha, const float* beta, const void* grad_costs, int64_t grad_costs_stride,
                            void* grad_logits, cudaStream_t stream);
// forced_align.cu
size_t forced_align_workspace_bytes_impl(const b200a_forced_align_desc* d);
int forced_align_check_impl(const b200a_forced_align_desc* d, const void* targets, const void* input_lengths,
                            const void* target_lengths, int64_t* out, void* ws, size_t ws_bytes, cudaStream_t stream);
int forced_align_run_impl(const b200a_forced_align_desc* d, const void* log_probs, const void* targets,
                          const void* input_lengths, const void* target_lengths, void* paths, void* scores, void* ws,
                          size_t ws_bytes, cudaStream_t stream);
// ctc_decoder.cu
size_t ctc_decoder_workspace_bytes_impl(const b200a_ctc_decoder_desc* d);
int ctc_decoder_run_impl(const b200a_ctc_decoder_desc* d, const float* log_prob, const int32_t* lengths,
                         int32_t* tokens, int32_t* token_lengths, float* scores, int32_t* status, void* ws,
                         size_t ws_bytes, cudaStream_t stream);
// masking.cu
size_t mask_workspace_bytes_impl(const b200a_mask_desc* d);
int mask_run_impl(const b200a_mask_desc* d, const b200a_mask_spec* masks, const float* in, float* out,
                  const float* fill_ptr, void* ws, size_t ws_bytes, cudaStream_t stream);
int mask_backward_impl(const b200a_mask_desc* d, const b200a_mask_spec* masks, const float* grad_out, float* grad_in,
                       float* grad_fill, void* ws, size_t ws_bytes, cudaStream_t stream);
size_t istft_backward_scratch(const b200a_frontend_desc* d, int64_t rows, int64_t frames);
int istft_backward_impl(const b200a_frontend_desc* d, const void* ws, const float* grad, int64_t rows, int64_t g_row_stride,
                        int64_t start, int64_t g_len, int64_t frames, void* scratch, float* grad_spec, cudaStream_t stream);
int mfcc_finish_impl(const b200a_frontend_desc* d, const void* ws, const float* feat, int64_t rows, int64_t frames,
                     const float* group_max, int64_t rows_per_group, float top_db, float* out, cudaStream_t stream);
// The RNN-T feature chain in the epilogue of the Stockham kernel (every n_fft), per-row lengths, fill frames past T(L_r)
int rnnt_features_impl(const b200a_frontend_desc* d, const void* ws, const float* wave, int64_t rows, int64_t length,
                       int64_t row_stride, const int64_t* lengths, const float* stats, float gain, int64_t out_frames,
                       float* out, float* mel_out, cudaStream_t stream);
int rnnt_backward_impl(const float* stats, float gain, const float* mel, const float* grad, int64_t gs_row,
                       int64_t gs_frame, int64_t gs_col, int64_t rows, int64_t frames, int n_mels, float* grad_mel,
                       cudaStream_t stream);
size_t kaldi_backward_scratch(const b200a_kaldi_desc* kd, const b200a_frontend_desc* d, int stage, int64_t rows,
                              int64_t length, int64_t frames);
int kaldi_backward_impl(const b200a_kaldi_desc* kd, const b200a_frontend_desc* d, const void* ws, int stage,
                        const float* wave, int64_t rows, int64_t length, int64_t row_stride, int64_t frames,
                        const float* grad, int64_t gs_row, int64_t gs_frame, int64_t gs_col, void* scratch,
                        float* grad_wave, int64_t grad_row_stride, cudaStream_t stream);

// frontend_pow2.cu: the register-FFT path.  frontend_run_pow2, istft_frames_pow2 and istft_backward_pow2 return
// kPathDeclined when it does not take the call.
size_t pow2_workspace_extra(const b200a_frontend_desc* d);
int pow2_prepare(const b200a_frontend_desc* d, void* ws, size_t ws_bytes, cudaStream_t stream);
int frontend_run_pow2(const b200a_frontend_desc* d, const void* ws, int stage, const float* wave, int64_t rows,
                      int64_t length, int64_t row_stride, int64_t frames, float* out, float* group_max,
                      int64_t rows_per_group, cudaStream_t stream, const b200a_kaldi_desc* kd, bool kaldi_prelog);
int istft_frames_pow2(const b200a_frontend_desc* d, const void* ws, const float* spec, int64_t rows, int64_t frames,
                      int64_t stride_row, int64_t stride_bin, int64_t stride_frame, float* frame_buf, cudaStream_t stream);
bool backward_fused_applicable(const b200a_frontend_desc* d, int stage);
bool kaldi_backward_fused_applicable(const b200a_frontend_desc* d, const b200a_kaldi_desc* kd, int stage, int64_t length);
// kd: the Kaldi gradient, or null; taken only where backward_fused_applicable / kaldi_backward_fused_applicable hold.
int frontend_backward_pow2(const b200a_frontend_desc* d, const void* ws, int stage, const float* wave, int64_t rows,
                           int64_t length, int64_t row_stride, int64_t frames, const float* grad, int64_t gs_row,
                           int64_t gs_frame, int64_t gs_col, float* frame_buf, cudaStream_t stream,
                           const b200a_kaldi_desc* kd);
bool istft_backward_fused_applicable(const b200a_frontend_desc* d, int64_t frames);
int istft_backward_pow2(const b200a_frontend_desc* d, const void* ws, const float* grad, int64_t rows, int64_t g_row_stride,
                        int64_t start, int64_t g_len, int64_t frames, float* grad_spec, cudaStream_t stream);

// standalone.cu
int fill_impl(float* dst, int64_t n, float v, cudaStream_t stream);
int ratio_impl(const float* pairs, int64_t n, float* out, cudaStream_t stream);
int apply_fbank_impl(const float* spec, int64_t rows, int64_t n_bins, int64_t frames, int64_t stride_row,
                     int64_t stride_bin, int64_t stride_frame, const float* fb, int n_filters, float* out,
                     cudaStream_t stream);
int amplitude_to_db_impl(const float* x, int64_t groups, int64_t group_elems, float mult, float amin, float offset,
                         float top_db, float* scratch, float* out, cudaStream_t stream);
int subtract_column_mean_impl(float* x, int64_t rows, int64_t frames, int64_t width, cudaStream_t stream);
int griffinlim_update_impl(const float* mag, int64_t ms_row, int64_t ms_bin, int64_t ms_frame, float inv_power,
                           const float* rebuilt, const float* tprev, float momentum, int normalize, float* proj,
                           int64_t rows, int64_t bins, int64_t frames, cudaStream_t stream);
int phase_vocoder_impl(const float* spec, int64_t s_row, int64_t s_bin, int64_t s_frame, int64_t rows, int64_t bins,
                       int64_t frames_in, double rate, const float* phase_advance, float* out, int64_t frames_out,
                       cudaStream_t stream);
int phase_vocoder_backward_impl(const float* spec, int64_t s_row, int64_t s_bin, int64_t s_frame, int64_t rows,
                                int64_t bins, int64_t frames_in, double rate, const float* out, const float* grad,
                                int64_t g_row, int64_t g_bin, int64_t g_frame, float* grad_spec, int64_t frames_out,
                                cudaStream_t stream);

// feature_backward.cu: input gradients of MFCC / LFCC after the mel stage, AmplitudeToDB, MelScale, SpectralCentroid
size_t mfcc_backward_scratch(int64_t rows, int64_t frames, int64_t rows_per_group);
int mfcc_backward_impl(const b200a_frontend_desc* d, const void* ws, const float* grad, int64_t gs_row, int64_t gs_frame,
                       int64_t gs_col, const float* feat, const float* mel, const float* group_max, int64_t rows,
                       int64_t frames, int64_t rows_per_group, float top_db, void* scratch, float* grad_mel,
                       cudaStream_t stream);
size_t amplitude_to_db_backward_scratch(int64_t groups, int64_t group_elems);
int amplitude_to_db_backward_impl(const float* x, const float* grad, int64_t g_stride, int64_t groups, int64_t group_elems,
                                  float mult, float amin, float offset, float top_db, const float* group_max, void* scratch,
                                  float* grad_x, cudaStream_t stream);
int apply_fbank_backward_impl(const float* grad, int64_t rows, int64_t n_filters, int64_t frames, int64_t gs_row,
                              int64_t gs_filter, int64_t gs_frame, const float* fb, int64_t n_bins, float* grad_spec,
                              cudaStream_t stream);
int ratio_backward_impl(const float* pairs, const float* grad, int64_t rows, int64_t frames, int64_t gs_row,
                        int64_t gs_frame, float* grad_pairs, cudaStream_t stream);

// resample.cu
size_t resample_workspace_bytes_impl(int new_r, int taps);
int resample_prepare_impl(const float* kernel, int orig_r, int new_r, int width, void* ws, size_t ws_bytes,
                          cudaStream_t stream);
int resample_run_impl(const void* ws, const float* kernel, int orig_r, int new_r, int width, const float* wave,
                      int64_t rows, int64_t length, int64_t row_stride, float* out, int64_t out_row_stride,
                      int64_t out_len, cudaStream_t stream);
size_t resample_backward_workspace_bytes_impl(int orig_r, int new_r, int width);
int resample_backward_prepare_impl(const float* kernel, int orig_r, int new_r, int width, void* ws, size_t ws_bytes,
                                   cudaStream_t stream);
int resample_backward_impl(const void* ws, int orig_r, int new_r, int width, const float* grad, int64_t rows,
                           int64_t g_row_stride, int64_t out_len, float* grad_wave, int64_t length,
                           int64_t grad_row_stride, cudaStream_t stream);

// ---- device helpers -----------------------------------------------------------------------
// Index into the raw waveform row for sample i of the (constant `pad`-extended, then centre
// padded) signal; returns -1 for a zero sample.  Mirrors b200a_pad_index on the host.
__device__ __forceinline__ int64_t source_index(int64_t i, int64_t length, int pad, int half, int pad_mode) {
  const int64_t ext = length + 2 * (int64_t)pad;  // length after the constant pre-padding
  int64_t j = i - half;                           // index into the pre-padded signal
  if (j < 0 || j >= ext) {
    if (pad_mode == B200A_PAD_CONSTANT) return -1;
    if (pad_mode == B200A_PAD_REFLECT) {
      j = j < 0 ? -j : 2 * (ext - 1) - j;
    } else if (pad_mode == B200A_PAD_REPLICATE) {
      j = j < 0 ? 0 : ext - 1;
    } else {
      j %= ext;
      if (j < 0) j += ext;
    }
  }
  const int64_t s = j - pad;
  return (s >= 0 && s < length) ? s : -1;
}

// dL/dX of |X|^p for the upstream value s, as torch differentiates abs().pow(p): p |X|^(p-2) X s.  At X = 0 it is 0 for
// p >= 1 and NaN for p < 1 (0^(p-1) = inf times sgn(0) = 0).
__device__ __forceinline__ float2 power_vjp(float re, float im, float p, float s) {
  if (p == 2.f) return make_float2(2.f * re * s, 2.f * im * s);
  const float mag = hypotf(re, im);
  if (mag == 0.f) return p < 1.f ? make_float2(CUDART_NAN_F, CUDART_NAN_F) : make_float2(0.f, 0.f);
  const float c = (p == 1.f ? s : p * powf(mag, p - 1.f) * s) / mag;
  return make_float2(re * c, im * c);
}

// The overlap-added squared window at sample s of an iSTFT of `frames` frames, formed exactly as istft_ola_kernel forms
// it (float, fmaf, frames in ascending order); 0 where no frame covers s.
__device__ __forceinline__ float istft_envelope(const float* window, int n_fft, int hop, int64_t frames, int64_t s) {
  const int64_t t_lo = s - n_fft + 1 <= 0 ? 0 : (s - n_fft + hop) / hop;  // ceil((s - n_fft + 1) / hop)
  int64_t t_hi = s / hop;
  if (t_hi > frames - 1) t_hi = frames - 1;
  float env = 0.f;
  for (int64_t t = t_lo; t <= t_hi; ++t) {
    const float w = window[s - t * hop];
    env = fmaf(w, w, env);
  }
  return env;
}

// The filters [x, y) with a non-zero weight at bin k, from each filter's non-zero bin range bands[m] = [x, y); (0, 0)
// when none is.
__device__ __forceinline__ int2 filter_range(const int2* bands, int n_mels, int k) {
  int lo = n_mels, hi = 0;
  for (int m = 0; m < n_mels; ++m) {
    const int2 b = bands[m];
    if (b.x <= k && k < b.y) {
      lo = min(lo, m);
      hi = m + 1;
    }
  }
  return hi > lo ? make_int2(lo, hi) : make_int2(0, 0);
}

// AmplitudeToDB's map (functional.py:385-386): mult * log10(max(x, amin)) - offset.  to_db_kernel and the adjoint's
// recompute of it (feature_backward.cu) share this one expression, so the adjoint's ties with the forward's group maxima
// are exact.
__device__ __forceinline__ float db_value(float x, float mult, float amin, float offset) {
  return mult * log10f(fmaxf(x, amin)) - offset;
}

// The RNN-T feature chain of one mel value m (pipelines/rnnt_pipeline.py:20-23, :43-44, :322-324):
//   x = m * gain;  x[x > e] = log(x);  x[x <= e] /= e;  y = (x - mean) * invstddev
// with the reference's two in-place statements taken literally: the second mask is read after the first write, so
// there are three pieces -- x / e (x <= e), log(x) / e (e < x <= e^e) and log(x) (x > e^e) -- and a NaN stays NaN
// (piece 0).  Returns y; `x` receives m * gain and `piece` the branch.  The forward epilogue, its fill frames and
// rnnt_vjp_kernel all call this one expression, so the gradient's branch decisions are the forward's, bit for bit.
constexpr float kRnntE = 2.71828182845904523536f;
__device__ __forceinline__ float rnnt_value(float m, float gain, float mean, float invstd, float& x, int& piece) {
  x = m * gain;
  float y = x;
  piece = 0;
  if (x > kRnntE) {
    y = logf(x);
    piece = 3;
  }
  if (y <= kRnntE) {
    y = y / kRnntE;
    piece = piece == 3 ? 2 : 1;
  }
  return (y - mean) * invstd;
}

__device__ __forceinline__ void atomic_max_f32(float* addr, float v) {
  // total order trick: non-negative floats compare like ints, negative like reversed uints
  if (v >= 0.f) {
    atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
  } else {
    atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
  }
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace b200a
