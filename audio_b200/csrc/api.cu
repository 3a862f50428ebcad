// extern "C" surface of libb200audio.so -- see include/b200audio.h for the contract.
#include <cmath>

#include "common.cuh"

using namespace b200a;

#pragma GCC visibility push(default)
extern "C" {

int b200a_version(void) { return B200A_VERSION; }

const char* b200a_strerror(int status) {
  switch (status) {
    case B200A_OK: return "ok";
    case B200A_EINVAL: return "invalid argument";
    case B200A_EUNSUPPORTED: return "configuration not supported by libb200audio";
    case B200A_ESHORT: return "signal too short for this n_fft / padding mode";
    case B200A_EWORKSPACE: return "workspace too small or not prepared";
    case B200A_ECUDA: return "CUDA launch failed";
    case B200A_ESINGULAR: return "rank-deficient system (singular Gram matrix)";
    default: return "unknown status";
  }
}

int64_t b200a_num_frames(int64_t length, int32_t n_fft, int32_t hop, int32_t center, int32_t pad) {
  if (n_fft < 1 || hop < 1 || length < 0 || pad < 0) return -1;
  const int64_t span = length + 2 * (int64_t)pad + (center ? 2 * (int64_t)(n_fft / 2) : 0);
  if (span < n_fft) return -1;
  return 1 + (span - n_fft) / hop;
}

int64_t b200a_pad_index(int64_t i, int64_t n, int32_t pad_mode) {
  if (i >= 0 && i < n) return i;
  switch (pad_mode) {
    case B200A_PAD_CONSTANT: return -1;
    case B200A_PAD_REFLECT: return i < 0 ? -i : 2 * (n - 1) - i;
    case B200A_PAD_REPLICATE: return i < 0 ? 0 : n - 1;
    default: {
      int64_t j = i % n;
      return j < 0 ? j + n : j;
    }
  }
}

int32_t b200a_num_bins(int32_t n_fft, int32_t onesided) { return onesided ? n_fft / 2 + 1 : n_fft; }

int32_t b200a_resample_width(int32_t orig_r, int32_t new_r, int32_t lowpass_filter_width, double rolloff) {
  // python: base = min(o, n); base *= rolloff; ceil(lpw * o / base)   (functional.py:1346-1359)
  double base = (double)(orig_r < new_r ? orig_r : new_r);
  base *= rolloff;
  return (int32_t)std::ceil((double)lowpass_filter_width * (double)orig_r / base);
}

int64_t b200a_resample_len(int64_t length, int32_t orig_r, int32_t new_r) {
  // python: torch.ceil(torch.as_tensor(new * L / orig)): exact int product, true (double) division,
  // then as_tensor rounds the python float to the default dtype float32 BEFORE the ceil.
  const double q = (double)((int64_t)new_r * length) / (double)orig_r;
  return (int64_t)std::ceil((float)q);
}

int b200a_resample_support(int32_t orig_r, int32_t new_r, int32_t lowpass_filter_width, double rolloff, int32_t phase,
                           int32_t* first, int32_t* count) {
  // functional.py:1376-1400: tap i of phase j is the windowed sinc at t = (-j/new' + (i - width)/orig') * base,
  // clamped to +-lowpass_filter_width where the window is (numerically) zero: live taps have |t| < lpw.
  if (orig_r < 1 || new_r < 1 || lowpass_filter_width < 1 || !(rolloff > 0.0) || phase < 0 || phase >= new_r ||
      first == nullptr || count == nullptr)
    return B200A_EINVAL;
  const int32_t width = b200a_resample_width(orig_r, new_r, lowpass_filter_width, rolloff);
  const int32_t taps = 2 * width + orig_r;
  const double base = (double)(orig_r < new_r ? orig_r : new_r) * rolloff;
  int32_t lo = taps, hi = -1;
  for (int32_t i = 0; i < taps; ++i) {
    const double t = ((double)(i - width) / (double)orig_r - (double)phase / (double)new_r) * base;
    if (std::fabs(t) < (double)lowpass_filter_width) {
      if (i < lo) lo = i;
      hi = i;
    }
  }
  *first = hi < 0 ? 0 : lo;
  *count = hi < 0 ? 0 : hi - lo + 1;
  return B200A_OK;
}

size_t b200a_frontend_workspace_bytes(const b200a_frontend_desc* desc) {
  if (validate_desc(desc) != B200A_OK) return 0;
  return ws_layout(*desc).total + pow2_workspace_extra(desc);
}

int b200a_frontend_prepare(const b200a_frontend_desc* desc, const float* window, const float* fb, const float* dct,
                           void* workspace, size_t workspace_bytes, b200a_stream stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc = frontend_prepare_impl(desc, window, fb, dct, workspace, workspace_bytes, s);
  if (rc != B200A_OK) return rc;
  return pow2_prepare(desc, workspace, workspace_bytes, s);
}

// Checks of a forward or backward call on a valid descriptor that read no pointer: stage, power, rows, length and the
// padding torch accepts.  The frame count on success, else a negative status.
static int64_t frontend_frames(const b200a_frontend_desc* desc, int32_t stage, int64_t rows, int64_t length) {
  if (stage < B200A_STAGE_COMPLEX || stage > B200A_STAGE_FEAT) return B200A_EINVAL;
  if (stage >= B200A_STAGE_MEL && desc->n_mels <= 0) return B200A_EINVAL;
  if (stage != B200A_STAGE_COMPLEX && !(desc->power > 0.f)) return B200A_EINVAL;
  if (rows < 0 || length < 0) return B200A_EINVAL;
  const int64_t ext = length + 2 * (int64_t)desc->pad;
  if (desc->center && (desc->pad_mode == B200A_PAD_REFLECT || desc->pad_mode == B200A_PAD_CIRCULAR)) {
    // torch: "Padding size should be less than the corresponding input dimension" (reflect needs
    // pad < n, circular pad <= n); both are reported as ESHORT
    const int64_t half = desc->n_fft / 2;
    if (desc->pad_mode == B200A_PAD_REFLECT ? half >= ext : half > ext) return B200A_ESHORT;
  }
  const int64_t frames = b200a_num_frames(length, desc->n_fft, desc->hop, desc->center, desc->pad);
  return frames < 1 ? (int64_t)B200A_ESHORT : frames;
}

int b200a_frontend_run(const b200a_frontend_desc* desc, const void* workspace, int32_t stage, const float* wave,
                       int64_t rows, int64_t length, int64_t row_stride, float* out, float* group_max,
                       int64_t rows_per_group, b200a_stream stream) {
  const int rc = validate_desc(desc);
  if (rc != B200A_OK || rows == 0) return rc;  // empty batch: nothing to enqueue (pointers may be null)
  if (workspace == nullptr || wave == nullptr || out == nullptr || row_stride < length) return B200A_EINVAL;
  const int64_t frames = frontend_frames(desc, stage, rows, length);
  if (frames < 1) return (int)frames;
  return frontend_run_impl(desc, workspace, stage, wave, rows, length, row_stride, frames, out, group_max, rows_per_group,
                           static_cast<cudaStream_t>(stream), nullptr);
}

size_t b200a_frontend_backward_scratch_bytes(const b200a_frontend_desc* desc, int32_t stage, int64_t rows, int64_t length) {
  if (validate_desc(desc) != B200A_OK || stage == B200A_STAGE_FEAT) return 0;
  const int64_t frames = frontend_frames(desc, stage, rows, length);
  if (frames < 1) return 0;
  return frontend_backward_scratch(desc, stage, rows, frames);
}

int b200a_frontend_backward(const b200a_frontend_desc* desc, const void* workspace, int32_t stage, const float* wave,
                            int64_t rows, int64_t length, int64_t row_stride, const float* grad_out, int64_t g_stride_row,
                            int64_t g_stride_frame, int64_t g_stride_col, void* scratch, float* grad_wave,
                            int64_t grad_row_stride, b200a_stream stream) {
  int rc = validate_desc(desc);
  if (rc != B200A_OK) return rc;
  if (stage < B200A_STAGE_COMPLEX || stage > B200A_STAGE_FEAT) return B200A_EINVAL;
  if (stage == B200A_STAGE_FEAT) return B200A_EUNSUPPORTED;
  if (rows == 0) return B200A_OK;  // empty batch: nothing to enqueue (pointers may be null)
  if (workspace == nullptr || wave == nullptr || grad_out == nullptr || scratch == nullptr || grad_wave == nullptr)
    return B200A_EINVAL;
  if (row_stride < length || grad_row_stride < length) return B200A_EINVAL;
  const int64_t frames = frontend_frames(desc, stage, rows, length);
  if (frames < 1) return (int)frames;
  return frontend_backward_impl(desc, workspace, stage, wave, rows, length, row_stride, frames, grad_out, g_stride_row,
                                g_stride_frame, g_stride_col, scratch, grad_wave, grad_row_stride,
                                static_cast<cudaStream_t>(stream));
}

int b200a_rnnt_features_run(const b200a_frontend_desc* desc, const void* workspace, const float* wave, int64_t rows,
                            int64_t length, int64_t row_stride, const int64_t* lengths, const float* stats, float gain,
                            int64_t out_frames, float* out, float* mel_out, b200a_stream stream) {
  const int rc = validate_desc(desc);
  if (rc != B200A_OK) return rc;
  if (desc->n_mels <= 0 || !(desc->power > 0.f) || !std::isfinite(gain)) return B200A_EINVAL;
  if (rows < 0 || length < 0 || out_frames < 0 || row_stride < length) return B200A_EINVAL;
  if (rows == 0 || out_frames == 0) return B200A_OK;  // nothing to enqueue (pointers may be null)
  if (workspace == nullptr || wave == nullptr || stats == nullptr || out == nullptr) return B200A_EINVAL;
  if (lengths == nullptr) {  // one length for every row: torch.stft's padding rules hold for it
    const int64_t frames = frontend_frames(desc, B200A_STAGE_MEL, rows, length);
    if (frames < 1) return (int)frames;
  }
  return rnnt_features_impl(desc, workspace, wave, rows, length, row_stride, lengths, stats, gain, out_frames, out, mel_out,
                            static_cast<cudaStream_t>(stream));
}

int b200a_rnnt_features_backward(const float* stats, float gain, const float* mel, const float* grad, int64_t g_stride_row,
                                 int64_t g_stride_frame, int64_t g_stride_col, int64_t rows, int64_t frames, int32_t n_mels,
                                 float* grad_mel, b200a_stream stream) {
  if (rows < 0 || frames < 0 || n_mels < 1 || !std::isfinite(gain)) return B200A_EINVAL;
  if (g_stride_row < 0 || g_stride_frame < 0 || g_stride_col < 0) return B200A_EINVAL;
  if (rows == 0 || frames == 0) return B200A_OK;
  if (stats == nullptr || mel == nullptr || grad == nullptr || grad_mel == nullptr) return B200A_EINVAL;
  return rnnt_backward_impl(stats, gain, mel, grad, g_stride_row, g_stride_frame, g_stride_col, rows, frames, n_mels,
                            grad_mel, static_cast<cudaStream_t>(stream));
}

int b200a_mfcc_finish(const b200a_frontend_desc* desc, const void* workspace, const float* feat, int64_t rows,
                      int64_t frames, const float* group_max, int64_t rows_per_group, float top_db, float* out,
                      b200a_stream stream) {
  int rc = validate_desc(desc);
  if (rc != B200A_OK) return rc;
  if (desc->n_mels <= 0 || desc->n_mfcc <= 0) return B200A_EINVAL;
  if (workspace == nullptr || feat == nullptr || out == nullptr || rows < 0 || frames < 0) return B200A_EINVAL;
  return mfcc_finish_impl(desc, workspace, feat, rows, frames, group_max, rows_per_group, top_db, out,
                          static_cast<cudaStream_t>(stream));
}

int b200a_apply_fbank(const float* spec, int64_t rows, int64_t n_bins, int64_t frames, int64_t stride_row,
                      int64_t stride_bin, int64_t stride_frame, const float* fb, int32_t n_filters, float* out,
                      b200a_stream stream) {
  if (spec == nullptr || fb == nullptr || out == nullptr) return B200A_EINVAL;
  if (rows < 0 || n_bins < 1 || frames < 0 || n_filters < 1) return B200A_EINVAL;
  return apply_fbank_impl(spec, rows, n_bins, frames, stride_row, stride_bin, stride_frame, fb, n_filters, out,
                          static_cast<cudaStream_t>(stream));
}

int b200a_amplitude_to_db(const float* x, int64_t groups, int64_t group_elems, float multiplier, float amin,
                          float offset, float top_db, float* scratch, float* out, b200a_stream stream) {
  if (x == nullptr || out == nullptr || groups < 0 || group_elems < 0) return B200A_EINVAL;
  return amplitude_to_db_impl(x, groups, group_elems, multiplier, amin, offset, top_db, scratch, out,
                              static_cast<cudaStream_t>(stream));
}

size_t b200a_mfcc_backward_scratch_bytes(const b200a_frontend_desc* desc, int64_t rows, int64_t frames,
                                         int64_t rows_per_group) {
  if (validate_desc(desc) != B200A_OK || desc->n_mels <= 0 || desc->n_mfcc <= 0) return 0;
  if (rows < 0 || frames < 0 || rows_per_group < 1) return 0;
  return mfcc_backward_scratch(rows, frames, rows_per_group);
}

int b200a_mfcc_backward(const b200a_frontend_desc* desc, const void* workspace, const float* grad, int64_t g_stride_row,
                        int64_t g_stride_frame, int64_t g_stride_col, const float* feat, const float* mel,
                        const float* group_max, int64_t rows, int64_t frames, int64_t rows_per_group, float top_db,
                        void* scratch, float* grad_mel, b200a_stream stream) {
  int rc = validate_desc(desc);
  if (rc != B200A_OK) return rc;
  if (desc->n_mels <= 0 || desc->n_mfcc <= 0 || rows < 0 || frames < 0) return B200A_EINVAL;
  if (g_stride_row < 0 || g_stride_frame < 0 || g_stride_col < 0) return B200A_EINVAL;
  const bool clamp = !desc->log_mels && group_max != nullptr && top_db >= 0.f;
  if (clamp && rows_per_group < 1) return B200A_EINVAL;
  if (rows == 0 || frames == 0) return B200A_OK;  // nothing to enqueue (pointers may be null)
  if (workspace == nullptr || grad == nullptr || mel == nullptr || grad_mel == nullptr) return B200A_EINVAL;
  if (clamp && (feat == nullptr || scratch == nullptr)) return B200A_EINVAL;
  return mfcc_backward_impl(desc, workspace, grad, g_stride_row, g_stride_frame, g_stride_col, feat, mel, group_max, rows,
                            frames, rows_per_group, top_db, scratch, grad_mel, static_cast<cudaStream_t>(stream));
}

size_t b200a_amplitude_to_db_backward_scratch_bytes(int64_t groups, int64_t group_elems) {
  if (groups < 0 || group_elems < 0) return 0;
  return amplitude_to_db_backward_scratch(groups, group_elems);
}

int b200a_amplitude_to_db_backward(const float* x, const float* grad, int64_t g_stride, int64_t groups, int64_t group_elems,
                                   float multiplier, float amin, float offset, float top_db, const float* group_max,
                                   void* scratch, float* grad_x, b200a_stream stream) {
  if (groups < 0 || group_elems < 0 || (g_stride != 0 && g_stride != 1)) return B200A_EINVAL;
  if (groups == 0 || group_elems == 0) return B200A_OK;
  if (x == nullptr || grad == nullptr || grad_x == nullptr) return B200A_EINVAL;
  if (group_max != nullptr && top_db >= 0.f && scratch == nullptr) return B200A_EINVAL;
  return amplitude_to_db_backward_impl(x, grad, g_stride, groups, group_elems, multiplier, amin, offset, top_db, group_max,
                                       scratch, grad_x, static_cast<cudaStream_t>(stream));
}

int b200a_apply_fbank_backward(const float* grad, int64_t rows, int64_t n_filters, int64_t frames, int64_t stride_row,
                               int64_t stride_filter, int64_t stride_frame, const float* fb, int64_t n_bins, float* grad_spec,
                               b200a_stream stream) {
  if (rows < 0 || n_filters < 1 || n_filters > 0x7fffffffLL || frames < 0 || n_bins < 1) return B200A_EINVAL;
  if (stride_row < 0 || stride_filter < 0 || stride_frame < 0) return B200A_EINVAL;
  if (rows == 0 || frames == 0) return B200A_OK;
  if (grad == nullptr || fb == nullptr || grad_spec == nullptr) return B200A_EINVAL;
  return apply_fbank_backward_impl(grad, rows, n_filters, frames, stride_row, stride_filter, stride_frame, fb, n_bins,
                                   grad_spec, static_cast<cudaStream_t>(stream));
}

int b200a_ratio_backward(const float* pairs, const float* grad, int64_t rows, int64_t frames, int64_t stride_row,
                         int64_t stride_frame, float* grad_pairs, b200a_stream stream) {
  if (rows < 0 || frames < 0 || stride_row < 0 || stride_frame < 0) return B200A_EINVAL;
  if (rows == 0 || frames == 0) return B200A_OK;
  if (pairs == nullptr || grad == nullptr || grad_pairs == nullptr) return B200A_EINVAL;
  return ratio_backward_impl(pairs, grad, rows, frames, stride_row, stride_frame, grad_pairs, static_cast<cudaStream_t>(stream));
}

int b200a_istft_run(const b200a_frontend_desc* desc, const void* workspace, const float* spec, int64_t rows,
                    int64_t frames, int64_t stride_row, int64_t stride_bin, int64_t stride_frame, float* frame_buf,
                    float* out, int64_t out_row_stride, int64_t start, int64_t out_len, b200a_stream stream) {
  int rc = validate_desc(desc);
  if (rc != B200A_OK) return rc;
  if (!desc->onesided) return B200A_EUNSUPPORTED;
  if (rows < 0 || frames < 1 || out_len < 0 || start < 0 || out_row_stride < out_len) return B200A_EINVAL;
  if (rows == 0 || out_len == 0) return B200A_OK;
  if (workspace == nullptr || spec == nullptr || frame_buf == nullptr || out == nullptr) return B200A_EINVAL;
  return istft_run_impl(desc, workspace, spec, rows, frames, stride_row, stride_bin, stride_frame, frame_buf, out,
                        out_row_stride, start, out_len, static_cast<cudaStream_t>(stream));
}

size_t b200a_istft_backward_scratch_bytes(const b200a_frontend_desc* desc, int64_t rows, int64_t frames) {
  if (validate_desc(desc) != B200A_OK || !desc->onesided || rows < 0 || frames < 1) return 0;
  return istft_backward_scratch(desc, rows, frames);
}

int b200a_istft_backward(const b200a_frontend_desc* desc, const void* workspace, const float* grad, int64_t rows,
                         int64_t g_row_stride, int64_t start, int64_t g_len, int64_t frames, void* scratch, float* grad_spec,
                         b200a_stream stream) {
  int rc = validate_desc(desc);
  if (rc != B200A_OK) return rc;
  if (!desc->onesided) return B200A_EUNSUPPORTED;
  if (rows < 0 || frames < 1 || g_row_stride < 0 || start < 0 || g_len < 0) return B200A_EINVAL;
  if (rows == 0) return B200A_OK;  // empty batch: nothing to enqueue (pointers may be null)
  if (workspace == nullptr || grad == nullptr || grad_spec == nullptr) return B200A_EINVAL;
  if (scratch == nullptr && istft_backward_scratch(desc, rows, frames) > 0) return B200A_EINVAL;
  return istft_backward_impl(desc, workspace, grad, rows, g_row_stride, start, g_len, frames, scratch, grad_spec,
                             static_cast<cudaStream_t>(stream));
}

int b200a_griffinlim_update(const float* mag, int64_t stride_row, int64_t stride_bin, int64_t stride_frame, float inv_power,
                            const float* rebuilt, const float* tprev, float momentum, int32_t normalize, float* proj,
                            int64_t rows, int64_t bins, int64_t frames, b200a_stream stream) {
  if (rows < 0 || bins < 1 || frames < 1 || !(inv_power > 0.f)) return B200A_EINVAL;
  if (rows == 0) return B200A_OK;
  if (mag == nullptr || proj == nullptr || (tprev != nullptr && rebuilt == nullptr)) return B200A_EINVAL;
  return griffinlim_update_impl(mag, stride_row, stride_bin, stride_frame, inv_power, rebuilt, tprev, momentum, normalize,
                                proj, rows, bins, frames, static_cast<cudaStream_t>(stream));
}

int b200a_phase_vocoder(const float* spec, int64_t stride_row, int64_t stride_bin, int64_t stride_frame, int64_t rows,
                        int64_t bins, int64_t frames_in, double rate, const float* phase_advance, float* out,
                        int64_t frames_out, b200a_stream stream) {
  if (rows < 0 || bins < 1 || frames_in < 1 || frames_out < 0 || !(rate > 0.0)) return B200A_EINVAL;
  if (rows == 0 || frames_out == 0) return B200A_OK;
  if (spec == nullptr || phase_advance == nullptr || out == nullptr) return B200A_EINVAL;
  return phase_vocoder_impl(spec, stride_row, stride_bin, stride_frame, rows, bins, frames_in, rate, phase_advance, out,
                            frames_out, static_cast<cudaStream_t>(stream));
}

int b200a_phase_vocoder_backward(const float* spec, int64_t stride_row, int64_t stride_bin, int64_t stride_frame,
                                 int64_t rows, int64_t bins, int64_t frames_in, double rate, const float* out,
                                 const float* grad, int64_t g_stride_row, int64_t g_stride_bin, int64_t g_stride_frame,
                                 float* grad_spec, int64_t frames_out, b200a_stream stream) {
  if (rows < 0 || bins < 1 || frames_in < 1 || frames_out < 1 || !(rate > 0.0)) return B200A_EINVAL;
  if (g_stride_row < 0 || g_stride_bin < 0 || g_stride_frame < 0) return B200A_EINVAL;
  if (rows == 0) return B200A_OK;
  if (spec == nullptr || out == nullptr || grad == nullptr || grad_spec == nullptr) return B200A_EINVAL;
  return phase_vocoder_backward_impl(spec, stride_row, stride_bin, stride_frame, rows, bins, frames_in, rate, out, grad,
                                     g_stride_row, g_stride_bin, g_stride_frame, grad_spec, frames_out,
                                     static_cast<cudaStream_t>(stream));
}

int64_t b200a_kaldi_num_frames(int64_t length, int32_t window_size, int32_t window_shift, int32_t snip_edges) {
  if (length < 0 || window_size < 1 || window_shift < 1) return -1;
  if (snip_edges) return length < window_size ? 0 : 1 + (length - window_size) / window_shift;
  return (length + window_shift / 2) / window_shift;
}

// The descriptor checks b200a_kaldi_run and b200a_kaldi_backward share.
static int validate_kaldi(const b200a_kaldi_desc* kaldi, const b200a_frontend_desc* desc, int32_t stage) {
  if (kaldi == nullptr) return B200A_EINVAL;
  int rc = validate_desc(desc);
  if (rc != B200A_OK) return rc;
  if (kaldi->window_size < 2 || kaldi->window_shift < 1 || kaldi->padded_size < kaldi->window_size ||
      kaldi->padded_size % 2 != 0)
    return B200A_EINVAL;
  if (desc->n_fft != kaldi->padded_size || desc->win_length != kaldi->padded_size || desc->hop != kaldi->window_shift ||
      desc->center != 0 || desc->pad != 0 || !desc->onesided)
    return B200A_EINVAL;
  if (stage != B200A_STAGE_POWER && stage != B200A_STAGE_MEL) return B200A_EINVAL;
  if (stage == B200A_STAGE_MEL && desc->n_mels <= 0) return B200A_EINVAL;
  if (!(desc->power > 0.f) || !(kaldi->preemphasis >= 0.f && kaldi->preemphasis <= 1.f)) return B200A_EINVAL;
  if (kaldi->energy_mode < 0 || kaldi->energy_mode > 2 || kaldi->energy_floor < 0.f) return B200A_EINVAL;
  const int values = stage == B200A_STAGE_MEL ? desc->n_mels : desc->n_fft / 2 + 1;
  if (kaldi->out_col0 < 0 || kaldi->out_col0 + values > kaldi->out_width ||
      kaldi->energy_col >= kaldi->out_width)
    return B200A_EINVAL;
  return B200A_OK;
}

int b200a_kaldi_run(const b200a_kaldi_desc* kaldi, const b200a_frontend_desc* desc, const void* workspace,
                    int32_t stage, const float* wave, int64_t rows, int64_t length, int64_t row_stride,
                    float* out, b200a_stream stream) {
  const int rc = validate_kaldi(kaldi, desc, stage);
  if (rc != B200A_OK) return rc;
  if (rows == 0) return B200A_OK;
  if (workspace == nullptr || wave == nullptr || out == nullptr) return B200A_EINVAL;
  if (rows < 0 || length < 0 || row_stride < length) return B200A_EINVAL;
  if (length < kaldi->window_size) return B200A_ESHORT;  // kaldi.py:142-144
  const int64_t frames = b200a_kaldi_num_frames(length, kaldi->window_size, kaldi->window_shift, kaldi->snip_edges);
  if (frames < 1) return B200A_ESHORT;
  return frontend_run_impl(desc, workspace, stage, wave, rows, length, row_stride, frames, out, nullptr, 1,
                           static_cast<cudaStream_t>(stream), kaldi);
}

size_t b200a_kaldi_backward_scratch_bytes(const b200a_kaldi_desc* kaldi, const b200a_frontend_desc* desc, int32_t stage,
                                          int64_t rows, int64_t length) {
  if (validate_kaldi(kaldi, desc, stage) != B200A_OK || rows < 0 || length < kaldi->window_size) return 0;
  const int64_t frames = b200a_kaldi_num_frames(length, kaldi->window_size, kaldi->window_shift, kaldi->snip_edges);
  if (frames < 1) return 0;
  return kaldi_backward_scratch(kaldi, desc, stage, rows, length, frames);
}

int b200a_kaldi_backward(const b200a_kaldi_desc* kaldi, const b200a_frontend_desc* desc, const void* workspace,
                         int32_t stage, const float* wave, int64_t rows, int64_t length, int64_t row_stride,
                         const float* grad_out, int64_t g_stride_row, int64_t g_stride_frame, int64_t g_stride_col,
                         void* scratch, float* grad_wave, int64_t grad_row_stride, b200a_stream stream) {
  const int rc = validate_kaldi(kaldi, desc, stage);
  if (rc != B200A_OK) return rc;
  if (g_stride_row < 0 || g_stride_frame < 0 || g_stride_col < 0) return B200A_EINVAL;
  if (rows == 0) return B200A_OK;
  if (workspace == nullptr || wave == nullptr || grad_out == nullptr || scratch == nullptr || grad_wave == nullptr)
    return B200A_EINVAL;
  if (rows < 0 || length < 0 || row_stride < length || grad_row_stride < length) return B200A_EINVAL;
  if (length < kaldi->window_size) return B200A_ESHORT;
  const int64_t frames = b200a_kaldi_num_frames(length, kaldi->window_size, kaldi->window_shift, kaldi->snip_edges);
  if (frames < 1) return B200A_ESHORT;
  return kaldi_backward_impl(kaldi, desc, workspace, stage, wave, rows, length, row_stride, frames, grad_out, g_stride_row,
                             g_stride_frame, g_stride_col, scratch, grad_wave, grad_row_stride,
                             static_cast<cudaStream_t>(stream));
}

int b200a_subtract_column_mean(float* x, int64_t rows, int64_t frames, int64_t width, b200a_stream stream) {
  if (rows < 0 || frames < 0 || width < 0) return B200A_EINVAL;
  if (rows == 0 || frames == 0 || width == 0) return B200A_OK;
  if (x == nullptr) return B200A_EINVAL;
  return subtract_column_mean_impl(x, rows, frames, width, static_cast<cudaStream_t>(stream));
}

int b200a_ratio_f32(const float* pairs, int64_t n, float* out, b200a_stream stream) {
  if (n < 0) return B200A_EINVAL;
  if (n == 0) return B200A_OK;
  if (pairs == nullptr || out == nullptr) return B200A_EINVAL;
  return ratio_impl(pairs, n, out, static_cast<cudaStream_t>(stream));
}

int b200a_fill_f32(float* dst, int64_t n, float value, b200a_stream stream) {
  if (dst == nullptr || n < 0) return B200A_EINVAL;
  return fill_impl(dst, n, value, static_cast<cudaStream_t>(stream));
}

size_t b200a_resample_workspace_bytes(int32_t new_r, int32_t taps) {
  if (new_r < 1 || taps < 1) return 0;
  return resample_workspace_bytes_impl(new_r, taps);
}

int b200a_resample_prepare(const float* kernel, int32_t orig_r, int32_t new_r, int32_t width, void* workspace,
                           size_t workspace_bytes, b200a_stream stream) {
  return resample_prepare_impl(kernel, orig_r, new_r, width, workspace, workspace_bytes,
                               static_cast<cudaStream_t>(stream));
}

int b200a_resample_run(const void* workspace, const float* kernel, int32_t orig_r, int32_t new_r, int32_t width,
                       const float* wave, int64_t rows, int64_t length, int64_t row_stride, float* out,
                       int64_t out_row_stride, int64_t out_len, b200a_stream stream) {
  return resample_run_impl(workspace, kernel, orig_r, new_r, width, wave, rows, length, row_stride, out,
                           out_row_stride, out_len, static_cast<cudaStream_t>(stream));
}

size_t b200a_resample_backward_workspace_bytes(int32_t orig_r, int32_t new_r, int32_t width) {
  if (orig_r < 1 || new_r < 1 || width < 0) return 0;
  return resample_backward_workspace_bytes_impl(orig_r, new_r, width);
}

int b200a_resample_backward_prepare(const float* kernel, int32_t orig_r, int32_t new_r, int32_t width, void* workspace,
                                    size_t workspace_bytes, b200a_stream stream) {
  return resample_backward_prepare_impl(kernel, orig_r, new_r, width, workspace, workspace_bytes,
                                        static_cast<cudaStream_t>(stream));
}

int b200a_resample_backward(const void* workspace, int32_t orig_r, int32_t new_r, int32_t width, const float* grad,
                            int64_t rows, int64_t g_row_stride, int64_t out_len, float* grad_wave, int64_t length,
                            int64_t grad_row_stride, b200a_stream stream) {
  if (orig_r < 1 || new_r < 1 || width < 0 || rows < 0 || length < 0 || out_len < 0 || g_row_stride < 0)
    return B200A_EINVAL;
  if (out_len != b200a_resample_len(length, orig_r, new_r)) return B200A_EINVAL;
  if (rows == 0) return B200A_OK;  // empty batch: nothing to enqueue (pointers may be null)
  if (workspace == nullptr || grad == nullptr || grad_wave == nullptr || grad_row_stride < length) return B200A_EINVAL;
  if (length == 0) return B200A_OK;
  return resample_backward_impl(workspace, orig_r, new_r, width, grad, rows, g_row_stride, out_len, grad_wave, length,
                                grad_row_stride, static_cast<cudaStream_t>(stream));
}

size_t b200a_inverse_mel_plan_bytes(int32_t n_stft, int32_t n_mels) { return inverse_mel_plan_bytes_impl(n_stft, n_mels); }

int b200a_inverse_mel_plan(const float* fb, int32_t n_stft, int32_t n_mels, int32_t driver, void* plan, size_t plan_bytes,
                           int32_t* bandwidth, int32_t* pivot) {
  return inverse_mel_plan_impl(fb, n_stft, n_mels, driver, plan, plan_bytes, bandwidth, pivot);
}

int b200a_inverse_mel_run(const void* plan, int32_t n_stft, int32_t n_mels, const float* mel, int64_t rows, int64_t frames,
                          int64_t stride_row, int64_t stride_mel, int64_t stride_frame, float* out, b200a_stream stream) {
  return inverse_mel_run_impl(plan, n_stft, n_mels, mel, rows, frames, stride_row, stride_mel, stride_frame, out,
                              static_cast<cudaStream_t>(stream));
}

int b200a_inverse_mel_backward(const void* plan, int32_t n_stft, int32_t n_mels, const float* mel, int64_t rows,
                               int64_t frames, int64_t stride_row, int64_t stride_mel, int64_t stride_frame,
                               const float* grad, int64_t g_stride_row, int64_t g_stride_frame, int64_t g_stride_bin,
                               float* grad_mel, b200a_stream stream) {
  return inverse_mel_backward_impl(plan, n_stft, n_mels, mel, rows, frames, stride_row, stride_mel, stride_frame, grad,
                                   g_stride_row, g_stride_frame, g_stride_bin, grad_mel, static_cast<cudaStream_t>(stream));
}

size_t b200a_lfilter_workspace_bytes(int64_t rows, int64_t length, int32_t n_order, int32_t n_filters) {
  return lfilter_workspace_bytes_impl(rows, length, n_order, n_filters, false);
}

size_t b200a_lfilter_backward_workspace_bytes(int64_t rows, int64_t length, int32_t n_order, int32_t n_filters) {
  return lfilter_workspace_bytes_impl(rows, length, n_order, n_filters, true);
}

int b200a_lfilter_run(const float* a, const float* b, int32_t n_filters, int32_t n_order, const float* x, int64_t batch,
                      int64_t length, int64_t stride_batch, int64_t stride_filter, int32_t clamp, int32_t reverse,
                      float* y, float* y_unclamped, void* workspace, size_t workspace_bytes, b200a_stream stream) {
  return lfilter_run_impl(a, b, n_filters, n_order, x, batch, length, stride_batch, stride_filter, clamp != 0,
                          reverse != 0, y, y_unclamped, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int b200a_lfilter_backward(const float* a, const float* b, int32_t n_filters, int32_t n_order, const float* x,
                           int64_t batch, int64_t length, int64_t stride_batch, int64_t stride_filter,
                           const float* y_unclamped, const float* grad, int32_t clamp, int32_t reverse, float* grad_x,
                           float* grad_a, float* grad_b, void* workspace, size_t workspace_bytes, b200a_stream stream) {
  return lfilter_backward_impl(a, b, n_filters, n_order, x, batch, length, stride_batch, stride_filter, y_unclamped,
                               grad, clamp != 0, reverse != 0, grad_x, grad_a, grad_b, workspace, workspace_bytes,
                               static_cast<cudaStream_t>(stream));
}

size_t b200a_fftconvolve_workspace_bytes(const b200a_fftconvolve_desc* desc) {
  return fftconvolve_workspace_bytes_impl(desc, false);
}

size_t b200a_fftconvolve_backward_workspace_bytes(const b200a_fftconvolve_desc* desc) {
  return fftconvolve_workspace_bytes_impl(desc, true);
}

int b200a_fftconvolve_run(const b200a_fftconvolve_desc* desc, const float* x, const float* y, float* out,
                          void* workspace, size_t workspace_bytes, b200a_stream stream) {
  return fftconvolve_run_impl(desc, x, y, out, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int b200a_fftconvolve_backward(const b200a_fftconvolve_desc* desc, const float* x, const float* y, const float* grad,
                               float* grad_x, float* grad_y, void* workspace, size_t workspace_bytes,
                               b200a_stream stream) {
  return fftconvolve_backward_impl(desc, x, y, grad, grad_x, grad_y, workspace, workspace_bytes,
                                   static_cast<cudaStream_t>(stream));
}

size_t b200a_convolve_workspace_bytes(const b200a_convolve_desc* desc) {
  return convolve_workspace_bytes_impl(desc, false);
}

size_t b200a_convolve_backward_workspace_bytes(const b200a_convolve_desc* desc) {
  return convolve_workspace_bytes_impl(desc, true);
}

int b200a_convolve_run(const b200a_convolve_desc* desc, const float* x, const float* y, float* out, void* workspace,
                       size_t workspace_bytes, b200a_stream stream) {
  return convolve_run_impl(desc, x, y, out, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int b200a_convolve_backward(const b200a_convolve_desc* desc, const float* x, const float* y, const float* grad,
                            float* grad_x, float* grad_y, void* workspace, size_t workspace_bytes,
                            b200a_stream stream) {
  return convolve_backward_impl(desc, x, y, grad, grad_x, grad_y, workspace, workspace_bytes,
                                static_cast<cudaStream_t>(stream));
}

size_t b200a_vad_workspace_bytes(const b200a_vad_desc* desc, int64_t chunk) {
  return vad_workspace_bytes_impl(desc, chunk);
}

int b200a_vad_walk(const b200a_vad_desc* desc, int64_t chunk, int64_t frame0, int64_t frames, const float* spectrum,
                   const float* cepstrum_window, float* rows, void* workspace, size_t workspace_bytes,
                   b200a_stream stream) {
  return vad_walk_impl(desc, chunk, frame0, frames, spectrum, cepstrum_window, rows, workspace, workspace_bytes,
                       static_cast<cudaStream_t>(stream));
}

int b200a_vad_trigger(const b200a_vad_desc* desc, int64_t chunk, int64_t frame0, int64_t frames, const float* power,
                      float* measures, void* workspace, size_t workspace_bytes, b200a_stream stream) {
  return vad_trigger_impl(desc, chunk, frame0, frames, power, measures, workspace, workspace_bytes,
                          static_cast<cudaStream_t>(stream));
}

int b200a_rnnt_loss_check(int32_t batch, int32_t classes, const int32_t* targets, int64_t target_cols,
                          const int32_t* logit_lengths, const int32_t* target_lengths, int32_t* out,
                          b200a_stream stream) {
  return rnnt_loss_check_impl(batch, classes, targets, target_cols, logit_lengths, target_lengths, out,
                              static_cast<cudaStream_t>(stream));
}

size_t b200a_rnnt_loss_workspace_bytes(const b200a_rnnt_loss_desc* desc) { return rnnt_loss_workspace_bytes_impl(desc); }

int b200a_rnnt_loss_forward(const b200a_rnnt_loss_desc* desc, const void* logits, const int32_t* targets,
                            const int32_t* logit_lengths, const int32_t* target_lengths, void* costs, float* denom,
                            float* alpha, float* beta, void* workspace, size_t workspace_bytes, b200a_stream stream) {
  return rnnt_loss_forward_impl(desc, logits, targets, logit_lengths, target_lengths, costs, denom, alpha, beta,
                                workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int b200a_rnnt_loss_backward(const b200a_rnnt_loss_desc* desc, const void* logits, const int32_t* targets,
                             const int32_t* logit_lengths, const int32_t* target_lengths, const float* denom,
                             const float* alpha, const float* beta, const void* grad_costs, int64_t grad_costs_stride,
                             void* grad_logits, b200a_stream stream) {
  return rnnt_loss_backward_impl(desc, logits, targets, logit_lengths, target_lengths, denom, alpha, beta, grad_costs,
                                 grad_costs_stride, grad_logits, static_cast<cudaStream_t>(stream));
}

int b200a_forced_align_check(const b200a_forced_align_desc* desc, const void* targets, const void* input_lengths,
                             const void* target_lengths, int64_t* out, void* workspace, size_t workspace_bytes,
                             b200a_stream stream) {
  return forced_align_check_impl(desc, targets, input_lengths, target_lengths, out, workspace, workspace_bytes,
                                 static_cast<cudaStream_t>(stream));
}

size_t b200a_forced_align_workspace_bytes(const b200a_forced_align_desc* desc) {
  return forced_align_workspace_bytes_impl(desc);
}

int b200a_forced_align_run(const b200a_forced_align_desc* desc, const void* log_probs, const void* targets,
                           const void* input_lengths, const void* target_lengths, void* paths, void* scores,
                           void* workspace, size_t workspace_bytes, b200a_stream stream) {
  return forced_align_run_impl(desc, log_probs, targets, input_lengths, target_lengths, paths, scores, workspace,
                               workspace_bytes, static_cast<cudaStream_t>(stream));
}

size_t b200a_ctc_decoder_workspace_bytes(const b200a_ctc_decoder_desc* desc) {
  return ctc_decoder_workspace_bytes_impl(desc);
}

int b200a_ctc_decoder_run(const b200a_ctc_decoder_desc* desc, const float* log_prob, const int32_t* lengths,
                          int32_t* tokens, int32_t* token_lengths, float* scores, int32_t* status, void* workspace,
                          size_t workspace_bytes, b200a_stream stream) {
  return ctc_decoder_run_impl(desc, log_prob, lengths, tokens, token_lengths, scores, status, workspace,
                              workspace_bytes, static_cast<cudaStream_t>(stream));
}

size_t b200a_mask_workspace_bytes(const b200a_mask_desc* desc) { return mask_workspace_bytes_impl(desc); }

int b200a_mask_run(const b200a_mask_desc* desc, const b200a_mask_spec* masks, const float* in, float* out,
                   const float* fill_ptr, void* workspace, size_t workspace_bytes, b200a_stream stream) {
  return mask_run_impl(desc, masks, in, out, fill_ptr, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int b200a_mask_backward(const b200a_mask_desc* desc, const b200a_mask_spec* masks, const float* grad_out,
                        float* grad_in, float* grad_fill, void* workspace, size_t workspace_bytes,
                        b200a_stream stream) {
  return mask_backward_impl(desc, masks, grad_out, grad_in, grad_fill, workspace, workspace_bytes,
                            static_cast<cudaStream_t>(stream));
}

}  // extern "C"
#pragma GCC visibility pop
