/*
 * b200audio.h -- C ABI of libb200audio.so, the sm_90a implementation of torchaudio's DSP
 * front-end hot path (STFT -> |.|^p -> mel -> dB/log -> DCT, and the polyphase sinc resampler).
 *
 * This is the drop-in boundary.  pytorch/audio has no native op for this path (it is Python
 * over ATen: torch.stft / matmul / conv1d); the entry points below are what a native op for it
 * would bind, following the convention of the reference's own native ops
 * (src/libtorchaudio/lfilter.cpp:54-138, src/libtorchaudio/iir_cuda.cu:41-78):
 *   - the caller allocates every buffer, outputs included (Tensor(a!) style);
 *   - kernels are enqueued on the stream the caller passes (cuda_utils.h:9-15), never synchronise;
 *   - arguments are validated and an error CODE is returned (the reference throws via
 *     STD_TORCH_CHECK; a C ABI cannot, and it never aborts -- contrast rnnt/gpu/gpu_transducer.h:20-31).
 * No torch/ATen type crosses this boundary: plain pointers, sizes and one POD descriptor.
 *
 * Rules for every function taking a stream:
 *   - all data pointers are DEVICE pointers on the current device, 4-byte aligned, fp32 unless noted;
 *   - the library never allocates, frees or copies device memory behind the caller's back, and
 *     keeps no mutable global state except one-time cudaFuncSetAttribute calls;
 *   - calls are asynchronous; return value 0 (B200A_OK) means "enqueued", a negative value is
 *     one of the B200A_E* codes and nothing was enqueued;
 *   - re-entrant and thread-safe for distinct streams/workspaces.
 *
 * Layouts: spectra and features are FRAME-MAJOR, out[b][t][bin], which is the physical layout of
 * the tensors the reference returns (logical (..., bin, t) with strides (.., 1, n_bins):
 * functional.py:123-137 and transforms/_transforms.py:413 produce transposed views).
 *
 * Citations below are relative to src/torchaudio/ of the pytorch/audio tree.
 */
#ifndef B200AUDIO_H
#define B200AUDIO_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200A_VERSION 100 /* 0.1.0 */

typedef void* b200a_stream; /* cudaStream_t */

enum b200a_status {
  B200A_OK = 0,
  B200A_EINVAL = -1,       /* bad argument (null pointer, non-positive size, bad enum) */
  B200A_EUNSUPPORTED = -2, /* valid in the reference, not implemented here (documented) */
  B200A_ESHORT = -3,       /* signal too short: reflect/circular pad needs n_fft/2 < length, or < n_fft samples */
  B200A_EWORKSPACE = -4,   /* workspace too small / not prepared for this descriptor */
  B200A_ECUDA = -5,        /* CUDA runtime reported an error at launch (cudaGetLastError) */
  B200A_ESINGULAR = -6     /* the system is rank-deficient (b200a_inverse_mel_plan: singular Gram matrix) */
};

enum b200a_pad_mode { /* torch.nn.functional.pad modes accepted by torch.stft(center=True) */
  B200A_PAD_REFLECT = 0,
  B200A_PAD_CONSTANT = 1,
  B200A_PAD_REPLICATE = 2,
  B200A_PAD_CIRCULAR = 3
};

/* What the fused front-end kernel writes. */
enum b200a_stage {
  B200A_STAGE_COMPLEX = 0, /* power=None: complex64 STFT, out[b][t][bin][2]        (functional.py:145) */
  B200A_STAGE_POWER = 1,   /* |X|^power,            out[b][t][n_bins]               (functional.py:141-144) */
  B200A_STAGE_MEL = 2,     /* (|X|^power) @ fb,     out[b][t][n_mels]               (transforms/_transforms.py:413) */
  B200A_STAGE_FEAT = 3     /* dB (unclamped) or log(mel+1e-6), out[b][t][n_mels]    (_transforms.py:701-705) */
};

/* One descriptor for Spectrogram / MelSpectrogram / MFCC (the three share the STFT stage). */
typedef struct b200a_frontend_desc {
  int32_t n_fft;             /* FFT size, 2..8192 (any integer; powers of two take the register-FFT path) */
  int32_t win_length;        /* window length <= n_fft; centred zero padding as at::stft does */
  int32_t hop;               /* hop length >= 1 */
  int32_t pad;               /* two-sided constant pre-padding (functional.py:112-114) */
  int32_t center;            /* torch.stft center */
  int32_t pad_mode;          /* enum b200a_pad_mode (only read when center != 0) */
  int32_t onesided;          /* 1: n_bins = n_fft/2+1, 0: n_bins = n_fft */
  int32_t frame_length_norm; /* normalized == "frame_length": X *= n_fft^-1/2 (functional.py:116,131) */
  int32_t window_norm;       /* normalized == True/"window": X /= sqrt(sum w^2)   (functional.py:139-140) */
  float power;               /* exponent > 0; ignored for B200A_STAGE_COMPLEX */
  int32_t n_mels;            /* 0 when no mel stage */
  int32_t n_mfcc;            /* 0 when no DCT stage */
  int32_t log_mels;          /* MFCC: 1 -> log(mel + 1e-6); 0 -> 10*log10(max(mel,1e-10))   */
  float db_multiplier;       /* AmplitudeToDB: 10 (power) or 20 (magnitude) */
  float db_amin;             /* 1e-10 */
  float db_offset;           /* multiplier * log10(max(amin, ref)); 0 for ref = 1 */
} b200a_frontend_desc;

/* ---- library ---------------------------------------------------------------------------- */
int b200a_version(void);
const char* b200a_strerror(int status);

/* ---- integer bookkeeping (host, bit-exact with the reference's shapes) -------------------- */
/* Frames torch.stft yields (functional.py:123-134); -1 when the padded signal is shorter than n_fft. */
int64_t b200a_num_frames(int64_t length, int32_t n_fft, int32_t hop, int32_t center, int32_t pad);
/* Source index in [0,n) for index i of a padded signal, -1 for "zero" (torch/functional.py:675-680). */
int64_t b200a_pad_index(int64_t i, int64_t n, int32_t pad_mode);
/* n_fft/2+1 or n_fft. */
int32_t b200a_num_bins(int32_t n_fft, int32_t onesided);
/* FIR half-width ceil(lpw*orig'/(min(orig',new')*rolloff)) (functional.py:1359). */
int32_t b200a_resample_width(int32_t orig_r, int32_t new_r, int32_t lowpass_filter_width, double rolloff);
/* ceil(new'*L/orig') evaluated as the reference does (functional.py:1427). */
int64_t b200a_resample_len(int64_t length, int32_t orig_r, int32_t new_r);
/* Live taps [first, first + count) of output phase `phase` of the (new', 2*width+orig') sinc kernel: the taps whose
 * window argument lies strictly inside +-lowpass_filter_width (functional.py:1376-1400); every other tap of the row
 * is (numerically) zero.  ~2*lpw*orig'/min(orig',new') taps.  Returns 0 or B200A_EINVAL. */
int b200a_resample_support(int32_t orig_r, int32_t new_r, int32_t lowpass_filter_width, double rolloff, int32_t phase,
                           int32_t* first, int32_t* count);

/* ---- fused front end -------------------------------------------------------------------- */
/* Bytes of caller-owned device workspace that b200a_frontend_prepare fills for this descriptor. */
size_t b200a_frontend_workspace_bytes(const b200a_frontend_desc* desc);

/*
 * Build the device-side constant tables (centre-padded window, twiddles, normalisation scale,
 * filterbank band table + copy, DCT copy) from the module's buffers.  Must be re-run whenever
 * `window`, `fb` or `dct` change (the Python modules track tensor versions).
 *   window : [win_length]           Spectrogram.window           (_transforms.py:86-87)
 *   fb     : [n_bins][n_mels] or NULL   MelScale.fb              (_transforms.py:400-401)
 *   dct    : [n_mels][n_mfcc] or NULL   MFCC.dct_mat             (_transforms.py:688-689)
 */
int b200a_frontend_prepare(const b200a_frontend_desc* desc, const float* window, const float* fb,
                           const float* dct, void* workspace, size_t workspace_bytes,
                           b200a_stream stream);

/*
 * Fused STFT front end: replaces F.spectrogram (functional.py:54-145) [+ MelScale.forward
 * (_transforms.py:403-415)] [+ the dB/log step of MFCC.forward (_transforms.py:701-705)].
 *   wave        : [rows] utterances of `length` samples, row r at wave + r*row_stride
 *   stage       : enum b200a_stage
 *   out         : [rows][T][n_bins] (POWER), [rows][T][n_bins][2] (COMPLEX), [rows][T][n_mels] (MEL/FEAT)
 *   group_max   : FEAT only, may be NULL: [ceil(rows/rows_per_group)] running maxima of the dB
 *                 features, combined with atomic max -- the caller initialises them to -inf
 *                 (b200a_fill_f32).  This is the `amax` of functional.py:399; rows_per_group
 *                 encodes the reference's packing rule (functional.py:395-397).
 */
int b200a_frontend_run(const b200a_frontend_desc* desc, const void* workspace, int32_t stage,
                       const float* wave, int64_t rows, int64_t length, int64_t row_stride,
                       float* out, float* group_max, int64_t rows_per_group, b200a_stream stream);

/*
 * Waveform gradient of b200a_frontend_run (the backward of F.spectrogram [+ MelScale]) for stage COMPLEX, POWER or MEL,
 * with the workspace the forward ran with.  With X = scale * DFT(w * frame) and g the upstream gradient:
 *   G_k = g_k (COMPLEX), p |X_k|^(p-2) X_k s_k with s_k = g_k (POWER) or sum_m fb[k][m] g_m (MEL); G_k = 0 at X_k = 0
 *   for p >= 1 and NaN for p < 1 (as torch's abs().pow(p) backward, which then makes the whole frame NaN);
 *   dframe = scale * w * N * irfft(H),  H_k = (G_k + conj G_{N-k}) / 2,  G = 0 outside the output bins;
 *   grad_wave = dframe overlap-added onto the padded signal and folded back onto the source samples (reflect mirrors,
 *   replicate adds to the edge samples, circular wraps, constant and `pad` padding drop); samples no frame covers get 0.
 *   wave       : the forward's input, as given to b200a_frontend_run
 *   grad_out   : [rows][T][width] with element strides (stride 0 allowed: expanded gradients); for COMPLEX the strides
 *                count complex elements, as in b200a_istft_run
 *   scratch    : caller-owned device memory of b200a_frontend_backward_scratch_bytes(desc, stage, rows, length) bytes
 *   grad_wave  : [rows] rows of `length` samples, row r at grad_wave + r * grad_row_stride (every sample written)
 * Deterministic: no atomics, every row independent of the others.  B200A_STAGE_FEAT: B200A_EUNSUPPORTED.
 */
int b200a_frontend_backward(const b200a_frontend_desc* desc, const void* workspace, int32_t stage, const float* wave,
                            int64_t rows, int64_t length, int64_t row_stride, const float* grad_out, int64_t g_stride_row,
                            int64_t g_stride_frame, int64_t g_stride_col, void* scratch, float* grad_wave,
                            int64_t grad_row_stride, b200a_stream stream);
/* Bytes of scratch b200a_frontend_backward needs: rows * T * n_fft floats of frame gradients (n_fft = 256 / 512 / 1024,
 * one-sided), plus the complex spectrum and a per-frame flag for every other size; 0 for an invalid request. */
size_t b200a_frontend_backward_scratch_bytes(const b200a_frontend_desc* desc, int32_t stage, int64_t rows, int64_t length);

/*
 * Second MFCC stage: top_db clamp + DCT-II, replaces functional.py:399 + _transforms.py:708.
 *   feat      : [rows][T][n_mels] from B200A_STAGE_FEAT
 *   group_max : [groups] maxima (after any cross-rank all-reduce), NULL or top_db < 0 => no clamp
 *   out       : [rows][T][n_mfcc]
 * With a clamp the product runs on the tensor pipe in error-compensated TF32 (~2^-21 relative to sum |feat * dct|, inside
 * the 1e-4 bar of the dB path); without one (log-mel MFCC, Kaldi MFCC) in FP32 FMAs.
 */
int b200a_mfcc_finish(const b200a_frontend_desc* desc, const void* workspace, const float* feat,
                      int64_t rows, int64_t frames, const float* group_max, int64_t rows_per_group,
                      float top_db, float* out, b200a_stream stream);

/* ---- RNN-T feature chain (pipelines/rnnt_pipeline.py:20-47, :310-343) ------------------------- */
/*
 * MelSpectrogram -> x = m * gain -> piecewise log -> (x - mean) * invstddev in one launch, with the workspace
 * b200a_frontend_prepare built for a MEL descriptor (window and filterbank).  The piecewise log is the reference's two
 * in-place statements, so it has three pieces, decided in float32:
 *   y = x / e (x <= e),  log(x) / e (e < x, log(x) <= e),  log(x) (log(x) > e);  a NaN stays NaN.
 * Row r has L_r = clamp(lengths[r], 0, length) samples (lengths NULL: L_r = length for every row) and
 * T(L_r) = b200a_num_frames(L_r, ...) frames of features; frames T(L_r) <= t < out_frames get chain(0) =
 * (0 - mean) * invstddev, the features of zero mel values (the recipes pad the mel batch with zeros).  The kernel never
 * reads outside [0, L_r) of row r.  With lengths, torch.stft's per-row rules (reflect needs L_r > n_fft/2) are the
 * caller's to check; without, they are checked here as in b200a_frontend_run (B200A_ESHORT).
 *   lengths  : NULL, or a DEVICE array of rows int64 lengths
 *   stats    : [2][n_mels]: mean, then invstddev
 *   gain     : the float32 multiplier (the reference's 32767^2 rounds to 1073676288)
 *   out      : [rows][out_frames][n_mels], every element written
 *   mel_out  : NULL, or [rows][out_frames][n_mels]: m before the chain (0 on fill frames), for the gradient
 * Every n_fft, powers of two included, runs the shared-memory Stockham kernel.  Bit-identical reruns; a row's output
 * does not depend on the other rows or on out_frames.
 */
int b200a_rnnt_features_run(const b200a_frontend_desc* desc, const void* workspace, const float* wave, int64_t rows,
                            int64_t length, int64_t row_stride, const int64_t* lengths, const float* stats, float gain,
                            int64_t out_frames, float* out, float* mel_out, b200a_stream stream);
/*
 * Mel gradient of the chain, elementwise, in torch's order: g * invstddev, then / e on the first two pieces, then / x
 * on the last two, then * gain (a NaN's piece passes g * invstddev * gain).  The pieces are decided from `mel` by the
 * forward's own expression.
 *   mel      : [rows][frames][n_mels], the forward's mel_out
 *   grad     : [rows][frames][n_mels] at element strides (0 allowed: expanded gradients)
 *   grad_mel : [rows][frames][n_mels], every element written; feed it to b200a_frontend_backward(B200A_STAGE_MEL)
 */
int b200a_rnnt_features_backward(const float* stats, float gain, const float* mel, const float* grad, int64_t g_stride_row,
                                 int64_t g_stride_frame, int64_t g_stride_col, int64_t rows, int64_t frames, int32_t n_mels,
                                 float* grad_mel, b200a_stream stream);

/* ---- stand-alone stages (MelScale / AmplitudeToDB modules used on their own) ---------------- */
/*
 * out[r][t][m] = sum_k spec[r][k][t] * fb[k][m] for a spectrogram given in the reference's LOGICAL
 * layout (.., n_bins, T) with arbitrary element strides (MelScale.forward, _transforms.py:403-415).
 */
int b200a_apply_fbank(const float* spec, int64_t rows, int64_t n_bins, int64_t frames,
                      int64_t stride_row, int64_t stride_bin, int64_t stride_frame, const float* fb,
                      int32_t n_filters, float* out, b200a_stream stream);

/*
 * F.amplitude_to_DB (functional.py:356-404) over `groups` contiguous chunks of `group_elems` floats:
 * y = mult*log10(max(x, amin)) - offset; if top_db >= 0, y = max(y, max_over_group(y) - top_db).
 * `scratch` holds `groups` floats.
 */
int b200a_amplitude_to_db(const float* x, int64_t groups, int64_t group_elems, float multiplier,
                          float amin, float offset, float top_db, float* scratch, float* out,
                          b200a_stream stream);

int b200a_fill_f32(float* dst, int64_t n, float value, b200a_stream stream);

/* ---- input gradients of the feature stages (MFCC / LFCC, AmplitudeToDB, MelScale, SpectralCentroid) -------------- */
/*
 * The top_db clamp c = max(d, thr), thr = group_max[g] - top_db (functional.py:399), differentiates as torch's maximum
 * and amax do: an element keeps its gradient where d > thr and half of it where d == thr; the rest goes to thr, is
 * summed over the group (R_g) and split evenly over the count_g elements equal to group_max[g]:
 *   g_d[e] = g[e] ([d > thr] + 1/2 [d == thr]) + [d == group_max[g]] R_g / count_g.
 * Deterministic: R_g is summed in a fixed order through `scratch` (per-tile partials, then one fixed-order reduction per
 * group), never with float atomics, so reruns are bit-identical.  Without a clamp the call is one elementwise pass.
 */
/* Bytes of scratch b200a_mfcc_backward needs with a clamp (per-tile partials + one float per group); 0 for an invalid
 * request. */
size_t b200a_mfcc_backward_scratch_bytes(const b200a_frontend_desc* desc, int64_t rows, int64_t frames,
                                         int64_t rows_per_group);
/*
 * Mel-stage gradient of b200a_mfcc_finish o (the dB / log map of B200A_STAGE_FEAT), with the forward's workspace:
 *   g_d[r][t][m] = sum_j dct[m][j] g[r][t][j]                               (the DCT, _transforms.py:708)
 *   log_mels:  grad_mel = g_d / (mel + 1e-6)
 *   dB:        grad_mel = g_d' * db_multiplier / (ln10 mel) where mel >= db_amin, else 0 (clamp(min=amin) passes the
 *              gradient at mel == amin);  g_d' = g_d through the top_db clamp above when group_max != NULL, top_db >= 0
 *   grad      : [rows][T][n_mfcc] cepstral gradient at element strides (0 allowed: expanded gradients)
 *   feat      : [rows][T][n_mels] the forward's B200A_STAGE_FEAT output (pre-clamp d): masks and ties read it
 *   mel       : [rows][T][n_mels] b200a_frontend_run(B200A_STAGE_MEL) of the same waveform: the derivative reads it
 *   group_max : the maxima the forward clamped with; rows_per_group as in b200a_frontend_run
 *   scratch   : b200a_mfcc_backward_scratch_bytes(desc, rows, T, rows_per_group) bytes (clamp only, else may be NULL)
 *   grad_mel  : [rows][T][n_mels], every element written; feed it to b200a_frontend_backward(B200A_STAGE_MEL)
 * The DCT is staged in shared memory: B200A_EUNSUPPORTED when n_mels x n_mfcc needs more than ~200 KB.
 */
int b200a_mfcc_backward(const b200a_frontend_desc* desc, const void* workspace, const float* grad, int64_t g_stride_row,
                        int64_t g_stride_frame, int64_t g_stride_col, const float* feat, const float* mel,
                        const float* group_max, int64_t rows, int64_t frames, int64_t rows_per_group, float top_db,
                        void* scratch, float* grad_mel, b200a_stream stream);
/* Bytes of scratch b200a_amplitude_to_db_backward needs with a clamp; 0 for an invalid request. */
size_t b200a_amplitude_to_db_backward_scratch_bytes(int64_t groups, int64_t group_elems);
/*
 * Gradient of b200a_amplitude_to_db: d = mult * log10(max(x, amin)) - offset is recomputed from x by the expression the
 * forward uses, so ties with the forward's maxima are exact; then grad_x = g_d' * mult / (ln10 x) where x >= amin, else 0.
 *   x         : the forward's input, `groups` contiguous chunks of `group_elems` floats
 *   grad      : grad[e * g_stride], g_stride 1 (contiguous) or 0 (expanded scalar)
 *   group_max : the forward's `scratch` ([groups] maxima) when it clamped (top_db >= 0), else NULL
 *   scratch   : b200a_amplitude_to_db_backward_scratch_bytes(groups, group_elems) bytes (clamp only)
 *   grad_x    : groups * group_elems floats, every element written
 */
int b200a_amplitude_to_db_backward(const float* x, const float* grad, int64_t g_stride, int64_t groups, int64_t group_elems,
                                   float multiplier, float amin, float offset, float top_db, const float* group_max,
                                   void* scratch, float* grad_x, b200a_stream stream);
/*
 * Spectrogram gradient of b200a_apply_fbank (the transpose of MelScale.forward):
 *   grad_spec[r][t][k] = sum_m fb[k][m] grad[r][m][t]
 *   grad      : logical [rows][n_filters][T] at element strides (0 allowed)
 *   fb        : [n_bins][n_filters], row-major
 *   grad_spec : FRAME-MAJOR [rows][T][n_bins], every element written.  No atomics; rows <= 65535.
 */
int b200a_apply_fbank_backward(const float* grad, int64_t rows, int64_t n_filters, int64_t frames, int64_t stride_row,
                               int64_t stride_filter, int64_t stride_frame, const float* fb, int64_t n_bins, float* grad_spec,
                               b200a_stream stream);
/*
 * Gradient of b200a_ratio_f32 for SpectralCentroid: y = N / D per frame gives
 *   grad_pairs[r][t] = (g / D, -g N / D^2),  (N, D) = pairs[r][t],  g = grad[r * stride_row + t * stride_frame]
 * which b200a_frontend_backward(B200A_STAGE_MEL) with the [f | 1] filterbank takes back to the waveform.
 *   pairs, grad_pairs : [rows][T][2]
 */
int b200a_ratio_backward(const float* pairs, const float* grad, int64_t rows, int64_t frames, int64_t stride_row,
                         int64_t stride_frame, float* grad_pairs, b200a_stream stream);

/*
 * out[i] = pairs[i][0] / pairs[i][1].  Last step of F.spectral_centroid (functional.py:1257-1299): the
 * fused front end is run with the two-column "filterbank" [bin frequency | 1] on the magnitude
 * spectrogram, which yields (sum_k f_k |X_k|, sum_k |X_k|) per frame; this divides them.
 */
int b200a_ratio_f32(const float* pairs, int64_t n, float* out, b200a_stream stream);

/* ---- inverse STFT ---------------------------------------------------------------------------- */
/*
 * torch.istft as F.inverse_spectrogram calls it (functional/functional.py:148-225): Hermitian inverse FFT of every
 * frame (C2R: the imaginary parts of bins 0 and n_fft/2 are ignored), x window, overlap-add, division by the
 * overlap-added squared window, for the output positions [start, start + out_len) of the n_fft + hop*(frames-1)
 * long signal (start = n_fft/2 when center).  The workspace is the one b200a_frontend_prepare built for the same
 * descriptor (window, twiddles, normalisation: `normalized` modes are undone here).  onesided descriptors only.
 *   spec      : complex64, logical [rows][n_fft/2+1][frames], strides in complex elements
 *   frame_buf : caller-owned scratch of rows * frames * n_fft floats (the windowed time frames)
 *   out       : [rows] signals of out_len samples, row r at out + r*out_row_stride
 * The caller checks the window envelope (NOLA) -- torch raises when its minimum is < 1e-11; this library divides.
 */
int b200a_istft_run(const b200a_frontend_desc* desc, const void* workspace, const float* spec, int64_t rows,
                    int64_t frames, int64_t stride_row, int64_t stride_bin, int64_t stride_frame,
                    float* frame_buf, float* out, int64_t out_row_stride, int64_t start, int64_t out_len,
                    b200a_stream stream);

/*
 * Spectrogram gradient of b200a_istft_run (the backward of torch.istft as F.inverse_spectrogram calls it), with the
 * workspace the forward ran with.  With X = scale * DFT(w * frame) the forward normalisation, N = n_fft,
 * env[s] = sum_t w^2[s - t hop] and g the upstream gradient of the returned samples:
 *   g_hat[s] = g[s - start] / env[s] for start <= s < start + g_len and s < N + hop (frames - 1), else 0;
 *   grad_spec[t][k] = c_k / (N scale) * sum_n w[n] g_hat[t hop + n] e^(-2 pi i k n / N),
 *   c_0 = 1, c_{N/2} = 1 (even N), c_k = 2 otherwise: the imaginary parts at bins 0 and N/2 are exactly 0
 * (torch's complex-gradient convention dL/dRe + i dL/dIm).  `start` counts the returned signal's offset in the
 * overlap-added one: n_fft/2 when centred, plus the `pad` F.inverse_spectrogram slices off.
 *   grad      : [rows] rows of g_len floats, row r at grad + r * g_row_stride (0 allowed: expanded gradients)
 *   scratch   : caller-owned device memory of b200a_istft_backward_scratch_bytes(desc, rows, frames) bytes (NULL when 0)
 *   grad_spec : complex64, frame-major [rows][frames][n_fft/2+1] (every element written)
 * Deterministic: no atomics, every row independent of the others.  onesided descriptors only; any n_fft (one kernel for
 * 256 / 512 / 1024 with hop <= ~n_fft, three for every other size).
 */
int b200a_istft_backward(const b200a_frontend_desc* desc, const void* workspace, const float* grad, int64_t rows,
                         int64_t g_row_stride, int64_t start, int64_t g_len, int64_t frames, void* scratch, float* grad_spec,
                         b200a_stream stream);
/* Bytes of scratch b200a_istft_backward needs: 0 on the register-FFT path, rows * (N + hop (frames - 1)) floats of g_hat
 * otherwise; also 0 for an invalid request (which b200a_istft_backward then rejects). */
size_t b200a_istft_backward_scratch_bytes(const b200a_frontend_desc* desc, int64_t rows, int64_t frames);

/*
 * One phase step of F.griffinlim (functional/functional.py:330-341):
 *   proj = mag^inv_power * angles,  angles = d / (|d| + 1e-16),  d = rebuilt - momentum * tprev
 * with angles = 1 when rebuilt is NULL (the first inversion, rand_init = False), d = rebuilt when tprev is NULL, and
 * angles = rebuilt as is when normalize == 0 (the first inversion with a random initial phase, :310-311).
 *   mag                   : |X|^power, logical [rows][bins][frames] with element strides (the user's tensor)
 *   rebuilt, tprev, proj  : complex64 frame-major [rows][frames][bins] (what b200a_frontend_run(COMPLEX) writes and
 *                           b200a_istft_run reads with strides (frames*bins, 1, bins))
 */
int b200a_griffinlim_update(const float* mag, int64_t stride_row, int64_t stride_bin, int64_t stride_frame,
                            float inv_power, const float* rebuilt, const float* tprev, float momentum,
                            int32_t normalize, float* proj, int64_t rows, int64_t bins, int64_t frames,
                            b200a_stream stream);

/*
 * F.phase_vocoder (functional/functional.py:713-803): time-stretch a complex spectrogram by `rate` without changing
 * pitch.  Output frame t' interpolates the magnitudes of input frames trunc(ts), trunc(ts + 1), ts = float(rate * t'),
 * and carries the accumulated phase advance; frames_out = ceil(frames_in / rate) (torch.arange(0, frames_in, rate)).
 *   spec          : complex64, logical [rows][bins][frames_in], strides in complex elements
 *   phase_advance : [bins] expected phase advance per hop (linspace(0, pi * hop, bins))
 *   out           : complex64 frame-major [rows][frames_out][bins]
 */
int b200a_phase_vocoder(const float* spec, int64_t stride_row, int64_t stride_bin, int64_t stride_frame, int64_t rows,
                        int64_t bins, int64_t frames_in, double rate, const float* phase_advance, float* out,
                        int64_t frames_out, b200a_stream stream);
/*
 * Spectrogram gradient of b200a_phase_vocoder: grad_spec = dL/dRe X + i dL/dIm X for the upstream gradient g of `out`,
 * torch's complex autograd convention.  With the forward's time grid (i0(t), i1(t), alpha_t) and o_t its output:
 *   a_t = Im g_t Re o_t - Re g_t Im o_t              (dL/dphi_t)
 *   m_t = Re(conj(g_t) sgn(o_t)), sgn(0) = 0         (dL/dmag_t)
 *   S_t = sum_{u >= t} a_u,  S_{frames_out} = 0      (adjoint of the phase cumsum; the last phase step is dropped)
 *   M_i = sum_{i0(t)=i} (1 - alpha_t) m_t + sum_{i1(t)=i} alpha_t m_t
 *   P_i = sum_{i1(t)=i} S_{t+1} - sum_{i0(t)=i} S_{t+1} + [i = 0] S_0
 *   grad_spec[i] = sgn(X_i) M_i + (i X_i / |X_i|^2) P_i,  exactly 0 at X_i = 0 (no NaN)
 * The phase wrap and phase_advance have zero gradient; contributions to the two zero pad frames are dropped, and frames
 * no step touches (rate > 2) get 0.
 *   spec      : the forward's input, logical [rows][bins][frames_in], strides in complex elements
 *   out       : the forward's output, complex64 frame-major [rows][frames_out][bins]
 *   grad      : logical [rows][bins][frames_out], strides in complex elements (0 allowed: expanded gradients)
 *   grad_spec : complex64 frame-major [rows][frames_in][bins] (every element written)
 * Deterministic: no atomics, every element written once by the thread of its (row, bin).  rows <= 65535.
 */
int b200a_phase_vocoder_backward(const float* spec, int64_t stride_row, int64_t stride_bin, int64_t stride_frame,
                                 int64_t rows, int64_t bins, int64_t frames_in, double rate, const float* out,
                                 const float* grad, int64_t g_stride_row, int64_t g_stride_bin, int64_t g_stride_frame,
                                 float* grad_spec, int64_t frames_out, b200a_stream stream);

/* ---- Kaldi-compatible features (compliance/kaldi.py: spectrogram :229-316, fbank :514-645, mfcc :669-813) -------- */
/*
 * Per-frame conditioning and output placement of the Kaldi front end; the transform itself (window, FFT size,
 * |X| or |X|^2, mel matrix) is described by a b200a_frontend_desc with center = 0, n_fft = win_length = padded_size,
 * hop = window_shift, and a workspace prepared by b200a_frontend_prepare from
 *   window : [padded_size]  the Kaldi window (_feature_window_function, :86-113) followed by zeros (:206-211)
 *   fb     : [padded_size/2+1][n_mels]  get_mel_banks(...) transposed, last row zero (:436-511, :623-624), or NULL.
 */
typedef struct b200a_kaldi_desc {
  int32_t window_size;      /* samples per frame, int(sample_frequency * frame_length * 0.001)          (:139) */
  int32_t window_shift;     /* int(sample_frequency * frame_shift * 0.001)                             (:138) */
  int32_t padded_size;      /* FFT size: next power of two of window_size, or window_size; even        (:140) */
  int32_t snip_edges;       /* 1: only frames inside the signal; 0: mirror-extended signal             (:44-83) */
  int32_t remove_dc_offset; /* subtract each frame's mean                                              (:181-184) */
  float preemphasis;        /* s[j] -= c * s[max(0, j-1)]; 0 disables                                  (:191-197) */
  int32_t energy_mode;      /* 0 none, 1 raw (after DC removal, before pre-emphasis), 2 after the window (:186-189,:213-215) */
  float energy_floor;       /* log energy >= log(energy_floor); 0: no floor                            (:116-123) */
  int32_t energy_col;       /* output column that receives the log energy, -1: none                   */
  int32_t out_width;        /* floats per output frame                                                 */
  int32_t out_col0;         /* output column of the first spectral / mel value                         */
  int32_t use_log;          /* log(max(v, FLT_EPSILON)) on the spectral / mel values                   (:310, :629-631) */
} b200a_kaldi_desc;

/* m of _get_strided (:62-68): 1 + (L - win)/shift (0 if L < win) when snip_edges, else (L + shift/2)/shift. */
int64_t b200a_kaldi_num_frames(int64_t length, int32_t window_size, int32_t window_shift, int32_t snip_edges);

/*
 * Fused Kaldi front end: frames -> DC removal -> [raw log energy] -> pre-emphasis -> window -> zero pad -> rFFT ->
 * |X|^power -> [mel] -> [log] for `rows` signals.  stage = B200A_STAGE_POWER (spectrogram) or B200A_STAGE_MEL (fbank).
 *   out : [rows][m][out_width]; spectral value k goes to column out_col0 + k unless that is energy_col.
 * Dither is not offered: the reference draws it with torch.randn per frame element (:176-178), which no
 * other generator reproduces; callers pass dither = 0.
 */
int b200a_kaldi_run(const b200a_kaldi_desc* kaldi, const b200a_frontend_desc* desc, const void* workspace,
                    int32_t stage, const float* wave, int64_t rows, int64_t length, int64_t row_stride,
                    float* out, b200a_stream stream);

/*
 * Waveform gradient of b200a_kaldi_run (stage POWER or MEL): torch's autograd of the reference op sequence, ties
 * included -- log(max(v, FLT_EPSILON)) gives 1/v above, half of 1/FLT_EPSILON on the tie and 0 below, and the energy
 * floor splits the same way; the decisions are taken from the pre-log values recomputed by the forward's own kernel.
 *   grad_out  : [rows][m][out_width] at element strides g_stride_* (0 allowed: an expanded gradient)
 *   grad_wave : [rows][length] at row stride grad_row_stride >= length; every sample is written
 *   scratch   : b200a_kaldi_backward_scratch_bytes(...) bytes
 * Status codes as b200a_kaldi_run; B200A_EINVAL also for a null grad_out, scratch or grad_wave.  No atomics: reruns
 * are bit-identical and a row's gradient does not depend on the other rows.
 */
int b200a_kaldi_backward(const b200a_kaldi_desc* kaldi, const b200a_frontend_desc* desc, const void* workspace,
                         int32_t stage, const float* wave, int64_t rows, int64_t length, int64_t row_stride,
                         const float* grad_out, int64_t g_stride_row, int64_t g_stride_frame, int64_t g_stride_col,
                         void* scratch, float* grad_wave, int64_t grad_row_stride, b200a_stream stream);
/* Scratch bytes of b200a_kaldi_backward: the recomputed pre-log rows, the per-frame energy gradient and NaN flag, the
 * complex spectrum and the frame gradients (rows * m * padded_size floats).  0 for an invalid request. */
size_t b200a_kaldi_backward_scratch_bytes(const b200a_kaldi_desc* kaldi, const b200a_frontend_desc* desc, int32_t stage,
                                          int64_t rows, int64_t length);

/* x[r][t][c] -= mean_t x[r][t][c], in place, for each of `rows` feature matrices (_subtract_column_mean, :219-226). */
int b200a_subtract_column_mean(float* x, int64_t rows, int64_t frames, int64_t width, b200a_stream stream);

/* ---- InverseMelScale (transforms/_transforms.py:418-503) ------------------------------------------------------- */
/*
 * x = relu(lstsq(fb^T, m).solution) per frame.  For n_mels <= n_stft and a nonsingular Gram matrix G = fb^T fb every
 * LAPACK driver returns the minimum-norm solution x = relu(fb G^-1 m).  A bin of a mel (or linear) bank overlaps at most
 * two adjacent filters, so G is banded; the plan factors it as banded L D L^T.
 */
#define B200A_INVERSE_MEL_MAX_BANDWIDTH 4 /* Gram bandwidth cap (mel and LFCC linear banks have 1) */
#define B200A_INVERSE_MEL_MAX_MELS 512    /* n_mels cap: the backward stages two 32-frame tiles in shared memory */
enum b200a_lstsq_driver { B200A_GELS = 0, B200A_GELSY = 1, B200A_GELSD = 2, B200A_GELSS = 3 };

/* Bytes of the plan blob for this size (its layout depends on n_stft and n_mels alone); 0 for non-positive sizes. */
size_t b200a_inverse_mel_plan_bytes(int32_t n_stft, int32_t n_mels);
/*
 * HOST-only: build the plan from a HOST copy of fb ([n_stft][n_mels], row-major float32; the caller copies it from the
 * device once per fb version and uploads the blob once).  In double precision: each bin's nonzero filter span and each
 * filter's nonzero bin span (read from fb, any bank), the Gram bandwidth, then G = L D L^T; stored as float32 factors
 * (L, 1/D), the per-bin table (first filter, count, fb values) and the per-filter table (first bin, count).
 *   plan      : HOST buffer of b200a_inverse_mel_plan_bytes(n_stft, n_mels) bytes (B200A_EWORKSPACE if smaller)
 *   bandwidth : out, the Gram bandwidth found (-1 if not reached)
 *   pivot     : out, the first zero pivot (0-based filter) on B200A_ESINGULAR, or for an overdetermined bank with gels
 *               the first empty bin; else -1
 * Returns B200A_ESINGULAR for a singular G (n_mels <= n_stft; the gels driver fails there too) and for n_mels > n_stft
 * with B200A_GELS and an all-zero bin; B200A_EUNSUPPORTED for any other n_mels > n_stft, a bandwidth above
 * B200A_INVERSE_MEL_MAX_BANDWIDTH or n_mels above B200A_INVERSE_MEL_MAX_MELS; B200A_EINVAL for null pointers,
 * non-positive sizes or a bad driver.
 */
int b200a_inverse_mel_plan(const float* fb, int32_t n_stft, int32_t n_mels, int32_t driver, void* plan, size_t plan_bytes,
                           int32_t* bandwidth, int32_t* pivot);
/*
 * out[r][t][k] = relu(sum_m fb[k][m] z[r][t][m]),  G z[r][t] = mel[r][:, t]  (one banded solve per frame, FP32)
 *   plan : the blob of b200a_inverse_mel_plan in DEVICE memory
 *   mel  : logical [rows][n_mels][frames] at element strides (the frame-major view MelSpectrogram returns and a
 *          contiguous tensor both load coalesced)
 *   out  : FRAME-MAJOR [rows][frames][n_stft], every element written
 */
int b200a_inverse_mel_run(const void* plan, int32_t n_stft, int32_t n_mels, const float* mel, int64_t rows, int64_t frames,
                          int64_t stride_row, int64_t stride_mel, int64_t stride_frame, float* out, b200a_stream stream);
/*
 * Mel gradient of b200a_inverse_mel_run: z and the pre-relu values are recomputed by the forward's code (the relu mask
 * is bit-identical to the forward's), u[m] = sum_{k in filter m} fb[k][m] [x_k > 0] g[k] in a fixed order, then
 * grad_mel = G^-1 u with the same factors.  No atomics: reruns are bit-identical.
 *   grad     : logical [rows][frames][n_stft] at element strides (0 allowed: expanded gradients)
 *   grad_mel : FRAME-MAJOR [rows][frames][n_mels], every element written
 */
int b200a_inverse_mel_backward(const void* plan, int32_t n_stft, int32_t n_mels, const float* mel, int64_t rows,
                               int64_t frames, int64_t stride_row, int64_t stride_mel, int64_t stride_frame,
                               const float* grad, int64_t g_stride_row, int64_t g_stride_frame, int64_t g_stride_bin,
                               float* grad_mel, b200a_stream stream);

/* ---- IIR filtering: lfilter (functional/filtering.py:1032-1099) ------------------------------------------------ */
/*
 * Rows are (batch, filter) pairs, row r = bi * n_filters + f uses filter f.  With n_order coefficients (filter order
 * N = n_order - 1) and the float32-normalised coefficients a^ = a / a0, b^ = b / a0 (one float division each, as the
 * reference normalises):
 *   v[t] = sum_{k=0..N} b^_k x[t-k],   y[t] = v[t] - sum_{k=1..N} a^_k y[t-k],   zero history before t = 0;
 * with `reverse` the recurrence runs from t = length-1 downward (x[t+k], y[t+k], zero history past the end), which is
 * filtfilt's second pass without flip copies.  `clamp` applies clamp(y, -1, 1) once at the end.
 * The recurrence is a chunked scan: every thread runs 32 samples serially from a zero history, chunk and tile carries
 * are joined through the N-sample output history with the carry map M and its powers built from a^ in DOUBLE, and
 * each chunk re-runs from its true starting history rounded to float32.  The scan order is fixed and the chunk length
 * depends on N alone: reruns are bit-identical and a row's output does not depend on the other rows.  No atomics.
 */
#define B200A_LFILTER_MAX_ORDER 16 /* filter order cap N = n_order - 1 (B200A_EUNSUPPORTED above) */

/* Workspace bytes of b200a_lfilter_run for `rows` = batch * n_filters rows of `length` samples; 0 for an invalid or
 * unsupported request.  b200a_lfilter_backward needs b200a_lfilter_backward_workspace_bytes instead. */
size_t b200a_lfilter_workspace_bytes(int64_t rows, int64_t length, int32_t n_order, int32_t n_filters);
size_t b200a_lfilter_backward_workspace_bytes(int64_t rows, int64_t length, int32_t n_order, int32_t n_filters);
/*
 *   a, b        : DEVICE [n_filters][n_order] raw coefficients (read on the device: no host synchronisation)
 *   x           : row (bi, f) at x + bi * stride_batch + f * stride_filter, unit element stride; stride_filter may be 0
 *                 (one waveform row for every filter: batching=False without a stacked copy)
 *   y           : [batch][n_filters][length] contiguous, every element written (clamped when `clamp`)
 *   y_unclamped : the same before the clamp, or NULL
 * B200A_EINVAL for null pointers, non-positive n_order / n_filters or negative sizes; B200A_EUNSUPPORTED for
 * n_order - 1 > B200A_LFILTER_MAX_ORDER; B200A_EWORKSPACE when workspace_bytes is too small.  batch == 0 or
 * length == 0 enqueues nothing.
 */
int b200a_lfilter_run(const float* a, const float* b, int32_t n_filters, int32_t n_order, const float* x, int64_t batch,
                      int64_t length, int64_t stride_batch, int64_t stride_filter, int32_t clamp, int32_t reverse,
                      float* y, float* y_unclamped, void* workspace, size_t workspace_bytes, b200a_stream stream);
/*
 * Gradients of b200a_lfilter_run.  g_y = grad * (-1 <= y_unclamped <= 1) when `clamp` (torch.clamp's inclusive rule),
 * else grad; u = the IIR recurrence run in the opposite direction on g_y (the mask is fused into its input read);
 *   grad_x[t] = sum_k b^_k u[t+k],  d a^_k = -sum_t u[t] y[t-k],  d b^_k = sum_t u[t] x[t-k]  (k toward the past of
 * the forward's direction), the last two summed over the rows of each filter, then taken through a0 to the raw a, b.
 *   y_unclamped : [batch][n_filters][length] contiguous (the forward's unclamped output)
 *   grad        : [batch][n_filters][length] contiguous
 *   grad_x      : [batch][n_filters][length] contiguous, or NULL;  grad_a, grad_b : [n_filters][n_order], or NULL
 * The coefficient gradients are reduced over rows and tiles in a fixed order (double partial sums): reruns are
 * bit-identical, and grad_x of a row does not depend on the other rows.  Statuses as b200a_lfilter_run.
 */
int b200a_lfilter_backward(const float* a, const float* b, int32_t n_filters, int32_t n_order, const float* x,
                           int64_t batch, int64_t length, int64_t stride_batch, int64_t stride_filter,
                           const float* y_unclamped, const float* grad, int32_t clamp, int32_t reverse, float* grad_x,
                           float* grad_a, float* grad_b, void* workspace, size_t workspace_bytes, b200a_stream stream);

/* ---- FFT convolution: fftconvolve (functional/functional.py:2189-2258) ------------------------------------------ */
/*
 * out[r][i] = sum_k x_r[k] y_r[start + i - k],  i < out_len, the slice [start, start + out_len) of the full
 * (n + m - 1)-sample linear convolution of output row r's operands x_r = x + x_index[r] * x_stride (n samples) and
 * y_r = y + y_index[r] * y_stride (m samples).  The index vectors express broadcasting: operand rows shared by several
 * output rows are transformed once.
 * Uniformly partitioned overlap-save: the shorter operand (the filter, K = min(n, m) taps; y when n == m) is cut into
 * P = ceil(K / B) partitions of B samples, B = the next power of two of K clamped to [256, 2048], and every FFT is 2B
 * points.  B depends on K alone and every sum runs in a fixed order without atomics: reruns are bit-identical and a
 * row's output does not depend on the other rows.
 */
#define B200A_FFTCONVOLVE_MAX_PARTITIONS 128 /* P cap: filters up to 128 * 2048 = 262144 taps (B200A_EUNSUPPORTED above) */

typedef struct b200a_fftconvolve_desc {
  int64_t n, m;            /* operand lengths, >= 1 each; n + m - 1 <= INT32_MAX */
  int64_t out_len, start;  /* the output slice of the full range: start >= 0, start + out_len <= n + m - 1 */
  int64_t rows;            /* output rows */
  int64_t x_rows, y_rows;  /* operand rows (>= 1); x_index[r] < x_rows, y_index[r] < y_rows */
  const int64_t* x_index;  /* DEVICE [rows] */
  const int64_t* y_index;  /* DEVICE [rows] */
  int64_t x_stride, y_stride; /* element stride between operand rows; unit stride in time */
} b200a_fftconvolve_desc;

/* Workspace bytes of b200a_fftconvolve_run / b200a_fftconvolve_backward for `desc`; 0 for an invalid or unsupported
 * descriptor. */
size_t b200a_fftconvolve_workspace_bytes(const b200a_fftconvolve_desc* desc);
size_t b200a_fftconvolve_backward_workspace_bytes(const b200a_fftconvolve_desc* desc);
/*
 *   out : [rows][out_len] contiguous, every element written once
 * B200A_EINVAL for a null pointer, a length < 1, negative sizes or strides, or a slice outside the full range;
 * B200A_EUNSUPPORTED above B200A_FFTCONVOLVE_MAX_PARTITIONS or for n + m - 1 > INT32_MAX; B200A_EWORKSPACE when
 * workspace_bytes is too small.  rows == 0 or out_len == 0 enqueues nothing.
 */
int b200a_fftconvolve_run(const b200a_fftconvolve_desc* desc, const float* x, const float* y, float* out,
                          void* workspace, size_t workspace_bytes, b200a_stream stream);
/*
 * Gradients of b200a_fftconvolve_run for the upstream gradient g = grad[r] placed at `start` of the full range (zero
 * elsewhere), per OUTPUT row:  grad_x[r][k] = sum_j g[k + j] y_r[j],  grad_y[r][j] = sum_k g[k + j] x_r[k].  The
 * caller sums the rows that share an operand.
 *   grad   : [rows][out_len] contiguous
 *   grad_x : [rows][n] contiguous;  grad_y : [rows][m] contiguous
 * Statuses as b200a_fftconvolve_run; out_len == 0 zero-fills both gradients.
 */
int b200a_fftconvolve_backward(const b200a_fftconvolve_desc* desc, const float* x, const float* y, const float* grad,
                               float* grad_x, float* grad_y, void* workspace, size_t workspace_bytes,
                               b200a_stream stream);

/* ---- direct convolution: convolve (functional/functional.py:2261-2314) ------------------------------------------ */
/*
 * The same result as b200a_fftconvolve_run, by the direct method: the filter (the shorter operand, K = min(n, m) taps;
 * y when n == m) times the signal as a banded Toeplitz product on TF32 x 3 tensor-core MMAs (round-to-nearest splits
 * and per-k-step round-to-nearest accumulation: float32 grade), 128 consecutive outputs per m16n8 tile over ceil((K + 7) / 8) k-steps.  Tile sizes depend on K alone and
 * nothing is atomic: reruns are bit-identical and a row's output does not depend on the other rows.  The descriptor is
 * b200a_fftconvolve_desc with the same meaning.
 */
#define B200A_CONVOLVE_MAX_TAPS 4096 /* K cap (B200A_EUNSUPPORTED above): past it fftconvolve does less work */

typedef b200a_fftconvolve_desc b200a_convolve_desc;

/* Workspace bytes of b200a_convolve_run / b200a_convolve_backward for `desc`; 0 for an invalid or unsupported
 * descriptor. */
size_t b200a_convolve_workspace_bytes(const b200a_convolve_desc* desc);
size_t b200a_convolve_backward_workspace_bytes(const b200a_convolve_desc* desc);
/*
 *   out : [rows][out_len] contiguous, every element written once
 * B200A_EINVAL for a null pointer, a length < 1, negative sizes or strides, or a slice outside the full range;
 * B200A_EUNSUPPORTED for K > B200A_CONVOLVE_MAX_TAPS or n + m - 1 > INT32_MAX; B200A_EWORKSPACE when workspace_bytes
 * is too small.  rows == 0 or out_len == 0 enqueues nothing.
 */
int b200a_convolve_run(const b200a_convolve_desc* desc, const float* x, const float* y, float* out, void* workspace,
                       size_t workspace_bytes, b200a_stream stream);
/*
 * Gradients of b200a_convolve_run, per OUTPUT row, as b200a_fftconvolve_backward defines them:
 *   grad_x[r][k] = sum_j g[k + j] y_r[j],  grad_y[r][j] = sum_k g[k + j] x_r[k]
 * with g = grad[r] placed at `start` of the full range.  The signal gradient is the forward kernel on g with the
 * reversed filter; the filter gradient is a tensor-core correlation per 2048-sample tile, whose partials are summed in
 * tile order.  The caller sums the rows that share an operand.
 *   grad   : [rows][out_len] contiguous
 *   grad_x : [rows][n] contiguous;  grad_y : [rows][m] contiguous
 * Statuses as b200a_convolve_run; out_len == 0 zero-fills both gradients.
 */
int b200a_convolve_backward(const b200a_convolve_desc* desc, const float* x, const float* y, const float* grad,
                            float* grad_x, float* grad_y, void* workspace, size_t workspace_bytes, b200a_stream stream);

/* ---- voice-activity trim: vad (functional/filtering.py:1414-1702) ---------------------------------------------- */
/*
 * The measurement loop of SoX's vad, run over `frames` consecutive measurement frames (a chunk) of `channels` channels
 * at a time.  Per frame f (global index g = frame0 + f) and channel c:
 *   1. |X| = b200a_frontend_run(B200A_STAGE_POWER, power 1) of the frame (the caller's pass: n_fft = dft_len,
 *      win_length = measure_len_ws, hop = period, center 0)
 *   2. b200a_vad_walk, per bin k of [spectrum_start, spectrum_end), in float32 with one rounding per operation:
 *        mult = b / (1 + b) while booting (b = g while g <= boot_count_max, or always when that is negative), else
 *        measure_smooth_mult;  S = S mult + |X| (1 - mult);  d = S^2;  nm = 0 while booting, else (d > N ? up : down);
 *        N = N nm + d (1 - nm);  r = sqrt(max(0, d - noise_reduction_amount N));  row[k] = r * cepstrum_window[k - s0]
 *   3. P = b200a_frontend_run(B200A_STAGE_MEL) of the rows (the caller's pass: n_fft = win_length = hop = dft_len / 2,
 *      window of ones, power 2, one filter of ones on [cepstrum_start, cepstrum_end))
 *   4. b200a_vad_trigger: meas = max(0, 21 + log(P / (cepstrum_end - cepstrum_start))) in double (0 for P <= 0), stored
 *      as float32;  mean = mean * trigger_mult + meas * (1 - trigger_mult) in float32;  the first (frame, channel) in
 *      frame-major order with mean >= trigger_level triggers, and the reference's flush scan over the last
 *      measures_len measures runs for that channel and every later one at that frame.
 * Chunks must be run in order on one workspace: frame0 == 0 starts from zero state, a later chunk continues the state
 * the previous one left exactly.  (The front end packs two frames into one complex FFT within a launch, so |X| and P
 * next to a chunk edge can differ in the last bits from a run with other chunk boundaries.)
 */
typedef struct b200a_vad_desc {
  int32_t channels;                      /* >= 1 */
  int32_t dft_len;                       /* power of two, 16..8192 (B200A_EUNSUPPORTED above) */
  int32_t spectrum_start, spectrum_end;  /* 1 <= start <= end <= dft_len / 2 */
  int32_t cepstrum_start, cepstrum_end;  /* 0 <= start < end <= dft_len / 4 */
  int32_t measures_len;                  /* ring length ceil(search_time * measure_freq) >= 1 */
  int32_t gap_len;                       /* int(allowed_gap * measure_freq + 0.5) */
  int32_t boot_count_max;                /* int(boot_time * measure_freq - 0.5) */
  int32_t period;                        /* measure_period_ns >= 1 */
  int64_t fixed_pre_trigger;             /* fixed_pre_trigger_len_ns */
  double noise_up_mult, noise_down_mult; /* rounded to float32 where used, as the reference's float32 tensors */
  double noise_reduction_amount;
  double measure_smooth_mult, trigger_mult;
  double trigger_level;                  /* compared in float32 */
} b200a_vad_desc;

/* Workspace bytes for `chunk` frames per call: the 16-byte status, the carried spectra, means and measure ring, and
 * per-chunk scratch; 0 for an invalid or unsupported descriptor. */
size_t b200a_vad_workspace_bytes(const b200a_vad_desc* desc, int64_t chunk);
/*
 *   spectrum        : [channels][frames][dft_len / 2 + 1] |X| of the chunk's frames
 *   cepstrum_window : [spectrum_end - spectrum_start]
 *   rows            : [channels][chunk][dft_len / 2]; bins [spectrum_start, spectrum_end) of the first `frames` rows
 *                     of each channel are written, the rest is left as it is (the caller zeroes it once)
 */
int b200a_vad_walk(const b200a_vad_desc* desc, int64_t chunk, int64_t frame0, int64_t frames, const float* spectrum,
                   const float* cepstrum_window, float* rows, void* workspace, size_t workspace_bytes,
                   b200a_stream stream);
/*
 *   power    : [channels][frames] cepstral band powers P
 *   measures : [channels][frames] the measures, float32
 * Writes the workspace's first 16 bytes: int64 {g, start} with g the triggering frame and start the first sample the
 * trim keeps, or {-1, 0} when no frame of the chunk triggered.  One CTA; no atomics.
 * Both calls: B200A_EINVAL for a null pointer or descriptor, a field outside its range, frame0 < 0 or frames outside
 * [0, chunk]; B200A_EUNSUPPORTED for dft_len > 8192, more than 65535 channels or chunk > 2^20; B200A_EWORKSPACE when
 * workspace_bytes is too small.  frames == 0 enqueues nothing.
 */
int b200a_vad_trigger(const b200a_vad_desc* desc, int64_t chunk, int64_t frame0, int64_t frames, const float* power,
                      float* measures, void* workspace, size_t workspace_bytes, b200a_stream stream);

/* ---- RNN-T loss: rnnt_loss (functional.py:1747-1796, rnnt/cpu/cpu_kernels.h) -------------------------------- */
/*
 * The transducer loss of a joiner output logits[batch][max_t][max_u][classes] (max_u = max target length + 1) in
 * float32 or float16; every step is float32.  Per sequence b with T = logit_lengths[b] >= 1 and U =
 * target_lengths[b] + 1, on the valid rows t < T, u < U:
 *   denom(t, u) = log sum_k exp(logits[b][t][u][k])                         (fused only)
 *   skip(t, u) = logits[..][blank] - denom,  emit(t, u) = logits[..][targets[b][u]] - denom  (u < U - 1; raw logits
 *   when fused == 0);  alpha / beta by the reference's recursions and lse (max + log1p(exp(min - max)), so the lse of
 *   two -inf is NaN);  cost[b] = -beta(0, 0).
 * The logit gradient (b200a_rnnt_loss_backward) is the reference CPU's formula per element, clamped to [-clamp, clamp]
 * when clamp > 0, times grad_costs[b]; rows outside (T, U) and every row of a sequence whose cost is not finite are 0.
 * No atomics in the loss kernels: reruns are bit-identical.
 */
#define B200A_DTYPE_F32 0
#define B200A_DTYPE_F16 1
#define B200A_RNNT_MAX_U 8192 /* max_u cap (B200A_EUNSUPPORTED above): the alpha / beta CTA stages 24 bytes per column */

typedef struct b200a_rnnt_loss_desc {
  int32_t batch;   /* >= 1 */
  int32_t max_t;   /* logits.shape[1] = max(logit_lengths) >= 1 */
  int32_t max_u;   /* logits.shape[2] = max(target_lengths) + 1; targets is [batch][max_u - 1] */
  int32_t classes; /* >= 1 */
  int32_t blank;   /* in [0, classes) */
  int32_t dtype;   /* B200A_DTYPE_F32 or B200A_DTYPE_F16: logits, costs, grad_costs and grad_logits */
  int32_t fused;   /* 1: log-softmax inside the loss; 0: the logits are log-probabilities already */
  float clamp;     /* gradient clamp when > 0 */
} b200a_rnnt_loss_desc;

/*
 * Input check, one CTA: out[0..4] = {max, min of logit_lengths; max, min of target_lengths; 1 if a target
 * targets[b][j] with j < target_lengths[b] (and j < target_cols) lies outside [0, classes), else 0}.  batch == 0 gives
 * {INT32_MIN, INT32_MAX, INT32_MIN, INT32_MAX, 0}.  targets is [batch][target_cols] contiguous.
 */
int b200a_rnnt_loss_check(int32_t batch, int32_t classes, const int32_t* targets, int64_t target_cols,
                          const int32_t* logit_lengths, const int32_t* target_lengths, int32_t* out,
                          b200a_stream stream);
/* Workspace bytes of b200a_rnnt_loss_forward: the (skip, emit) pair of every row; 0 for an invalid descriptor. */
size_t b200a_rnnt_loss_workspace_bytes(const b200a_rnnt_loss_desc* desc);
/*
 *   costs              : [batch] in the logits' dtype
 *   denom, alpha, beta : [batch][max_t][max_u] float32, the valid rows written; all null for a forward without a
 *                        gradient (only beta is walked), else alpha and beta, and denom when fused
 * The lengths and targets must have passed b200a_rnnt_loss_check's conditions (lengths within the shape, T >= 1,
 * U >= 1, targets in range); nothing here reads them back.  B200A_EINVAL for null pointers or fields out of range,
 * B200A_EUNSUPPORTED for max_u > B200A_RNNT_MAX_U, B200A_EWORKSPACE for a short workspace.
 */
int b200a_rnnt_loss_forward(const b200a_rnnt_loss_desc* desc, const void* logits, const int32_t* targets,
                            const int32_t* logit_lengths, const int32_t* target_lengths, void* costs, float* denom,
                            float* alpha, float* beta, void* workspace, size_t workspace_bytes, b200a_stream stream);
/*
 * grad_logits[b][t][u][k] for every element, written once; grad_costs[b * grad_costs_stride] (0: an expanded scalar).
 * denom may be null when fused == 0.  Statuses as b200a_rnnt_loss_forward.
 */
int b200a_rnnt_loss_backward(const b200a_rnnt_loss_desc* desc, const void* logits, const int32_t* targets,
                             const int32_t* logit_lengths, const int32_t* target_lengths, const float* denom,
                             const float* alpha, const float* beta, const void* grad_costs, int64_t grad_costs_stride,
                             void* grad_logits, b200a_stream stream);

/* ---- CTC forced alignment: forced_align (functional/_alignment.py, forced_align/cpu/compute.cpp) --------------- */
/*
 * The Viterbi alignment of targets[batch][max_l] to log_probs[batch][max_t][classes] (float32, float16 or float64),
 * per sequence b with T_b = input_lengths[b] >= 1 and L_b = target_lengths[b]: the reference CPU's band, its tie rules
 * and its arithmetic in the input dtype, so every row equals the reference's alignment of that row alone, bit for bit.
 *   paths  : [batch][max_t] in the targets' dtype; frames t >= T_b hold blank, a row with L_b = 0 is all blank
 *   scores : [batch][max_t] in the log-probs' dtype, log_probs[b][t][paths[b][t]]; 0 for t >= T_b
 * One CTA per sequence in one launch, no atomics: reruns are bit-identical.
 */
#define B200A_DTYPE_F64 2
#define B200A_INDEX_I32 0
#define B200A_INDEX_I64 1
/* max_l cap (B200A_EUNSUPPORTED above): 2 max_l + 1 states in the registers of 512 threads */
#define B200A_FORCED_ALIGN_MAX_L 8191

typedef struct b200a_forced_align_desc {
  int32_t batch;        /* >= 1 */
  int32_t max_t;        /* log_probs.shape[1] >= 1 */
  int32_t max_l;        /* targets.shape[1] >= 0 */
  int32_t classes;      /* >= 1 */
  int32_t blank;        /* in [0, classes) (any value for b200a_forced_align_check) */
  int32_t dtype;        /* B200A_DTYPE_F32, B200A_DTYPE_F16 or B200A_DTYPE_F64: log_probs and scores */
  int32_t target_dtype; /* B200A_INDEX_I32 or B200A_INDEX_I64: targets and paths */
  int32_t length_dtype; /* B200A_INDEX_I32 or B200A_INDEX_I64: input_lengths and target_lengths */
} b200a_forced_align_desc;

/*
 * Input check, one CTA: out[0..10] = {max, min of input_lengths; max, min of target_lengths; 1 if a target
 * targets[b][j] with j < min(target_lengths[b], max_l) is >= classes, else 0; the same for < 0; the same for == blank;
 * the first b with input_lengths[b] < target_lengths[b] + R_b (R_b: the repeats targets[b][j] == targets[b][j - 1]
 * among those targets) or -1, and that sequence's (T_b, L_b, R_b)}.  Writes R_b as int32 to workspace[0 .. batch), the
 * walk's input: the workspace of b200a_forced_align_run, or at least 4 * batch bytes.  Accepts max_l above the cap.
 */
int b200a_forced_align_check(const b200a_forced_align_desc* desc, const void* targets, const void* input_lengths,
                             const void* target_lengths, int64_t* out, void* workspace, size_t workspace_bytes,
                             b200a_stream stream);
/* Workspace bytes of b200a_forced_align_run (R_b and 2-bit backpointers per frame and state); 0 for an invalid
 * descriptor or max_l above B200A_FORCED_ALIGN_MAX_L. */
size_t b200a_forced_align_workspace_bytes(const b200a_forced_align_desc* desc);
/*
 * The workspace must hold b200a_forced_align_check's R_b for these targets and lengths, and the lengths must have
 * passed its conditions (1 <= T_b <= max_t, 0 <= L_b <= max_l, T_b >= L_b + R_b, targets in [0, classes)); nothing here
 * reads them back.  B200A_EINVAL for null pointers or fields out of range, B200A_EUNSUPPORTED for max_l above
 * B200A_FORCED_ALIGN_MAX_L, B200A_EWORKSPACE for a short workspace.
 */
int b200a_forced_align_run(const b200a_forced_align_desc* desc, const void* log_probs, const void* targets,
                           const void* input_lengths, const void* target_lengths, void* paths, void* scores,
                           void* workspace, size_t workspace_bytes, b200a_stream stream);

/* ---- CUDA CTC prefix beam search: cuda_ctc_decoder (models/decoder/_cuda_ctc_decoder.py, cuctc/) ------------- */
/*
 * The reference's CTC prefix beam search over log_prob[batch][max_t][vocab] (float32, contiguous), blank 0.  Per
 * sequence b with T_b = lengths[b], the steps are the frames t < T_b with log_prob[b][t][0] < threshold (the log of
 * the blank-skip threshold); candidates, merges and lse follow the reference's operation order, and among
 * bit-equal keys the lower beam * vocab + token wins (the stay entry counts as token 0).  Outputs, best first:
 *   tokens        : [batch][beam][max_t] int32; the first token_lengths[b][r] of each row are the hypothesis
 *   token_lengths : [batch][beam] int32
 *   scores        : [batch][beam] float32; a row without a selected frame has every hypothesis empty with score 0
 *   status        : [batch] int32; 1 where lengths[b] is outside [0, max_t] (that row is not read), else 0
 * One CTA per sequence in one launch, no atomics across CTAs: a row's result does not depend on the batch.
 */
/* beam cap (B200A_EINVAL above): one CTA's candidate list */
#define B200A_CTC_DECODER_MAX_BEAM 128
/* vocab cap (B200A_EINVAL above): beam * vocab + token in 31 bits */
#define B200A_CTC_DECODER_MAX_VOCAB (1 << 24)

typedef struct b200a_ctc_decoder_desc {
  int32_t batch;   /* >= 1 */
  int32_t max_t;   /* log_prob.shape[1] >= 0 */
  int32_t vocab;   /* log_prob.shape[2], in [1, B200A_CTC_DECODER_MAX_VOCAB] */
  int32_t beam;    /* in [1, min(vocab, B200A_CTC_DECODER_MAX_BEAM)] */
  float threshold; /* a frame is a step when log_prob[b][t][0] < threshold; not NaN */
} b200a_ctc_decoder_desc;

/* Workspace bytes of b200a_ctc_decoder_run (selected frames and the token trie); 0 for an invalid descriptor. */
size_t b200a_ctc_decoder_workspace_bytes(const b200a_ctc_decoder_desc* desc);
/* B200A_EINVAL for an invalid descriptor or null pointers (log_prob and tokens may be null when max_t is 0),
 * B200A_EWORKSPACE for a short workspace.  Nothing is read back: check status after the stream's work. */
int b200a_ctc_decoder_run(const b200a_ctc_decoder_desc* desc, const float* log_prob, const int32_t* lengths,
                          int32_t* tokens, int32_t* token_lengths, float* scores, int32_t* status, void* workspace,
                          size_t workspace_bytes, b200a_stream stream);

/* ---- SpecAugment masking: mask_along_axis(_iid), FrequencyMasking, TimeMasking, SpecAugment -------------------- */
/*
 * out[r][f][t] = fill where (f, t) lies in any mask of row r, else in[r][f][t] bit for bit (NaNs included), over
 * rows x freq x time float32 with 64-bit element strides; row r = r0 * rows1 + r1.  A mask covers the indices i of its
 * axis with (float)start <= (float)i < (float)end.  Its [start, end) is either shared by every row, or per row from two
 * uniform draws u, w (the reference's mask_along_axis_iid, in float32 without contraction):
 *   value = u[r] * (float)mask_param,  lo = w[r] * ((float)size - value),
 *   start = trunc(lo),  end = trunc(lo) + trunc(value)      (size: freq or time; start may be negative)
 * All masks of one call share the fill, so their union is what sequential application of each would give.
 * Tiles go through shared memory when the input's and the output's unit-stride axes differ, so both sides are
 * coalesced.  No atomics: reruns are bit-identical.
 */
#define B200A_MASK_AXIS_FREQ 0
#define B200A_MASK_AXIS_TIME 1

typedef struct b200a_mask_spec {
  int32_t axis;              /* B200A_MASK_AXIS_FREQ or B200A_MASK_AXIS_TIME */
  int32_t mask_param;        /* per-row masks: the limited mask_param, >= 1; unused for a shared interval */
  int64_t start, end;        /* the shared interval when value_draws is null */
  const float* value_draws;  /* per-row masks: [rows] device draws u, or null for the shared interval */
  const float* start_draws;  /* per-row masks: [rows] device draws w */
} b200a_mask_spec;

typedef struct b200a_mask_desc {
  int64_t rows0, rows1;      /* >= 0; rows = rows0 * rows1 */
  int64_t freq, time;        /* >= 0 */
  int64_t in_stride[4];      /* elements, for (r0, r1, f, t) */
  int64_t out_stride[4];
  int32_t n_masks;           /* >= 0 */
  float fill;                /* the fill when fill_ptr is null (b200a_mask_run) */
} b200a_mask_desc;

/* Workspace bytes of b200a_mask_run and b200a_mask_backward (the mask table and the backward's per-CTA partial
 * sums); 0 for an invalid descriptor. */
size_t b200a_mask_workspace_bytes(const b200a_mask_desc* desc);
/*
 * masks: n_masks host records, copied into the workspace on the stream (the caller may free them on return).
 * fill_ptr: a device float32 read on the stream in place of desc->fill, or null.  B200A_EINVAL for null pointers
 * (in and out may be null when the tensor is empty), negative sizes, a bad axis or a per-row mask with mask_param
 * below 1 or a null start_draws; B200A_EWORKSPACE for a short workspace.
 */
int b200a_mask_run(const b200a_mask_desc* desc, const b200a_mask_spec* masks, const float* in, float* out,
                   const float* fill_ptr, void* workspace, size_t workspace_bytes, b200a_stream stream);
/*
 * The gradient: grad_in = grad_out with every masked element 0 (desc->in_stride describes grad_out, which may have
 * zero strides; desc->out_stride describes grad_in, which may be null when grad_fill is not).  grad_fill, when not
 * null, receives the sum of grad_out over the masked elements: per-CTA partial sums in a fixed order, then a one-CTA
 * fold in a fixed order, in double.  Statuses as b200a_mask_run.
 */
int b200a_mask_backward(const b200a_mask_desc* desc, const b200a_mask_spec* masks, const float* grad_out,
                        float* grad_in, float* grad_fill, void* workspace, size_t workspace_bytes,
                        b200a_stream stream);

/* ---- polyphase sinc resampler ------------------------------------------------------------- */
/* Workspace bytes for b200a_resample_prepare (per-phase tap supports + compacted taps). */
size_t b200a_resample_workspace_bytes(int32_t new_r, int32_t taps);
/*
 * Analyse the cached kernel (Resample.kernel, _transforms.py:955-968; functional.py:1305-1402):
 * find each phase's contiguous non-negligible tap range and write the compacted table.
 *   kernel : [new_r][taps], taps = 2*width + orig_r
 */
int b200a_resample_prepare(const float* kernel, int32_t orig_r, int32_t new_r, int32_t width,
                           void* workspace, size_t workspace_bytes, b200a_stream stream);
/*
 * F._apply_sinc_resample_kernel (functional.py:1405-1432):
 *   out[r][f*new_r + j] = sum_i kernel[j][i] * xpad[r][f*orig_r + i],  xpad = width zeros | x | zeros,
 * for the first out_len = b200a_resample_len(length, orig_r, new_r) outputs of each row.
 */
int b200a_resample_run(const void* workspace, const float* kernel, int32_t orig_r, int32_t new_r,
                       int32_t width, const float* wave, int64_t rows, int64_t length,
                       int64_t row_stride, float* out, int64_t out_row_stride, int64_t out_len,
                       b200a_stream stream);

/*
 * Waveform gradient of b200a_resample_run.  With o' = orig_r, n' = new_r, w = width, taps = 2w + o', K the kernel
 * masked to each phase's live taps (the support b200a_resample_prepare finds) and g the upstream gradient:
 *   G[f][j] = g[f n' + j] for f n' + j < out_len, else 0;   D = G K   (frames x taps);
 *   grad_wave[s] = sum_f D[f][s + w - f o']  over the frames with 0 <= s + w - f o' < taps,  0 <= s < length.
 * The forward workspace and b200a_resample_prepare are unchanged: a resampler that never differentiates pays nothing.
 */
/* Bytes of the backward workspace for this ratio; 0 for an invalid one. */
size_t b200a_resample_backward_workspace_bytes(int32_t orig_r, int32_t new_r, int32_t width);
/* Adjoint tables from the cached kernel [new_r][2*width + orig_r]: per-phase supports (same rule as the forward),
 * per-tap live phase ranges + the transposed masked taps (direct kernel), the per-8-tap-column k-step plan and TF32
 * hi/lo B fragments (mma kernel).  The backward never reads the live `kernel` buffer afterwards.
 * B200A_EWORKSPACE when workspace_bytes < b200a_resample_backward_workspace_bytes(orig_r, new_r, width). */
int b200a_resample_backward_prepare(const float* kernel, int32_t orig_r, int32_t new_r, int32_t width,
                                    void* workspace, size_t workspace_bytes, b200a_stream stream);
/* grad_wave[r][s], s < length, every sample written; grad row r at grad + r*g_row_stride (0 allowed: expanded
 * gradients), unit element stride, out_len = b200a_resample_len(length, orig_r, new_r) values per row.
 * Deterministic, no atomics, every row independent; the kernel is chosen by the ratio alone. */
int b200a_resample_backward(const void* workspace, int32_t orig_r, int32_t new_r, int32_t width,
                            const float* grad, int64_t rows, int64_t g_row_stride, int64_t out_len,
                            float* grad_wave, int64_t length, int64_t grad_row_stride, b200a_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* B200AUDIO_H */
