"""Float64 numpy restatement of the waveform gradients (vector-Jacobian products) of the Kaldi spectrogram, fbank and
mfcc, built on oracle/kaldi_oracle.py.  tests/test_kaldi_grad_oracle.py checks it against torch.autograd through the
reference's op sequence (compliance/kaldi.py:44-83, 116-123, 154-216, 220-226, 292-316, 600-645, 760-813), restated here
in torch (``torch_kaldi``): float64 is the autograd reference, float32 on the CPU the yardstick of float32 round-off.
tests/test_gpu_kaldi_grad.py checks the GPU kernels against it."""
import math

import numpy as np
import torch

from oracle import kaldi_oracle as KO

EPS = KO.EPS
DEFAULTS = dict(blackman_coeff=0.42, energy_floor=1.0, frame_length=25.0, frame_shift=10.0, high_freq=0.0,
                htk_compat=False, low_freq=20.0, num_mel_bins=23, preemphasis_coefficient=0.97, raw_energy=True,
                remove_dc_offset=True, round_to_power_of_two=True, sample_frequency=16000.0, snip_edges=True,
                subtract_mean=False, use_energy=False, use_log_fbank=True, use_power=True, vtln_high=-500.0,
                vtln_low=100.0, vtln_warp=1.0, window_type="povey", num_ceps=13, cepstral_lifter=22.0)


def options(kind, kw):
    """Every option of `kind` with the reference's defaults (spectrogram: the energy column is always on)."""
    o = dict(DEFAULTS)
    o.update({k: v for k, v in kw.items() if k not in ("dither", "channel", "min_duration")})
    if kind == "spectrogram":
        o.update(use_energy=True, use_log_fbank=True, use_power=True, htk_compat=False)
    if kind == "mfcc":
        o.update(use_log_fbank=True, use_power=True)
    return o


def frame_index(n, size, shift, snip):
    """(m, size) source sample of every frame element (kaldi.py:44-83), mirrored edges included."""
    return KO.get_strided(np.arange(n, dtype=np.float64), size, shift, snip).astype(np.int64)


def _geometry(n, o):
    shift, size, padded = KO.window_properties(n, o["sample_frequency"], o["frame_shift"], o["frame_length"],
                                               o["round_to_power_of_two"], o["preemphasis_coefficient"])
    return shift, size, padded, frame_index(n, size, shift, o["snip_edges"])


def _banks(o, padded):
    b, _ = KO.get_mel_banks(o["num_mel_bins"], padded, o["sample_frequency"], o["low_freq"], o["high_freq"], o["vtln_low"],
                            o["vtln_high"], o["vtln_warp"])
    return np.concatenate([b, np.zeros((b.shape[0], 1))], axis=1)  # (n_mels, padded/2 + 1)


def finish_matrix(o):
    """(inputs, outputs) matrix from the fbank-layout row [log mels | energy] to the mfcc row (kaldi.py:760-813)."""
    n_mels, ceps = o["num_mel_bins"], o["num_ceps"]
    m = KO.dct_matrix(ceps, n_mels)
    if o["cepstral_lifter"] != 0.0:
        m = m * KO.lifter_coeffs(ceps, o["cepstral_lifter"])[None, :]
    if o["use_energy"]:
        m[:, 0] = 0.0
        route = np.zeros((1, ceps))
        route[0, 0] = 1.0
        m = np.concatenate([m, route], axis=0)
    if o["htk_compat"]:
        first = m[:, :1] if o["use_energy"] else m[:, :1] * math.sqrt(2)
        m = np.concatenate([m[:, 1:], first], axis=1)
    return m


def _log_vjp(v, g):
    """d log(maximum(v, eps)) / dv times g with torch's tie rule."""
    return np.where(v > EPS, g / np.where(v > EPS, v, 1.0), np.where(v == EPS, 0.5 * g / EPS, 0.0))


def kaldi_vjp(kind, wave, grad, **kw):
    """Gradient of sum(grad * kind(wave, **kw)) with respect to the 1-D `wave` (float64)."""
    o = options(kind, kw)
    x = np.asarray(wave, dtype=np.float64).reshape(-1)
    n = x.shape[0]
    shift, size, padded, idx = _geometry(n, o)
    c = o["preemphasis_coefficient"]
    w = KO.feature_window(o["window_type"], size, o["blackman_coeff"])
    fr = x[idx]
    s = fr - fr.mean(1, keepdims=True) if o["remove_dc_offset"] else fr
    prev = np.concatenate([s[:, :1], s[:, :-1]], axis=1)
    v = (s - c * prev) * w[None, :] if c != 0.0 else s * w[None, :]
    vp = np.concatenate([v, np.zeros((v.shape[0], padded - size))], axis=1)
    X = np.fft.rfft(vp, axis=1)
    E = (s ** 2).sum(1) if o["raw_energy"] else (vp ** 2).sum(1)
    g = np.asarray(grad, dtype=np.float64).reshape(idx.shape[0], -1)
    if o["subtract_mean"]:
        g = g - g.mean(0, keepdims=True)
    use_energy = o["use_energy"]
    n_mels = o["num_mel_bins"]
    if kind == "mfcc":  # to the fbank layout [log mels | energy]
        g = g @ finish_matrix(o).T
        g_vals, g_e = g[:, :n_mels], (g[:, n_mels] if use_energy else None)
    elif kind == "fbank":
        off = int(use_energy and not o["htk_compat"])
        g_vals = g[:, off:off + n_mels]
        g_e = None if not use_energy else g[:, n_mels if o["htk_compat"] else 0]
    else:
        g_vals, g_e = g.copy(), g[:, 0]
        g_vals[:, 0] = 0.0  # bin 0 holds the log energy
    power = 2.0 if o["use_power"] else 1.0
    mag = np.abs(X)
    spec = mag ** power
    if kind == "spectrogram":
        g_p = _log_vjp(spec, g_vals)
    else:
        banks = _banks(o, padded)
        mel = spec @ banks.T
        g_mel = _log_vjp(mel, g_vals) if o["use_log_fbank"] else g_vals
        g_p = g_mel @ banks
    if power == 2.0:
        g_x = 2.0 * g_p * np.conj(X)
    else:
        g_x = np.where(mag > 0, g_p * np.conj(X) / np.where(mag > 0, mag, 1.0), 0.0)
    k = np.arange(padded // 2 + 1)[:, None]
    basis = np.exp(-2j * math.pi * k * np.arange(padded)[None, :] / padded)
    d_v = np.real(g_x @ basis)[:, :size]
    g_E = np.zeros(idx.shape[0])
    if g_e is not None:
        le = np.log(np.maximum(E, EPS))
        g_le = g_e
        if o["energy_floor"] != 0.0:
            fl = math.log(o["energy_floor"])
            g_le = np.where(le > fl, g_e, np.where(le == fl, 0.5 * g_e, 0.0))
        g_E = _log_vjp(E, g_le)
    if not o["raw_energy"]:
        d_v = d_v + 2.0 * v * g_E[:, None]
    d_p = d_v * w[None, :]
    if c != 0.0:
        d_s = d_p.copy()
        d_s[:, :-1] -= c * d_p[:, 1:]
        d_s[:, 0] -= c * d_p[:, 0]
    else:
        d_s = d_p
    if o["raw_energy"]:
        d_s = d_s + 2.0 * s * g_E[:, None]
    if o["remove_dc_offset"]:
        d_s = d_s - d_s.mean(1, keepdims=True)
    out = np.zeros(n)
    np.add.at(out, idx.reshape(-1), d_s.reshape(-1))
    return out


# ---- the reference's op sequence in torch (autograd ground truth) ------------------------------------------------
def torch_kaldi(kind, wave, **kw):
    """kind(wave) of a (..., n) torch tensor in its dtype, with the reference's ops on the last two dims (frames,
    samples), so autograd gives its gradient; leading dims are rows computed together."""
    o = options(kind, kw)
    dt = wave.dtype
    n = wave.shape[-1]
    shift, size, padded, idx = _geometry(n, o)
    dev = wave.device
    eps = torch.tensor(EPS, dtype=dt, device=dev)
    fr = wave[..., torch.from_numpy(idx).to(dev)]
    if o["remove_dc_offset"]:
        fr = fr - torch.mean(fr, dim=-1).unsqueeze(-1)

    def log_energy(f):
        le = torch.max(f.pow(2).sum(-1), eps).log()
        if o["energy_floor"] == 0.0:
            return le
        return torch.max(le, torch.tensor(math.log(o["energy_floor"]), dtype=dt, device=dev))

    if o["raw_energy"]:
        le = log_energy(fr)
    c = o["preemphasis_coefficient"]
    if c != 0.0:  # the reference's replicate pad by one sample on the left (kaldi.py:195-198)
        off = torch.cat((fr[..., :1], fr), dim=-1)
        fr = fr - c * off[..., :-1]
    fr = fr * torch.from_numpy(KO.feature_window(o["window_type"], size, o["blackman_coeff"])).to(dev, dt)
    if padded != size:
        fr = torch.nn.functional.pad(fr, (0, padded - size), mode="constant", value=0)
    if not o["raw_energy"]:
        le = log_energy(fr)
    X = torch.fft.rfft(fr)
    if kind == "spectrogram":
        out = torch.max(X.abs().pow(2.0), eps).log()
        out[..., 0] = le
    else:
        spec = X.abs()
        if o["use_power"]:
            spec = spec.pow(2.0)
        mel = torch.matmul(spec, torch.from_numpy(_banks(o, padded)).to(dev, dt).T)
        if o["use_log_fbank"]:
            mel = torch.max(mel, eps).log()
        if o["use_energy"]:
            e = le.unsqueeze(-1)
            mel = torch.cat((mel, e), -1) if o["htk_compat"] else torch.cat((e, mel), -1)
        out = mel
        if kind == "mfcc":
            n_mels, ceps = o["num_mel_bins"], o["num_ceps"]
            if o["use_energy"]:
                sle = out[..., n_mels if o["htk_compat"] else 0]
                m0 = int(not o["htk_compat"])
                out = out[..., m0:n_mels + m0]
            out = out.matmul(torch.from_numpy(KO.dct_matrix(ceps, n_mels)).to(dev, dt))
            if o["cepstral_lifter"] != 0.0:
                out = out * torch.from_numpy(KO.lifter_coeffs(ceps, o["cepstral_lifter"])).to(dev, dt)
            if o["use_energy"]:
                out[..., 0] = sle
            if o["htk_compat"]:
                energy = out[..., 0].unsqueeze(-1)
                out = out[..., 1:]
                if not o["use_energy"]:
                    energy = energy * math.sqrt(2)
                out = torch.cat((out, energy), dim=-1)
    if o["subtract_mean"]:
        out = out - torch.mean(out, dim=-2).unsqueeze(-2)
    return out


def torch_vjp(kind, wave, grad, dtype=torch.float64, **kw):
    """torch.autograd of torch_kaldi in `dtype` on the CPU: the gradient of sum(grad * out) as float64 numpy."""
    x = torch.tensor(np.asarray(wave).reshape(-1), dtype=dtype, requires_grad=True)
    out = torch_kaldi(kind, x, **kw)
    out.backward(torch.as_tensor(np.asarray(grad), dtype=dtype).reshape(out.shape))
    return x.grad.double().numpy()
