"""Float64 numpy restatement of the waveform gradient (vector-Jacobian product) of the polyphase resampler, the adjoint
of oracle.frontend_oracle.apply_sinc_resample_kernel.  tests/test_resample_grad_oracle.py checks it against
torch.autograd through the reference's op sequence; tests/test_gpu_resample_grad.py checks the GPU kernels against it."""
import numpy as np


def resample_vjp(g, orig_freq, new_freq, gcd, kernel, width, length) -> np.ndarray:
    """Gradient of sum(g * resample(x)) with respect to x of `length` samples, float64.  With o' = orig/gcd,
    n' = new/gcd, taps = 2 width + o':
        G[f][j] = g[f n' + j] (0 past the returned outputs),   D = G K   (frames x taps),
        dx_pad[f o' + i] += D[f][i]  over the frames of the (width, width + o') zero-padded signal,
    and the padding is dropped: dx = dx_pad[width : width + length]."""
    g = np.asarray(g, dtype=np.float64)
    lead, out_len = g.shape[:-1], g.shape[-1]
    flat = g.reshape(-1, out_len)
    o = int(orig_freq) // gcd
    n = int(new_freq) // gcd
    k = np.asarray(kernel, dtype=np.float64).reshape(n, -1)
    taps = k.shape[1]
    padded = length + 2 * width + o
    frames = (padded - taps) // o + 1
    assert out_len <= frames * n
    G = np.zeros((flat.shape[0], frames * n))
    G[:, :out_len] = flat
    D = np.einsum("bfp,pt->bft", G.reshape(-1, frames, n), k)
    idx = np.arange(taps)[None, :] + o * np.arange(frames)[:, None]  # (frames, taps) positions in the padded signal
    dxp = np.zeros((flat.shape[0], padded))
    for b in range(flat.shape[0]):
        np.add.at(dxp[b], idx.ravel(), D[b].ravel())
    return dxp[:, width:width + length].reshape(lead + (length,))
