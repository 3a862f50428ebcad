"""Host-buffer pipeline: run a front-end module over waveforms that live in (pinned) HOST memory.

An H100 turns 256 x 10 s of audio into mel features in a fraction of a millisecond, but the same
batch takes milliseconds to cross PCIe.  ``HostPipeline`` splits the batch into row chunks and keeps three
CUDA streams busy -- host->device copies, the fused kernel, device->host copies -- so the end-to-end
time approaches the slower of the two PCIe directions instead of their sum plus the compute.
Consecutive calls overlap too: the H2D copies of call k+1 start while the D2H copies of call k drain.

    pipe = HostPipeline(T.MelSpectrogram(16000, n_fft=1024, hop_length=256, n_mels=80).cuda())
    feats = pipe(wave_host)              # (B, n_mels, T) view of a pinned frame-major (B, T, n_mels) buffer
    pipe.synchronize()                   # host waits; or pipe.join() to make the current stream wait

Rows are independent on this path (SURVEY.md 8e), so chunking never changes results -- with ONE
exception the caller must respect: ``MFCC`` / ``LFCC`` on a 2-D batch share one top_db maximum over the
whole batch (reference functional.py:395-399); chunking such a call would change it, so it is refused.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import transforms as T

_N_BUF = 3


class HostPipeline:
    def __init__(self, module: torch.nn.Module, chunk_rows: int = 64, device: Optional[torch.device] = None):
        if (isinstance(module, T.MFCC) and not module.log_mels) or (isinstance(module, T.LFCC) and not module.log_lf):
            raise ValueError(
                "HostPipeline cannot chunk MFCC / LFCC with the batch-global top_db clamp (reference "
                "functional.py:395-399: one maximum over a 2-D batch); pass (B, 1, time) inputs through the module "
                "directly or use log_mels=True / log_lf=True"
            )
        params = list(module.buffers())
        self.device = device if device is not None else (params[0].device if params else torch.device("cuda"))
        if self.device.type != "cuda":
            raise RuntimeError("HostPipeline needs the module on a CUDA device (no CPU fallback)")
        self.module = module
        self.chunk_rows = int(chunk_rows)
        if self.chunk_rows < 1:
            raise ValueError("chunk_rows must be positive")
        self._s_in = torch.cuda.Stream(self.device)
        self._s_run = torch.cuda.Stream(self.device)
        self._s_out = torch.cuda.Stream(self.device)
        self._dev_in = None
        self._buf_free: List[Optional[torch.cuda.Event]] = [None] * _N_BUF  # kernel that last read each staging buffer
        self._next_buf = 0
        self._host_out = None

    def synchronize(self) -> None:
        """Block the host until every result enqueued so far sits in its host buffer."""
        self._s_out.synchronize()

    def join(self) -> None:
        """Make the CURRENT stream wait for everything enqueued so far (no host synchronisation)."""
        torch.cuda.current_stream(self.device).wait_stream(self._s_out)

    @torch.inference_mode()
    def __call__(self, wave_host: torch.Tensor, out_host: Optional[torch.Tensor] = None) -> torch.Tensor:
        if wave_host.is_cuda or wave_host.dim() != 2 or wave_host.dtype != torch.float32:
            raise TypeError("HostPipeline expects a 2-D float32 CPU tensor (pin it for asynchronous copies)")
        rows, length = wave_host.shape
        step = max(1, min(self.chunk_rows, rows))
        n_chunks = (rows + step - 1) // step
        if self._dev_in is None or tuple(self._dev_in.shape[1:]) != (step, length):
            self.synchronize()  # nobody may still be reading the buffers we are about to drop
            with torch.cuda.device(self.device):
                self._dev_in = torch.empty((_N_BUF, step, length), dtype=torch.float32, device=self.device)
            self._buf_free = [None] * _N_BUF
        # work the caller enqueued before this call (e.g. writing wave_host from the device) is respected;
        # results of EARLIER calls are not waited for here -- that is what lets consecutive calls overlap
        self._s_in.wait_stream(torch.cuda.current_stream(self.device))
        result = out_host
        for i in range(n_chunks):
            lo, hi = i * step, min(rows, (i + 1) * step)
            b = self._next_buf
            self._next_buf = (b + 1) % _N_BUF
            buf = self._dev_in[b, : hi - lo]
            ev_in, ev_run = torch.cuda.Event(), torch.cuda.Event()
            with torch.cuda.stream(self._s_in):
                if self._buf_free[b] is not None:
                    self._s_in.wait_event(self._buf_free[b])  # the kernel that read this buffer has finished
                buf.copy_(wave_host[lo:hi], non_blocking=True)
                ev_in.record(self._s_in)
            with torch.cuda.stream(self._s_run):
                self._s_run.wait_event(ev_in)
                y = self.module(buf)  # logical (rows, W, T) view of frame-major (rows, T, W) memory
                ev_run.record(self._s_run)
            self._buf_free[b] = ev_run
            y_fm = y.transpose(-1, -2)
            if result is None:
                result = torch.empty((rows,) + tuple(y_fm.shape[1:]), dtype=y.dtype).pin_memory()
            with torch.cuda.stream(self._s_out):
                self._s_out.wait_event(ev_run)
                y_fm.record_stream(self._s_out)
                result[lo:hi].copy_(y_fm, non_blocking=True)
        self._host_out = result
        return result.transpose(-1, -2)
