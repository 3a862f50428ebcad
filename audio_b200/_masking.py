"""SpecAugment masking (reference functional/functional.py:806-957, transforms/_transforms.py:1167-1349) on the kernel of
``csrc/masking.cu``.

Every entry point makes the reference's random draws itself, with the reference's calls, shapes, devices, dtypes and
order (``mask_along_axis_iid``: two ``torch.rand`` of the batch shape on the input's device; ``mask_along_axis``: two
``torch.rand(1)`` from the CPU generator, whose interval is computed here with the reference's CPU tensor arithmetic),
and skips them where the reference does.  The masks then go to one launch, which recomputes each per-row interval from
its draws in the reference's float32 arithmetic.  All masks of one call share the fill, so applying their union at once
equals the reference's sequential application.

The output is a fresh tensor with the strides the reference's op sequence gives for the same input, found by replaying
that sequence (its non-random ops only) on ``meta`` tensors (empty CPU tensors for an empty input), cached per shape,
strides and op sequence.
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Tuple, Union

import torch
from torch import Tensor
from torch.autograd.function import once_differentiable

from . import _lib
from ._plans import _require_cuda_f32, _stream_ptr


def _get_mask_param(mask_param: int, p: float, axis_length: int) -> int:
    """The mask length limit: ``mask_param``, capped at ``int(axis_length * p)`` unless ``p == 1.0``."""
    if p == 1.0:
        return mask_param
    return min(mask_param, int(axis_length * p))


def _check_axis_and_p(dim: int, axis: int, p: float) -> None:
    if axis not in [dim - 2, dim - 1]:
        raise ValueError(
            "Only Frequency and Time masking are supported"
            f" (axis {dim - 2} and axis {dim - 1} supported; {axis} given)."
        )
    if not 0.0 <= p <= 1.0:
        raise ValueError(f"The value of p must be between 0.0 and 1.0 ({p} given).")


def _check_inputs(x: Tensor, mask_value) -> None:
    _require_cuda_f32(x, "specgram")
    if isinstance(mask_value, Tensor):
        if mask_value.dtype != torch.float32 or mask_value.numel() != 1 or mask_value.device != x.device:
            raise RuntimeError(
                "audio_b200: a tensor mask_value must be a one-element float32 tensor on the input's device "
                f"(got {mask_value.dtype}, {mask_value.numel()} elements, on {mask_value.device})"
            )


class _Mask:
    """One mask of a fused launch: per-row draws (``value``, ``low``) or an interval shared by every row."""

    __slots__ = ("time", "mask_param", "start", "end", "value", "low")

    def __init__(self, time: bool, mask_param: int = 0, start: int = 0, end: int = 0,
                 value: Optional[Tensor] = None, low: Optional[Tensor] = None):
        self.time, self.mask_param, self.start, self.end, self.value, self.low = (time, mask_param, start, end,
                                                                                  value, low)

    def spec(self) -> _lib.MaskSpec:
        axis = _lib.MASK_AXIS_TIME if self.time else _lib.MASK_AXIS_FREQ
        if self.value is None:
            return _lib.MaskSpec(axis, 0, self.start, self.end, None, None)
        return _lib.MaskSpec(axis, self.mask_param, 0, 0, self.value.data_ptr(), self.low.data_ptr())


def draw_iid(specgrams: Tensor, mask_param: int, mask_value, axis: int, p: float) -> Optional[_Mask]:
    """The checks and draws of ``mask_along_axis_iid``; None where the reference returns its input."""
    dim = specgrams.dim()
    if dim < 3:
        raise ValueError(f"Spectrogram must have at least three dimensions ({dim} given).")
    _check_axis_and_p(dim, axis, p)
    mask_param = _get_mask_param(mask_param, p, specgrams.shape[axis])
    if mask_param < 1:
        return None
    _check_inputs(specgrams, mask_value)
    shape = specgrams.shape[: (dim - 2)]
    value = torch.rand(shape, device=specgrams.device, dtype=specgrams.dtype)
    low = torch.rand(shape, device=specgrams.device, dtype=specgrams.dtype)
    return _Mask(axis == dim - 1, mask_param=mask_param, value=value, low=low)


def draw_shared(specgram: Tensor, mask_param: int, mask_value, axis: int, p: float) -> Optional[_Mask]:
    """The checks and CPU draws of ``mask_along_axis``; None where the reference returns its input."""
    dim = specgram.dim()
    if dim < 2:
        raise ValueError(f"Spectrogram must have at least two dimensions (time and frequency) ({dim} given).")
    _check_axis_and_p(dim, axis, p)
    size = specgram.shape[axis]
    mask_param = _get_mask_param(mask_param, p, size)
    if mask_param < 1:
        return None
    # the reference packs the batch before drawing: its error for an ambiguous empty shape comes first
    torch.empty_strided(specgram.shape, specgram.stride(), device="meta").reshape([-1] + list(specgram.shape[-2:]))
    _check_inputs(specgram, mask_value)
    value = torch.rand(1) * mask_param
    min_value = torch.rand(1) * (size - value)
    start = int(min_value.long())
    end = int(min_value.long() + value.long())
    if end - start >= mask_param:
        raise ValueError("Number of columns to be masked should be less than mask_param")
    return _Mask(axis == dim - 1, start=start, end=end)


# ---- output layout: the reference's op sequence replayed on meta tensors ------------------------------------------
_LAYOUTS: "dict[tuple, Tuple[tuple, tuple]]" = {}


def _replay(shape, stride, steps, fill_shape) -> Tuple[tuple, tuple]:
    # Empty tensors run on the CPU, where there is nothing to compute: some ops lay out an empty result differently
    # on meta tensors.
    dev = "cpu" if 0 in shape else "meta"
    x = torch.empty_strided(shape, stride, device=dev)
    fill = 0.0 if fill_shape is None else torch.empty(fill_shape, device=dev)
    for iid, ax in steps:
        dim = x.dim()
        if iid:  # mask_along_axis_iid
            start = torch.empty(x.shape[: dim - 2], dtype=torch.long, device=dev)[..., None, None]
            idx = torch.arange(0, x.size(ax), device=dev, dtype=x.dtype)
            mask = (idx >= start) & (idx < start + start)
            xt = x.transpose(ax, -1)
            y = torch.where(mask, fill.repeat(xt.shape), xt) if fill_shape is not None else xt.masked_fill(mask, fill)
            x = y.transpose(ax, -1)
        else:  # mask_along_axis
            full = x.size()
            s = x.reshape([-1] + list(full[-2:]))
            start = torch.zeros((), dtype=torch.long, device=dev)
            mask = torch.arange(0, s.shape[ax - dim + 3], device=dev, dtype=x.dtype)
            mask = (mask >= start) & (mask < start + start)
            if ax == dim - 2:
                mask = mask.unsqueeze(-1)
            y = s.masked_fill(mask, fill)
            x = y.reshape(full[:-2] + y.shape[-2:])
    return tuple(x.shape), tuple(x.stride())


def _layout(x: Tensor, steps, fill) -> Tuple[tuple, tuple]:
    fill_shape = tuple(fill.shape) if isinstance(fill, Tensor) else None
    key = (tuple(x.shape), tuple(x.stride()), tuple(steps), fill_shape)
    out = _LAYOUTS.get(key)
    if out is None:
        if len(_LAYOUTS) >= 256:
            _LAYOUTS.pop(next(iter(_LAYOUTS)))
        out = _LAYOUTS[key] = _replay(x.shape, x.stride(), steps, fill_shape)
    return out


# ---- launch ---------------------------------------------------------------------------------------------------------
_I64x4 = ctypes.c_int64 * 4


def _row_groups(shape, a_stride, b_stride):
    """The batch dimensions as at most two (size, stride a, stride b) groups with row-major row order, or None."""
    groups: List[Tuple[int, int, int]] = []
    for n, sa, sb in zip(shape, a_stride, b_stride):
        if n == 1:
            continue
        if groups and groups[-1][1] == sa * n and groups[-1][2] == sb * n:
            groups[-1] = (groups[-1][0] * n, sa, sb)
        else:
            groups.append((n, sa, sb))
    if len(groups) > 2:
        return None
    while len(groups) < 2:
        groups.insert(0, (1, 0, 0))
    return groups


def _desc(src: Tensor, dst_shape, dst_stride, n_masks: int, fill: float):
    """The descriptor for src -> a tensor of dst_stride, and src (copied to contiguous when its batch dimensions and
    the destination's do not collapse to two strides each)."""
    groups = _row_groups(src.shape[:-2], src.stride()[:-2], dst_stride[:-2])
    if groups is None:
        src = src.contiguous()
        groups = _row_groups(src.shape[:-2], src.stride()[:-2], dst_stride[:-2])
        if groups is None:
            raise RuntimeError(f"audio_b200: masking does not support the output layout {dst_stride} of shape "
                               f"{tuple(dst_shape)}: its batch dimensions do not collapse to two strides")
    (n0, a0, b0), (n1, a1, b1) = groups
    F, T = dst_shape[-2:]
    desc = _lib.MaskDesc(n0, n1, F, T, _I64x4(a0, a1, *src.stride()[-2:]),
                         _I64x4(b0, b1, *dst_stride[-2:]), n_masks, fill)
    return desc, src


def _specs(masks):
    arr = (_lib.MaskSpec * max(len(masks), 1))()
    for i, m in enumerate(masks):
        arr[i] = m.spec()
    return arr


def _workspace(desc, device) -> Tensor:
    return torch.empty(_lib.lib().b200a_mask_workspace_bytes(desc), dtype=torch.uint8, device=device)


def _forward(x: Tensor, masks, fill, shape, stride) -> Tensor:
    dev = x.device
    with torch.cuda.device(dev):
        out = torch.empty_strided(shape, stride, dtype=x.dtype, device=dev)
        desc, src = _desc(x, shape, stride, len(masks), 0.0 if isinstance(fill, Tensor) else float(fill))
        ws = _workspace(desc, dev)
        rc = _lib.lib().b200a_mask_run(desc, _specs(masks), src.data_ptr(), out.data_ptr(),
                                       fill.data_ptr() if isinstance(fill, Tensor) else None, ws.data_ptr(),
                                       ws.numel(), _stream_ptr(dev))
    _lib.check(rc, "mask_along_axis")
    return out


class _MaskFunction(torch.autograd.Function):
    """The fused masking with the gradients of the input (g with the masked elements zeroed) and of a tensor fill (the
    sum of g over the masked elements).  Saved: the masks' draws or intervals, nothing input-sized."""

    @staticmethod
    def forward(ctx, x, fill_tensor, fill, masks, shape, stride):
        ctx.masks, ctx.fill_shape, ctx.dev = masks, None if fill_tensor is None else fill_tensor.shape, x.device
        return _forward(x, masks, fill, shape, stride)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        want_x, want_fill = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        dev = ctx.dev
        if g.dtype != torch.float32:
            g = g.float()
        with torch.cuda.device(dev):
            grad_x = torch.empty(g.shape, dtype=torch.float32, device=dev) if want_x else None
            grad_fill = torch.empty((), dtype=torch.float32, device=dev) if want_fill else None
            dst = grad_x.stride() if want_x else g.stride()
            desc, src = _desc(g, g.shape, dst, len(ctx.masks), 0.0)
            ws = _workspace(desc, dev)
            rc = _lib.lib().b200a_mask_backward(desc, _specs(ctx.masks), src.data_ptr(),
                                                grad_x.data_ptr() if want_x else None,
                                                grad_fill.data_ptr() if want_fill else None, ws.data_ptr(),
                                                ws.numel(), _stream_ptr(dev))
        _lib.check(rc, "mask_along_axis backward")
        if want_fill:
            grad_fill = grad_fill.reshape(ctx.fill_shape)
        return grad_x, grad_fill, None, None, None, None


def apply_masks(x: Tensor, masks: List[_Mask], steps, fill: Union[float, Tensor]) -> Tensor:
    """One launch for every mask in ``masks`` (``steps``: the reference op sequence they stand for, as
    (iid, axis) pairs); the input itself when there is none."""
    if not masks:
        return x
    shape, stride = _layout(x, steps, fill)
    fill_tensor = fill if isinstance(fill, Tensor) else None
    if torch.is_grad_enabled() and (x.requires_grad or (fill_tensor is not None and fill_tensor.requires_grad)):
        return _MaskFunction.apply(x, fill_tensor, fill, masks, shape, stride)
    return _forward(x, masks, fill, shape, stride)


def mask_along_axis_iid(specgrams: Tensor, mask_param: int, mask_value: Union[float, Tensor], axis: int,
                        p: float = 1.0) -> Tensor:
    """Mask ``[v_0, v_0 + v)`` along ``axis`` (one of the last two of a ``(..., freq, time)`` tensor with at least 3
    dimensions), independently per example: ``v ~ uniform(0, max_v)``, ``v_0 ~ uniform(0, size - v)`` from two
    ``torch.rand`` of the batch shape on the input's device, ``max_v = mask_param`` when ``p == 1.0`` and
    ``min(mask_param, int(size * p))`` otherwise.  Returns the input itself when ``max_v < 1``.  CUDA float32 input; a
    tensor ``mask_value`` is one float32 element on the same device and receives a gradient."""
    m = draw_iid(specgrams, mask_param, mask_value, axis, p)
    if m is None:
        return specgrams
    return apply_masks(specgrams, [m], [(True, axis)], mask_value)


def mask_along_axis(specgram: Tensor, mask_param: int, mask_value: Union[float, Tensor], axis: int,
                    p: float = 1.0) -> Tensor:
    """Mask ``[v_0, v_0 + v)`` along ``axis`` (one of the last two, at least 2 dimensions), one interval for every
    example, drawn with two ``torch.rand(1)`` from the CPU generator whatever the device; otherwise as
    :func:`mask_along_axis_iid`."""
    m = draw_shared(specgram, mask_param, mask_value, axis, p)
    if m is None:
        return specgram
    return apply_masks(specgram, [m], [(False, axis)], mask_value)


def spec_augment(specgram: Tensor, n_time_masks: int, time_mask_param: int, n_freq_masks: int, freq_mask_param: int,
                 iid_masks: bool, p: float, zero_masking: bool) -> Tensor:
    """``SpecAugment.forward`` in one launch: the reference's ``mean()`` and draws in its order, then every mask."""
    mask_value = 0.0 if zero_masking else specgram.mean()
    time_dim = specgram.dim() - 1
    freq_dim = time_dim - 1
    iid = specgram.dim() > 2 and iid_masks is True
    draw = draw_iid if iid else draw_shared
    masks, steps = [], []
    for n, param, axis in ((n_time_masks, time_mask_param, time_dim), (n_freq_masks, freq_mask_param, freq_dim)):
        for _ in range(n):
            m = draw(specgram, param, mask_value, axis, p)
            if m is not None:
                masks.append(m)
                steps.append((iid, axis))
    return apply_masks(specgram, masks, steps, mask_value)
