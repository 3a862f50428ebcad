"""A device-agnostic torch restatement of SpecAugment masking: ``mask_along_axis_iid``, ``mask_along_axis``,
``FrequencyMasking``, ``TimeMasking`` and ``SpecAugment`` (reference functional.py:806-957, _transforms.py:1167-1349).

It is the contract audio_b200's fused kernel is held to, written as the reference's op sequence so that values, output
strides, autograd and random-number consumption all follow from it:
- the mask length limit is ``mask_param``, or ``min(mask_param, int(size * p))`` when ``p != 1``; below 1 the input
  object itself comes back and nothing is drawn;
- per-example masks draw ``u`` then ``w``, each ``torch.rand`` of the batch shape on the input's device and dtype; the
  interval is ``[long(w * (size - u * mask_param)), that + long(u * mask_param))`` in float32, compared against a float32
  index ramp; a tensor fill goes through ``where`` with the fill repeated to the (transposed) shape, a number through
  ``masked_fill``;
- shared masks draw two ``torch.rand(1)`` from the CPU generator, apply one interval to every example of the
  ``(-1, freq, time)`` packed view with ``masked_fill``, and raise when the interval is not shorter than the limit;
- ``SpecAugment`` takes ``mean()`` once (unless ``zero_masking``), then applies every time mask, then every frequency
  mask, per example when the input has more than 2 dimensions and ``iid_masks``.

``make_input`` and ``run_case`` rebuild the cases of tests/golden/specaugment_ref_cases.npz against any namespace
holding the five entry points.
"""
from types import SimpleNamespace

import torch
from torch import Tensor


def _limit(mask_param, p, size):
    return mask_param if p == 1.0 else min(mask_param, int(size * p))


def _checks(dim, axis, p, min_dim, what):
    if dim < min_dim:
        raise ValueError(what.format(dim))
    if axis not in [dim - 2, dim - 1]:
        raise ValueError(
            f"Only Frequency and Time masking are supported (axis {dim - 2} and axis {dim - 1} supported; {axis} given)."
        )
    if not 0.0 <= p <= 1.0:
        raise ValueError(f"The value of p must be between 0.0 and 1.0 ({p} given).")


def _ramp_mask(size, start, end, like):
    ramp = torch.arange(0, size, device=like.device, dtype=like.dtype)
    return (ramp >= start) & (ramp < end)


def mask_along_axis_iid(specgrams, mask_param, mask_value, axis, p=1.0):
    dim = specgrams.dim()
    _checks(dim, axis, p, 3, "Spectrogram must have at least three dimensions ({} given).")
    limit = _limit(mask_param, p, specgrams.shape[axis])
    if limit < 1:
        return specgrams
    batch = specgrams.shape[: dim - 2]
    u = torch.rand(batch, device=specgrams.device, dtype=specgrams.dtype) * limit
    w = torch.rand(batch, device=specgrams.device, dtype=specgrams.dtype) * (specgrams.size(axis) - u)
    start = w.long()
    end = start + u.long()
    mask = _ramp_mask(specgrams.size(axis), start[..., None, None], end[..., None, None], specgrams)
    moved = specgrams.transpose(axis, -1)
    if isinstance(mask_value, Tensor):
        moved = torch.where(mask, mask_value.repeat(moved.shape), moved)
    else:
        moved = moved.masked_fill(mask, mask_value)
    return moved.transpose(axis, -1)


def mask_along_axis(specgram, mask_param, mask_value, axis, p=1.0):
    dim = specgram.dim()
    _checks(dim, axis, p, 2, "Spectrogram must have at least two dimensions (time and frequency) ({} given).")
    limit = _limit(mask_param, p, specgram.shape[axis])
    if limit < 1:
        return specgram
    shape = specgram.size()
    packed = specgram.reshape([-1] + list(shape[-2:]))
    size = packed.size(axis - dim + 3)
    u = torch.rand(1) * limit
    w = torch.rand(1) * (size - u)
    start = w.long().squeeze()
    end = (w.long() + u.long()).squeeze()
    mask = _ramp_mask(size, start, end, packed)
    if axis == dim - 2:
        mask = mask.unsqueeze(-1)
    if end - start >= limit:
        raise ValueError("Number of columns to be masked should be less than mask_param")
    packed = packed.masked_fill(mask, mask_value)
    return packed.reshape(shape[:-2] + packed.shape[-2:])


class _AxisMasking(torch.nn.Module):
    def __init__(self, mask_param, axis, iid_masks, p=1.0):
        super().__init__()
        self.mask_param, self.axis, self.iid_masks, self.p = mask_param, axis, iid_masks, p

    def forward(self, specgram, mask_value=0.0):
        axis = self.axis + specgram.dim() - 3
        if self.iid_masks:
            return mask_along_axis_iid(specgram, self.mask_param, mask_value, axis, p=self.p)
        value = float(mask_value) if isinstance(mask_value, Tensor) else mask_value
        return mask_along_axis(specgram, self.mask_param, value, axis, p=self.p)


class FrequencyMasking(_AxisMasking):
    def __init__(self, freq_mask_param, iid_masks=False):
        super().__init__(freq_mask_param, 1, iid_masks)


class TimeMasking(_AxisMasking):
    def __init__(self, time_mask_param, iid_masks=False, p=1.0):
        if not 0.0 <= p <= 1.0:
            raise ValueError(f"The value of p must be between 0.0 and 1.0 ({p} given).")
        super().__init__(time_mask_param, 2, iid_masks, p=p)


class SpecAugment(torch.nn.Module):
    def __init__(self, n_time_masks, time_mask_param, n_freq_masks, freq_mask_param, iid_masks=True, p=1.0,
                 zero_masking=False):
        super().__init__()
        self.n_time_masks, self.time_mask_param = n_time_masks, time_mask_param
        self.n_freq_masks, self.freq_mask_param = n_freq_masks, freq_mask_param
        self.iid_masks, self.p, self.zero_masking = iid_masks, p, zero_masking

    def forward(self, specgram):
        value = 0.0 if self.zero_masking else specgram.mean()
        t_axis = specgram.dim() - 1
        fn = mask_along_axis_iid if specgram.dim() > 2 and self.iid_masks is True else mask_along_axis
        for _ in range(self.n_time_masks):
            specgram = fn(specgram, self.time_mask_param, value, t_axis, p=self.p)
        for _ in range(self.n_freq_masks):
            specgram = fn(specgram, self.freq_mask_param, value, t_axis - 1, p=self.p)
        return specgram


ORACLE = SimpleNamespace(mask_along_axis_iid=mask_along_axis_iid, mask_along_axis=mask_along_axis,
                         FrequencyMasking=FrequencyMasking, TimeMasking=TimeMasking, SpecAugment=SpecAugment)


# ---- the fixture's cases ------------------------------------------------------------------------------------------
def make_input(spec, device="cpu"):
    """spec = {"shape", "seed"[, "view"][, "nan"]}: seeded normal values on the CPU, moved to ``device``, then viewed:
    "t" transposes the last two dimensions, "step" keeps every other time column, "perm" moves dimension 1 last."""
    x = torch.randn(spec["shape"], generator=torch.Generator().manual_seed(spec["seed"]))
    for i in spec.get("nan", ()):
        x.view(-1)[i] = float("nan")
    x = x.to(device)
    view = spec.get("view")
    if view == "t":
        x = x.transpose(-1, -2)
    elif view == "step":
        x = x[..., ::2]
    elif view == "perm":
        x = x.movedim(1, -1)
    return x


def run_case(ns, op, x):
    """op = (name, *args): "iid" / "axis" (mask_param, fill, axis, p), "freq" (param, iid, fill), "time" (param, iid,
    p, fill) or "spec" (n_time, time_param, n_freq, freq_param, iid, p, zero).  A fill ("t", v) is a 0-d tensor on
    the input's device."""
    name, *a = op

    def fill(v):
        return torch.tensor(v[1], dtype=torch.float32, device=x.device) if isinstance(v, tuple) else v

    if name == "iid":
        return ns.mask_along_axis_iid(x, a[0], fill(a[1]), a[2], p=a[3])
    if name == "axis":
        return ns.mask_along_axis(x, a[0], fill(a[1]), a[2], p=a[3])
    if name == "freq":
        return ns.FrequencyMasking(a[0], iid_masks=a[1])(x, fill(a[2]))
    if name == "time":
        return ns.TimeMasking(a[0], iid_masks=a[1], p=a[2])(x, fill(a[3]))
    if name == "spec":
        return ns.SpecAugment(*a[:4], iid_masks=a[4], p=a[5], zero_masking=a[6])(x)
    raise KeyError(name)
