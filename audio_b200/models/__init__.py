"""Model-side components on the GPU: ``models.decoder`` (the CUDA CTC prefix beam-search decoder)."""
from . import decoder  # noqa: F401
