"""mit_b200 -- H100-native (sm_90a) detect -> OCR -> inpaint hot path for manga-image-translator.

Python host code over the C-ABI library ``libmitb.so`` (hand-written CUDA, see ../csrc and /include/mitb.h).
Importing this package never imports CUDA code; ``Engine`` / the plugin classes fail loudly when the extension or a
Hopper GPU is missing (there is no CPU fallback).
"""
from ._lib import MitbError, LIB_PATH  # noqa: F401

__all__ = ["MitbError", "LIB_PATH"]
