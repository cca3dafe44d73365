"""byol_b200 — H100-native (sm_90a) BYOL training step behind the jramapuram/BYOL Python API.

Importing the package loads the mandatory C-ABI CUDA library (``libbyol_b200.so``); there is no fallback.
"""
from . import _lib  # noqa: F401  (fails loudly when the CUDA extension is missing)

__all__ = ["_lib"]
