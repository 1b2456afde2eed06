"""wav2lip_b200 — H100-native compute core for the Wav2Lip hot path.

Python host side: a ctypes binding of libw2l.so (include/w2l.h) plus mirrors of the reference's
`models` package and `audio.melspectrogram` with the same names and call signatures.  PyTorch is
used for device memory and streams only; all arithmetic happens in the hand-written sm_90a kernels
behind the C-ABI.  There is no CPU fallback: without the built library or without an H100 every
compute call raises.
"""
from . import _lib  # noqa: F401
from ._lib import W2LError, lib_path  # noqa: F401

__all__ = ["_lib", "W2LError", "lib_path", "models", "audio"]


def __getattr__(name):  # lazy: `models` imports torch
    if name in ("models", "audio"):
        import importlib
        return importlib.import_module("." + name, __name__)
    raise AttributeError(name)
