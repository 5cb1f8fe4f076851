"""sam_audio_b200 — H100-native (sm_90a) implementation of the SAMAudio.separate() hot path.

Public surface mirrors the reference package (reference: sam_audio/__init__.py:3-4):
``SAMAudio``, ``SAMAudioProcessor`` (+ ``Batch``, ``SeparationResult``).
"""
from .config import SAMAudioConfig, stand_in_config  # noqa: F401
from .processor import Batch, SAMAudioProcessor  # noqa: F401


def __getattr__(name):
    # model.py binds the CUDA library lazily so that host-only tools can import the package
    if name in ("SAMAudio", "SeparationResult", "build_synthetic_model", "DFLT_ODE_OPT"):
        from . import model
        return getattr(model, name)
    raise AttributeError(name)


__all__ = ["SAMAudio", "SAMAudioProcessor", "Batch", "SeparationResult", "SAMAudioConfig"]
