"""fastlivo_b200 -- H100-native FAST-LIVO measurement / iterated-ESKF hot path.

The product is ``libfastlivo_b200.so`` (hand-written sm_90a CUDA behind the C ABI of
``include/fastlivo_b200.h``).  This Python package is only the thin ctypes binding the
tests and ``bench.py`` drive it through, plus the synthetic-frame generator.  The
directory name contains a hyphen, so import it through ``fastlivo_loader.load()`` at
the repo root (registers it as module ``fastlivo_b200``).
"""
from . import capi, synth  # noqa: F401
from .capi import Handle, FlbError, build, lib_path  # noqa: F401
