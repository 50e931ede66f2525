"""Stands in for the torch_pitch_shift package (1.2) that the app imports (app.py:59): the same two names, running on
the GPU kernels of vampnet_b200.pitch."""
from vampnet_b200.pitch import get_fast_shifts, pitch_shift

__all__ = ["pitch_shift", "get_fast_shifts"]
