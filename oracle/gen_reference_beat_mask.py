"""Run the ORIGINAL project's ``Interface.make_beat_mask`` once, with a tracker that returns fixed beat and downbeat
times, and store its masks and the torch draws that follow each call.

    VAMPNET_REFERENCE_ROOT=<checkout of the original vampnet> python -m oracle.gen_reference_beat_mask

Writes tests/golden/reference_beat_mask.npz.  tests/test_beat_mask_cpu.py rebuilds each mask with
``vampnet_b200.beats.beat_mask`` from the same times and seeds and compares, so it needs no checkout of the original.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_shims  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
SR, HOP, N_CODEBOOKS, DURATION = 44100, 768, 14, 6.3
BEATS = np.arange(0.0, 6.0, 0.4) + np.array([0.0, 0.013] * 8)[:15]
DOWNBEATS = np.concatenate([BEATS[::4], [5.95]])
# (beats, downbeats, kwargs) per case; shared with the test
CASES = [
    ("empty", np.zeros(0), np.zeros(0), {}),
    ("no_downbeats", BEATS, np.zeros(0), {}),
    ("overlap", BEATS, DOWNBEATS, {}),
    ("before", BEATS, DOWNBEATS, dict(before_beat_s=0.1, after_beat_s=0.05)),
    ("factors_dropout", BEATS, DOWNBEATS, dict(beat_downsample_factor=2, downbeat_downsample_factor=3, dropout=0.3)),
    ("factors_dropout_noinvert", BEATS, DOWNBEATS,
     dict(beat_downsample_factor=3, downbeat_downsample_factor=2, dropout=0.3, invert=False)),
    ("no_upbeats", BEATS, DOWNBEATS, dict(mask_upbeats=False, after_beat_s=0.1)),
    ("no_downbeats_masked", BEATS, DOWNBEATS, dict(mask_downbeats=False, before_beat_s=0.05, dropout=0.5)),
    ("before_dropout", BEATS, DOWNBEATS, dict(before_beat_s=0.2, dropout=0.3)),
]


def s2t_stub(s2t):
    """An object carrying what make_beat_mask reads from the Interface besides the tracker."""
    stub = types.SimpleNamespace(codec=types.SimpleNamespace(sample_rate=SR, hop_length=HOP), device="cpu",
                                 c2f=types.SimpleNamespace(n_codebooks=N_CODEBOOKS), coarse=None)
    stub.s2t = lambda s: s2t(stub, s)
    return stub


def main():
    if not ref_shims.available():
        raise SystemExit(f"the original project is not at {ref_shims.REFERENCE_ROOT} (set VAMPNET_REFERENCE_ROOT)")
    try:
        Ref = ref_shims.load_reference_interface().Interface
        out = {}
        for k, (name, beats, downbeats, kw) in enumerate(CASES):
            stub = s2t_stub(Ref.s2t)
            stub.beat_tracker = types.SimpleNamespace(extract_beats=lambda sig, b=beats, d=downbeats: (b, d))
            torch.manual_seed(100 + k)
            mask = Ref.make_beat_mask(stub, types.SimpleNamespace(duration=DURATION), **kw)
            out[f"{name}_mask"] = mask.numpy().astype(np.int8)
            out[f"{name}_next"] = torch.rand(8).numpy()
            print(name, tuple(mask.shape), int(mask.sum()))
        np.savez_compressed(os.path.join(GOLDEN, "reference_beat_mask.npz"), **out)
    finally:
        ref_shims.uninstall()


if __name__ == "__main__":
    main()
