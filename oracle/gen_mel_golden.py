"""TEST INFRASTRUCTURE — write tests/golden/mel_*.npz: seeded signal pairs and their multi-scale mel distance from
oracle/mel_oracle.py in float64.

    python -m oracle.gen_mel_golden

Each file holds the signals x and y (B, C, N) float32, the sample rate, the scales as rows (n_mels, fmin, fmax, w)
(fmax = sr / 2 where audiotools' default None applies), the float64 loss and per-item losses, and one scale's float64
mel spectrogram of x (the first scale).
"""
from __future__ import annotations

import os

import numpy as np

from . import mel_oracle as mo

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

CASES = {
    # the default loss (150 / 80 bands, 2048 / 512 windows) on two 0.3 s mono pairs at 44.1 kHz
    "mel_default": dict(sr=44100, n=13230, B=2, C=1, scales=mo.DEFAULT_SCALES),
    # seven scales from 32 to 2048 samples, empty bands at 32 and 64, on one 0.25 s stereo pair at 48 kHz
    "mel_seven": dict(sr=48000, n=12000, B=1, C=2, scales=mo.SEVEN_SCALES),
}


def make(name: str) -> dict:
    c = CASES[name]
    pairs = [mo.test_pair(c["n"], c["sr"], seed=b, channels=c["C"]) for b in range(c["B"])]
    x = np.stack([p[0] for p in pairs])
    y = np.stack([p[1] for p in pairs])
    loss, items = mo.mel_loss(x, y, c["sr"], c["scales"])
    scales = np.array([(m, lo, c["sr"] / 2 if hi is None else hi, w) for m, lo, hi, w in c["scales"]], dtype=np.float64)
    m, lo, hi, w = c["scales"][0]
    spec = mo.mel_spectrogram(x.astype(np.float64), c["sr"], m, lo, hi, w, w // 4)
    return dict(x=x, y=y, sr=np.int64(c["sr"]), scales=scales, loss=np.float64(loss), item_loss=items, spec=spec)


def main():
    for name in CASES:
        path = os.path.join(OUT, f"{name}.npz")
        np.savez_compressed(path, **make(name))
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
