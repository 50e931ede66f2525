"""TEST INFRASTRUCTURE — write tests/golden/beat_<signal>.npz: the float64 beat oracle's envelope, tempo, tempo lag,
beat frames and decision margins for each synthetic signal of oracle.beat_oracle.SIGNALS (44.1 kHz, hop 512).

    python -m oracle.gen_beat_golden

Data only: the signals are regenerated from their seeds by oracle.beat_oracle.test_signal.
"""
from __future__ import annotations

import os

import numpy as np

from . import beat_oracle as bo

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
SR, HOP = 44100, 512
MARGINS = ("margin", "margin_tempo", "margin_dp", "margin_last", "margin_trim")


def main():
    for name in bo.SIGNALS:
        r = bo.beat_track(bo.test_signal(name), SR, HOP)
        np.savez_compressed(os.path.join(OUT, f"beat_{name}.npz"), envelope=r["envelope"], tempo=np.float64(r["tempo"]),
                            lag=np.int64(r["lag"]), beats=r["beats"], sr=np.int64(SR), hop=np.int64(HOP),
                            **{m: np.float64(r[m]) for m in MARGINS})
        print(name, r["tempo"], r["beats"].tolist(), f"margin {r['margin']:.2e}")


if __name__ == "__main__":
    main()
