"""TEST INFRASTRUCTURE — write tests/golden/onset_<signal>.npz: the float64 onset oracle's normalised envelope, onset
frames and smallest decision margin for each synthetic signal of oracle.onset_oracle.SIGNALS (44.1 kHz, hop 768).

    python -m oracle.gen_onset_golden

Data only: the signals are regenerated from their seeds by oracle.onset_oracle.test_signal.
"""
from __future__ import annotations

import os

import numpy as np

from . import onset_oracle as oo

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
SR, HOP = 44100, 768


def main():
    for name in oo.SIGNALS:
        r = oo.onset_detect(oo.test_signal(name), SR, HOP)
        np.savez_compressed(os.path.join(OUT, f"onset_{name}.npz"), envelope=r["envelope"], onsets=r["onsets"],
                            margin=np.float64(r["margin"]), sr=np.int64(SR), hop=np.int64(HOP))
        print(name, r["onsets"].tolist())


if __name__ == "__main__":
    main()
