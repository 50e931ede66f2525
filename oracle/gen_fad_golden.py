"""Writes tests/golden/fad_*.npz: for each case, the weight seed, the 16 kHz signals of a background and an evaluation
set, and the float64 oracle's embeddings, moments and distance (oracle/fad_oracle.py).  The weights (72 M
parameters) are not stored: fad_oracle.random_state_dict(seed) regenerates them.

    python -m oracle.gen_fad_golden
"""
from __future__ import annotations

import os

import numpy as np

from oracle import fad_oracle as fo

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
# per set, the signal lengths in samples at 16 kHz: 1 to 3 examples each, and one too short to give any
CASES = {
    "fad_tones": dict(seed=11, background=[15600, 31000, 15600, 12000], eval=[15600, 31000, 15600, 31000]),
}


def make(name, seed, background, eval):
    sd = fo.random_state_dict(seed)
    out = dict(seed=np.int64(seed))
    moments = []
    for side, lengths in (("background", background), ("eval", eval)):
        sigs = [fo.test_signal(n, 1000 * seed + 10 * i + (side == "eval")) for i, n in enumerate(lengths)]
        if side == "eval":  # louder, with a second tone: a different distribution
            sigs = [np.clip(1.5 * s + fo.test_signal(len(s), 7 + i), -1, 1) for i, s in enumerate(sigs)]
        # stored as float16 to keep the fixture small; the oracle sees the same (rounded) samples
        sigs = [s.astype(np.float16).astype(np.float32) for s in sigs]
        ex = np.concatenate([fo.examples(s) for s in sigs])
        emb = fo.embed(ex, sd)
        mu, sigma = fo.stats(emb)
        moments.append((mu, sigma))
        out[f"{side}_lengths"] = np.array(lengths, np.int64)
        out[f"{side}_signal"] = np.concatenate(sigs).astype(np.float16)
        out[f"{side}_embeddings"] = emb
    out["score"] = np.float64(fo.frechet_distance(*moments[0], *moments[1]))
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **out)
    print(name, "score", float(out["score"]), "examples", len(out["background_embeddings"]), len(out["eval_embeddings"]))


if __name__ == "__main__":
    for name, c in CASES.items():
        make(name, **c)
