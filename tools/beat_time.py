"""CUDA-event time of beat tracking (vampnet_b200.beats.beat_track at 44.1 kHz, hop 512) for 1, 4 and 16 rows of 10 s
clips and for one 30 s and one 100 s clip (the app accepts uploads up to 100 s), and the envelope's distance to the
float64 oracle:

    python tools/beat_time.py [--iters 20] [--out FILE]

Each configuration is warmed, then timed over --iters back-to-back calls between two CUDA events, three times; the
median is reported in us per call and per clip.  The card's name, power limit and SM clocks are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import beat_oracle as bo  # noqa: E402
from tools.onset_time import time_us  # noqa: E402

SR, HOP = 44100, 512


def main():
    from vampnet_b200.beats import beat_track
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    res = {"clip": dict(sr=SR, hop=HOP), "runs": [], "envelope_error": {}}
    for name in bo.SIGNALS:
        y = bo.test_signal(name)
        got = beat_track(torch.from_numpy(y).cuda(), SR, HOP)
        want = bo.beat_track(y, SR, HOP)
        env = got.envelope[0].cpu().double().numpy()
        res["envelope_error"][name] = dict(
            max_rel=float(np.abs(env - want["envelope"]).max() / max(want["envelope"].max(), 1e-30)),
            oracle_margin=float(want["margin"]), beats_equal=got.frames[0, :int(got.counts[0])].cpu().numpy().tolist()
            == want["beats"].tolist())
    shapes = [(1, 10.0), (4, 10.0), (16, 10.0), (1, 30.0), (1, 100.0)]
    for B, seconds in shapes:
        x = torch.from_numpy(np.stack([bo.test_signal(f"bursts_{seconds:g}", seed=s) for s in range(B)])).cuda()
        us, runs = time_us(lambda: beat_track(x, SR, HOP), a.iters)
        res["runs"].append(dict(B=B, seconds=seconds, frames=1 + x.shape[1] // HOP, us=round(us, 1),
                                us_per_clip=round(us / B, 1), runs_us=[round(r, 1) for r in runs]))
    q = os.popen("nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv,noheader").read().strip()
    res["card"] = torch.cuda.get_device_name(0)
    res["nvidia_smi"] = q
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
