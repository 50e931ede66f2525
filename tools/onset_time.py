"""CUDA-event time of onset detection and onset-mask building for B clips of 10 s at 44.1 kHz, hop 768 (576 frames,
the app's analysis shape), and the envelope's distance to the float64 oracle on the same clips:

    python tools/onset_time.py [--batch 1 4 16] [--iters 50] [--out FILE]

Each configuration is warmed, then timed over --iters back-to-back calls between two CUDA events, three times; the
median is reported in us per call and per clip.  "detect" is vampnet_b200.onset.onset_detect (spectrogram, mel, dB,
flux, peak picking and backtracking); "mask" is onset_mask for (B, 14, 575) codes.  The card's name, power limit and
SM clocks are read in the same run.
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

from oracle import onset_oracle as oo  # noqa: E402

SR, HOP, N = 44100, 768, 441600


def time_us(fn, iters, reps=3):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        out.append(1e3 * e0.elapsed_time(e1) / iters)
    return sorted(out)[len(out) // 2], out


def main():
    from vampnet_b200.onset import onset_detect, onset_mask
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    clips = np.stack([oo.test_signal(f"bursts_{N}", seed=s) for s in range(max(a.batch))])
    res = {"clip": dict(sr=SR, hop=HOP, samples=N, frames=oo.n_frames(N, HOP)), "runs": [], "envelope_error": {}}
    for name in oo.SIGNALS:
        y = oo.test_signal(name)
        got = onset_detect(torch.from_numpy(y).cuda(), SR, HOP).envelope[0].cpu().double().numpy()
        want = oo.onset_detect(y, SR, HOP)
        res["envelope_error"][name] = dict(max_abs=float(np.abs(got - want["envelope"]).max()),
                                           oracle_margin=float(want["margin"]))
    for B in a.batch:
        x = torch.from_numpy(clips[:B]).cuda()
        z = torch.zeros(B, 14, -(-N // HOP), dtype=torch.int64, device="cuda")
        det = onset_detect(x, SR, HOP)
        d_us, d_runs = time_us(lambda: onset_detect(x, SR, HOP), a.iters)
        m_us, m_runs = time_us(lambda: onset_mask(det, z, 2), a.iters)
        res["runs"].append(dict(B=B, detect_us=round(d_us, 2), detect_us_per_clip=round(d_us / B, 2),
                                detect_runs_us=[round(r, 2) for r in d_runs], mask_us=round(m_us, 2),
                                mask_runs_us=[round(r, 2) for r in m_runs]))
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
