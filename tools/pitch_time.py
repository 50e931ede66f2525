"""CUDA-event time of pitch shift (vampnet_b200.pitch.pitch_shift at 44.1 kHz, n_fft 689, hop 21) for 1, 4 and 16 rows
of 10 s clips and one 30 s clip, at -11, -1, +5 and +12 semitones, and, where torchaudio imports, of the reference's own
fp32 composition on CUDA (torch_pitch_shift 1.2's steps) for the shifts whose resampler table fits in memory:

    python tools/pitch_time.py [--iters 5] [--out FILE]

Each configuration is warmed, then timed over --iters back-to-back calls between two CUDA events, three times; the
median is reported in ms per call and per clip.  The card's name, power limit and SM clocks are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import gen_pitch_golden as gg  # noqa: E402
from oracle import pitch_oracle as po  # noqa: E402
from tools.onset_time import time_us  # noqa: E402

SR = 44100
SHIFTS = (-11, -1, 5, 12)
TABLE_LIMIT = 2e9  # bytes of one float64 intermediate of torchaudio's resampler table


def reference_fp32(x, shift):
    """torch_pitch_shift 1.2's pitch_shift on x (B, C, N) fp32 CUDA, as that package composes it."""
    import torchaudio
    B, C, N = x.shape
    n_fft, hop, new_freq, rate = po.shift_params(shift, SR)
    y = torch.stft(x.reshape(B * C, N), n_fft, hop, return_complex=True)[None]
    y = torchaudio.transforms.TimeStretch(fixed_rate=rate, n_freq=y.shape[2], hop_length=hop).to(x.device)(y)
    y = torch.istft(y[0], n_fft, hop)
    y = torchaudio.transforms.Resample(SR, new_freq).to(x.device)(y)
    y = y[:, :N] if y.shape[1] >= N else torch.nn.functional.pad(y, (0, N - y.shape[1]))
    return y.reshape(B, C, N)


def table_bytes(shift):
    _, _, new, _ = po.shift_params(shift, SR)
    g = math.gcd(SR, new)
    o, n = SR // g, new // g
    return 8 * n * (o + 2 * math.ceil(6 * o / (min(o, n) * 0.99)))


def main():
    from vampnet_b200.pitch import pitch_shift
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    try:
        import torchaudio  # noqa: F401
        have_ta = True
    except Exception:
        have_ta = False
    res = {"clip": dict(sr=SR, n_fft=689, hop=21), "runs": [], "reference_fp32": [], "torchaudio": have_ta}
    for B, seconds in [(1, 10.0), (4, 10.0), (16, 10.0), (1, 30.0)]:
        x = torch.from_numpy(np.stack([gg.signal(SR, seconds, s) for s in range(B)])[:, None]).cuda()
        for shift in SHIFTS:
            us, runs = time_us(lambda: pitch_shift(x, shift, SR), a.iters)
            res["runs"].append(dict(B=B, seconds=seconds, shift=shift, ms=round(us / 1e3, 3),
                                    ms_per_clip=round(us / 1e3 / B, 3), runs_ms=[round(r / 1e3, 3) for r in runs]))
            if have_ta and B == 1 and seconds == 10.0:
                if table_bytes(shift) > TABLE_LIMIT:
                    res["reference_fp32"].append(dict(shift=shift, ms=None, table_bytes=table_bytes(shift)))
                else:
                    us, runs = time_us(lambda: reference_fp32(x, shift), a.iters)
                    res["reference_fp32"].append(dict(shift=shift, ms=round(us / 1e3, 3),
                                                      table_bytes=table_bytes(shift)))
        del x
        torch.cuda.empty_cache()
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
