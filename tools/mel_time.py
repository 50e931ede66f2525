"""CUDA-event time of the default multi-scale mel distance (DESIGN.md §13) on 10 s mono pairs at 44.1 kHz:

    python tools/mel_time.py [--batch 1 16 64] [--iters 20] [--out FILE]

For each batch size, times MelSpectrogramLoss()(x, y) (csrc/mel.cu) and, on the same GPU and signals, the fp32 torch
composition audiotools runs: torch.stft with a periodic Hann window, the magnitude, a matmul with the filterbank and
nn.L1Loss, at both scales.  Each is warmed, then timed over --iters back-to-back calls between two CUDA events, three
times; the median is reported.  The card's name, power limit and SM clocks are read in the same run.
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

from tools.onset_time import time_us  # noqa: E402


def torch_composition(sr, device):
    """audiotools' MelSpectrogramLoss() forward as fp32 torch ops, with the same float32 Slaney filterbanks."""
    from oracle.mel_oracle import DEFAULT_SCALES, hann, mel_filterbank
    scales = [(w, torch.from_numpy(hann(w)).float().to(device),
               torch.from_numpy(mel_filterbank(sr, m, w, lo, hi)).to(device)) for m, lo, hi, w in DEFAULT_SCALES]
    l1 = torch.nn.L1Loss()

    def mel(s, w, win, fb):
        B, C, N = s.shape
        S = torch.stft(s.reshape(-1, N), w, w // 4, window=win, center=True, pad_mode="reflect",
                       return_complex=True).abs()
        return (S.transpose(1, 2) @ fb.T).transpose(1, 2).reshape(B, C, fb.shape[0], -1)

    def loss(x, y):
        out = 0.0
        for w, win, fb in scales:
            X, Y = mel(x, w, win, fb), mel(y, w, win, fb)
            out = out + l1(X.clamp(1e-5).pow(2.0).log10(), Y.clamp(1e-5).pow(2.0).log10())
            out = out + l1(X, Y)
        return out
    return loss


def main():
    from oracle.mel_oracle import test_pair
    from vampnet_b200.audio import AudioSignal
    from vampnet_b200.metrics import MelSpectrogramLoss
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 16, 64])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    card = os.popen("nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv,noheader").read().strip()
    sr, n = 44100, 441000
    ours, ref = MelSpectrogramLoss(), torch_composition(sr, "cuda")
    res = dict(card=card, sr=sr, samples=n, iters=a.iters, batches={})
    for B in a.batch:
        pairs = [test_pair(n, sr, seed=b) for b in range(B)]
        x = torch.from_numpy(np.stack([p[0] for p in pairs])).cuda()
        y = torch.from_numpy(np.stack([p[1] for p in pairs])).cuda()
        xs, ys = AudioSignal(x, sr), AudioSignal(y, sr)
        t_ours, runs_ours = time_us(lambda: ours(xs, ys), a.iters)
        t_ref, runs_ref = time_us(lambda: ref(x, y), a.iters)
        v_ours, v_ref = ours(xs, ys).item(), float(ref(x, y))
        res["batches"][B] = dict(ours_us=t_ours, ours_runs_us=runs_ours, torch_us=t_ref, torch_runs_us=runs_ref,
                                 loss=v_ours, torch_loss=v_ref)
        print(f"B={B:3d} pairs of 10 s: mel.cu {t_ours:9.1f} us ({t_ours / B:8.1f} per pair)   torch fp32 "
              f"{t_ref:9.1f} us ({t_ref / B:8.1f} per pair)   loss {v_ours:.7f} vs {v_ref:.7f}")
    print(f"card: {card}")
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
