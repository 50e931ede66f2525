"""Write tests/golden/pitch_*.npz: torch_pitch_shift's composition run in float64 by torch and torchaudio themselves.

    python -m oracle.gen_pitch_golden

``torch_composition`` is torch_pitch_shift 1.2's pitch_shift with every tensor in float64: torch.stft ->
torchaudio.transforms.TimeStretch (its float32 phase advance) -> torch.istft -> torchaudio.functional.resample.  The
vocoder's time steps are the float32 values the reference computes on CUDA (oracle.pitch_oracle.time_steps), not a
float64 arange.  Each file holds the fp32 input ``x``, the shift (``shift`` in semitones, or ``num``/``den`` for a
Fraction), the sample rate, the composition's output ``out`` (rounded to float32) and the oracle's conditioning
figure ``cond``.
"""
from __future__ import annotations

import math
import os
from fractions import Fraction

import numpy as np

from oracle import pitch_oracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")


def signal(sr, seconds, seed, silence_s=0.0):
    """A few partials with a slow vibrato, onsets and a seeded noise floor (1e-3), peaking below 1; optionally digital
    silence first."""
    rng = np.random.default_rng(seed)
    n = int(sr * seconds)
    t = np.arange(n) / sr
    x = np.zeros(n)
    for f, a in zip(rng.uniform(110, 2000, 4), (0.3, 0.2, 0.15, 0.1)):
        x += a * np.sin(2 * np.pi * f * t + 3 * np.sin(2 * np.pi * 5 * t) / 5 + rng.uniform(0, 2 * np.pi))
    x *= 0.6 + 0.4 * np.cos(2 * np.pi * 1.5 * t) ** 2
    x += 1e-3 * rng.standard_normal(n)
    if silence_s:
        x[:int(sr * silence_s)] = 0.0
    return (x / (1.05 * np.abs(x).max())).astype(np.float32)


def torch_composition(x, shift, sample_rate, bins_per_octave=12):
    """x (B, C, N) float32 numpy -> float64 numpy, by torch and torchaudio in float64."""
    import torch
    import torchaudio
    B, C, N = x.shape
    n_fft, hop, new_freq, rate = po.shift_params(shift, sample_rate, bins_per_octave)
    y = torch.from_numpy(np.asarray(x, dtype=np.float64).reshape(B * C, N))
    spec = torch.stft(y, n_fft, hop, return_complex=True)
    stretcher = torchaudio.transforms.TimeStretch(fixed_rate=rate, n_freq=spec.shape[-2], hop_length=hop)
    arange = torch.arange

    def fp32_steps(start, end, step, dtype=None, device=None):  # the reference's float32 time steps, held in float64
        assert start == 0
        return torch.from_numpy(po.time_steps(end, step)).to(dtype)

    torch.arange = fp32_steps
    try:
        spec = stretcher(spec[None])[0]
    finally:
        torch.arange = arange
    y = torch.istft(spec, n_fft, hop)
    y = torchaudio.functional.resample(y, sample_rate, new_freq)
    out = torch.zeros(B * C, N, dtype=torch.float64)
    n = min(N, y.shape[1])
    out[:, :n] = y[:, :n]
    return out.reshape(B, C, N).numpy()


CASES = [  # name, sample rate, seconds, seed, shift, leading silence (s)
    ("m12", 44100, 0.5, 1, -12, 0.0),
    ("m7", 44100, 0.5, 2, -7, 0.0),
    ("m2", 44100, 0.5, 3, -2, 0.0),
    ("p2", 44100, 0.5, 4, 2, 0.0),
    ("p9", 44100, 0.5, 5, 9, 0.0),
    ("p12", 44100, 0.5, 6, 12, 0.0),
    ("frac4_3", 44100, 0.5, 7, Fraction(4, 3), 0.0),
    ("sr48k_p9", 48000, 0.5, 8, 9, 0.0),
    ("silence_m2", 44100, 0.5, 9, -2, 0.2),
]


def main():
    for name, sr, seconds, seed, shift, silence in CASES:
        x = signal(sr, seconds, seed, silence)[None, None]
        out = torch_composition(x, shift, sr)
        _, cond = po.pitch_shift(x, shift, sr)
        frac = isinstance(shift, Fraction)
        np.savez_compressed(os.path.join(GOLDEN, f"pitch_{name}.npz"), x=x, out=out.astype(np.float32),
                            sample_rate=sr, cond=cond, shift=0 if frac else shift,
                            num=shift.numerator if frac else 0, den=shift.denominator if frac else 0)
        print(name, f"cond {cond:.2e}", f"max |out| {np.abs(out).max():.3f}")


def load(path):
    """(x, shift, sample_rate, out, cond) of a golden file."""
    z = np.load(path)
    shift = Fraction(int(z["num"]), int(z["den"])) if int(z["den"]) else int(z["shift"])
    return z["x"], shift, int(z["sample_rate"]), z["out"], float(z["cond"])


if __name__ == "__main__":
    main()
