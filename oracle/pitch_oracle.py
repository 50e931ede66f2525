"""torch_pitch_shift 1.2's pitch_shift restated in float64 numpy (DESIGN.md §11).

    torch.stft(x, n_fft, hop, return_complex=True)           rectangular window, center=True, reflect padding
    TimeStretch(fixed_rate=1/ratio, n_freq, hop)              torchaudio.functional.phase_vocoder, phase advance
                                                              linspace(0, pi hop, n_bins) in float32
    torch.istft(., n_fft, hop)                                rectangular window, center=True, length=None
    torchaudio.functional.resample(., sr, int(sr / ratio))    sinc_interp_hann, width 6, rolloff 0.99
    cut or zero-pad to N

Everything is float64 except the vocoder's time steps, which are the float32 values torch.arange(0, F, rate) gives
on CUDA (float(rate) * float(i)); ``time_steps`` states them.  ``pitch_shift`` also returns the conditioning figure:
the smallest bin magnitude, relative to its frame's largest, among the bins of non-silent frames whose angle enters
the phase accumulation.  An angle decided by rounding stays in every later frame's phase, so a signal is a fair test
of a float64 implementation only where that figure is well above the float64 epsilon (1e-8 is used).
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np


def shift_params(shift, sample_rate, bins_per_octave=12, n_fft=0, hop_length=0):
    n_fft = int(n_fft) or int(sample_rate) // 64
    hop = int(hop_length) or n_fft // 32
    ratio = shift if isinstance(shift, Fraction) else 2.0 ** (float(shift) / bins_per_octave)
    return n_fft, hop, int(sample_rate / ratio), float(1 / ratio)


def time_steps(F, rate):
    n = math.ceil(F / rate)
    return (np.float32(rate) * np.arange(n, dtype=np.float32)).astype(np.float32)


def phase_advance(nb, hop):
    """torch.linspace(0, pi * hop, nb) in float32, from both ends as torch computes it."""
    end = np.float32(math.pi * hop)
    step = np.float32(end / np.float32(nb - 1))
    k = np.arange(nb)
    lo = step * k.astype(np.float32)
    hi = end - step * (nb - 1 - k).astype(np.float32)
    return np.where(k < nb // 2, lo, hi).astype(np.float32).astype(np.float64)


def stft(x, n_fft, hop):
    """(rows, N) -> (rows, F, n_bins) complex128."""
    pad = n_fft // 2
    xp = np.pad(x, ((0, 0), (pad, pad)), mode="reflect")
    F = 1 + (x.shape[1] + 2 * pad - n_fft) // hop  # 1 + (N - 1) // hop for odd n_fft
    idx = np.arange(F)[:, None] * hop + np.arange(n_fft)[None, :]
    return np.fft.rfft(xp[:, idx], axis=-1)


def phase_vocoder(spec, rate, hop, ts=None):
    """(rows, F, nb) -> (rows, F', nb), and the conditioning figure."""
    if rate == 1.0:
        return spec, math.inf
    rows, F, nb = spec.shape
    ts = time_steps(F, rate) if ts is None else ts
    alphas = (ts % np.float32(1.0)).astype(np.float64)[None, :, None]
    i0 = np.floor(ts).astype(np.int64)
    padded = np.concatenate([spec, np.zeros((rows, 2, nb), spec.dtype)], axis=1)
    s0, s1 = padded[:, i0], padded[:, i0 + 1]
    adv = phase_advance(nb, hop)[None, None, :]
    ph = np.angle(s1) - np.angle(s0) - adv
    ph = ph - 2 * math.pi * np.round(ph / (2 * math.pi))
    ph = ph + adv
    ph = np.concatenate([np.angle(spec[:, :1]), ph[:, :-1]], axis=1)
    acc = np.cumsum(ph, axis=1)
    mag = alphas * np.abs(s1) + (1 - alphas) * np.abs(s0)
    # conditioning: frames whose angles enter (frame 0, and both gathered frames of every kept increment)
    used = np.zeros(F + 2, bool)
    used[0] = True
    used[i0[:-1]] = True
    used[i0[:-1] + 1] = True
    a = np.abs(spec[:, used[:F]])
    peak = a.max(axis=-1, keepdims=True)
    live = np.broadcast_to(peak > 0, a.shape)
    cond = float((a / np.where(peak > 0, peak, 1.0))[live].min()) if live.any() else math.inf
    return mag * np.exp(1j * acc), cond


def istft(spec, n_fft, hop):
    """(rows, F', nb) -> (rows, L), L = n_fft - 2 (n_fft // 2) + hop (F' - 1)."""
    rows, F2, _ = spec.shape
    frames = np.fft.irfft(spec, n=n_fft, axis=-1)
    total = n_fft + hop * (F2 - 1)
    y = np.zeros((rows, total))
    cnt = np.zeros(total)
    for f in range(F2):
        y[:, f * hop:f * hop + n_fft] += frames[:, f]
        cnt[f * hop:f * hop + n_fft] += 1
    s = n_fft // 2
    return y[:, s:total - s] / cnt[s:total - s]


def resample(y, orig, new):
    """torchaudio.functional.resample(y, orig, new) with its defaults, each output from its taps with |t| < 6."""
    if orig == new:
        return y
    g = math.gcd(int(orig), int(new))
    o_g, n_g = int(orig) // g, int(new) // g
    base = min(o_g, n_g) * 0.99
    width = math.ceil(6 * o_g / base)
    rows, L = y.shape
    target = int(math.ceil(np.float32(n_g * L / o_g)))
    o = np.arange(target)
    c, j = o // n_g, o % n_g
    reach = 6 * o_g / base
    centre = o_g * (j / n_g)
    u0 = np.maximum(-width, np.floor(centre - reach).astype(np.int64) - 1)
    T = int(math.ceil(2 * reach)) + 4
    u = u0[:, None] + np.arange(T)[None, :]
    t = ((-j)[:, None] / n_g + u / o_g) * base
    ok = (np.abs(t) < 6) & (u <= width + o_g - 1)
    p = c[:, None] * o_g + u
    ok &= (p >= 0) & (p < L)
    w = np.cos(t * math.pi / 6 / 2) ** 2
    tp = t * math.pi
    with np.errstate(invalid="ignore", divide="ignore"):
        k = np.where(tp == 0, 1.0, np.sin(tp) / tp)
    k = k * (w * (base / o_g))
    k = np.where(ok, k, 0.0)
    return np.einsum("rot,ot->ro", y[:, np.clip(p, 0, L - 1)], k)


def pitch_shift(x, shift, sample_rate, bins_per_octave=12, n_fft=0, hop_length=0):
    """x (B, C, N) -> (out (B, C, N) float64, conditioning figure)."""
    x = np.asarray(x, dtype=np.float64)
    B, C, N = x.shape
    n_fft, hop, new_freq, rate = shift_params(shift, sample_rate, bins_per_octave, n_fft, hop_length)
    rows = x.reshape(B * C, N)
    spec, cond = phase_vocoder(stft(rows, n_fft, hop), rate, hop)
    y = resample(istft(spec, n_fft, hop), sample_rate, new_freq)
    out = np.zeros((B * C, N))
    n = min(N, y.shape[1])
    out[:, :n] = y[:, :n]
    return out.reshape(B, C, N), cond
