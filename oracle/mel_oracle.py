"""TEST INFRASTRUCTURE — float64 restatement of audiotools' ``AudioSignal.mel_spectrogram`` and
``metrics.spectral.MelSpectrogramLoss`` (the audio metric of the reference's scripts/exp/eval.py).

audiotools is not installed and the reference does not pin it, so the definition is written out as a contract
(DESIGN.md §13), and the GPU path is tested against this file:

1. Window: periodic Hann, ``scipy.signal.get_window("hann", w)`` rounded to float32 (audiotools moves it to the
   device as a float32 tensor).
2. ``torch.stft(x, n_fft=w, hop_length=hop, window, center=True, pad_mode="reflect")``: the signal reflect-padded by
   w // 2 on both sides, F = 1 + N // hop frames, magnitude of the 1 + w // 2 bins.
3. Projection on ``librosa.filters.mel(sr, n_fft=w, n_mels, fmin, fmax or sr / 2)``: Slaney scale and norm, the
   weights rounded to float32 as librosa stores them.  At (2048, 128, 0, sr / 2) this is onset_oracle.mel_filterbank.
4. The loss, per scale: log_weight * mean|log10(max(X, eps) ** pow) - log10(max(Y, eps) ** pow)|
   + mag_weight * mean|X - Y|, the means over all B * C * n_mels * F elements, summed over the scales.

Everything after the float32 window and weights is float64 here.
"""
from __future__ import annotations

import numpy as np
import scipy.signal

from oracle.onset_oracle import _hz_to_mel, _mel_to_hz

DEFAULT_SCALES = ((150, 0.0, None, 2048), (80, 0.0, None, 512))  # (n_mels, fmin, fmax, window length)


def hann(w: int) -> np.ndarray:
    """Step 1, as float64 values of the float32 window."""
    return scipy.signal.get_window("hann", w).astype(np.float32).astype(np.float64)


def mel_filterbank(sr: float, n_mels: int, n_fft: int, fmin: float = 0.0, fmax: float = None) -> np.ndarray:
    """Step 3: (n_mels, 1 + n_fft // 2) float32, as librosa.filters.mel(sr=sr, n_fft=n_fft, n_mels=n_mels, fmin=fmin,
    fmax=fmax or sr / 2, htk=False, norm="slaney") builds it."""
    fmax = 0.5 * sr if fmax is None else fmax
    fftfreqs = np.fft.rfftfreq(n_fft, d=1.0 / sr)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    w = np.zeros((n_mels, 1 + n_fft // 2), dtype=np.float32)
    for i in range(n_mels):
        w[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    return (w.astype(np.float64) * enorm[:, None]).astype(np.float32)


def stft(y: np.ndarray, n_fft: int, hop: int, window: np.ndarray = None) -> np.ndarray:
    """Step 2 for (..., N) float64 samples: complex (..., 1 + n_fft // 2, F).  N must exceed n_fft // 2."""
    y = np.asarray(y, dtype=np.float64)
    N = y.shape[-1]
    if N <= n_fft // 2:
        raise ValueError(f"N = {N} must exceed n_fft // 2 = {n_fft // 2}")
    window = hann(n_fft) if window is None else np.asarray(window, dtype=np.float64)
    pad = [(0, 0)] * (y.ndim - 1) + [(n_fft // 2, n_fft // 2)]
    yp = np.pad(y, pad, mode="reflect")
    F = 1 + N // hop
    idx = np.arange(F)[:, None] * hop + np.arange(n_fft)[None, :]
    X = np.fft.rfft(yp[..., idx] * window, axis=-1)  # (..., F, bins)
    return np.swapaxes(X, -1, -2)


def mel_spectrogram(y: np.ndarray, sr: int, n_mels: int, fmin: float, fmax, n_fft: int, hop: int) -> np.ndarray:
    """Steps 1-3: (..., N) -> (..., n_mels, F) float64."""
    fb = mel_filterbank(sr, n_mels, n_fft, fmin, fmax).astype(np.float64)
    return np.matmul(fb, np.abs(stft(y, n_fft, hop)))


def mel_loss(x: np.ndarray, y: np.ndarray, sr: int, scales=DEFAULT_SCALES, clamp_eps: float = 1e-5, pow: float = 2.0,
             log_weight: float = 1.0, mag_weight: float = 1.0):
    """Step 4 for (B, C, N) signals: (loss, per-item losses (B,)), float64.  scales: (n_mels, fmin, fmax, w) with
    hop = w // 4."""
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    loss, items = 0.0, np.zeros(x.shape[0])
    for n_mels, fmin, fmax, w in scales:
        X = mel_spectrogram(x, sr, n_mels, fmin, fmax, w, w // 4)
        Y = mel_spectrogram(y, sr, n_mels, fmin, fmax, w, w // 4)
        dlog = np.abs(np.log10(np.maximum(X, clamp_eps) ** pow) - np.log10(np.maximum(Y, clamp_eps) ** pow))
        dmag = np.abs(X - Y)
        loss += log_weight * dlog.mean() + mag_weight * dmag.mean()
        items += log_weight * dlog.reshape(x.shape[0], -1).mean(1) + mag_weight * dmag.reshape(x.shape[0], -1).mean(1)
    return float(loss), items


# ------------------------------------------------------------------------------------------------ test signals
def test_pair(n: int, sr: int, seed: int = 0, channels: int = 1):
    """Two seeded float32 (channels, n) signals: a tone over noise with a silent first tenth, and noise brick-wall
    low-passed at 0.36 sr (16 kHz at 44.1 kHz)."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    a = 0.4 * np.sin(2 * np.pi * 440.0 * t)[None] + 0.05 * rng.standard_normal((channels, n))
    a[:, : n // 10] = 0.0
    noise = rng.standard_normal((channels, n))
    spec = np.fft.rfft(noise, axis=-1)
    spec[:, np.fft.rfftfreq(n, 1.0 / sr) > 0.36 * sr] = 0.0
    b = 0.2 * np.fft.irfft(spec, n=n, axis=-1)
    return a.astype(np.float32), b.astype(np.float32)


# Seven scales from 32 to 2048 samples with 5 to 320 bands; at 48 kHz the 32 and 64 windows have an empty band each
SEVEN_SCALES = tuple((m, 0.0, None, w) for m, w in zip((5, 10, 20, 40, 80, 160, 320), (32, 64, 128, 256, 512, 1024, 2048)))
