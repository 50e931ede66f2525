"""TEST INFRASTRUCTURE — float64 restatement of librosa 0.10.x ``onset.onset_detect(y, sr, hop_length=H,
backtrack=True)`` with every other argument at its default, the detector behind the reference's ``mask.onset_mask``
(reference vampnet/mask.py:203-226) and the app's ``onsets()`` helper (app.py:69-78).

librosa is not a dependency of this project, so the algorithm is written out from the 0.10 sources as a contract:

1. ``stft(n_fft=2048, hop=H, window="hann", center=True, pad_mode="constant")``: periodic Hann window, the signal
   zero-padded by n_fft // 2 on both sides, 1 + N // H frames, power |X|^2 for 1 + n_fft // 2 bins.
2. 128 Slaney mel bands, fmin = 0, fmax = 0.5 * sr (set by ``onset_strength_multi``), ``norm="slaney"``, the weights
   rounded to float32 exactly as ``filters.mel`` does.
3. ``power_to_db(S, ref=1, amin=1e-10, top_db=80)``: clamped below at the clip's maximum minus 80.
4. Spectral flux with lag 1 and max_size 1, averaged over the bands, left-padded by lag + n_fft // (2 H), trimmed.
5. Normalised to [0, 1]: minus the minimum, over (maximum + tiny(float32)).  All-zero or non-finite: no onsets.
6. ``util.peak_pick`` with pre_max = 0.03 sr // H, post_max = 1, pre_avg = 0.10 sr // H, post_avg = pre_avg + 1,
   wait = 0.03 sr // H (each rounded up to an int), delta = 0.07.
7. ``onset_backtrack`` onto the preceding local minimum of the normalised envelope (frame 0 always a candidate).
8. The reference's mask: ``mask[:, :, idx - w:idx + w] = 0`` with Python slice semantics.

Versions before 0.10 used fmax = 11025 Hz and ``pad_mode="reflect"``; those are not what is restated here.
Parity with librosa itself is not checked (it is not installed); the GPU path is tested against this file.

Every decision of steps 6-7 is also reported with its margin, the distance by which it was taken, so that a test
can tell a robust decision from a knife-edge one.
"""
from __future__ import annotations

import math

import numpy as np

N_FFT = 2048
N_MELS = 128
AMIN = 1e-10
TOP_DB = 80.0
DELTA = 0.07
TINY32 = float(np.finfo(np.float32).tiny)


# ------------------------------------------------------------------------------------------------ 1. spectrogram
def hann_periodic(n: int = N_FFT) -> np.ndarray:
    k = np.arange(n, dtype=np.float64)
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * k / n)


def n_frames(n_samples: int, hop: int) -> int:
    return 1 + n_samples // hop


def power_spectrum(y: np.ndarray, hop: int) -> np.ndarray:
    """|STFT|^2, (1 + n_fft // 2, F) float64."""
    y = np.asarray(y, dtype=np.float64)
    F = n_frames(y.shape[-1], hop)
    yp = np.pad(y, (N_FFT // 2, N_FFT // 2 + hop * F))  # right side: room for the last frame at any length
    idx = np.arange(F)[:, None] * hop + np.arange(N_FFT)[None, :]
    X = np.fft.rfft(yp[idx] * hann_periodic()[None, :], axis=-1)
    return (X.real ** 2 + X.imag ** 2).T


# ------------------------------------------------------------------------------------------------ 2. mel
def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-300) / min_log_hz) / logstep, f / f_sp)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_filterbank(sr: float, n_mels: int = N_MELS) -> np.ndarray:
    """(n_mels, 1 + n_fft // 2) float32, as librosa.filters.mel(sr=sr, n_fft=2048, fmax=sr / 2) builds it."""
    fftfreqs = np.fft.rfftfreq(N_FFT, d=1.0 / sr)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(0.0), _hz_to_mel(0.5 * sr), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    w = np.zeros((n_mels, 1 + N_FFT // 2), dtype=np.float32)
    for i in range(n_mels):
        w[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    return (w.astype(np.float64) * enorm[:, None]).astype(np.float32)


# ------------------------------------------------------------------------------------------------ 3-5. envelope
def onset_strength(y: np.ndarray, sr: float, hop: int) -> np.ndarray:
    """Raw (unnormalised) onset envelope, (F,) float64."""
    P = power_spectrum(y, hop)
    S = mel_filterbank(sr).astype(np.float64) @ P
    db = 10.0 * np.log10(np.maximum(AMIN, S))
    db = np.maximum(db, db.max() - TOP_DB)
    flux = np.maximum(0.0, db[:, 1:] - db[:, :-1]).mean(axis=0)
    pad = 1 + N_FFT // (2 * hop)
    return np.concatenate([np.zeros(pad), flux])[:S.shape[1]]


def normalise(env: np.ndarray) -> np.ndarray:
    env = env - env.min()
    return env / (env.max() + TINY32)


# ------------------------------------------------------------------------------------------------ 6. peak_pick
def peak_params(sr: float, hop: int) -> dict:
    """onset_detect's defaults (float expressions with Python's float //), rounded up as peak_pick does."""
    c = lambda v: int(math.ceil(v))  # noqa: E731
    return dict(pre_max=c(0.03 * sr // hop), post_max=c(0.00 * sr // hop + 1), pre_avg=c(0.10 * sr // hop),
                post_avg=c(0.10 * sr // hop + 1), wait=c(0.03 * sr // hop), delta=DELTA)


def peak_pick(x: np.ndarray, pre_max: int, post_max: int, pre_avg: int, post_avg: int, delta: float, wait: int):
    """Returns (peaks, margin).  Windows are truncated at both ends: frame i compares against x[i - pre : i + post].
    This is what librosa's maximum_filter1d(cval=x.min()) and its corrected uniform_filter1d compute for the defaults
    (post_max = 1 and post_avg = pre_avg + 1, where both filters have origin 0).

    margin: the smallest distance by which any frame's keep decision (x == mov_max and x >= mov_avg + delta) was
    taken.  For x == mov_max that is the gap between x[i] and the largest other value in its window."""
    x = np.asarray(x, dtype=np.float64)
    F = x.shape[0]
    keep = np.zeros(F, dtype=bool)
    margin = np.inf
    for i in range(F):
        lo, hi = max(0, i - pre_max), min(F, i + post_max)
        others = np.concatenate([x[lo:i], x[i + 1:hi]])
        a = x[i] - others.max() if others.size else np.inf       # >= 0: x[i] is the window's maximum
        lo, hi = max(0, i - pre_avg), min(F, i + post_avg)
        b = x[i] - (x[lo:hi].mean() + delta)                      # >= 0: above the threshold
        keep[i] = a >= 0 and b >= 0 and x[i] != 0
        m = min(a, b) if keep[i] else max(v for v in (-a, -b) if v > 0) if (a < 0 or b < 0) else np.inf
        margin = min(margin, m)
    peaks, last = [], -np.inf
    for i in np.flatnonzero(keep):
        if i > last + wait:
            peaks.append(int(i))
            last = i
    return np.array(peaks, dtype=np.int64), float(margin)


# ------------------------------------------------------------------------------------------------ 7. backtrack
def onset_backtrack(events: np.ndarray, energy: np.ndarray, exact_prefix: int = 0):
    """Each event moves to the latest frame m <= event with energy[m] <= energy[m-1] and energy[m] < energy[m+1]
    (frame 0 always qualifies).  Returns (frames, margin): margin is the smallest distance by which a minimum test
    was decided on the frames that decide some event, [chosen minimum, event].  A comparison between two of the
    first `exact_prefix` frames (the envelope's zero padding, exact in any precision) has no margin to lose."""
    e = np.asarray(energy, dtype=np.float64)
    F = e.shape[0]
    is_min = np.zeros(F, dtype=bool)
    is_min[0] = True
    gap = np.full(F, np.inf)
    for i in range(1, F - 1):
        a, b = e[i - 1] - e[i], e[i + 1] - e[i]   # minimum iff a >= 0 and b > 0
        is_min[i] = a >= 0 and b > 0
        if i < exact_prefix:
            a = np.inf if a == 0 else a
            b = np.inf if b == 0 and i + 1 < exact_prefix else b
        gap[i] = min(abs(a), abs(b)) if is_min[i] else max((v for v in (-a, -b) if v >= 0), default=np.inf)
    out, margin = [], np.inf
    for ev in np.asarray(events, dtype=np.int64):
        m = int(np.flatnonzero(is_min[:ev + 1])[-1])
        out.append(m)
        margin = min(margin, gap[m:ev + 1].min())
    return np.array(out, dtype=np.int64), float(margin)


# ------------------------------------------------------------------------------------------------ steps 1-7
def onset_detect(y: np.ndarray, sr: float, hop: int, backtrack: bool = True) -> dict:
    """envelope: the normalised envelope (F,); onsets: frame indices; margin: smallest decision margin (inf when
    nothing was decided)."""
    env = normalise(onset_strength(y, sr, hop))
    if not env.any() or not np.all(np.isfinite(env)):
        return dict(envelope=env, onsets=np.zeros(0, dtype=np.int64), margin=np.inf)
    p = peak_params(sr, hop)
    peaks, margin = peak_pick(env, **p)
    if backtrack:
        peaks, m2 = onset_backtrack(peaks, env, exact_prefix=1 + N_FFT // (2 * hop))
        margin = min(margin, m2)
    return dict(envelope=env, onsets=peaks, margin=margin)


# ------------------------------------------------------------------------------------------------ 8. mask
def onset_mask(onsets, width: int, shape) -> np.ndarray:
    """The reference's loop, verbatim: ones, then mask[:, :, idx - width:idx + width] = 0 per onset."""
    mask = np.ones(shape, dtype=np.int64)
    for idx in onsets:
        mask[:, :, int(idx) - width:int(idx) + width] = 0
    return mask


# ------------------------------------------------------------------------------------------------ test signals
def test_signal(name: str, sr: int = 44100, seed: int = 0) -> np.ndarray:
    """Seeded synthetic float32 clips used by the tests and the golden files."""
    rng = np.random.default_rng(seed)
    if name == "clicks":
        y = 1e-3 * rng.standard_normal(int(2.0 * sr))
        for t in (0.25, 0.61, 1.02, 1.37, 1.80):
            y[int(t * sr)] += 0.9
    elif name == "bursts":
        n = int(3.0 * sr)
        y = 0.01 * rng.standard_normal(n)
        tt = np.arange(n) / sr
        for k, t0 in enumerate((0.3, 0.9, 1.55, 2.2, 2.7)):
            on = tt >= t0
            y += on * 0.5 * np.exp(-6.0 * np.maximum(tt - t0, 0)) * np.sin(2 * np.pi * (220 * (k + 1)) * tt)
    elif name == "silence":
        y = np.zeros(int(1.0 * sr))
    elif name == "dc":
        y = np.full(int(1.0 * sr), 0.25)
    elif name == "short":
        y = 0.3 * rng.standard_normal(1500)
    elif name.startswith("bursts_"):  # bursts_<n samples>
        n = int(name.split("_")[1])
        y = 0.01 * rng.standard_normal(n)
        tt = np.arange(n) / sr
        for k, t0 in enumerate(np.arange(0.4, n / sr - 0.2, 0.85)):
            on = tt >= t0
            y += on * 0.5 * np.exp(-8.0 * np.maximum(tt - t0, 0)) * np.sin(2 * np.pi * (180 * (k % 5 + 1)) * tt)
    else:
        raise KeyError(name)
    return y.astype(np.float32)


SIGNALS = ("clicks", "bursts", "silence", "dc", "short", "bursts_441000", "bursts_441600", "bursts_132300")
