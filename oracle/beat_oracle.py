"""TEST INFRASTRUCTURE — float64 restatement of librosa 0.10.1's ``beat.beat_track(y=y, sr=sr, hop_length=H)`` with
every other argument at its default (start_bpm = 120, tightness = 100, trim = True, frame units), the classical beat
tracker behind ``vampnet_b200.beats`` (DESIGN.md §10).

librosa is not a dependency of this project, so the algorithm is written out from the 0.10.1 sources as a contract:

1. ``onset_strength(y, sr, hop_length=H, aggregate=np.median)``: the onset-detect envelope of oracle.onset_oracle
   (steps 1-4 there) before normalisation, with the median over the 128 mel bands in place of the mean.
2. ``feature.tempo`` (ac_size = 8 s, std_bpm = 1, max_tempo = 320, aggregate = mean): W = int(8 sr) // H lags; the
   envelope padded by W // 2 frames of linear ramp from 0 on both sides, cut into one W-frame window per envelope frame,
   times a periodic Hann window, autocorrelated (lags 0..W-1), each frame divided by its largest |value| (left alone
   when that is below tiny(float64)), averaged over frames; then the argmax over lags of
   log1p(1e6 tg) - 0.5 (log2 bpm - log2 120)^2, lags at or above 320 BPM excluded (lag 0 is inf BPM).
3. ``__beat_tracker``: period = round(60 sr / H / bpm) (round half to even); the envelope divided by its standard
   deviation (ddof = 1) when that is > 0; the local score is that convolved ("same") with exp(-0.5 (32 j / period)^2),
   j = -period..period; the dynamic programme over predecessors i + w, w = -2 period .. -round(period / 2), weighted
   -tightness log(-w / period)^2, a predecessor before frame 0 contributing its weight alone; first maximum wins; a
   frame starts no chain (backlink -1) while the first-beat flag is up and its local score is below 0.01 max; the last
   beat is the last local maximum of the cumulative score (x[i] > x[i-1], x[i] >= x[i+1], edge-padded) whose double
   exceeds the median of those maxima; the backlink chain from there; the trim: the local score at the beats smoothed
   by [0.5, 1, 0.5] (scipy's Hann(5) without its zero ends), threshold 0.5 RMS, and ``beats[valid.min():valid.max()]``
   (the last valid beat is dropped, as librosa 0.10.1 does).
4. An all-zero envelope: tempo 0 and no beats.  Where librosa 0.10.1 raises instead of answering (no local maximum of
   the cumulative score, no beat above the trim threshold, a period below one frame) the answer here is no beats.

librosa 0.10.2 rewrote the tracker (numba kernels): the DP there scans predecessors nearest first and skips those
before frame 0, and the trim keeps the last valid beat, so its beats can differ; that release is not restated.
librosa computes the envelope's standard deviation in float32 and its autocorrelation by FFT; here everything after
the envelope is float64, and the smoothing sums run in the order written below.  Parity with librosa itself is not
checked (it is not installed); the GPU path is tested against this file.

Every decision is reported with its margin, relative to the quantities compared: |a - b| / max(|a|, |b|) (an exact
tie of two zeros has no margin to lose).
"""
from __future__ import annotations

import numpy as np

from . import onset_oracle as oo

START_BPM = 120.0
STD_BPM = 1.0
AC_SIZE = 8.0
MAX_TEMPO = 320.0
TIGHTNESS = 100.0


def _rel(a: float, b: float) -> float:
    s = max(abs(a), abs(b))
    return abs(a - b) / s if s > 0 else np.inf


# ------------------------------------------------------------------------------------------------ 1. envelope
def onset_strength(y: np.ndarray, sr: float, hop: int) -> np.ndarray:
    """Raw onset strength with the median over bands, (F,) float64."""
    P = oo.power_spectrum(y, hop)
    S = oo.mel_filterbank(sr).astype(np.float64) @ P
    db = 10.0 * np.log10(np.maximum(oo.AMIN, S))
    db = np.maximum(db, db.max() - oo.TOP_DB)
    flux = np.median(np.maximum(0.0, db[:, 1:] - db[:, :-1]), axis=0)
    pad = 1 + oo.N_FFT // (2 * hop)
    return np.concatenate([np.zeros(pad), flux])[:S.shape[1]]


# ------------------------------------------------------------------------------------------------ 2. tempo
def tempo_lags(sr: float, hop: int) -> int:
    """time_to_frames(8.0, sr, hop): int(8 sr) // hop."""
    return int(AC_SIZE * sr) // hop


def bpm_grid(sr: float, hop: int) -> np.ndarray:
    W = tempo_lags(sr, hop)
    b = np.zeros(W)
    b[0] = np.inf
    b[1:] = 60.0 * sr / (hop * np.arange(1.0, W))
    return b


def log_prior(sr: float, hop: int, start_bpm: float = START_BPM) -> np.ndarray:
    bpms = bpm_grid(sr, hop)
    lp = -0.5 * ((np.log2(bpms) - np.log2(start_bpm)) / STD_BPM) ** 2
    lp[:int(np.argmax(bpms < MAX_TEMPO))] = -np.inf
    return lp


def hann_window(W: int) -> np.ndarray:
    """scipy.signal.get_window("hann", W, fftbins=True): 0.5 + 0.5 cos of linspace(-pi, pi, W + 1)[:W]."""
    fac = np.linspace(-np.pi, np.pi, W + 1)[:W]
    return 0.5 + 0.5 * np.cos(fac)


def tempogram_mean(env: np.ndarray, W: int) -> np.ndarray:
    """The autocorrelation tempogram, normalised per frame by its maximum and averaged over frames, (W,)."""
    env = np.asarray(env, dtype=np.float64)
    n, half = env.shape[0], W // 2
    ramp = lambda e: np.linspace(0.0, e, half, endpoint=False)  # noqa: E731  (numpy's linear_ramp)
    p = np.concatenate([ramp(env[0]), env, ramp(env[-1])[::-1]])
    frames = np.lib.stride_tricks.sliding_window_view(p, W)[:n] * hann_window(W)[None, :]
    n_pad = 2 * W - 1
    ac = np.fft.irfft(np.abs(np.fft.rfft(frames, n=n_pad, axis=1)) ** 2, n=n_pad, axis=1)[:, :W]
    length = np.abs(ac).max(axis=1, keepdims=True)
    length[length < np.finfo(np.float64).tiny] = 1.0
    return (ac / length).mean(axis=0)


def estimate_tempo(env: np.ndarray, sr: float, hop: int, start_bpm: float = START_BPM):
    """Returns (bpm, lag index, margin)."""
    W = tempo_lags(sr, hop)
    score = np.log1p(1e6 * tempogram_mean(env, W)) + log_prior(sr, hop, start_bpm)
    k = int(np.argmax(score))
    rest = np.delete(score, k)
    rest = rest[np.isfinite(rest)]
    margin = _rel(score[k], rest.max()) if rest.size else np.inf
    return float(bpm_grid(sr, hop)[k]), k, margin


# ------------------------------------------------------------------------------------------------ 3. tracker
def local_score(env: np.ndarray, period: int) -> np.ndarray:
    env = np.asarray(env, dtype=np.float64)
    norm = env.std(ddof=1) if env.shape[0] > 1 else np.nan
    if norm > 0:
        env = env / norm
    g = np.exp(-0.5 * (np.arange(-period, period + 1) * 32.0 / period) ** 2)
    F = env.shape[0]
    xp = np.concatenate([np.zeros(period), env, np.zeros(period)])
    out = np.zeros(F)
    for j in range(2 * period + 1):  # out[i] = sum_j env[i + j - period] g[j], j ascending
        out = out + xp[j:j + F] * g[j]
    return out


def track(env: np.ndarray, sr: float, hop: int, bpm: float, tightness: float = TIGHTNESS, trim: bool = True) -> dict:
    """beats (frames), period, and the smallest margin of the DP path, last-beat and trim decisions."""
    none = dict(beats=np.zeros(0, dtype=np.int64), period=0, margin_dp=np.inf, margin_last=np.inf,
                margin_trim=np.inf)
    period = round(60.0 * (float(sr) / hop) / bpm)
    if period < 1:
        return none
    none["period"] = period
    ls = local_score(env, period)
    F = ls.shape[0]
    lo, hi = -2 * period, -int(np.round(period / 2))
    offs = np.arange(lo, hi + 1)
    txwt = -tightness * np.log(-offs / period) ** 2
    cum = np.zeros(F)
    back = np.zeros(F, dtype=np.int64)
    gap = np.full(F, np.inf)
    thr = 0.01 * ls.max()
    first, first_margin = True, np.inf
    for i in range(F):
        idx = i + offs
        cand = txwt + np.where((idx >= 0) & (idx < i), cum[np.clip(idx, 0, None)], 0.0)
        b = int(np.argmax(cand))
        cum[i] = ls[i] + cand[b]
        if cand.size > 1:
            gap[i] = _rel(cand[b], np.delete(cand, b).max())
        if first:
            first_margin = min(first_margin, _rel(ls[i], thr))
        if first and ls[i] < thr:
            back[i] = -1
        else:
            back[i] = i + offs[b]
            first = False
    # last beat: util.localmax with edge padding
    prev = np.concatenate([cum[:1], cum[:-1]])
    nxt = np.concatenate([cum[1:], cum[-1:]])
    maxes = (cum > prev) & (cum >= nxt)
    if not maxes.any():
        return none
    med = np.median(cum[maxes])
    sel = np.flatnonzero(maxes & (2.0 * cum > med))
    if sel.size == 0:
        return none
    margin_last = min(min(_rel(cum[i], prev[i]) for i in range(1, F)) if F > 1 else np.inf,
                      min(_rel(2.0 * cum[i], med) for i in np.flatnonzero(maxes)))
    chain = [int(sel[-1])]
    while back[chain[-1]] >= 0:
        chain.append(int(back[chain[-1]]))
    beats = np.array(chain[::-1], dtype=np.int64)
    margin_dp = min(first_margin, gap[beats].min())
    # trim
    x = ls[beats]
    xp = np.concatenate([[0.0], x, [0.0]])
    smooth = (xp[:-2] * 0.5 + xp[1:-1]) + xp[2:] * 0.5
    t = 0.5 * np.sqrt(np.sum(smooth ** 2) / smooth.size) if trim else 0.0
    valid = np.flatnonzero(smooth > t)
    if valid.size == 0:
        return dict(none, margin_dp=margin_dp, margin_last=margin_last)
    lo_v, hi_v = int(valid.min()), int(valid.max())
    decided = list(range(0, lo_v + 1)) + list(range(hi_v, smooth.size))
    margin_trim = min(_rel(smooth[j], t) for j in decided)
    return dict(beats=beats[lo_v:hi_v], period=period, margin_dp=margin_dp, margin_last=margin_last,
                margin_trim=margin_trim)


def beat_track_envelope(env: np.ndarray, sr: float, hop: int, start_bpm: float = START_BPM,
                        tightness: float = TIGHTNESS, trim: bool = True) -> dict:
    """Steps 2-4 on a given envelope: tempo (BPM, 0 for an all-zero envelope), lag, beats, margin (the smallest)."""
    env = np.asarray(env, dtype=np.float64)
    if not env.any():
        return dict(tempo=0.0, lag=0, beats=np.zeros(0, dtype=np.int64), margin=np.inf, margin_tempo=np.inf,
                    margin_dp=np.inf, margin_last=np.inf, margin_trim=np.inf)
    bpm, lag, mt = estimate_tempo(env, sr, hop, start_bpm)
    r = track(env, sr, hop, bpm, tightness, trim)
    margin = min(mt, r["margin_dp"], r["margin_last"], r["margin_trim"])
    return dict(tempo=bpm, lag=lag, beats=r["beats"], margin=margin, margin_tempo=mt, margin_dp=r["margin_dp"],
                margin_last=r["margin_last"], margin_trim=r["margin_trim"])


def beat_track(y: np.ndarray, sr: float, hop: int = 512, **kw) -> dict:
    """Steps 1-4.  envelope: the float64 envelope; the decisions are taken on it rounded to float32, the precision
    the GPU envelope is delivered in."""
    env = onset_strength(y, sr, hop)
    r = beat_track_envelope(env.astype(np.float32), sr, hop, **kw)
    r["envelope"] = env
    return r


def frames_to_time(frames, sr: float, hop: int) -> np.ndarray:
    return np.asarray(frames, dtype=np.int64) * hop / float(sr)


# ------------------------------------------------------------------------------------------------ test signals
def click_train(period_samples: float, seconds: float, sr: int = 44100, seed: int = 0, offset: float = 0.1,
                noise: float = 1e-3) -> np.ndarray:
    rng = np.random.default_rng(seed)
    n = int(seconds * sr)
    y = noise * rng.standard_normal(n)
    t = offset * sr
    while t < n:
        i = int(round(t))
        y[i:i + 32] += 0.9 * np.hanning(32)[:n - i]
        t += period_samples
    return y.astype(np.float32)


def test_signal(name: str, sr: int = 44100, seed: int = 0) -> np.ndarray:
    """Seeded synthetic float32 clips used by the tests and the golden files."""
    rng = np.random.default_rng(seed)
    if name.startswith("clicks"):   # clicks<bpm>
        return click_train(60.0 * sr / float(name[6:]), 6.0, sr, seed)
    if name.startswith("bursts_"):  # bursts_<seconds>: tone bursts at a 0.52 s beat over noise
        n = int(float(name[7:]) * sr)
        y = 0.01 * rng.standard_normal(n)
        tt = np.arange(n) / sr
        for k, t0 in enumerate(np.arange(0.2, n / sr - 0.1, 0.52)):
            on = tt >= t0
            y += on * 0.5 * np.exp(-10.0 * np.maximum(tt - t0, 0)) * np.sin(2 * np.pi * (180 * (k % 4 + 1)) * tt)
        return y.astype(np.float32)
    if name in ("silence", "dc", "short"):
        return oo.test_signal(name, sr, seed)
    raise KeyError(name)


SIGNALS = ("clicks90", "clicks120", "clicks150", "bursts_4", "silence", "dc", "short", "bursts_10", "bursts_30")
