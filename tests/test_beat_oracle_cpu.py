"""CPU: the float64 restatement of librosa 0.10.1's beat_track (oracle/beat_oracle.py) on probes whose answers are
exact, and against its own golden files (tests/golden/beat_*.npz, written by oracle/gen_beat_golden.py)."""
import os

import numpy as np
import pytest

from oracle import beat_oracle as bo

SR, HOP = 44100, 512
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def test_click_train_with_a_whole_frame_period():
    """Clicks every 43 frames: tempo = tempo_frequencies[43] and one beat per click, 1-2 frames after it (the flux
    peaks where the click enters the analysis window, shifted by the envelope's padding), except the last click,
    which the trim drops."""
    y = bo.click_train(43 * HOP, 8.0, SR, offset=0.1)
    r = bo.beat_track(y, SR, HOP)
    assert r["lag"] == 43 and r["tempo"] == 60.0 * SR / (HOP * 43.0)
    clicks = (0.1 * SR + 43 * HOP * np.arange(16)) / HOP
    clicks = clicks[clicks < y.shape[0] / HOP]
    beats = r["beats"]
    assert len(beats) == len(clicks) - 1
    lag = beats - clicks[:len(beats)]
    assert np.all((lag > 1) & (lag <= 2)), lag
    assert r["margin"] > 1e-4


def test_impulse_envelope():
    """An envelope of unit impulses every 40 frames: the tempo lag is 40 and every impulse but the last is a beat."""
    env = np.zeros(800)
    env[5::40] = 1.0
    r = bo.beat_track_envelope(env, SR, HOP)
    assert r["lag"] == 40 and r["tempo"] == 60.0 * SR / (HOP * 40.0)
    assert r["beats"].tolist() == list(range(5, 765, 40))


@pytest.mark.parametrize("name", ["silence", "dc"])
def test_silence_and_dc_give_no_tempo_and_no_beats(name):
    r = bo.beat_track(bo.test_signal(name), SR, HOP)
    assert not r["envelope"].any()
    assert r["tempo"] == 0.0 and len(r["beats"]) == 0


@pytest.mark.parametrize("n", [1, 300, 1500, 2047])
def test_clip_shorter_than_n_fft(n):
    y = (0.3 * np.random.default_rng(n).standard_normal(n)).astype(np.float32)
    r = bo.beat_track(y, SR, HOP)
    assert r["envelope"].shape == (1 + n // HOP,)
    if r["envelope"].any():
        assert r["tempo"] > 0 and np.all((r["beats"] >= 0) & (r["beats"] < r["envelope"].shape[0]))
    else:
        assert r["tempo"] == 0.0 and len(r["beats"]) == 0


def test_tempo_prior_and_window():
    lp = bo.log_prior(SR, HOP)
    bpms = bo.bpm_grid(SR, HOP)
    assert bo.tempo_lags(SR, HOP) == 689 == len(bpms)
    assert np.all(np.isneginf(lp[bpms >= bo.MAX_TEMPO])) and np.all(np.isfinite(lp[bpms < bo.MAX_TEMPO]))
    w = bo.hann_window(8)
    assert np.allclose(w, 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(8) / 8), atol=1e-15)


def test_trim_drops_the_last_valid_beat():
    """beats[valid.min():valid.max()] drops the last valid beat.  The chain ends on a beat after the last impulse:
    without the trim (threshold 0) that extra beat is the one dropped; with it,
    the extra beat falls below 0.5 RMS and the last impulse, now the last valid beat, is dropped."""
    env = np.zeros(400)
    env[10::30] = 1.0
    r0 = bo.beat_track_envelope(env, SR, HOP, trim=False)
    r1 = bo.beat_track_envelope(env, SR, HOP, trim=True)
    assert r0["beats"].tolist() == list(range(10, 371, 30))
    assert r1["beats"].tolist() == list(range(10, 341, 30))


@pytest.mark.parametrize("name", bo.SIGNALS)
def test_oracle_reproduces_golden(name):
    g = np.load(os.path.join(GOLDEN, f"beat_{name}.npz"))
    r = bo.beat_track(bo.test_signal(name), int(g["sr"]), int(g["hop"]))
    np.testing.assert_allclose(r["envelope"], g["envelope"], rtol=1e-12, atol=1e-12)
    assert r["tempo"] == float(g["tempo"]) and r["lag"] == int(g["lag"])
    assert r["beats"].tolist() == g["beats"].tolist()
    assert r["margin"] == pytest.approx(float(g["margin"]), rel=1e-6)
