"""CPU: the float64 onset oracle (oracle/onset_oracle.py, librosa 0.10's onset_detect restated) checked piece by piece:
its mel filterbank and power spectrum against torchaudio / torch, peak_pick and onset_backtrack on hand-made envelopes,
the reference's onset-mask slice semantics, and the golden files it wrote."""
import os

import numpy as np
import pytest
import torch

from oracle import onset_oracle as oo

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
PP = dict(pre_max=1, post_max=1, pre_avg=5, post_avg=6, delta=0.07, wait=1)


def test_peak_params_at_the_app_rate():
    assert oo.peak_params(44100, 768) == PP
    assert oo.peak_params(22050, 512) == dict(pre_max=1, post_max=1, pre_avg=4, post_avg=5, delta=0.07, wait=1)


@pytest.mark.parametrize("sr", [44100, 22050, 48000])
def test_mel_filterbank_matches_torchaudio(sr):
    torchaudio = pytest.importorskip("torchaudio")
    want = torchaudio.functional.melscale_fbanks(1025, 0.0, sr / 2, 128, sr, norm="slaney", mel_scale="slaney").T
    got = oo.mel_filterbank(sr)
    assert got.dtype == np.float32 and got.shape == (128, 1025)
    assert np.abs(got - want.numpy()).max() <= 1e-6 * np.abs(want.numpy()).max() * 5


@pytest.mark.parametrize("n", [441600, 441000, 1500, 3000])
def test_power_spectrum_matches_torch_stft(n):
    y = np.random.default_rng(n).standard_normal(n)
    X = torch.stft(torch.from_numpy(y), 2048, 768, window=torch.hann_window(2048, periodic=True, dtype=torch.float64),
                   center=True, pad_mode="constant", return_complex=True)
    P = oo.power_spectrum(y, 768)
    assert P.shape == (1025, oo.n_frames(n, 768)) == tuple(X.shape)
    np.testing.assert_allclose(P, X.abs().numpy() ** 2, rtol=1e-9, atol=1e-9 * P.max())


def _pick(x, **kw):
    return oo.peak_pick(np.asarray(x, dtype=np.float64), **{**PP, **kw})[0].tolist()


def test_peak_pick_wait_suppresses_the_next_frame():
    x = np.zeros(30)
    x[10], x[12] = 1.0, 0.9   # frame 12 > 10 + wait: both kept
    assert _pick(x) == [10, 12]
    x = np.zeros(30)
    x[10], x[11] = 0.9, 1.0   # the max window looks one frame back only: both are peaks, 11 is within the wait
    assert _pick(x) == [10]
    assert _pick(np.r_[np.zeros(10), 1.0, 0.0, 1.0, np.zeros(10)], wait=2) == [10]


def test_peak_pick_plateaus_and_ties():
    x = np.zeros(30)
    x[10] = x[11] = 1.0       # plateau: both equal their window maximum; wait keeps the first only
    assert _pick(x) == [10]
    x[12] = 1.0               # 12 > 10 + 1
    assert _pick(x) == [10, 12]


def test_peak_pick_first_and_last_frame_and_truncated_means():
    x = np.zeros(20)
    x[0] = 1.0                # truncated max window [0, 1) and mean over x[0:6]
    x[19] = 1.0               # truncated mean over x[14:20]
    assert _pick(x) == [0, 19]
    # truncated means at both ends: (5 * 0.2 + 0.3) / 6 + 0.07 = 0.287 <= 0.3 keeps the frame; the untruncated
    # nearest-mode mean (5 * 0.2 + 6 * 0.3) / 11 + 0.07 = 0.325 would not
    y = np.full(20, 0.2)
    y[19] = 0.3
    assert _pick(y) == [19]
    y = np.full(20, 0.2)
    y[0] = 0.3
    assert _pick(y) == [0]


def test_onset_backtrack():
    e = np.array([0.0, 0.0, 0.5, 0.2, 0.1, 0.4, 1.0, 0.3, 0.3, 0.8, 0.2])
    got, _ = oo.onset_backtrack(np.array([6, 9, 2]), e)
    assert got.tolist() == [4, 8, 1]    # 1: 0 <= 0 and 0 < 0.5; 8: 0.3 <= 0.3 and 0.3 < 0.8
    got, _ = oo.onset_backtrack(np.array([0, 10]), e)
    assert got.tolist() == [0, 8]       # frame 0 always qualifies; the last frame never does
    got, _ = oo.onset_backtrack(np.array([3]), np.array([0.5, 0.6, 0.7, 0.8]))
    assert got.tolist() == [0]


@pytest.mark.parametrize("width", [0, 1, 2, 3])
def test_onset_mask_slice_semantics(width):
    T = 10
    got = oo.onset_mask([0, 1, 5, 9, 11], width, (2, 3, T))
    ref = np.ones((2, 3, T), dtype=np.int64)
    for idx in [0, 1, 5, 9, 11]:
        lo, hi = idx - width, idx + width
        start = lo + T if lo < 0 else lo               # the wrapped start of a negative bound
        start = min(max(start, 0), T)
        stop = min(max(hi + T if hi < 0 else hi, 0), T)
        ref[:, :, start:stop] = 0
    assert np.array_equal(got, ref)
    if width >= 1:
        # idx - w < 0: the slice starts at T + idx - w and usually selects nothing before it
        assert oo.onset_mask([0], width, (1, 1, T))[0, 0, :T - width].all()
    if width == 0:
        assert got.all()
    # idx + w > T: truncated at T
    assert not oo.onset_mask([9], 3, (1, 1, T))[0, 0, 6:].any()


@pytest.mark.parametrize("name", oo.SIGNALS)
def test_golden_files_match_the_oracle(name):
    g = np.load(os.path.join(GOLDEN, f"onset_{name}.npz"))
    r = oo.onset_detect(oo.test_signal(name), int(g["sr"]), int(g["hop"]))
    np.testing.assert_allclose(r["envelope"], g["envelope"], rtol=0, atol=1e-12)
    assert r["onsets"].tolist() == g["onsets"].tolist()
    assert r["margin"] == pytest.approx(float(g["margin"]), rel=1e-9) or r["margin"] == float(g["margin"])
