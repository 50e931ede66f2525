"""CPU: the mel-distance oracle (oracle/mel_oracle.py) against torch and torchaudio in float64, its goldens, and the
host logic of the eval CLI (vampnet_b200.eval) with the loss injected."""
import csv
import math

import numpy as np
import pytest
import torch
import torchaudio

from oracle import gen_mel_golden as gm
from oracle import mel_oracle as mo
from oracle import onset_oracle as oo


@pytest.mark.parametrize("n_fft,hop,N", [(32, 8, 17), (512, 128, 4000), (2048, 512, 1025), (4096, 1024, 9000),
                                          (256, 100, 3001)])
def test_stft_matches_torch_float64(n_fft, hop, N):
    y = np.random.default_rng(n_fft).standard_normal((2, N))
    win = torch.hann_window(n_fft, periodic=True, dtype=torch.float64)
    want = torch.stft(torch.from_numpy(y), n_fft, hop, window=win, center=True, pad_mode="reflect",
                      return_complex=True).numpy()
    got = mo.stft(y, n_fft, hop, window=win.numpy())
    assert got.shape == want.shape == (2, n_fft // 2 + 1, 1 + N // hop)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


def test_stft_refuses_short_input():
    with pytest.raises(ValueError):
        mo.stft(np.zeros(1024), 2048, 512)


def test_window_is_scipy_hann_in_float32():
    import scipy.signal
    for w in (32, 512, 2048, 4096):
        assert np.array_equal(mo.hann(w), scipy.signal.get_window("hann", w).astype(np.float32).astype(np.float64))
        # the same fp32 values as the periodic Hann that onset_oracle and the device tables evaluate
        assert np.array_equal(mo.hann(w).astype(np.float32), oo.hann_periodic(w).astype(np.float32))


# (sr, n_fft, n_mels, fmin, fmax)
BANKS = [(44100, 2048, 150, 0.0, None), (44100, 512, 80, 0.0, None), (16000, 512, 80, 0.0, None),
         (22050, 1024, 64, 100.0, 8000.0), (48000, 32, 5, 0.0, None), (44100, 4096, 320, 30.0, 20000.0)]


@pytest.mark.parametrize("sr,n_fft,n_mels,fmin,fmax", BANKS)
def test_filterbank_matches_torchaudio(sr, n_fft, n_mels, fmin, fmax):
    """torchaudio builds the band edges with a float32 linspace, so it agrees with librosa's float64 construction to
    about 1e-5 of the largest weight (1.1e-5 measured at 4096 / 320 bands)."""
    got = mo.mel_filterbank(sr, n_mels, n_fft, fmin, fmax)
    assert got.dtype == np.float32 and got.shape == (n_mels, n_fft // 2 + 1)
    with pytest.warns(UserWarning) if n_fft == 32 else _nothing():
        want = torchaudio.functional.melscale_fbanks(n_fft // 2 + 1, fmin, fmax or sr / 2, n_mels, sr, norm="slaney",
                                                     mel_scale="slaney").T.numpy()
    assert np.abs(got - want).max() <= 2e-5 * np.abs(want).max()


class _nothing:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


@pytest.mark.parametrize("sr", [16000, 22050, 44100, 48000])
def test_filterbank_defaults_are_onsets(sr):
    assert np.array_equal(mo.mel_filterbank(sr, 128, 2048, 0.0, sr / 2), oo.mel_filterbank(sr))
    assert np.array_equal(mo.mel_filterbank(sr, 128, 2048, 0.0, None), oo.mel_filterbank(sr))


def test_seven_scales_have_empty_bands_at_48k():
    empty = [int((mo.mel_filterbank(48000, m, w, 0.0, None) == 0).all(1).sum()) for m, _, _, w in mo.SEVEN_SCALES]
    assert empty == [1, 1, 0, 0, 0, 0, 0]


def _torch_loss(x, y, sr, scales, eps=1e-5, pw=2.0):
    """The audiotools composition in float64 torch: torch.stft, the filterbank, nn.L1Loss."""
    x, y = torch.from_numpy(x.astype(np.float64)), torch.from_numpy(y.astype(np.float64))
    B, C, N = x.shape
    loss, l1 = 0.0, torch.nn.L1Loss()
    for n_mels, fmin, fmax, w in scales:
        win = torch.from_numpy(mo.hann(w))
        fb = torch.from_numpy(mo.mel_filterbank(sr, n_mels, w, fmin, fmax).astype(np.float64))

        def mel(s):
            S = torch.stft(s.reshape(-1, N), w, w // 4, window=win, center=True, pad_mode="reflect",
                           return_complex=True).abs()
            return (S.transpose(1, 2) @ fb.T).transpose(1, 2).reshape(B, C, n_mels, -1)
        X, Y = mel(x), mel(y)
        loss = loss + l1(X.clamp(eps).pow(pw).log10(), Y.clamp(eps).pow(pw).log10())
        loss = loss + l1(X, Y)
    return float(loss)


@pytest.mark.parametrize("name", list(gm.CASES))
def test_loss_matches_torch_float64_and_golden(name):
    g = np.load(f"{gm.OUT}/{name}.npz")
    c = gm.CASES[name]
    x, y, sr = g["x"], g["y"], int(g["sr"])
    loss, items = mo.mel_loss(x, y, sr, c["scales"])
    want = _torch_loss(x, y, sr, c["scales"])
    assert abs(loss - want) <= 1e-12 * abs(want)
    assert abs(items.mean() - loss) <= 1e-12 * loss
    fresh = gm.make(name)
    assert np.array_equal(fresh["x"], x) and np.array_equal(fresh["y"], y)
    assert loss == float(g["loss"]) and np.array_equal(items, g["item_loss"])


def test_loss_is_zero_for_equal_signals_and_symmetric():
    x, y = mo.test_pair(4000, 16000)
    assert mo.mel_loss(x[None], x[None], 16000)[0] == 0.0
    assert mo.mel_loss(x[None], y[None], 16000)[0] == mo.mel_loss(y[None], x[None], 16000)[0]


# ------------------------------------------------------------------------------------------------ eval CLI, host side
def _write(path, data, sr):
    from vampnet_b200.audio import AudioSignal
    AudioSignal(torch.from_numpy(np.asarray(data, dtype=np.float32)), sr).write(path)


def _fake_loss(calls):
    """Per item: the mean of |x - y| and the length, so the test sees what each pair was scored on."""
    def loss(x, y):
        calls.append((tuple(x.audio_data.shape), x.sample_rate))
        return ((x.audio_data - y.audio_data).abs().mean((1, 2)) + 1000.0 * x.signal_length).double()
    return loss


def _exp(tmp_path, sr=8000, n=800):
    rng = np.random.default_rng(0)
    base = [0.5 * rng.standard_normal((1, n)).clip(-0.9, 0.9) for _ in range(3)]
    for i, b in enumerate(base):
        _write(tmp_path / "baseline" / f"{i}.wav", b, sr)
        _write(tmp_path / "plain" / f"{i}.wav", b * 0.5, sr)
    for i in (0, 1):  # a condition with fewer files: the baseline list is cut to 2 for it
        _write(tmp_path / "inpaint_0.01" / f"{i}.wav", base[i] * 0.25, sr)
    return base


def test_eval_pairs_trims_and_writes_csvs(tmp_path):
    from vampnet_b200 import eval as ev
    for d in ("baseline", "plain", "inpaint_0.01"):
        (tmp_path / d).mkdir()
    _exp(tmp_path)
    calls = []
    rows = ev.evaluate(tmp_path, loss=_fake_loss(calls))
    # conditions sorted by name, files by int(stem), one call per condition (all pairs share a shape)
    assert [(c, f) for _, c, f in rows] == [("inpaint_0.01", "0"), ("inpaint_0.01", "1"), ("plain", "0"),
                                            ("plain", "1"), ("plain", "2")]
    assert calls == [((2, 1, 800 - 2 * 80), 8000), ((3, 1, 800), 8000)]  # int(0.01 * 8000) = 80 trimmed from each end
    with open(tmp_path / "metrics-all.csv") as f:
        got = list(csv.reader(f))
    assert got[0] == ["mel", "condition", "file"]
    assert [r[1:] for r in got[1:]] == [[c, s] for _, c, s in rows]
    assert [float(r[0]) for r in got[1:]] == [m for m, _, _ in rows]
    with open(tmp_path / "stats-mel.csv") as f:
        stats = list(csv.reader(f))
    assert stats[0] == ["condition", "mean", "count", "std"]
    for row, cond in zip(stats[1:], ("inpaint_0.01", "plain")):
        v = np.array([m for m, c, _ in rows if c == cond])
        assert row[0] == cond and float(row[1]) == v.mean() and int(row[2]) == v.size
        assert float(row[3]) == np.std(v, ddof=1)


def test_eval_single_file_condition_has_empty_std(tmp_path):
    from vampnet_b200 import eval as ev
    for d in ("baseline", "one"):
        (tmp_path / d).mkdir()
    _write(tmp_path / "baseline" / "0.wav", np.zeros((1, 400)), 8000)
    _write(tmp_path / "one" / "0.wav", np.zeros((1, 400)), 8000)
    ev.evaluate(tmp_path, loss=_fake_loss([]))
    with open(tmp_path / "stats-mel.csv") as f:
        assert list(csv.reader(f))[1][2:] == ["1", ""]


def test_eval_resamples_and_truncates_condition(tmp_path):
    from vampnet_b200 import eval as ev
    for d in ("baseline", "up"):
        (tmp_path / d).mkdir()
    _write(tmp_path / "baseline" / "0.wav", np.zeros((1, 800)), 8000)
    _write(tmp_path / "up" / "0.wav", np.zeros((1, 2000)), 16000)  # 2000 at 16 kHz -> 1000 at 8 kHz -> cut to 800
    calls = []
    ev.evaluate(tmp_path, loss=_fake_loss(calls))
    assert calls == [((1, 1, 800), 8000)]


def test_eval_stem_mismatch_and_missing_baseline(tmp_path):
    from vampnet_b200 import eval as ev
    for d in ("baseline", "bad"):
        (tmp_path / d).mkdir()
    _write(tmp_path / "baseline" / "0.wav", np.zeros((1, 400)), 8000)
    _write(tmp_path / "bad" / "7.wav", np.zeros((1, 400)), 8000)
    with pytest.raises(ValueError, match="do not match"):
        ev.evaluate(tmp_path, loss=_fake_loss([]))
    with pytest.raises(ValueError, match="not found"):
        ev.evaluate(tmp_path, baseline_key="nope", loss=_fake_loss([]))


def test_eval_short_condition_is_refused(tmp_path):
    from vampnet_b200 import eval as ev
    for d in ("baseline", "short"):
        (tmp_path / d).mkdir()
    _write(tmp_path / "baseline" / "0.wav", np.zeros((1, 400)), 8000)
    _write(tmp_path / "short" / "0.wav", np.zeros((1, 300)), 8000)
    with pytest.raises(ValueError, match="differs from the baseline"):
        ev.evaluate(tmp_path, loss=_fake_loss([]))


# ------------------------------------------------------------------------------------------------ options, host side
def test_loss_refuses_unsupported_options():
    from vampnet_b200.metrics import MelSpectrogramLoss
    MelSpectrogramLoss()
    MelSpectrogramLoss(window_type="hann", n_mels=[5] * 7, window_lengths=[2 ** k for k in range(5, 12)],
                       mel_fmin=[0.0] * 7, mel_fmax=[None] * 7)
    for kw in (dict(loss_fn=torch.nn.MSELoss()), dict(loss_fn=torch.nn.L1Loss(reduction="sum")),
               dict(match_stride=True), dict(window_type="sqrt_hann"), dict(window_lengths=[2048, 500]),
               dict(window_lengths=[8192, 512]), dict(window_lengths=[16, 512]), dict(n_mels=[150])):
        with pytest.raises(ValueError):
            MelSpectrogramLoss(**kw)


def test_default_stft_is_audiotools():
    from vampnet_b200.metrics import default_stft
    assert default_stft(44100) == (2048, 512)
    assert default_stft(16000) == (512, 128)
    assert default_stft(48000) == (2048, 512)
    assert default_stft(22050) == (1024, 256)
    assert all(w == int(2 ** math.ceil(math.log2(0.032 * sr))) for sr in (8000, 24000, 32000, 96000)
               for w in [default_stft(sr)[0]])


def test_truncate_samples():
    from vampnet_b200.audio import AudioSignal
    s = AudioSignal(torch.arange(10.0)[None, None], 8000).truncate_samples(4)
    assert s.audio_data.tolist() == [[[0.0, 1.0, 2.0, 3.0]]]
