"""CPU: the float64 pitch-shift oracle (oracle/pitch_oracle.py) against torch and torchaudio themselves, the golden
outputs, the shapes and formulas it states, get_fast_shifts, and the torch_pitch_shift import name."""
import math
import os
from fractions import Fraction

import numpy as np
import pytest

from oracle import gen_pitch_golden as gg
from oracle import pitch_oracle as po

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("shift", [-12, -7, -2, 0, 2, 10, 12, Fraction(4, 3)])
def test_oracle_equals_torchaudio_composition(shift):
    pytest.importorskip("torchaudio")
    x = gg.signal(44100, 0.5, 11)[None, None]
    want = gg.torch_composition(x, shift, 44100)
    got, _ = po.pitch_shift(x, shift, 44100)
    assert np.abs(got - want).max() < 1e-11


@pytest.mark.parametrize("name", [n for n, *_ in gg.CASES])
def test_oracle_equals_goldens(name):
    x, shift, sr, out, cond = gg.load(os.path.join(GOLDEN, f"pitch_{name}.npz"))
    got, c = po.pitch_shift(x, shift, sr)
    assert c > 1e-8 and math.isclose(c, cond, rel_tol=1e-9)
    assert np.abs(got - out).max() < 1e-7  # out is stored in float32


def test_time_steps_formula():
    ts = po.time_steps(1051, 2 ** (-7 / 12))
    assert ts.dtype == np.float32 and ts.size == math.ceil(1051 / 2 ** (-7 / 12))
    assert np.array_equal(ts, np.float32(2 ** (-7 / 12)) * np.arange(ts.size, dtype=np.float32))
    assert po.time_steps(10, 0.5).tolist() == [i * 0.5 for i in range(20)]


def test_lengths():
    # 1 s at 44.1 kHz: n_fft 689 (odd), hop 21; torch.stft's frame count is 1 + (N - 1) // hop for odd n_fft
    spec = po.stft(np.zeros((1, 44100)), 689, 21)
    assert spec.shape == (1, 2100, 345)
    assert po.stft(np.zeros((1, 48000)), 750, 23).shape == (1, 1 + 48000 // 23, 376)
    # istft: n_fft - 2 (n_fft // 2) + hop (F' - 1)
    assert po.istft(np.zeros((1, 10, 345), complex), 689, 21).shape == (1, 1 + 21 * 9)
    assert po.istft(np.zeros((1, 10, 376), complex), 750, 23).shape == (1, 23 * 9)
    # resample: ceil(new_g L / orig_g), the quotient rounded to float32 first
    assert po.resample(np.zeros((1, 44101)), 44100, 39288).shape == (1, math.ceil(np.float32(3274 * 44101 / 3675)))
    # +2 semitones on a 1 s clip ends a few samples short of N; the tail is zero
    n_fft, hop, new, rate = po.shift_params(2, 44100)
    assert (n_fft, hop, new) == (689, 21, 39288)
    x = gg.signal(44100, 1.0, 12)[None, None]
    out, _ = po.pitch_shift(x, 2, 44100)
    F2 = math.ceil(2100 / rate)
    target = math.ceil(np.float32(3274 * (1 + 21 * (F2 - 1)) / 3675))
    assert target < 44100 and np.all(out[..., target:] == 0) and np.any(out[..., target - 1] != 0)


def test_shift_params():
    assert po.shift_params(-12, 44100) == (689, 21, 88200, 2.0)
    assert po.shift_params(12, 44100) == (689, 21, 22050, 0.5)
    assert po.shift_params(Fraction(4, 3), 44100) == (689, 21, 33075, 0.75)
    assert po.shift_params(0, 48000) == (750, 23, 48000, 1.0)


def test_get_fast_shifts():
    from vampnet_b200.pitch import get_fast_shifts, shift_params
    fs = get_fast_shifts(44100)
    assert all(isinstance(f, Fraction) and 0.5 <= f <= 2 and f != 1 for f in fs)
    for f in (Fraction(1, 2), Fraction(2), Fraction(4, 3), Fraction(3, 4), Fraction(49, 50), Fraction(25, 18)):
        assert f in fs
    assert Fraction(11, 10) not in fs and Fraction(1, 3) not in fs  # 11 does not divide 44100; 1/3 is below 0.5
    assert fs == sorted(set(fs))
    assert get_fast_shifts(44100, lambda f: f == Fraction(7, 5)) == [Fraction(7, 5)]
    assert get_fast_shifts(9973) == []  # a prime rate: no ratio other than 1
    assert shift_params(Fraction(4, 3), 44100) == po.shift_params(Fraction(4, 3), 44100)
    assert shift_params(-5, 44100) == po.shift_params(-5, 44100)


def test_torch_pitch_shift_name_resolves_here():
    ns = {}
    exec("from torch_pitch_shift import pitch_shift, get_fast_shifts", ns)
    import vampnet_b200.pitch
    assert ns["pitch_shift"] is vampnet_b200.pitch.pitch_shift
    assert ns["get_fast_shifts"] is vampnet_b200.pitch.get_fast_shifts
    import torch_pitch_shift
    assert sorted(torch_pitch_shift.__all__) == ["get_fast_shifts", "pitch_shift"]
    assert os.path.dirname(os.path.dirname(torch_pitch_shift.__file__)) == os.path.dirname(os.path.dirname(__file__))


def test_cpu_input_without_cuda_raises():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    from vampnet_b200.pitch import pitch_shift
    with pytest.raises(RuntimeError):
        pitch_shift(torch.zeros(1, 1, 4000), 2, 44100)


def test_silence_then_tone_angles_are_zero():
    # digital silence gives all-zero frames: angle 0 on both sides, and they leave the conditioning figure alone
    x = gg.signal(44100, 0.5, 9, 0.2)
    spec = po.stft(x[None].astype(np.float64), 689, 21)
    silent = np.abs(spec).max(axis=-1) == 0
    assert silent[0, :100].all() and np.all(np.angle(spec[silent]) == 0)
