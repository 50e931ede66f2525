"""GPU: pitch shift (vampnet_b200/pitch.py, csrc/pitch.cu) against the float64 restatement of torch_pitch_shift 1.2's
composition in oracle/pitch_oracle.py, and the golden outputs of torch and torchaudio themselves in float64.

Everything between the fp32 ends runs in float64, so the outputs are compared within ATOL, absolute, on signals peaking
below 1.  The vocoder's running phase keeps any rounding of a quiet bin's angle for the rest of the clip, so every
signal's conditioning figure (the smallest relative bin magnitude whose angle enters that sum) is asserted above
COND_MIN: a signal that would make the comparison a test of rounding fails loudly instead."""
import ctypes
import os
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import gen_pitch_golden as gg
from oracle import pitch_oracle as po

pytestmark = pytest.mark.gpu

SR = 44100
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
ATOL = 1e-6
COND_MIN = 1e-8
_worst = {}


def _shift(x, shift, sr=SR, **kw):
    from vampnet_b200.pitch import pitch_shift
    return pitch_shift(torch.from_numpy(np.ascontiguousarray(x)).cuda(), shift, sr, **kw)


def _check(x, shift, sr=SR, name=""):
    want, cond = po.pitch_shift(x, shift, sr)
    assert cond > COND_MIN, f"{name}: conditioning {cond:.2e}"
    got = _shift(x, shift, sr).cpu().numpy().astype(np.float64)
    err = float(np.abs(got - want).max())
    _worst[name] = err
    assert err <= ATOL, f"{name}: max |device - oracle| = {err:.3e}"
    return err


@pytest.mark.parametrize("shift", range(-12, 13))
def test_every_semitone_2s(shift):
    _check(gg.signal(SR, 2.0, 100 + shift)[None, None], shift, name=f"2s {shift:+d}")


@pytest.mark.parametrize("shift", [-11, -1, 5, 12])
def test_ten_second_clips(shift):
    _check(gg.signal(SR, 10.0, 200 + shift)[None, None], shift, name=f"10s {shift:+d}")


def test_48k_and_fraction():
    _check(gg.signal(48000, 1.0, 300)[None, None], 5, 48000, name="48k +5")
    from vampnet_b200.pitch import get_fast_shifts
    frac = get_fast_shifts(SR)[7]
    assert isinstance(frac, Fraction)
    _check(gg.signal(SR, 1.0, 301)[None, None], frac, name=f"fraction {frac}")


@pytest.mark.parametrize("name", [n for n, *_ in gg.CASES])
def test_goldens(name):
    x, shift, sr, out, cond = gg.load(os.path.join(GOLDEN, f"pitch_{name}.npz"))
    assert cond > COND_MIN
    got = _shift(x, shift, sr).cpu().numpy().astype(np.float64)
    # the golden output is stored in float32: half an ulp below 1 on top of the float64 agreement
    err = float(np.abs(got - out).max())
    _worst[f"golden {name}"] = err
    assert err <= ATOL + 6e-8, f"{name}: {err:.3e}"


def test_time_steps_equal_cuda_arange():
    from vampnet_b200.pitch import shift_params, time_steps
    for shift in (-12, -11, -5, -1, 1, 7, 12, Fraction(4, 3)):
        _, _, _, rate = shift_params(shift, SR)
        for F in (2, 1051, 21001, 63001):
            want = torch.arange(0, F, rate, dtype=torch.float32, device="cuda")
            assert torch.equal(time_steps(F, rate), want), (shift, F)
            assert torch.equal(want.cpu(), torch.from_numpy(po.time_steps(F, rate))), (shift, F)


def test_batch_rows_equal_rows_alone_and_repeat():
    x = np.stack([gg.signal(SR, 1.0 + 0.25 * i, 400 + i)[:SR] for i in range(6)]).reshape(2, 3, SR)
    for shift in (-7, 3, Fraction(3, 2)):
        a = _shift(x, shift)
        b = _shift(x, shift)
        assert a.shape == (2, 3, SR)
        assert torch.equal(a, b), "two runs differ"
        for i in range(2):
            for c in range(3):
                alone = _shift(x[i:i + 1, c:c + 1], shift)
                assert torch.equal(a[i, c], alone[0, 0]), (shift, i, c)


def test_no_host_sync():
    from vampnet_b200.pitch import pitch_shift
    x = torch.from_numpy(gg.signal(SR, 1.0, 500)[None, None]).cuda()
    pitch_shift(x, 4, SR)  # first call for this n_fft uploads the bases
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for shift in (-3, 0, 4, Fraction(4, 3)):
            pitch_shift(x, shift, SR)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_cpu_input_returns_on_cpu():
    from vampnet_b200.pitch import pitch_shift
    x = torch.from_numpy(gg.signal(SR, 1.0, 600)[None, None])
    out = pitch_shift(x, -5, SR)
    assert out.device.type == "cpu" and out.shape == x.shape
    assert torch.equal(out, pitch_shift(x.cuda(), -5, SR).cpu())


def test_zero_shift_is_the_stft_round_trip():
    x = gg.signal(SR, 1.0, 700)[None, None]
    err = _check(x, 0, name="0 (identity vocoder and resampler)")
    assert err < ATOL


@pytest.fixture(scope="module")
def cache(tmp_path_factory):
    from tests.dropin_cache import write_cache
    root = tmp_path_factory.mktemp("cache") / "models" / "vampnet"
    write_cache(root)
    old = os.environ.get("VAMPNET_MODELS_DIR")
    os.environ["VAMPNET_MODELS_DIR"] = str(root)
    for k in [k for k in sys.modules if k == "vampnet" or k.startswith("vampnet.")]:
        del sys.modules[k]
    yield root
    if old is None:
        os.environ.pop("VAMPNET_MODELS_DIR", None)
    else:
        os.environ["VAMPNET_MODELS_DIR"] = old


def test_app_pitch_shift_sequence(cache):
    """app.py:180-190 with pitch_shift_amt = 3: _preprocess, shift_pitch (app.py:60-66) on the CPU signal, encode,
    build_mask, vamp, decode, through the vampnet and torch_pitch_shift import names."""
    ns = {}
    exec("from torch_pitch_shift import pitch_shift, get_fast_shifts", ns)
    import vampnet_b200.pitch
    assert ns["pitch_shift"] is vampnet_b200.pitch.pitch_shift
    from vampnet.interface import AudioSignal, Interface
    interface = Interface.default(device="cuda")
    y = gg.signal(SR, 229 * 768 / SR, 800)
    sig = interface._preprocess(AudioSignal(torch.from_numpy(y)[None, None], SR))
    before = sig.samples.clone()
    sig.samples = ns["pitch_shift"](sig.samples, shift=3, sample_rate=sig.sample_rate)
    assert sig.samples.device == before.device and sig.samples.shape == before.shape
    assert torch.equal(sig.samples.cpu(), vampnet_b200.pitch.pitch_shift(before.cuda(), 3, sig.sample_rate).cpu())
    codes = interface.encode(sig)
    mask = interface.build_mask(codes, sig=sig, periodic_prompt=7, upper_codebook_mask=3)
    z = interface.vamp(codes, mask, return_mask=False, _sampling_steps=3, seed=2, temperature=1.0)
    assert z.shape == codes.shape and not (z == 1024).any()
    out = interface.decode(z)
    assert torch.isfinite(out.samples).all()


def test_refusals():
    from vampnet_b200 import _lib
    from vampnet_b200.pitch import pitch_shift
    x = torch.zeros(1, 1, 4000, device="cuda")
    for bad in (lambda: pitch_shift(x.double(), 2, SR), lambda: pitch_shift(x[0], 2, SR),
                lambda: pitch_shift(x[:, :, :300], 2, SR),  # N <= n_fft // 2
                lambda: pitch_shift(x, 2, SR, n_fft=8), lambda: pitch_shift(x, 2, SR, n_fft=5000),
                lambda: pitch_shift(x, 2, SR, n_fft=512, hop_length=513),
                lambda: pitch_shift(torch.zeros(1, 65536, 400, device="cuda"), 2, SR),
                lambda: pitch_shift(x, Fraction(SR * 2, 1), SR)):  # new_freq = 0
        with pytest.raises(RuntimeError):
            bad()
    L = _lib.lib()
    need = ctypes.c_uint64(0)
    good = (1, 4000, SR, 39288, 689, 21, 0.9)
    assert L.vnb_pitch_workspace_bytes(*good, ctypes.byref(need)) == 0
    ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    out = torch.empty(1, 4000, device="cuda")
    call = lambda a=good, xp=_lib.ptr(x), w=_lib.ptr(ws), n=need.value, o=_lib.ptr(out): L.vnb_pitch_shift(  # noqa
        xp, *a, w, n, o, None)
    assert call(xp=None) != 0 and call(w=None) != 0 and call(o=None) != 0
    assert call(n=need.value - 1) != 0
    for bad in ((0, 4000, SR, 39288, 689, 21, 0.9), (65536, 4000, SR, 39288, 689, 21, 0.9),
                (1, 344, SR, 39288, 689, 21, 0.9), (1, 4000, SR, 39288, 689, 0, 0.9),
                (1, 4000, SR, 39288, 15, 1, 0.9), (1, 4000, SR, 39288, 4097, 21, 0.9),
                (1, 4000, SR, 0, 689, 21, 0.9), (1, 4000, SR, 39288, 689, 21, 0.0),
                (1, 4000, SR, 39288, 689, 21, -1.0)):
        assert L.vnb_pitch_workspace_bytes(*bad, ctypes.byref(need)) != 0, bad
        assert call(a=bad) != 0, bad
    assert L.vnb_pitch_workspace_bytes(*good, None) != 0
    assert call() == 0  # the same call with good arguments goes through
    torch.cuda.synchronize()


def test_report_worst_error():
    """Runs last in this file: prints the largest error measured against the oracle and the goldens."""
    if _worst:
        name = max(_worst, key=_worst.get)
        print(f"\npitch: largest max|device - reference| {_worst[name]:.3e} ({name}) over {len(_worst)} signals")
