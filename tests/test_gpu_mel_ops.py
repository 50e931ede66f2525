"""GPU: the mel spectrogram kernel (csrc/mel.cu) through the C ABI, against oracle/mel_oracle.py in float64, across
every supported window (32 to 4096 samples), sample rates of 16 to 48 kHz, non-default fmin / fmax, empty Slaney
bands, hops of 1 and of non-divisors, and the smallest accepted N = n_fft / 2 + 1, where the reflect padding reaches
the signal's far end.  Also: a batched row equals the row alone, bit for bit, and every refusal returns an error
without a launch and without touching the output."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import mel_oracle as mo
from vampnet_b200 import _lib

pytestmark = pytest.mark.gpu

# error bound relative to the largest oracle value of the same frame (row, f): the device's fp32 FFT and band sums
# reached 2.2e-7 of it at most on these cases (H100 80GB HBM3, DESIGN.md §13)
SPEC_TOL = 1e-6

# (n_fft, hop, n_mels, sr, fmin, fmax, N)
CASES = [
    (32, 8, 5, 48000, 0.0, None, 17),           # N = n_fft / 2 + 1; band 0 is empty at 48 kHz
    (64, 16, 10, 48000, 0.0, None, 2000),        # an empty band
    (128, 32, 20, 16000, 0.0, None, 3000),
    (256, 64, 40, 22050, 50.0, 8000.0, 5000),    # fmin and fmax
    (512, 128, 80, 44100, 0.0, None, 257),       # N = n_fft / 2 + 1
    (512, 1, 64, 16000, 0.0, None, 700),         # hop 1
    (1024, 256, 160, 48000, 0.0, None, 9000),
    (2048, 512, 150, 44100, 0.0, None, 1025),    # the default loss's first scale at N = n_fft / 2 + 1
    (2048, 512, 320, 44100, 20.0, 16000.0, 20000),
    (4096, 1024, 128, 48000, 0.0, None, 2049),   # N = n_fft / 2 + 1
    (4096, 1000, 256, 16000, 0.0, 7000.0, 30000),  # a hop that does not divide N
]
IDS = [f"w{c[0]}_h{c[1]}_m{c[2]}_sr{c[3]}_N{c[6]}" for c in CASES]


def signal(rows, N, sr, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(N) / sr
    x = 0.3 * np.sin(2 * np.pi * 440.0 * (1 + np.arange(rows))[:, None] * t) + 0.05 * rng.standard_normal((rows, N))
    return x.astype(np.float32)


def scale(n_fft, hop, n_mels, sr, fmin, fmax):
    return _lib.MelScale(n_fft, hop, n_mels, fmin, sr / 2 if fmax is None else fmax)


def spec(x, sr, sc):
    L = _lib.lib()
    xd = torch.from_numpy(x).cuda()
    rows, N = x.shape
    out = torch.full((rows, sc.n_mels, 1 + N // sc.hop), float("nan"), device="cuda")
    _lib.check(L.vnb_mel_spectrogram(_lib.ptr(xd), rows, N, sr, C.byref(sc), _lib.ptr(out), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("n_fft,hop,n_mels,sr,fmin,fmax,N", CASES, ids=IDS)
def test_spectrogram_matches_oracle(n_fft, hop, n_mels, sr, fmin, fmax, N):
    x = signal(2, N, sr)
    got = spec(x, sr, scale(n_fft, hop, n_mels, sr, fmin, fmax))
    want = mo.mel_spectrogram(x.astype(np.float64), sr, n_mels, fmin, fmax, n_fft, hop)
    assert got.shape == want.shape == (2, n_mels, 1 + N // hop)
    frame_max = want.max(axis=1, keepdims=True)
    assert (frame_max > 0).all()
    ratio = float((np.abs(got - want) / frame_max).max())
    assert ratio <= SPEC_TOL, f"error {ratio:.3e} of the frame's largest value"
    empty = (mo.mel_filterbank(sr, n_mels, n_fft, fmin, fmax) == 0).all(1)
    assert (got[:, empty] == 0).all()


def test_cases_cover_empty_bands_and_reflect_edges():
    assert any((mo.mel_filterbank(sr, m, w, lo, hi) == 0).all(1).any() for w, _, m, sr, lo, hi, _ in CASES)
    assert {w for w, *_ in CASES} == {32, 64, 128, 256, 512, 1024, 2048, 4096}
    assert sum(N == w // 2 + 1 for w, *_, N in CASES) >= 3


@pytest.mark.parametrize("n_fft,hop,n_mels", [(32, 8, 5), (512, 128, 80), (2048, 512, 150), (4096, 1024, 64)])
def test_batched_row_equals_row_alone(n_fft, hop, n_mels):
    sr, N = 44100, 12345
    x = signal(5, N, sr, seed=3)
    sc = scale(n_fft, hop, n_mels, sr, 0.0, None)
    batch = spec(x, sr, sc)
    for r in (0, 2, 4):
        assert np.array_equal(spec(x[r:r + 1], sr, sc)[0], batch[r])
    assert np.array_equal(spec(x, sr, sc), batch)


def test_refusals_do_not_launch():
    L = _lib.lib()
    x = torch.zeros(2, 4096, device="cuda")
    out = torch.full((2, 8, 64), 7.0, device="cuda")
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    loss = torch.full((1,), 7.0, device="cuda")
    good = dict(n_fft=512, hop=128, n_mels=8, fmin=0.0, fmax=8000.0)

    def sp(samples=x, rows=2, N=4096, sr=16000, o=out, **kw):
        sc = _lib.MelScale(**{**good, **kw})
        return L.vnb_mel_spectrogram(_lib.ptr(samples), rows, N, sr, C.byref(sc), _lib.ptr(o), _lib.stream_ptr())

    def ml(xp=x, yp=x, B=1, Ch=2, N=4096, sr=16000, n_scales=1, eps=1e-5, pw=2.0, lw=1.0, mw=1.0, w=ws,
           wbytes=1 << 20, lo=loss, scales=True, **kw):
        sc = (_lib.MelScale * 17)(*[_lib.MelScale(**{**good, **kw})] * 17)
        return L.vnb_mel_loss(_lib.ptr(xp), _lib.ptr(yp), B, Ch, N, sr, sc if scales else None, n_scales, eps, pw, lw,
                              mw, _lib.ptr(w), wbytes, _lib.ptr(lo), None, _lib.stream_ptr())

    def nbytes(B=1, Ch=2, N=4096, sr=16000, n_scales=1, **kw):
        sc = (_lib.MelScale * 17)(*[_lib.MelScale(**{**good, **kw})] * 17)
        v = C.c_uint64()
        return L.vnb_mel_workspace_bytes(B, Ch, N, sr, sc, n_scales, C.byref(v))

    assert sp() == 0 and ml() == 0 and nbytes() == 0
    torch.cuda.synchronize()
    out.fill_(7.0)
    loss.fill_(7.0)
    refused_spec = [dict(samples=None), dict(o=None), dict(rows=0), dict(rows=65536), dict(sr=0), dict(n_fft=16),
                    dict(n_fft=8192), dict(n_fft=500), dict(N=256), dict(hop=0), dict(n_mels=0), dict(n_mels=4097),
                    dict(fmin=-1.0), dict(fmax=0.0), dict(fmin=100.0, fmax=100.0), dict(fmax=float("nan")),
                    dict(fmax=float("inf"))]
    refused_loss = [dict(xp=None), dict(yp=None), dict(w=None), dict(lo=None), dict(scales=False), dict(B=0),
                    dict(Ch=0), dict(B=2, Ch=40000), dict(n_scales=0), dict(n_scales=17), dict(N=256),
                    dict(n_fft=100), dict(hop=0), dict(n_mels=0), dict(fmin=-1.0), dict(fmax=0.0), dict(sr=0),
                    dict(eps=0.0), dict(eps=float("nan")), dict(pw=float("inf")), dict(lw=float("nan")),
                    dict(mw=float("inf")), dict(wbytes=16)]
    refused_bytes = [dict(B=0), dict(B=2, Ch=40000), dict(n_scales=17), dict(n_fft=64, N=32), dict(n_mels=0)]
    before = L.vnb_launch_count()
    for kw in refused_spec:
        assert sp(**kw) != 0, kw
        assert L.vnb_last_error()
    for kw in refused_loss:
        assert ml(**kw) != 0, kw
    for kw in refused_bytes:
        assert nbytes(**kw) != 0, kw
    v = C.c_uint64()
    assert L.vnb_mel_workspace_bytes(1, 1, 4096, 16000, None, 1, C.byref(v)) != 0
    assert L.vnb_mel_workspace_bytes(1, 1, 4096, 16000, C.byref(_lib.MelScale(**good)), 1, None) != 0
    assert L.vnb_launch_count() == before
    torch.cuda.synchronize()
    assert (out == 7.0).all() and (loss == 7.0).all()
    assert sp() == 0 and ml() == 0  # the library still works
