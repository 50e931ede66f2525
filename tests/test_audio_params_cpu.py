"""CPU: the parameter cases of the audio op tests (tests/test_gpu_pitch_ops.py, tests/test_gpu_beat_ops.py,
tests/test_gpu_onset_ops.py) and of the bits record (tools/audio_bits.py) are what they claim to be, checked without a
GPU: each pitch plan is accepted or refused by vnb_pitch_workspace_bytes and vnb_dbg_pitch_layout as documented and its
shapes are the oracle's; the cases together cover the n_fft, hop, N, frame-count residues, rates and rate pairs they
are meant to; every beat (sr, hop) gives its tempo window W; and every chosen signal and envelope clears its margin or
conditioning guard on the float64 oracles, so a badly chosen case fails here rather than on an H100."""
import math

import numpy as np
import pytest

from oracle import beat_oracle as bo
from oracle import mel_oracle as mo
from oracle import onset_oracle as oo
from oracle import pitch_oracle as po
from tests import test_gpu_beat_ops as B
from tests import test_gpu_onset_ops as O
from tests import test_gpu_pitch_ops as P
from tools import audio_bits as AB


@pytest.fixture(scope="module")
def built():
    from vampnet_b200 import build
    return build.build()


def documented_refusal(rows, N, sr, new_freq, rate, n_fft, hop):
    """vnb_pitch_workspace_bytes' refusals as include/vampnet_b200.h lists them."""
    if not (1 <= rows <= 65535 and 16 <= n_fft <= 4096 and 1 <= hop <= n_fft and N > n_fft // 2):
        return True
    if sr < 1 or new_freq < 1 or not (rate > 0 and math.isfinite(rate)):
        return True
    F = 1 + (N + 2 * (n_fft // 2) - n_fft) // hop
    F2 = math.ceil(F / rate) if rate != 1.0 else F
    return not 1 <= F2 <= 1 << 30 or n_fft - 2 * (n_fft // 2) + hop * (F2 - 1) < 1


ALL_PITCH = [c[1:] for c in P.CASES] + list(AB.PITCH_CASES.values())
REFUSED = [  # rows, N, sr, new_freq, rate, n_fft, hop
    (1, 1025, 44100, 44100, 1.0, 2048, 2048),   # one frame of even n_fft: an empty istft signal
    (1, 1025, 44100, 44100, 2.0, 2048, 2048),   # the same after the vocoder: ceil(1 / 2) = 1 frame
    (1, 8, 44100, 44100, 1.0, 16, 1),           # N = n_fft // 2
    (1, 4000, 44100, 44100, 1.0, 15, 1), (1, 4000, 44100, 44100, 1.0, 4097, 21),
    (1, 4000, 44100, 44100, 1.0, 64, 65), (1, 4000, 44100, 44100, 1.0, 64, 0),
    (0, 4000, 44100, 44100, 1.0, 64, 16), (65536, 4000, 44100, 44100, 1.0, 64, 16),
    (1, 4000, 44100, 0, 1.0, 64, 16), (1, 4000, 44100, 44100, 0.0, 64, 16),
    (1, 4000, 44100, 44100, math.inf, 64, 16),
]


@pytest.mark.parametrize("case", ALL_PITCH + REFUSED)
def test_pitch_plan_accepted_or_refused_as_documented(built, case):
    rows, N, sr, new_freq, rate, n_fft, hop = case
    plan = AB.pitch_plan(rows, N, sr, new_freq, n_fft, hop, rate)
    assert (plan is None) == documented_refusal(*case)
    if plan is None:
        return
    need, offs, dims = plan
    assert tuple(dims) == P.plan_dims(N, sr, new_freq, rate, n_fft, hop)
    F, F2, L, _ = dims
    nb = n_fft // 2 + 1
    assert (offs[1] < 0) == (rate == 1.0)
    sizes = [rows * F * nb * 16, rows * F2 * nb * 16, rows * F2 * n_fft * 8, rows * L * 8]
    regions = sorted((o, o + s) for o, s in zip(offs, sizes) if o >= 0)
    assert all(o % 256 == 0 for o, _ in regions) and regions[0][0] == 0
    assert all(a[1] <= b[0] for a, b in zip(regions, regions[1:])), "overlapping intermediates"
    assert regions[-1][1] <= need


def test_pitch_cases_cover_the_edges():
    cases = [dict(zip(("rows", "N", "sr", "new_freq", "rate", "n_fft", "hop"), c[1:])) for c in P.CASES]
    dims = [P.plan_dims(c["N"], c["sr"], c["new_freq"], c["rate"], c["n_fft"], c["hop"]) for c in cases]
    assert {c["n_fft"] for c in cases} >= {16, 17, 63, 64, 65, 127, 128, 129, 689, 750, 1024, 2047, 2048, 4095, 4096}
    hops = {(c["n_fft"], c["hop"]) for c in cases}
    for rule in (lambda n: n // 4, lambda n: n // 2, lambda n: n - 1, lambda n: n):
        assert any(h == rule(n) for n, h in hops)
    small = [c for c in cases if c["hop"] <= 2]
    assert {1, 2} <= {c["hop"] for c in small} and all(c["n_fft"] <= 256 and c["N"] <= 300 for c in small)
    assert any(c["N"] == c["n_fft"] // 2 + 1 for c in cases)
    assert {0, 1, 63} <= {F % 64 for F, *_ in dims}
    assert {0, 1, 31} <= {F2 % 32 for _, F2, *_ in dims}
    r12 = 2.0 ** (1 / 12)
    rates = {c["rate"] for c in cases}
    assert {0.5, 2.0, r12, 1 / r12} <= rates
    assert any(F2 == 2 * F for (F, F2, *_), c in zip(dims, cases) if c["rate"] == 0.5)
    near = [c for c in cases if c["rate"] not in (1.0, 0.5, 2.0, r12, 1 / r12)]
    assert near, "a rate whose time steps land close to whole frames"
    for c in near:
        ts = po.time_steps(P.plan_dims(c["N"], c["sr"], c["new_freq"], c["rate"], c["n_fft"], c["hop"])[0], c["rate"])
        frac = ts % np.float32(1.0)
        assert ((frac > 0) & (np.minimum(frac, 1 - frac) < 1e-5)).any()
    pairs = {(c["sr"], c["new_freq"]) for c in cases if c["rate"] == 1.0 and c["sr"] != c["new_freq"]}
    assert pairs >= {(44100, 41625), (44100, 44101), (48000, 96000), (16000, 15999), (8000, 16001)}
    rs = [(c["N"], d[3]) for c, d in zip(cases, dims) if c["sr"] != c["new_freq"]]
    assert any(t > N for N, t in rs) and any(t < N for N, t in rs)
    assert {1, 3} <= {c["rows"] for c in cases} and P.BATCHED


@pytest.mark.parametrize("i", range(len(P.END_TO_END)))
def test_pitch_end_to_end_signals_are_well_conditioned(i):
    x, shift, sr, n_fft, hop = P.e2e_case(i)
    _, cond = po.pitch_shift(x, shift, sr, n_fft=n_fft, hop_length=hop)
    assert cond > P.COND_MIN, f"conditioning {cond:.2e}"


def test_beat_windows():
    for W, (sr, hop) in B.WINDOWS.items():
        assert bo.tempo_lags(sr, hop) == W
    assert set(B.WINDOWS) >= {2, 3, 31, 255, 256, 257, 459, 689, 1024, 4095, 4096}
    assert B.WINDOWS[459] == (44100, 768)
    assert bo.tempo_lags(1000, 8000) == 1 and bo.tempo_lags(4097, 8) == 4097


@pytest.mark.parametrize("W,F,seed", B.RANGE_CASES, ids=[f"W{W}_F{F}" for W, F, _ in B.RANGE_CASES])
def test_beat_envelopes_clear_the_margin(W, F, seed):
    sr, hop = B.WINDOWS[W]
    r = bo.beat_track_envelope(B.envelope(W, F, seed), sr, hop)
    assert r["margin"] > B.MARGIN_MIN, r["margin"]


@pytest.mark.parametrize("name,build,sr,hop,kw", B.BOUNDARY_CASES, ids=[c[0] for c in B.BOUNDARY_CASES])
def test_beat_boundary_cases_decide_what_they_test(name, build, sr, hop, kw):
    r = bo.beat_track_envelope(build(), sr, hop, **kw)
    assert r["margin"] > B.MARGIN_MIN, r["margin"]
    grid = bo.bpm_grid(sr, hop)
    max_idx = int(np.argmax(grid < 320.0))
    if name == "pulse_at_320bpm_lag30":
        assert grid[30] == 320.0 and max_idx == 31 and r["lag"] != 30
    if name == "pulse_at_max_idx_lag31":
        assert r["lag"] == max_idx == 31
    if name == "period_one_frame":
        assert sr / hop < 320.0 / 60.0 and r["lag"] == max_idx == 1
        assert round(60.0 * sr / hop / r["tempo"]) == 1 and len(r["beats"]) > 2


@pytest.mark.parametrize("sr,hop,name", B.END_TO_END)
def test_beat_end_to_end_signals_clear_the_margin(sr, hop, name):
    assert bo.beat_track(bo.test_signal(name, sr), sr, hop)["margin"] > 2 * B.ENV_RTOL


@pytest.mark.parametrize("backtrack", [True, False])
@pytest.mark.parametrize("sr,hop,name", O.CASES, ids=O.IDS)
def test_onset_signals_clear_the_margin(sr, hop, name, backtrack):
    _, _, margin = O.oracle(sr, hop, name, backtrack)
    assert margin > 2 * O.ENV_TOL, margin


def test_onset_geometry_corners():
    O.test_geometry_corners_are_covered()
    assert {sr for sr, _, _ in O.CASES} >= {8000, 16000, 22050, 44100, 48000, 96000}
    assert {h for _, h, _ in O.CASES} >= {32, 64, 256, 512, 768, 1024, 1025, 1323, 1324, 2048, 4096}
    assert oo.peak_params(44100, 32)["wait"] == 41


def test_mel_bits_cases_cover_every_window_and_empty_bands():
    spec = list(AB.MEL_SPEC_CASES.values())
    assert {w for w, *_ in spec} == {32, 64, 128, 256, 512, 1024, 2048, 4096}
    assert any((mo.mel_filterbank(sr, m, w) == 0).all(1).any() for w, _, m, sr, _ in spec)
    assert any(N == w // 2 + 1 for w, *_, N in spec)
    for sr, _, _, _, scales in AB.MEL_LOSS_CASES.values():
        if scales == mo.SEVEN_SCALES:
            assert sr == 48000 and any((mo.mel_filterbank(sr, m, w) == 0).all(1).any() for m, _, _, w in scales)
    assert any(scales == mo.DEFAULT_SCALES for *_, scales in AB.MEL_LOSS_CASES.values())
