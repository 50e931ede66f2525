"""GPU: the beat tracker's decisions (csrc/beat.cu, through vnb_dbg_beat_from_envelope) across the whole tempo-window
range the ABI accepts, W = int(8 sr) // hop from 2 to 4096, against oracle/beat_oracle.py in float64.

The kernels are built around that range: LAGS_PER_THREAD lag accumulators per thread, a shared window of
BEAT_MAX_LAGS doubles, Gaussian and transition tables of 2 BEAT_MAX_LAGS, frames chunked by fpc = ceil(W / 256) with a
256 F + W workspace bound, max_idx (the first lag below 320 BPM), and period-1 tempi, where the dynamic programme
reads librosa's zero at q == i.  Everything after the envelope is float64, so fed the same envelope the kernels take
the oracle's decisions exactly: tempo and beat frames are compared with ==, on envelopes whose smallest relative
decision margin is asserted above 1e-9 (a thinner one fails rather than skips).  End to end, beat_track is compared at
two more (sr, hop) pairs within test_gpu_beats.py's ENV_RTOL."""
import numpy as np
import pytest
import torch

from oracle import beat_oracle as bo
from tools import audio_bits as AB

pytestmark = pytest.mark.gpu

MARGIN_MIN = 1e-9
ENV_RTOL = 1e-5

# W: (sr, hop) with int(8 sr) // hop == W
WINDOWS = {2: (1000, 4000), 3: (1500, 4000), 31: (1000, 258), 255: (16000, 501), 256: (8000, 250),
           257: (8000, 249), 459: (44100, 768), 689: (44100, 512), 1024: (16000, 125), 4095: (4095, 8),
           4096: (2048, 4)}


def frame_counts(W):
    """1, 2, W - 1, W, W + 1 and, where the float64 oracle's (F, 2 W) FFT stays small, multiples of W."""
    fs = [1, 2, W] if W == 4095 else [1, 2, W - 1, W, W + 1] + ([2 * W, 3 * W + 7] if W <= 1024 else [])
    return sorted({f for f in fs if f >= 1})


def envelope(W, F, seed):
    """A random onset envelope (F,) float32 with pulses every W / 25 .. W / 8 frames (0.3 to 1 s at any W)."""
    rng = np.random.default_rng(seed)
    env = rng.exponential(0.3, F) * (rng.random(F) < 0.7)
    period = max(1, int(round(W * rng.uniform(1 / 25, 1 / 8))))
    phase = int(rng.integers(0, period))
    env[phase::period] += rng.uniform(1.0, 4.0, len(env[phase::period]))
    return env.astype(np.float32)


def pulses(F, period, seed, noise=0.05):
    """Unit pulses every `period` frames over a weak random floor, (F,) float32: a tempo chosen by its lag."""
    rng = np.random.default_rng(seed)
    env = noise * rng.random(F)
    env[3::period] += 1.0
    return env.astype(np.float32)


RANGE_CASES = [(W, F, 100 * W + F) for W in WINDOWS for F in frame_counts(W)]
# (name, envelope builder, sr, hop, keyword arguments)
BOUNDARY_CASES = [
    # sr 16000, hop 100: exactly 320 BPM at lag 30, which the prior excludes, and lag 31 = max_idx, the first it
    # allows; the prior is centred on the pulses' own tempo
    ("pulse_at_320bpm_lag30", lambda: pulses(900, 30, 1), 16000, 100, dict(start_bpm=320.0)),
    ("pulse_at_max_idx_lag31", lambda: pulses(900, 31, 2), 16000, 100, dict(start_bpm=9600 / 31)),
    # sr 1000, hop 250: 4 frames per second, so 240 BPM (lag 1, max_idx) is a period of one frame
    ("period_one_frame", lambda: pulses(120, 1, 3, noise=0.5), 1000, 250, dict(start_bpm=240.0)),
    # the other arguments at W = 4096
    ("w4096_no_trim", lambda: envelope(4096, 4200, 5), 2048, 4, dict(trim=False)),
    ("w4096_start_bpm_30_tight_1", lambda: envelope(4096, 4200, 6), 2048, 4, dict(start_bpm=30.0, tightness=1.0)),
    ("w4096_start_bpm_300_tight_5000", lambda: envelope(4096, 4200, 7), 2048, 4,
     dict(start_bpm=300.0, tightness=5000.0)),
]
# end to end: (sr, hop, signal)
END_TO_END = [(44100, 768, "bursts_4"), (22050, 256, "clicks120")]


def _compare(env, sr, hop, **kw):
    want = bo.beat_track_envelope(env, sr, hop, **kw)
    assert want["margin"] > MARGIN_MIN, f"oracle decision margin {want['margin']:.3e}"
    tempo, beats = AB.beat_from_envelope(env[None], sr, hop, **kw)
    assert tempo[0] == want["tempo"], (tempo[0], want["tempo"])
    assert beats[0].tolist() == want["beats"].tolist()
    return want


@pytest.mark.parametrize("W,F,seed", RANGE_CASES, ids=[f"W{W}_F{F}" for W, F, _ in RANGE_CASES])
def test_tempo_window_range(W, F, seed):
    sr, hop = WINDOWS[W]
    assert bo.tempo_lags(sr, hop) == W
    _compare(envelope(W, F, seed), sr, hop)


@pytest.mark.parametrize("name,build,sr,hop,kw", BOUNDARY_CASES, ids=[c[0] for c in BOUNDARY_CASES])
def test_tempo_boundaries_and_arguments(name, build, sr, hop, kw):
    want = _compare(build(), sr, hop, **kw)
    if name == "pulse_at_320bpm_lag30":
        assert bo.bpm_grid(sr, hop)[30] == 320.0 and want["lag"] != 30
    if name == "pulse_at_max_idx_lag31":
        assert want["lag"] == int(np.argmax(bo.bpm_grid(sr, hop) < 320.0)) == 31
    if name == "period_one_frame":
        assert round(60.0 * sr / hop / want["tempo"]) == 1 and len(want["beats"]) > 2


def test_batched_rows_at_w4096_equal_rows_alone():
    envs = np.stack([envelope(4096, 4500, s) for s in (11, 12, 13)])
    tempo, beats = AB.beat_from_envelope(envs, 2048, 4)
    for b in range(3):
        t1, b1 = AB.beat_from_envelope(envs[b:b + 1], 2048, 4)
        assert tempo[b] == t1[0] and beats[b].tolist() == b1[0].tolist()


def test_window_outside_2_to_4096_is_refused():
    from vampnet_b200 import _lib
    L = _lib.lib()
    env = torch.ones(64, device="cuda")
    ws = torch.empty(1 << 22, dtype=torch.uint8, device="cuda")
    outs = [torch.empty(64, dtype=t, device="cuda") for t in (torch.float64, torch.int32, torch.int32)]
    for sr, hop, ok in ((1000, 8000, False), (4097, 8, False), (1000, 4000, True), (2048, 4, True)):
        W = bo.tempo_lags(sr, hop)
        assert (2 <= W <= 4096) == ok, W
        rc = L.vnb_dbg_beat_from_envelope(_lib.ptr(env), 1, 64, sr, hop, 120.0, 100.0, 1, _lib.ptr(ws), ws.numel(),
                                          *map(_lib.ptr, outs), _lib.stream_ptr())
        assert (rc == 0) == ok, (sr, hop, W)
    torch.cuda.synchronize()


@pytest.mark.parametrize("sr,hop,name", END_TO_END, ids=[f"{sr}_{hop}" for sr, hop, _ in END_TO_END])
def test_end_to_end(sr, hop, name):
    y = bo.test_signal(name, sr)
    want = bo.beat_track(y, sr, hop)
    assert want["margin"] > 2 * ENV_RTOL, f"oracle decision margin {want['margin']:.3e} is too thin"
    env, tempo, beats = AB.beat_track(y[None], sr, hop)
    err = float(np.abs(env[0].double().numpy() - want["envelope"]).max() / want["envelope"].max())
    assert err <= ENV_RTOL, f"relative envelope error {err:.3e}"
    assert float(tempo[0]) == want["tempo"]
    assert beats[0].numpy().tolist() == want["beats"].tolist()
