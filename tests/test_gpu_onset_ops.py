"""GPU: the onset detector (csrc/onset.cu) across (sample rate, hop), against oracle/onset_oracle.py in float64.

onset_geometry derives peak_pick's pre_max, wait, pre_avg and the envelope's padding from (sr, hop), and onset_tables
builds the mel filterbank from sr; test_gpu_onset.py runs only 44100 / 768.  The pairs here reach the corners of that
geometry: pre_max = wait = 0 (hop > 0.03 sr), pad = 1 (hop > 1024), wait longer than the greedy walk's 32-frame ballot
step (44100 / 32 gives 41), and frames that skip samples (hop > 2048).  The envelope is held to test_gpu_onset.py's
ENV_TOL; onset frames are compared exactly, with and without backtracking, on signals whose oracle decision margin
exceeds twice ENV_TOL (a thinner one fails rather than skips)."""
import numpy as np
import pytest

from oracle import onset_oracle as oo
from tools import audio_bits as AB

pytestmark = pytest.mark.gpu

ENV_TOL = 5e-6

# (sr, hop, signal)
CASES = [
    (8000, 64, "bursts_132300"), (8000, 256, "bursts"),
    (16000, 32, "clicks"), (16000, 512, "bursts"),        # 16000 / 512: pre_max = wait = 0
    (22050, 1024, "bursts"), (22050, 1025, "bursts"),     # 1025: pad = 1
    (44100, 32, "bursts"),                                # wait = 41 > 32
    (44100, 1323, "bursts"), (44100, 1324, "bursts"),     # wait = 1, then 0
    (48000, 768, "clicks"), (48000, 2048, "bursts"),
    (96000, 64, "clicks"), (96000, 4096, "bursts"),       # 4096 > 2048: frames skip samples
]
IDS = [f"{sr}_{hop}_{sig}" for sr, hop, sig in CASES]


def oracle(sr, hop, name, backtrack):
    """The oracle's envelope, onsets and decision margin, with or without backtracking."""
    r = oo.onset_detect(oo.test_signal(name, sr), sr, hop, backtrack=backtrack)
    return r["envelope"], r["onsets"], r["margin"]


@pytest.mark.parametrize("backtrack", [True, False], ids=["backtrack", "peaks"])
@pytest.mark.parametrize("sr,hop,name", CASES, ids=IDS)
def test_onsets_match_oracle(sr, hop, name, backtrack):
    env_want, onsets_want, margin = oracle(sr, hop, name, backtrack)
    assert margin > 2 * ENV_TOL, f"oracle decision margin {margin:.3e} is too thin to test"
    env, onsets = AB.onset_detect(oo.test_signal(name, sr)[None], sr, hop, backtrack=backtrack)
    assert env.shape == (1, oo.n_frames(oo.test_signal(name, sr).shape[0], hop))
    err = float(np.abs(env[0].double().numpy() - env_want).max())
    assert err <= ENV_TOL, f"envelope error {err:.3e}"
    assert onsets[0].numpy().tolist() == onsets_want.tolist()


def test_geometry_corners_are_covered():
    p = [oo.peak_params(sr, hop) for sr, hop, _ in CASES]
    pads = [1 + oo.N_FFT // (2 * hop) for _, hop, _ in CASES]
    assert any(q["pre_max"] == q["wait"] == 0 for q in p)
    assert any(q["wait"] > 32 for q in p)
    assert 1 in pads and any(hop > 2048 for _, hop, _ in CASES)
