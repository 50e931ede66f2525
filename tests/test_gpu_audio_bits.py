"""GPU: the audio kernels reproduce, bit for bit, the outputs recorded in tests/golden/audio_bits.npz by
tools/audio_bits.py: the pitch shift's fp32 output and its four float64 intermediates (spectrum, stretched spectrum,
inverse-DFT frames, overlap-added signal) at eight parameter points, the beat tracker's envelope, tempo and beats at
three tempo windows, the onset detector's envelope and onsets at three (sr, hop), the mel spectrogram at every window
length, and the mel loss and per-item losses at two scale sets.  Schedule, tiling and the order
of stores may change; the float operations on every output and their order may not."""
import os

import numpy as np
import pytest

from tools import audio_bits as AB

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "audio_bits.npz"))


@pytest.mark.parametrize("name", AB.CASES)
def test_audio_output_bits_match_record(golden, name):
    outs = AB.run_named(name)
    got = AB.digest(outs)
    want = str(golden["sha256_" + name])
    if got != want:
        vals = AB.sample_values(outs, name)
        ref = golden["sample_" + name]
        same = (vals == ref) | (np.isnan(vals) & np.isnan(ref))
        pytest.fail(f"{name}: sha256 {got} != recorded {want}; sampled values of the first output: "
                    f"{int((~same).sum())} of {vals.size} differ, max |diff| {np.nanmax(np.abs(vals - ref)):.3e}")
