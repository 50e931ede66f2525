"""CPU: the beat-synced mask built from beat times (vampnet_b200.beats.beat_mask) against the reference's own
Interface.make_beat_mask, run with a tracker returning fixed times (tests/golden/reference_beat_mask.npz, written by
oracle/gen_reference_beat_mask.py): the masks and the torch draws that follow each call."""
import os
import types

import numpy as np
import pytest
import torch

from oracle.gen_reference_beat_mask import CASES, DURATION, HOP, N_CODEBOOKS, SR
from vampnet_b200.audio import AudioSignal
from vampnet_b200.beats import beat_mask
from vampnet_b200.interface import Interface

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_beat_mask.npz"))


def _s2t():
    stub = types.SimpleNamespace(codec=types.SimpleNamespace(sample_rate=SR, hop_length=HOP))
    return lambda s: Interface.s2t(stub, s)


@pytest.mark.parametrize("k", range(len(CASES)), ids=[c[0] for c in CASES])
def test_beat_mask_equals_reference(k):
    name, beats, downbeats, kw = CASES[k]
    torch.manual_seed(100 + k)
    mask = beat_mask(beats, downbeats, DURATION, _s2t(), N_CODEBOOKS, "cpu", **kw)
    nxt = torch.rand(8)
    assert mask.dtype == torch.int64
    assert np.array_equal(mask.numpy(), GOLDEN[f"{name}_mask"].astype(np.int64)), name
    assert np.array_equal(nxt.numpy(), GOLDEN[f"{name}_next"]), name


def test_downsample_factor_below_one_is_refused():
    for kw in (dict(beat_downsample_factor=0), dict(downbeat_downsample_factor=0)):
        with pytest.raises(ValueError):
            beat_mask(np.array([0.5]), np.zeros(0), 2.0, _s2t(), 4, "cpu", **kw)


def test_trim_has_audiotools_meaning():
    sig = AudioSignal(torch.arange(10.0)[None, None], 10)
    assert sig.clone().trim(2, 3).audio_data[0, 0].tolist() == [2.0, 3.0, 4.0, 5.0, 6.0]
    assert sig.clone().trim(4, 0).audio_data[0, 0].tolist() == [4.0, 5.0, 6.0, 7.0, 8.0, 9.0]
