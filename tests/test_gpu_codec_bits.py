"""GPU: the codec kernels reproduce, bit for bit, the outputs recorded in tests/golden/codec_bits.npz by
tools/codec_bits.py: each epilogue variant x MMA width of conv_wgmma_kernel, the transposed convolutions' store, the
two edge layers, the RVQ in its three modes, the fp32 convolution and a short full-size encode + decode.  Schedule,
tiling and the order of stores may change; the float operations on every output and their order may not."""
import os

import numpy as np
import pytest

from tools import codec_bits as CB

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "codec_bits.npz"))


@pytest.mark.parametrize("name", CB.CASES)
def test_codec_output_bits_match_record(golden, name):
    outs = CB.run_named(name)
    got = CB.digest(outs)
    want = str(golden["sha256_" + name])
    if got != want:
        vals = CB.sample_values(outs, name)
        ref = golden["sample_" + name]
        same = (vals == ref) | (np.isnan(vals) & np.isnan(ref))
        pytest.fail(f"{name}: sha256 {got} != recorded {want}; sampled values of the first output: "
                    f"{int((~same).sum())} of {vals.size} differ, max |diff| {np.nanmax(np.abs(vals - ref)):.3e}")
