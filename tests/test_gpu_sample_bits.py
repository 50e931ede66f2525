"""GPU: the sampling step (vnb_dbg_sample, every path) reproduces, bit for bit, the tokens, confidences and re-masked
zcur recorded in tests/golden/sample_bits.npz by tools/sample_bits.py.  Schedule and register allocation may change;
the float operations, their order and every decision may not, so every hash must match."""
import os

import numpy as np
import pytest

from tools import sample_bits as SB

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "sample_bits.npz"))


@pytest.mark.parametrize("case", SB.CASES, ids=[c[0] for c in SB.CASES])
def test_sample_output_bits_match_record(golden, case):
    name = case[0]
    outs = SB.run_case(*case)
    got = SB.digest(outs)
    want = str(golden["sha256_" + name])
    if got != want:
        vals = SB.sample_values(outs, name)
        ref = golden["sample_" + name]
        same = (vals == ref) | (np.isnan(vals) & np.isnan(ref))
        pytest.fail(f"{name}: sha256 {got} != recorded {want}; sampled confidences: {int((~same).sum())} of "
                    f"{vals.size} differ")
