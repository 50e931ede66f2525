"""GPU: the fused attention kernel reproduces, bit for bit, the outputs recorded in tests/golden/attention_bits.npz by
tools/attention_bits.py.  Schedule, register allocation and address arithmetic of the kernel may change; the float
operations on every score and their order may not, so every output hash must match."""
import os

import numpy as np
import pytest

from tools import attention_bits as AB

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "attention_bits.npz"))


@pytest.mark.parametrize("B,T,H,sat", AB.CASES, ids=[AB.case_name(*c) for c in AB.CASES])
def test_attention_output_bits_match_record(golden, B, T, H, sat):
    name = AB.case_name(B, T, H, sat)
    out = AB.run_case(B, T, H, sat)
    got = AB.digest(out)
    want = str(golden["sha256_" + name])
    if got != want:
        flat = out.float().reshape(-1).numpy()
        idx = AB.sample_index(flat.size, name)
        ref = golden["sample_" + name]
        diff = np.abs(flat[idx] - ref)
        pytest.fail(f"{name}: sha256 {got} != recorded {want}; sampled values: {int((flat[idx] != ref).sum())} of "
                    f"{idx.size} differ, max |diff| {np.nanmax(diff):.3e}, NaN {int(np.isnan(flat).sum())}")
