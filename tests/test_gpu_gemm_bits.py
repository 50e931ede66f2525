"""GPU: the GEMM family's fused epilogues reproduce, bit for bit, the outputs recorded in tests/golden/gemm_bits.npz by
tools/gemm_bits.py, with both tile variants (one CTA per tile and CTA pairs, vnb_set_option "gemm_pair").  Schedule,
register allocation and the order of the epilogue's stores may change; the float operations on every output and their
order may not, so every hash must match."""
import os

import numpy as np
import pytest

from tools import gemm_bits as GB

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "gemm_bits.npz"))


@pytest.fixture(params=[0, 1], ids=["single_cta", "cta_pair"])
def pair(request):
    prev = GB.set_pair(request.param)
    yield request.param
    GB.set_pair(prev)


@pytest.mark.parametrize("case", GB.CASES, ids=[GB.case_name(*c) for c in GB.CASES])
def test_gemm_fused_output_bits_match_record(golden, pair, case):
    name = GB.case_name(*case)
    outs = GB.run_case(*case)
    got = GB.digest(outs)
    want = str(golden["sha256_" + name])
    if got != want:
        vals = GB.sample_values(outs, name)
        ref = golden["sample_" + name]
        same = (vals == ref) | (np.isnan(vals) & np.isnan(ref))
        pytest.fail(f"{name}: sha256 {got} != recorded {want}; sampled values of the first output: "
                    f"{int((~same).sum())} of {vals.size} differ, max |diff| {np.nanmax(np.abs(vals - ref)):.3e}")
