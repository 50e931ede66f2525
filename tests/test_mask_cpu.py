"""CPU: vampnet_b200.mask against the ORIGINAL project's vampnet/mask.py under the same torch seeds (its outputs are
stored in tests/golden/reference_mask.npz by oracle/gen_reference_golden.py), plus checks of our own (including
the reference's only fixture for this code, scratch/rms_mask.txt: period 7, 3 unmasked-able codebooks)."""
import os

import numpy as np
import pytest
import torch

from oracle.gen_reference_golden import MASK_X_SEED, MASK_X_SHAPE, build_mask_chain, mask_cases
from vampnet_b200 import mask as pm


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "reference_mask.npz"))


def test_periodic_and_codebook_mask_shape_of_fixture():
    z = torch.zeros(1, 14, 100, dtype=torch.long)
    m = pm.mask_and(pm.linear_random(z, 1.0), pm.periodic_mask(z, 7, 1, random_roll=False))
    m = pm.codebook_mask(pm.codebook_unmask(m, 0), 3)
    assert m.shape == (1, 14, 100)
    assert (m[0, 3:] == 1).all()
    assert (m[0, :3, ::7] == 0).all() and m[0, :3].sum() == 3 * (100 - 15)


def test_apply_mask_and_inpaint():
    x = torch.randint(0, 1024, (2, 4, 20))
    m = pm.inpaint(x, 3, 5)
    assert (m[:, :, :3] == 0).all() and (m[:, :, -5:] == 0).all() and (m[:, :, 3:-5] == 1).all()
    y, _ = pm.apply_mask(x, m, 1024)
    assert torch.equal(y[:, :, :3], x[:, :, :3]) and (y[:, :, 3:-5] == 1024).all()
    with pytest.raises(AssertionError):
        pm.apply_mask(x, m * 2, 1024)
    with pytest.raises(AssertionError):
        pm.apply_mask(x, m.int(), 1024)


def test_against_reference_mask_module(golden):
    x = torch.randint(0, 1024, MASK_X_SHAPE, generator=torch.Generator().manual_seed(MASK_X_SEED))
    for i, fn in enumerate(mask_cases(pm, x)):
        torch.manual_seed(123 + i)
        got = fn()
        want = torch.from_numpy(golden[f"case{i}"])
        assert torch.equal(got, want if got.is_floating_point() else want.long()), f"case {i}"


def test_build_mask_rng_stream_matches_reference(golden):
    """Interface.build_mask composes the pieces; same seed -> same mask AND same RNG state afterwards."""
    x = torch.randint(0, 1024, (2, 14, 100), generator=torch.Generator().manual_seed(1))
    torch.manual_seed(7)
    b = build_mask_chain(pm, x)
    rb = torch.rand(4)
    assert torch.equal(b, torch.from_numpy(golden["chain"]).long())
    assert torch.equal(rb, torch.from_numpy(golden["chain_next_draws"]))
