"""GPU: Interface.vamp_many(mixed_lengths=True) equals the sequential vamp() calls bit for bit — tokens, returned masks
and the global RNG state afterwards — for requests whose coarse remainders (and so launches) have different lengths."""
import numpy as np
import pytest
import torch

from tests.test_gpu_interface import iface  # noqa: F401  (module fixture: tiny coarse / c2f / codec)
from tests.test_gpu_interface_many import reseed, rng_state

pytestmark = pytest.mark.gpu


def test_vamp_many_mixed_lengths_equals_sequential_vamp(iface):  # noqa: F811
    g = torch.Generator().manual_seed(13)
    reqs = []
    # coarse chunks of 35 frames: remainders of 13, 15, 20, 26 and 1 frames; fine-stage chunks of 15 (padded)
    for T, bs, fb, k, rm, kw in [(83, 2, 1, 1, True, dict(seed=3)), (50, 1, 2, 1, False, dict(temperature=0.8)),
                                 (20, 2, 2, 2, True, {}), (61, 1, 1, 1, False, dict(sample_cutoff=0.5, seed=9)),
                                 (36, 2, 1, 1, False, dict(top_p=0.9))]:
        z = torch.randint(0, 1024, (1, 14, T), generator=g).cuda()
        mask = (torch.rand(1, 14, T, generator=g) < 0.7).long().cuda()
        mask[:, :, ::6] = 0
        reqs.append(dict(codes=z, mask=mask, batch_size=bs, feedback_steps=fb, time_stretch_factor=k, return_mask=rm,
                         _sampling_steps=3, **kw))
    reseed(21)
    want = [iface.vamp(**r) for r in reqs]
    want_rng = rng_state()
    reseed(21)
    got = iface.vamp_many(reqs, mixed_lengths=True)
    got_rng = rng_state()
    for i, (r, a, b) in enumerate(zip(reqs, got, want)):
        if r["return_mask"]:
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), f"request {i} differs"
        else:
            assert torch.equal(a, b), f"request {i} differs"
    assert got_rng[0] == want_rng[0] and np.array_equal(got_rng[1][1], want_rng[1][1])
    assert torch.equal(got_rng[2], want_rng[2])
