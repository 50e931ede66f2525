"""GPU: Interface.vamp_many on the CUDA path equals the sequential vamp() calls bit for bit — tokens, returned masks and
the global RNG state afterwards — for requests of different lengths (several coarse chunks with a remainder, padded
fine-stage chunks), batch sizes 1-2, feedback passes 1-2, time stretch 1-2 and both return_mask values.  And
generate_many(return_signal=True) decodes each call like generate() does."""
import random

import numpy as np
import pytest
import torch

from tests.test_gpu_interface import iface  # noqa: F401  (module fixture: tiny coarse / c2f / codec)

pytestmark = pytest.mark.gpu


def rng_state():
    return random.getstate(), np.random.get_state(), torch.get_rng_state()


def reseed(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def test_vamp_many_equals_sequential_vamp(iface):  # noqa: F811
    g = torch.Generator().manual_seed(12)
    reqs = []
    # coarse chunks of 35 frames, fine-stage chunks of 15 (padded)
    for T, bs, fb, k, rm, kw in [(83, 2, 1, 1, True, dict(seed=3)), (50, 1, 2, 1, False, dict(temperature=0.8)),
                                 (20, 2, 2, 2, True, {}), (61, 1, 1, 1, False, dict(sample_cutoff=0.5, seed=9))]:
        z = torch.randint(0, 1024, (1, 14, T), generator=g).cuda()
        mask = (torch.rand(1, 14, T, generator=g) < 0.7).long().cuda()
        mask[:, :, ::6] = 0
        reqs.append(dict(codes=z, mask=mask, batch_size=bs, feedback_steps=fb, time_stretch_factor=k, return_mask=rm,
                         _sampling_steps=3, **kw))
    reseed(21)
    want = [iface.vamp(**r) for r in reqs]
    want_rng = rng_state()
    reseed(21)
    got = iface.vamp_many(reqs)
    got_rng = rng_state()
    for i, (r, a, b) in enumerate(zip(reqs, got, want)):
        if r["return_mask"]:
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), f"request {i} differs"
        else:
            assert torch.equal(a, b), f"request {i} differs"
    assert got_rng[0] == want_rng[0] and np.array_equal(got_rng[1][1], want_rng[1][1])
    assert torch.equal(got_rng[2], want_rng[2])


def test_generate_many_return_signal(iface):  # noqa: F811
    g = torch.Generator().manual_seed(2)
    calls = [dict(start_tokens=torch.randint(0, 1024, (b, 4, 30), generator=g).cuda(), _sampling_steps=3, seed=s,
                  return_signal=rs) for b, s, rs in [(1, 4, True), (2, None, False), (2, None, True)]]
    reseed(1)
    want = [iface.coarse.generate(iface.codec, **c) for c in calls]
    reseed(1)
    got = iface.coarse.generate_many(iface.codec, calls)
    for c, a, b in zip(calls, got, want):
        if c["return_signal"]:
            assert a.sample_rate == b.sample_rate and torch.equal(a.audio_data, b.audio_data)
        else:
            assert torch.equal(a, b)
