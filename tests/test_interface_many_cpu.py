"""CPU: Interface.vamp_many orchestration — every request's chunks run stage by stage through generate_many, and the
result, the keys each chunk gets and the global RNG state afterwards equal the sequential vamp() calls'.  The stub
models draw their key the way VampNet.generate does (draw_philox_key, or a given philox_key) and fold it into their
output, so a key handed to the wrong chunk, or drawn in the wrong order, changes the result."""
import random

import numpy as np
import pytest
import torch

from tests.test_interface_cpu import StubCodec, StubModel, fake_generate
from vampnet_b200.interface import Interface
from vampnet_b200.modules.transformer import draw_philox_key


class KeyedStub(StubModel):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.launches = []

    def generate(self, codec=None, time_steps=None, start_tokens=None, mask=None, return_signal=True, seed=None,
                 philox_key=None, **kwargs):
        assert return_signal is False
        key = philox_key if philox_key is not None else draw_philox_key(seed)
        self.calls.append(dict(time_steps=time_steps, shape=tuple(start_tokens.shape), key=key, kwargs=kwargs))
        return fake_generate(start_tokens, mask, self.salt + key % 1009)

    def generate_many(self, codec, calls):
        self.launches.append([tuple(c["start_tokens"].shape) for c in calls])
        return [self.generate(codec, **c) for c in calls]


def make_iface():
    coarse, c2f = KeyedStub(4, 0, salt=5), KeyedStub(14, 4, salt=9)
    return Interface.from_models(StubCodec(), coarse, c2f, device="cpu", coarse_chunk_size_s=0.6,
                                 coarse2fine_chunk_size_s=0.25)


def requests(seed):
    g = torch.Generator().manual_seed(seed)

    def case(T, keep_every):
        z = torch.randint(0, 1024, (1, 14, T), generator=g)
        mask = torch.ones_like(z)
        mask[:, :, ::keep_every] = 0
        return z, mask
    out = []
    for T, bs, fb, k, rm, kw in [(83, 2, 1, 1, True, dict(temperature=0.7)), (50, 1, 2, 1, False, dict(seed=4)),
                                 (20, 2, 2, 2, True, {}), (61, 1, 3, 1, False, dict(seed=8, top_p=0.9)),
                                 (35, 1, 1, 1, True, {})]:
        z, mask = case(T, 5 + T % 4)
        out.append(dict(codes=z, mask=mask, batch_size=bs, feedback_steps=fb, time_stretch_factor=k, return_mask=rm,
                        **kw))
    return out


def rng_state():
    return random.getstate(), np.random.get_state(), torch.get_rng_state()


def reseed(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


@pytest.mark.parametrize("order", [(0, 1, 2, 3, 4), (3, 4, 0, 2, 1), (2,)])
def test_vamp_many_equals_sequential_vamp(order):
    reqs = [requests(7)[i] for i in order]
    seq = make_iface()
    reseed(11)
    want = [seq.vamp(**r) for r in reqs]
    want_rng = rng_state()
    many = make_iface()
    reseed(11)
    got = many.vamp_many(reqs)
    got_rng = rng_state()
    assert len(got) == len(want)
    for r, a, b in zip(reqs, got, want):
        if r["return_mask"]:
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        else:
            assert torch.equal(a, b)
    assert got_rng[0] == want_rng[0] and np.array_equal(got_rng[1][1], want_rng[1][1])
    assert torch.equal(got_rng[2], want_rng[2])
    # every chunk got the key its sequential call drew, and the same generate arguments
    for m_seq, m_many in ((seq.coarse, many.coarse), (seq.c2f, many.c2f)):
        assert sorted((c["key"], c["shape"], str(c["kwargs"])) for c in m_seq.calls) == \
            sorted((c["key"], c["shape"], str(c["kwargs"])) for c in m_many.calls)


def test_vamp_many_launches_one_generate_many_per_stage():
    reqs = requests(3)
    iface = make_iface()
    iface.vamp_many(reqs)
    coarse_span, c2f_span = 35, 15

    def n_chunks(T, span):
        return -(-T // span)
    frames = [r["codes"].shape[-1] * r["time_stretch_factor"] for r in reqs]
    passes = max(r["feedback_steps"] for r in reqs)
    assert len(iface.coarse.launches) == passes and len(iface.c2f.launches) == 1
    for i, launch in enumerate(iface.coarse.launches):
        assert len(launch) == sum(n_chunks(f, coarse_span) for f, r in zip(frames, reqs) if r["feedback_steps"] > i)
        assert all(s[1] == 4 for s in launch)
    assert len(iface.c2f.launches[0]) == sum(n_chunks(f, c2f_span) for f in frames)
    assert all(s[1:] == (14, c2f_span) for s in iface.c2f.launches[0])
    # the fine stage keeps its pinned arguments; the coarse stage gets each request's own
    assert all(c["kwargs"] == {"cfg_guidance": None, "typical_filtering": True, "_sampling_steps": 2}
               for c in iface.c2f.calls)
    assert {str(c["kwargs"]) for c in iface.coarse.calls} == {"{'temperature': 0.7}", "{}", "{'top_p': 0.9}"}
