"""CPU: Interface.vamp_many(mixed_lengths=True) hands the flag to both stages' generate_many and still equals the
sequential vamp() calls (results, each chunk's key, RNG state); without the flag, generate_many is called as before,
with no extra argument."""
import numpy as np
import pytest
import torch

from tests.test_interface_many_cpu import KeyedStub, requests, reseed, rng_state
from tests.test_interface_cpu import StubCodec
from vampnet_b200.interface import Interface


class FlagStub(KeyedStub):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.flags = []

    def generate_many(self, codec, calls, **kw):
        self.flags.append(kw)
        return super().generate_many(codec, calls)


def make_iface():
    return Interface.from_models(StubCodec(), FlagStub(4, 0, salt=5), FlagStub(14, 4, salt=9), device="cpu",
                                 coarse_chunk_size_s=0.6, coarse2fine_chunk_size_s=0.25)


@pytest.mark.parametrize("mixed", [True, False])
def test_vamp_many_forwards_mixed_lengths(mixed):
    reqs = requests(7)
    seq = make_iface()
    reseed(11)
    want = [seq.vamp(**r) for r in reqs]
    want_rng = rng_state()
    many = make_iface()
    reseed(11)
    got = many.vamp_many(reqs, mixed_lengths=True) if mixed else many.vamp_many(reqs)
    got_rng = rng_state()
    for r, a, b in zip(reqs, got, want):
        if r["return_mask"]:
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        else:
            assert torch.equal(a, b)
    assert got_rng[0] == want_rng[0] and np.array_equal(got_rng[1][1], want_rng[1][1])
    assert torch.equal(got_rng[2], want_rng[2])
    expect = {"mixed_lengths": True} if mixed else {}
    assert many.coarse.flags and many.c2f.flags
    assert all(f == expect for f in many.coarse.flags + many.c2f.flags)
    for m_seq, m_many in ((seq.coarse, many.coarse), (seq.c2f, many.c2f)):
        assert sorted((c["key"], c["shape"], str(c["kwargs"])) for c in m_seq.calls) == \
            sorted((c["key"], c["shape"], str(c["kwargs"])) for c in m_many.calls)
