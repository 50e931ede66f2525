"""CPU: Interface.vamp_many(mixed_steps=True) hands the flag to both stages' generate_many and still equals the
sequential vamp() calls; VampNet._launch_calls(mixed_steps=True) buckets calls without their step counts, orders every
launch by steps, longest first (stable), and maps the results back to list order."""
import numpy as np
import pytest
import torch

from tests.test_interface_cpu import StubCodec
from tests.test_interface_many_cpu import KeyedStub, requests, reseed, rng_state
from vampnet_b200.interface import Interface
from vampnet_b200.modules import transformer as TR


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


@pytest.mark.parametrize("kw", [dict(mixed_steps=True), dict(mixed_steps=True, mixed_lengths=True),
                                dict(mixed_steps=False)], ids=["steps", "steps_lengths", "off"])
def test_vamp_many_forwards_mixed_steps(kw):
    reqs = requests(7)
    for i, r in enumerate(reqs):  # requests of different step counts
        r["_sampling_steps"] = (12, 24, 36, 48, 64)[i % 5]
    seq = make_iface()
    reseed(11)
    want = [seq.vamp(**r) for r in reqs]
    want_rng = rng_state()
    many = make_iface()
    reseed(11)
    got = many.vamp_many(reqs, **kw)
    got_rng = rng_state()
    for r, a, b in zip(reqs, got, want):
        if r["return_mask"]:
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        else:
            assert torch.equal(a, b)
    assert got_rng[0] == want_rng[0] and np.array_equal(got_rng[1][1], want_rng[1][1])
    assert torch.equal(got_rng[2], want_rng[2])
    expect = {k: True for k, v in kw.items() if v}
    assert many.coarse.flags and many.c2f.flags
    assert all(f == expect for f in many.coarse.flags + many.c2f.flags)
    for m_seq, m_many in ((seq.coarse, many.coarse), (seq.c2f, many.c2f)):
        assert sorted((c["key"], c["shape"], str(c["kwargs"])) for c in m_seq.calls) == \
            sorted((c["key"], c["shape"], str(c["kwargs"])) for c in m_many.calls)


class LaunchRecorder:
    """Stands in for a VampNet in _launch_calls: records every launch's calls and returns call i's result as a (B, 1, T)
    tensor filled with i."""

    def __init__(self):
        self.launches = []

    def _launch_group(self, calls, keep):
        self.launches.append(("group", [c["i"] for c in calls], [c["steps"] for c in calls]))
        return [torch.full((c["z"].shape[0], 1, c["z"].shape[-1]), c["i"]) for c in calls]

    def _launch_ragged(self, calls, keep):
        self.launches.append(("ragged", [c["i"] for c in calls], [c["steps"] for c in calls]))
        return [torch.full((c["z"].shape[0], 1, c["z"].shape[-1]), c["i"]) for c in calls]


def prepared(spec):
    return [dict(i=i, z=torch.zeros(B, 1, T, dtype=torch.int64), steps=s, top_p=tp)
            for i, (B, T, s, tp) in enumerate(spec)]


def run(calls, **kw):
    rec = LaunchRecorder()
    outs = TR.VampNet._launch_calls(rec, calls, **kw)
    for i, (c, o) in enumerate(zip(calls, outs)):  # results in list order
        assert o.shape == (c["z"].shape[0], 1, c["z"].shape[-1]) and bool((o == i).all())
    return rec.launches


SPEC = [(1, 50, 2, 0.0), (2, 50, 5, 0.0), (1, 50, 5, 0.9), (1, 50, 1, 0.0), (2, 50, 9, 0.0), (1, 50, 3, 0.9),
        (1, 50, 5, 0.0), (1, 30, 9, 0.0)]


def test_launch_calls_orders_each_launch_longest_steps_first():
    # T buckets stay without mixed_lengths; the steps no longer split a bucket
    assert run(prepared(SPEC), mixed_steps=True) == [("group", [4, 1, 6, 0, 3], [9, 5, 5, 2, 1]),
                                                     ("group", [2, 5], [5, 3]), ("group", [7], [9])]
    assert run(prepared(SPEC), mixed_steps=True, mixed_lengths=True) == [
        ("ragged", [4, 7, 1, 6, 0, 3], [9, 9, 5, 5, 2, 1]), ("ragged", [2, 5], [5, 3])]
    # without the flag: one launch per (T, steps, top-p) bucket, as before
    assert run(prepared(SPEC)) == [("group", [0], [2]), ("group", [1, 6], [5, 5]), ("group", [2], [5]),
                                   ("group", [3], [1]), ("group", [4], [9]), ("group", [5], [3]), ("group", [7], [9])]


def test_launch_calls_split_is_unchanged(monkeypatch):
    """MANY_MAX_ROWS packs the bucket in list order (mixed_lengths: longest T first) before each launch is ordered."""
    monkeypatch.setattr(TR, "MANY_MAX_ROWS", 200)
    assert run(prepared(SPEC), mixed_steps=True) == [("group", [1, 0, 3], [5, 2, 1]), ("group", [4, 6], [9, 5]),
                                                     ("group", [2, 5], [5, 3]), ("group", [7], [9])]
