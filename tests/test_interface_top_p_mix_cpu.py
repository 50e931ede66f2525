"""CPU: Interface.vamp_many(mixed_top_p=True) hands the flag to both stages' generate_many and still equals the
sequential vamp() calls; VampNet._launch_calls(mixed_top_p=True) buckets calls without their top-p state, keeps the
MANY_MAX_ROWS split and the longest-first orders of mixed_lengths / mixed_steps, and maps the results back to list
order.  Without the flag the grouping is the one before."""
import numpy as np
import pytest
import torch

from tests.test_interface_many_cpu import requests, reseed, rng_state
from tests.test_interface_steps_cpu import SPEC, make_iface, prepared, run
from vampnet_b200.modules import transformer as TR


@pytest.mark.parametrize("kw", [dict(mixed_top_p=True), dict(mixed_top_p=True, mixed_steps=True, mixed_lengths=True),
                                dict(mixed_top_p=False)], ids=["top_p", "top_p_steps_lengths", "off"])
def test_vamp_many_forwards_mixed_top_p(kw):
    reqs = requests(8)
    for i, r in enumerate(reqs):  # nucleus and plain requests, and top_p values that switch the filter off
        r["top_p"] = (0.8, None, 0.95, 0.0, 1.0)[i % 5]
    seq = make_iface()
    reseed(12)
    want = [seq.vamp(**r) for r in reqs]
    want_rng = rng_state()
    many = make_iface()
    reseed(12)
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


# SPEC (B, T, steps, top_p): calls 2 and 5 have top-p on
def test_launch_calls_mix_top_p_in_one_launch_per_bucket():
    # the (T, steps) buckets of the plain calls now take the nucleus calls of the same (T, steps)
    assert run(prepared(SPEC), mixed_top_p=True) == [("group", [0], [2]), ("group", [1, 2, 6], [5, 5, 5]),
                                                     ("group", [3], [1]), ("group", [4], [9]), ("group", [5], [3]),
                                                     ("group", [7], [9])]
    # with mixed steps: one launch per T, longest steps first (stable)
    assert run(prepared(SPEC), mixed_top_p=True, mixed_steps=True) == [
        ("group", [4, 1, 2, 6, 5, 0, 3], [9, 5, 5, 5, 3, 2, 1]), ("group", [7], [9])]
    # and with mixed lengths: every call in one launch, longest T first, then longest steps first
    assert run(prepared(SPEC), mixed_top_p=True, mixed_steps=True, mixed_lengths=True) == [
        ("ragged", [4, 7, 1, 2, 6, 5, 0, 3], [9, 9, 5, 5, 5, 3, 2, 1])]


def test_launch_calls_without_the_flag_is_unchanged():
    assert run(prepared(SPEC), mixed_top_p=False) == run(prepared(SPEC))
    assert run(prepared(SPEC), mixed_top_p=False, mixed_steps=True) == [
        ("group", [4, 1, 6, 0, 3], [9, 5, 5, 2, 1]), ("group", [2, 5], [5, 3]), ("group", [7], [9])]


def test_launch_calls_mixed_top_p_split_is_unchanged(monkeypatch):
    """MANY_MAX_ROWS packs each bucket in list order (mixed_lengths: longest T first) before each launch is ordered."""
    monkeypatch.setattr(TR, "MANY_MAX_ROWS", 200)
    # T = 50: list order 0, 1, 2 (4 rows); 3 would make 5 x 50 > 200: [3, 4, 5] (4 rows); then [6]; T = 30: [7]
    assert run(prepared(SPEC), mixed_top_p=True, mixed_steps=True) == [
        ("group", [1, 2, 0], [5, 5, 2]), ("group", [4, 5, 3], [9, 3, 1]), ("group", [6], [5]), ("group", [7], [9])]
