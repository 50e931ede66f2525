"""GPU: VampNet.generate_many — many independent generate() calls batched into one vnb_generate_many launch per
(T, steps, top-p on/off) bucket — equals the same calls made one by one, bit for bit, and leaves the global RNGs where
the sequential calls leave them.  Each row of a launch keeps its own call's N0, temperatures, schedules, top_p, Philox
key and row numbering, and the kernels' per-row arithmetic does not depend on the batch, so torch.equal is the
criterion, under both sampler paths (fused into the classifier epilogue, and from materialised logits)."""
import ctypes
import random

import numpy as np
import pytest
import torch

from tests.test_gpu_parity import TINY_C2F, TINY_COARSE, build

pytestmark = pytest.mark.gpu

FULL_COARSE = dict(n_heads=20, n_layers=20, n_codebooks=4, n_conditioning_codebooks=0, embedding_dim=1280)


def rng_state():
    return random.getstate(), np.random.get_state(), torch.get_rng_state()


def assert_same_rng(a, b):
    assert a[0] == b[0], "random state differs"
    assert a[1][0] == b[1][0] and np.array_equal(a[1][1], b[1][1]) and a[1][2:] == b[1][2:], "numpy state differs"
    assert torch.equal(a[2], b[2]), "torch state differs"


def reseed_globals(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def mix(cfg, seed):
    """A seeded mix of calls: B in {1, 2, 3}, seeds given and not, two temperatures, mask temperatures 10.5 and 0,
    sample cutoffs 1, 0.5 and -1 (true greedy), 3-D, 2-D and absent masks, two T buckets, a bucket with a different
    step count, and a top-p bucket whose calls use different top_p."""
    g = torch.Generator().manual_seed(seed)
    C, V = cfg["n_codebooks"], cfg.get("vocab_size", 1024)

    def z(B, T):
        return torch.randint(0, V, (B, C, T), generator=g).cuda()

    def m3(B, T):
        return (torch.rand(B, C, T, generator=g) < 0.6).long().cuda()

    def m2(B, T):
        return (torch.rand(B, T, generator=g) < 0.5).long().cuda()

    out = [
        dict(start_tokens=z(2, 40), mask=m3(2, 40), seed=11, temperature=1.0, mask_temperature=10.5),
        dict(start_tokens=z(1, 40), mask=m2(1, 40), temperature=0.7, mask_temperature=0.0, sample_cutoff=0.5),
        dict(start_tokens=z(3, 40), sample_cutoff=-1.0),
        dict(start_tokens=z(2, 24), mask=m3(2, 24), seed=5, temperature=0.7, sample_cutoff=0.5),
        dict(start_tokens=z(1, 24), mask=m2(1, 24), mask_temperature=0.0),
        dict(time_steps=24),
        dict(start_tokens=z(2, 40), mask=m3(2, 40), top_p=0.9),
        dict(start_tokens=z(1, 40), mask=m2(1, 40), top_p=0.8, seed=3, temperature=0.7),
        dict(start_tokens=z(2, 40), mask=m3(2, 40), _sampling_steps=3, sample_cutoff=-1.0),
        dict(start_tokens=z(1, 40), seed=7, _sampling_steps=3, mask_temperature=0.0),
    ]
    for c in out:
        c.setdefault("_sampling_steps", 4)
        c["return_signal"] = False
    return out


def set_fused(v):
    from vampnet_b200 import _lib as L
    prev = ctypes.c_int32(0)
    L.check(L.lib().vnb_get_option(b"fused_sampler", ctypes.byref(prev)))
    L.check(L.lib().vnb_set_option(b"fused_sampler", v))
    return prev.value


def sequential_and_batched(model, codec, calls, rng_seed):
    reseed_globals(rng_seed)
    want = [model.generate(codec, **c) for c in calls]
    want_rng = rng_state()
    reseed_globals(rng_seed)
    got = model.generate_many(codec, calls)
    return want, want_rng, got, rng_state()


@pytest.mark.parametrize("fused", [1, 0])
@pytest.mark.parametrize("tag,cfgd,lora", [("coarse", TINY_COARSE, False), ("c2f", TINY_C2F, False),
                                           ("coarse_lora", TINY_COARSE, True)])
def test_generate_many_equals_sequential_calls(tag, cfgd, lora, fused):
    _, _, model, _, codec = build(cfgd, lora=lora)
    prev = set_fused(fused)
    try:
        calls = mix(cfgd, seed=31)
        want, want_rng, got, got_rng = sequential_and_batched(model, codec, calls, rng_seed=123)
    finally:
        set_fused(prev)
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape and torch.equal(a, b), f"[{tag}] call {i} differs"
    assert_same_rng(got_rng, want_rng)


def test_generate_many_launches_one_per_bucket():
    """The mix above has four (T, steps, top-p) buckets: each is one launch with one group per call."""
    from vampnet_b200 import _lib as L
    _, _, model, _, codec = build(TINY_COARSE)
    calls = mix(TINY_COARSE, seed=5)
    seen = []
    real = L.lib
    lib = real()

    class Spy:
        def __getattr__(self, name):
            return getattr(lib, name)

        def vnb_generate_many(self, *a):
            seen.append((a[3], a[4], a[5], a[8]))  # B, T, steps, n_groups
            return lib.vnb_generate_many(*a)
    L.lib = lambda: Spy()
    try:
        model.generate_many(codec, calls)
    finally:
        L.lib = real
    assert sorted(seen) == sorted([(6, 40, 4, 3), (4, 24, 4, 3), (3, 40, 4, 2), (3, 40, 3, 2)]), seen


def test_full_size_coarse_app_shape():
    """The app's shape: the 20-layer d = 1280 coarse model at T = 575 (a 10 s chunk), eight calls of B = 2."""
    _, _, model, _, codec = build(FULL_COARSE)
    g = torch.Generator().manual_seed(8)
    calls = []
    for i in range(8):
        z = torch.randint(0, 1024, (2, 4, 575), generator=g).cuda()
        mask = (torch.rand(2, 4, 575, generator=g) < 0.7).long().cuda()
        calls.append(dict(start_tokens=z, mask=mask, _sampling_steps=12, return_signal=False,
                          seed=None if i % 3 else 100 + i, temperature=1.0 if i % 2 else 0.8))
    want, want_rng, got, got_rng = sequential_and_batched(model, codec, calls, rng_seed=9)
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), f"call {i} differs"
    assert_same_rng(got_rng, want_rng)


def test_regrouped_replay_needs_no_new_capture():
    """A (B, T) workspace replays its captured graph across groupings, seeds and temperatures: the grouping and the
    per-group table are written before every replay."""
    from vampnet_b200 import _lib as L
    _, _, model, _, codec = build(TINY_COARSE)
    g = torch.Generator().manual_seed(4)

    def calls(sizes, seeds, temps):
        return [dict(start_tokens=torch.randint(0, 1024, (b, 4, 40), generator=g).cuda(),
                     mask=(torch.rand(b, 4, 40, generator=g) < 0.6).long().cuda(), seed=s, temperature=t,
                     _sampling_steps=4, return_signal=False) for b, s, t in zip(sizes, seeds, temps)]
    model.generate_many(codec, calls([2, 1, 3], [1, None, 2], [1.0, 0.7, 1.0]))
    second = calls([1, 1, 2, 2], [None, 9, None, 10], [0.6, 1.0, 1.3, 0.9])
    before = L.lib().vnb_graph_capture_count()
    reseed_globals(77)
    got = model.generate_many(codec, second)
    assert L.lib().vnb_graph_capture_count() == before, "regrouping captured a new graph"
    got_rng = rng_state()
    reseed_globals(77)
    want = [model.generate(codec, **c) for c in second]
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    assert_same_rng(got_rng, rng_state())


def test_malformed_groups_raise():
    from vampnet_b200 import _lib as L
    _, _, model, _, codec = build(TINY_COARSE)
    model._ensure_handle(codec)
    B, T, steps = 3, 16, 2
    z = torch.randint(0, 1024, (B, 4, T)).cuda()
    out = torch.empty_like(z)
    gam = (ctypes.c_float * steps)(0.5, 0.1)
    tef = (ctypes.c_float * steps)(1.0, 0.0)
    dos = (ctypes.c_int32 * steps)(1, 1)

    def groups(*spec):
        arr = (L.GenGroup * max(len(spec), 1))()
        for g, (rows, top_p) in zip(arr, spec):
            g.rows, g.temperature, g.temp_eff, g.do_sample, g.seed_lo, g.seed_hi, g.top_p = rows, 1.0, tef, dos, 1, 0, top_p
        return arr

    def launch(arr, n, B=B, steps=steps):
        with torch.cuda.device(model.device):
            L.check(L.lib().vnb_generate_many(model._handle, L.ptr(z), None, B, T, steps, gam, arr, n, 0, L.ptr(out),
                                              L.stream_ptr(model.device)))
    launch(groups((1, 0.0), (2, 0.0)), 2)  # well formed
    cases = [
        (lambda: launch(groups((1, 0.0), (1, 0.0)), 2), "sum to 2"),
        (lambda: launch(groups((2, 0.0), (2, 0.0)), 2), "sum to 4"),
        (lambda: launch(groups((3, 0.0)), 0), "n_groups 0"),
        (lambda: launch(groups(*[(1, 0.0)] * 4), 4), "n_groups 4"),
        (lambda: launch(groups((1, 0.0), (0, 0.0), (2, 0.0)), 3), "0 rows"),
        (lambda: launch(groups((3, 0.0)), 1, steps=0), "sampling_steps 0"),
        (lambda: launch(groups((3, 0.0)), 1, steps=257), "sampling_steps 257"),
        (lambda: launch(groups((1, 0.9), (2, 0.0)), 2), "mix top-p"),
    ]
    for fn, what in cases:
        with pytest.raises(RuntimeError, match="vampnet_b200"):
            fn()
    torch.cuda.synchronize()
    launch(groups((3, 0.0)), 1)  # the library still works after the rejections
    torch.cuda.synchronize()
