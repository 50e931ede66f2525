"""GPU: VampNet.generate_many(mixed_lengths=True) — calls of different T in one vnb_generate_ragged launch per
(sampling steps, top-p on/off) bucket — equals the same calls made one by one, bit for bit, and leaves the global RNGs
where the sequential calls leave them.

Each call is padded to its launch's longest T with kept frames (code 0, mask 0): they are never sampled, never count
in N0 and never re-masked, attention stops at the call's own length, and the QKV epilogue writes zero v^T columns for
them, so the real frames see exactly the operands of a launch of their own.  The lengths span the attention kernel's
64-key blocks and 128-query tiles (1, 63, 64, 65, 127, 128, 129, 200), with one call at the launch's full T."""
import ctypes

import pytest
import torch

from tests.test_gpu_adapters import base_with_adapters
from tests.test_gpu_generate_many import (FULL_COARSE, assert_same_rng, reseed_globals, rng_state, set_fused)
from tests.test_gpu_parity import TINY_C2F, TINY_COARSE, build

pytestmark = pytest.mark.gpu


def ragged_mix(cfg, seed, adapters=()):
    """Calls of T in {1, 63, 64, 65, 127, 128, 129, 200} and B in {1, 2}: seeds given and not, two temperatures, mask
    temperatures 10.5 and 0, sample cutoffs 1, 0.5 and -1, 3-D, 2-D and absent masks, start tokens absent; a bucket
    with a different step count and a top-p bucket, each of mixed T too.  `adapters` are spread over the calls."""
    g = torch.Generator().manual_seed(seed)
    C = cfg["n_codebooks"]

    def z(B, T):
        return torch.randint(0, 1024, (B, C, T), generator=g).cuda()

    def m3(B, T):
        return (torch.rand(B, C, T, generator=g) < 0.6).long().cuda()

    def m2(B, T):
        return (torch.rand(B, T, generator=g) < 0.5).long().cuda()

    out = [
        dict(start_tokens=z(2, 129), mask=m3(2, 129), seed=11, temperature=1.0, mask_temperature=10.5),
        dict(start_tokens=z(1, 200), mask=m2(1, 200), temperature=0.7, mask_temperature=0.0, sample_cutoff=0.5),
        dict(start_tokens=z(2, 63), sample_cutoff=-1.0),
        dict(start_tokens=z(1, 1), mask=m3(1, 1), seed=5, temperature=0.7),
        dict(start_tokens=z(2, 64), mask=m2(2, 64), mask_temperature=0.0),
        dict(time_steps=65),
        dict(start_tokens=z(1, 127), mask=m3(1, 127), seed=6),
        dict(start_tokens=z(1, 128), mask=m3(1, 128), temperature=1.3),
        dict(start_tokens=z(2, 200), mask=m3(2, 200), top_p=0.9),
        dict(start_tokens=z(1, 65), mask=m2(1, 65), top_p=0.8, seed=3, temperature=0.7),
        dict(start_tokens=z(1, 1), top_p=0.85),
        dict(start_tokens=z(2, 129), mask=m3(2, 129), _sampling_steps=3, sample_cutoff=-1.0),
        dict(start_tokens=z(1, 64), seed=7, _sampling_steps=3, mask_temperature=0.0),
        dict(start_tokens=z(1, 200), mask=m3(1, 200), _sampling_steps=3, seed=8),
    ]
    for i, c in enumerate(out):
        c.setdefault("_sampling_steps", 4)
        c["return_signal"] = False
        if adapters and adapters[i % len(adapters)] is not None:
            c["adapter"] = adapters[i % len(adapters)]
    return out


def sequential_and_mixed(model, codec, calls, rng_seed):
    reseed_globals(rng_seed)
    want = [model.generate(codec, **c) for c in calls]
    want_rng = rng_state()
    reseed_globals(rng_seed)
    got = model.generate_many(codec, calls, mixed_lengths=True)
    return want, want_rng, got, rng_state()


def assert_all_equal(got, want, tag):
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape and torch.equal(a, b), f"[{tag}] call {i} (T = {b.shape[-1]}) differs"


@pytest.mark.parametrize("fused", [1, 0])
@pytest.mark.parametrize("tag,cfgd,lora", [("coarse", TINY_COARSE, False), ("c2f", TINY_C2F, False),
                                           ("coarse_lora", TINY_COARSE, True)])
def test_mixed_lengths_equal_sequential_calls(tag, cfgd, lora, fused):
    _, _, model, _, codec = build(cfgd, lora=lora)
    prev = set_fused(fused)
    try:
        want, want_rng, got, got_rng = sequential_and_mixed(model, codec, ragged_mix(cfgd, seed=31), rng_seed=123)
    finally:
        set_fused(prev)
    assert_all_equal(got, want, tag)
    assert_same_rng(got_rng, want_rng)


@pytest.mark.parametrize("fused", [1, 0])
@pytest.mark.parametrize("tag,cfgd", [("coarse", TINY_COARSE), ("c2f", TINY_C2F)])
def test_mixed_lengths_with_adapters_equal_sequential_calls(tag, cfgd, fused):
    _, _, model, _, codec = base_with_adapters(cfgd, seed=2)
    prev = set_fused(fused)
    try:
        calls = ragged_mix(cfgd, seed=17, adapters=(None, "ft0", "ft1"))
        want, want_rng, got, got_rng = sequential_and_mixed(model, codec, calls, rng_seed=5)
    finally:
        set_fused(prev)
    assert_all_equal(got, want, tag + " adapters")
    assert_same_rng(got_rng, want_rng)


def test_full_size_coarse_app_shapes():
    """The 20-layer d = 1280 coarse model: B = 2 calls of a full 10 s chunk (575 frames) and three remainders."""
    _, _, model, _, codec = build(FULL_COARSE)
    g = torch.Generator().manual_seed(8)
    calls = []
    for i, T in enumerate((575, 502, 271, 133)):
        z = torch.randint(0, 1024, (2, 4, T), generator=g).cuda()
        mask = (torch.rand(2, 4, T, generator=g) < 0.7).long().cuda()
        calls.append(dict(start_tokens=z, mask=mask, _sampling_steps=12, return_signal=False,
                          seed=None if i % 3 else 100 + i, temperature=1.0 if i % 2 else 0.8))
    seen = []
    with spy_ragged(seen):
        want, want_rng, got, got_rng = sequential_and_mixed(model, codec, calls, rng_seed=9)
    assert [s[:2] for s in seen] == [(8, 575)], seen
    assert_all_equal(got, want, "full coarse")
    assert_same_rng(got_rng, want_rng)


class spy_ragged:
    """Records (B, T, steps, n_groups, frames) of every vnb_generate_ragged launch while installed."""

    def __init__(self, seen):
        from vampnet_b200 import _lib as L
        self.L, self.real, self.seen = L, L.lib, seen

    def __enter__(self):
        lib, seen = self.real(), self.seen

        class Spy:
            def __getattr__(self, name):
                return getattr(lib, name)

            def vnb_generate_ragged(self, *a):
                seen.append((a[3], a[4], a[5], a[8], tuple(a[9][:a[8]])))
                return lib.vnb_generate_ragged(*a)
        self.L.lib = lambda: Spy()
        return self

    def __exit__(self, *exc):
        self.L.lib = self.real


def test_mixed_lengths_launch_grouping(monkeypatch):
    """Mixed T with equal steps and top-p on/off is one launch at the longest T; the launch splits where rows x T would
    pass MANY_MAX_ROWS, longest calls first."""
    from vampnet_b200.modules import transformer as TR
    _, _, model, _, codec = build(TINY_COARSE)
    g = torch.Generator().manual_seed(3)
    calls = [dict(start_tokens=torch.randint(0, 1024, (B, 4, T), generator=g).cuda(), _sampling_steps=3,
                  return_signal=False, seed=i)
             for i, (B, T) in enumerate([(1, 65), (2, 129), (1, 1), (1, 200), (2, 64)])]
    seen = []
    with spy_ragged(seen):
        model.generate_many(codec, calls, mixed_lengths=True)
    assert seen == [(7, 200, 3, 5, (200, 129, 65, 64, 1))], seen
    seen.clear()
    monkeypatch.setattr(TR, "MANY_MAX_ROWS", 600)
    with spy_ragged(seen):
        reseed_globals(4)
        got = model.generate_many(codec, calls, mixed_lengths=True)
    # 200 x (1 + 2) = 600 fits; one more row would make 800: the rest is a launch at T = 65
    assert seen == [(3, 200, 3, 2, (200, 129)), (4, 65, 3, 3, (65, 64, 1))], seen
    reseed_globals(4)
    assert_all_equal(got, [model.generate(codec, **c) for c in calls], "split launch")


def test_new_lengths_on_a_captured_workspace_need_no_capture():
    """The frames table is written before every replay: a second mixed launch on the same (B, T) workspace with other
    lengths replays the captured graph and is still bit-identical to the sequential calls."""
    from vampnet_b200 import _lib as L
    _, _, model, _, codec = build(TINY_COARSE)
    g = torch.Generator().manual_seed(6)

    def calls(lengths, seeds):
        return [dict(start_tokens=torch.randint(0, 1024, (1, 4, T), generator=g).cuda(),
                     mask=(torch.rand(1, 4, T, generator=g) < 0.6).long().cuda(), seed=s, _sampling_steps=4,
                     return_signal=False) for T, s in zip(lengths, seeds)]
    model.generate_many(codec, calls([150, 129, 40], [1, None, 2]), mixed_lengths=True)
    second = calls([150, 20, 100], [None, 9, 10])
    before = L.lib().vnb_graph_capture_count()
    reseed_globals(77)
    got = model.generate_many(codec, second, mixed_lengths=True)
    assert L.lib().vnb_graph_capture_count() == before, "new lengths captured a new graph"
    got_rng = rng_state()
    reseed_globals(77)
    assert_all_equal(got, [model.generate(codec, **c) for c in second], "replay")
    assert_same_rng(got_rng, rng_state())


def test_ragged_refusals():
    from vampnet_b200 import _lib as L
    _, _, model, _, codec = build(TINY_COARSE)
    model._ensure_handle(codec)
    B, T, steps = 3, 16, 2
    z = torch.randint(0, 1024, (B, 4, T)).cuda()
    mask = torch.zeros(B, 4, T, dtype=torch.int32).cuda()
    mask[:, :, :4] = 1
    out = torch.empty_like(z)
    gam = (ctypes.c_float * steps)(0.5, 0.1)
    tef = (ctypes.c_float * steps)(1.0, 0.0)
    dos = (ctypes.c_int32 * steps)(1, 1)
    arr = (L.GenGroup * 2)()
    for gr, rows in zip(arr, (1, 2)):
        gr.rows, gr.temperature, gr.temp_eff, gr.do_sample, gr.seed_lo, gr.seed_hi, gr.top_p = rows, 1.0, tef, dos, 1, 0, 0.0

    def launch(frames, m=mask):
        fr = None if frames is None else (ctypes.c_int32 * 2)(*frames)
        with torch.cuda.device(model.device):
            L.check(L.lib().vnb_generate_ragged(model._handle, L.ptr(z), L.ptr(m), B, T, steps, gam, arr, 2, fr, None, 0,
                                                L.ptr(out), L.stream_ptr(model.device)))
    launch((16, 5))          # well formed
    launch((16, 16), None)   # no group shorter than T: the default mask is allowed
    launch(None, None)       # no table: vnb_generate_many
    cases = [
        (lambda: launch((16, 0)), "outside 1..T"),
        (lambda: launch((17, 5)), "outside 1..T"),
        (lambda: launch((-1, 16)), "outside 1..T"),
        (lambda: launch((16, 5), None), "needs a mask"),
    ]
    for fn, what in cases:
        with pytest.raises(RuntimeError, match=what):
            fn()
    torch.cuda.synchronize()
    launch((4, 16))  # the library still works after the rejections
    torch.cuda.synchronize()
