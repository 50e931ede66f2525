"""GPU: VampNet.generate_many(mixed_top_p=True) — nucleus (top-p) and plain-sampling calls in one
vnb_generate_mixed_top_p launch — equals the same calls made one by one, bit for bit, and leaves the global RNGs where
the sequential calls leave them.

With the fused sampler, such a launch runs the split classifier epilogue: the plain rows leave records and draw in the
combine, the nucleus rows store their logits and draw in the nucleus kernel.  Without it, every row draws in the
nucleus kernel from materialised logits.  Calls of one row at T = 40 alternate top-p on and off, so the 128-row tiles
of the classifier hold rows of both kinds; top_p 0, 1.0 and None are all "off"."""
import ctypes

import pytest
import torch

from tests.test_gpu_adapters import base_with_adapters
from tests.test_gpu_generate_many import FULL_COARSE, assert_same_rng, reseed_globals, rng_state, set_fused
from tests.test_gpu_generate_ragged import assert_all_equal
from tests.test_gpu_generate_steps import steps_mix
from tests.test_gpu_parity import TINY_C2F, TINY_COARSE, build

pytestmark = pytest.mark.gpu

ENTRIES = ("vnb_generate_many", "vnb_generate_many_adapted", "vnb_generate_ragged", "vnb_generate_steps",
           "vnb_generate_mixed_top_p")


class spy_launches:
    """Records (entry point, B, T, top-p on per group) of every generate launch while installed."""

    def __init__(self, seen):
        from vampnet_b200 import _lib as L
        self.L, self.real, self.seen = L, L.lib, seen

    def __enter__(self):
        lib, seen = self.real(), self.seen

        class Spy:
            def __getattr__(self, name):
                fn = getattr(lib, name)
                if name not in ENTRIES:
                    return fn

                def rec(*a):
                    groups, n = a[7], a[8]
                    seen.append((name, a[3], a[4], tuple(0.0 < groups[g].top_p < 1.0 for g in range(n))))
                    return fn(*a)
                return rec
        self.L.lib = lambda: Spy()
        return self

    def __exit__(self, *exc):
        self.L.lib = self.real


def top_p_mix(cfg, seed, n=10, T=40, steps=6, adapters=()):
    """Calls of one row (two for every fourth) at T frames: top_p cycling through 0.8, None, 0.9, 0, 1.0; greedy,
    sampled and cutoff schedules; seeds given and not; masks of both shapes and none."""
    g = torch.Generator().manual_seed(seed)
    C = cfg["n_codebooks"]
    out = []
    for i in range(n):
        B = 2 if i % 4 == 3 else 1
        c = dict(start_tokens=torch.randint(0, 1024, (B, C, T), generator=g).cuda(), _sampling_steps=steps,
                 top_p=(0.8, None, 0.9, 0.0, 1.0)[i % 5], sample_cutoff=(1.0, -1.0, 0.5)[i % 3],
                 temperature=(1.0, 0.7)[i % 2], return_signal=False)
        if i % 3 == 0:
            c["mask"] = (torch.rand(B, C, T, generator=g) < 0.6).long().cuda()
        elif i % 3 == 1:
            c["mask"] = (torch.rand(B, T, generator=g) < 0.5).long().cuda()
        if i % 2 == 0:
            c["seed"] = 40 + i
        if adapters and adapters[i % len(adapters)] is not None:
            c["adapter"] = adapters[i % len(adapters)]
        out.append(c)
    return out


def sequential_and_mixed(model, codec, calls, rng_seed, **kw):
    reseed_globals(rng_seed)
    want = [model.generate(codec, **c) for c in calls]
    want_rng = rng_state()
    reseed_globals(rng_seed)
    got = model.generate_many(codec, calls, mixed_top_p=True, **kw)
    return want, want_rng, got, rng_state()


@pytest.mark.parametrize("fused", [1, 0])
@pytest.mark.parametrize("tag,cfgd,lora", [("coarse", TINY_COARSE, False), ("c2f", TINY_C2F, False),
                                           ("coarse_lora", TINY_COARSE, True)])
def test_mixed_top_p_equal_sequential_calls(tag, cfgd, lora, fused):
    _, _, model, _, codec = build(cfgd, lora=lora)
    prev = set_fused(fused)
    seen = []
    try:
        with spy_launches(seen):
            want, want_rng, got, got_rng = sequential_and_mixed(model, codec, top_p_mix(cfgd, seed=21), rng_seed=7)
    finally:
        set_fused(prev)
    assert_all_equal(got, want, f"{tag} fused={fused}")
    assert_same_rng(got_rng, want_rng)
    batched = [s for s in seen if s[0] == "vnb_generate_mixed_top_p"]
    assert len(batched) == 1 and batched[0][1:3] == (12, 40), seen
    assert batched[0][3] == (True, False, True, False, False, True, False, True, False, False), batched


@pytest.mark.parametrize("fused", [1, 0])
@pytest.mark.parametrize("tag,cfgd", [("coarse", TINY_COARSE), ("c2f", TINY_C2F)])
def test_mixed_top_p_with_steps_lengths_and_adapters(tag, cfgd, fused):
    """Adapters, mixed lengths, mixed steps and mixed top-p in the same launches."""
    _, _, model, _, codec = base_with_adapters(cfgd, seed=2)
    prev = set_fused(fused)
    seen = []
    try:
        calls = steps_mix(cfgd, seed=19, adapters=(None, "ft0", "ft1"), lengths=True)
        with spy_launches(seen):
            want, want_rng, got, got_rng = sequential_and_mixed(model, codec, calls, rng_seed=5, mixed_lengths=True,
                                                                mixed_steps=True)
        calls = top_p_mix(cfgd, seed=22, adapters=("ft1", None, "ft0"))
        want2, want_rng2, got2, got_rng2 = sequential_and_mixed(model, codec, calls, rng_seed=6)
    finally:
        set_fused(prev)
    assert_all_equal(got, want, tag + " adapters + lengths + steps")
    assert_same_rng(got_rng, want_rng)
    # the sequential calls are one-call launches; the batched calls are one launch
    assert [s[0] for s in seen if s[0] not in ("vnb_generate_many", "vnb_generate_many_adapted")] == \
        ["vnb_generate_mixed_top_p"], seen
    assert_all_equal(got2, want2, tag + " adapters")
    assert_same_rng(got_rng2, want_rng2)


def test_full_size_coarse_app_shapes():
    """The 20-layer d = 1280 coarse model: B = 2 calls of a 10 s chunk (575 frames) and a remainder, top-p 0.9 / 0.8
    next to plain ones, in one launch."""
    _, _, model, _, codec = build(FULL_COARSE)
    g = torch.Generator().manual_seed(9)
    calls = []
    for i, (T, tp) in enumerate(zip((575, 575, 575, 271), (0.9, None, 0.8, None))):
        z = torch.randint(0, 1024, (2, 4, T), generator=g).cuda()
        mask = (torch.rand(2, 4, T, generator=g) < 0.7).long().cuda()
        calls.append(dict(start_tokens=z, mask=mask, _sampling_steps=12, return_signal=False, top_p=tp,
                          seed=None if i % 3 else 100 + i, temperature=1.0 if i % 2 else 0.8))
    seen = []
    with spy_launches(seen):
        want, want_rng, got, got_rng = sequential_and_mixed(model, codec, calls, rng_seed=9, mixed_lengths=True)
    assert [s for s in seen if s[0] == "vnb_generate_mixed_top_p"] == \
        [("vnb_generate_mixed_top_p", 8, 575, (True, False, True, False))], seen
    assert_all_equal(got, want, "full coarse")
    assert_same_rng(got_rng, want_rng)


def test_new_top_p_assignment_on_a_captured_workspace_needs_no_capture():
    """The group -> top-p assignment is read from the per-step table written before every replay: a second launch on
    the same (B, T, S) workspace with another assignment replays the captured graph and is still bit-identical."""
    from vampnet_b200 import _lib as L
    _, _, model, _, codec = build(TINY_COARSE)
    g = torch.Generator().manual_seed(6)

    def calls(tps, seeds):
        return [dict(start_tokens=torch.randint(0, 1024, (1, 4, 48), generator=g).cuda(),
                     mask=(torch.rand(1, 4, 48, generator=g) < 0.6).long().cuda(), seed=s, _sampling_steps=5,
                     top_p=tp, return_signal=False) for tp, s in zip(tps, seeds)]
    model.generate_many(codec, calls([0.9, None, None], [1, None, 2]), mixed_top_p=True)
    second = calls([None, 0.85, 0.7], [None, 9, 10])
    before = L.lib().vnb_graph_capture_count()
    reseed_globals(77)
    got = model.generate_many(codec, second, mixed_top_p=True)
    assert L.lib().vnb_graph_capture_count() == before, "a new top-p assignment captured a new graph"
    got_rng = rng_state()
    reseed_globals(77)
    assert_all_equal(got, [model.generate(codec, **c) for c in second], "replay")
    assert_same_rng(got_rng, rng_state())


def test_mixed_top_p_refusals():
    """vnb_generate_mixed_top_p refuses what vnb_generate_steps refuses, except a mix of top-p on and off."""
    from vampnet_b200 import _lib as L
    _, _, model, _, codec = build(TINY_COARSE)
    model._ensure_handle(codec)
    B, T = 3, 16
    z = torch.randint(0, 1024, (B, 4, T)).cuda()
    mask = torch.zeros(B, 4, T, dtype=torch.int32).cuda()
    mask[:, :, :4] = 1
    out = torch.empty_like(z)
    keep = []

    def launch(steps, gammas="ok", frames=None, m=mask, top_p=(0.9, 0.0), n_groups=2, rows=(1, 2)):
        arr = (L.GenGroup * 2)()
        for gr, r, n, tp in zip(arr, rows, steps, top_p):
            n_arr = max(n, 1)
            tef = (ctypes.c_float * n_arr)(*([1.0] * n_arr))
            dos = (ctypes.c_int32 * n_arr)(*([1] * n_arr))
            keep.extend([tef, dos])
            gr.rows, gr.temperature, gr.temp_eff, gr.do_sample, gr.seed_lo, gr.seed_hi, gr.top_p = r, 1.0, tef, dos, 1, 0, tp
        gam = [(ctypes.c_float * max(n, 1))(*([0.5] * max(n, 1))) for n in steps]
        keep.extend(gam)
        ptrs = None
        if gammas is not None:
            ptrs = (ctypes.POINTER(ctypes.c_float) * 2)(*[ctypes.cast(a, ctypes.POINTER(ctypes.c_float)) for a in gam])
            if gammas == "null_entry":
                ptrs[1] = ctypes.POINTER(ctypes.c_float)()
        st = (ctypes.c_int32 * 2)(*steps)
        fr = None if frames is None else (ctypes.c_int32 * 2)(*frames)
        with torch.cuda.device(model.device):
            L.check(L.lib().vnb_generate_mixed_top_p(model._handle, L.ptr(z), L.ptr(m), B, T, st, ptrs, arr, n_groups,
                                                     fr, None, 0, L.ptr(out), L.stream_ptr(model.device)))
    launch((5, 2))                               # a mix: accepted
    launch((3, 3), top_p=(0.0, 1.0), m=None)     # no group on, default mask
    launch((4, 4), top_p=(0.5, 0.99))            # every group on
    launch((4, 1), frames=(16, 7))               # with lengths
    cases = [
        (lambda: launch((2, 5)), "non-increasing"),
        (lambda: launch((0, 0)), "outside 1..256"),
        (lambda: launch((257, 3)), "outside 1..256"),
        (lambda: launch((3, 2), gammas=None), "required"),
        (lambda: launch((3, 2), gammas="null_entry"), "lacks its schedules"),
        (lambda: launch((3, 2), frames=(16, 17)), "outside 1..T"),
        (lambda: launch((3, 2), frames=(16, 5), m=None), "needs a mask"),
        (lambda: launch((3, 2), rows=(1, 1)), "sum to"),
        (lambda: launch((3, 2), n_groups=4), "out of range"),
    ]
    for fn, what in cases:
        with pytest.raises(RuntimeError, match=what):
            fn()
    torch.cuda.synchronize()
    launch((6, 1))  # the library still works after the refusals
    torch.cuda.synchronize()
