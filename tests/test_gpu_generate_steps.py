"""GPU: VampNet.generate_many(mixed_steps=True) — calls of different sampling-step counts in one vnb_generate_steps
launch — equals the same calls made one by one, bit for bit, and leaves the global RNGs where the sequential calls
leave them.

A launch runs as many iterations as its longest call.  A call of fewer steps is idle until its own steps fill the
launch's last iterations: its state is not touched, and then every step uses the call's own gamma, temperatures,
sampling flag, Philox step word and last-step flag.  The step counts cover 1 (live only on the last iteration), 2, 3,
7 and 12; sample cutoffs 1, 0.5 and -1 flip the sampling flag at different steps per call."""
import ctypes

import pytest
import torch

from tests.test_gpu_adapters import base_with_adapters
from tests.test_gpu_generate_many import FULL_COARSE, assert_same_rng, reseed_globals, rng_state, set_fused
from tests.test_gpu_generate_ragged import assert_all_equal
from tests.test_gpu_parity import TINY_C2F, TINY_COARSE, build

pytestmark = pytest.mark.gpu


def steps_mix(cfg, seed, adapters=(), lengths=False):
    """Calls of 1, 2, 3, 7 and 12 steps, B in {1, 2, 3}, seeds given and not, two temperatures, mask temperatures 10.5
    and 0, sample cutoffs 1, 0.5 and -1, 3-D, 2-D and absent masks; a top-p bucket of mixed steps.  lengths: the calls
    also have different T (a mask on every call, as mixed lengths need)."""
    g = torch.Generator().manual_seed(seed)
    C = cfg["n_codebooks"]

    def z(B, T):
        return torch.randint(0, 1024, (B, C, T), generator=g).cuda()

    def m3(B, T):
        return (torch.rand(B, C, T, generator=g) < 0.6).long().cuda()

    def m2(B, T):
        return (torch.rand(B, T, generator=g) < 0.5).long().cuda()

    def T_(t):
        return t if lengths else 40

    out = [
        dict(start_tokens=z(2, T_(40)), mask=m3(2, T_(40)), seed=11, _sampling_steps=7, mask_temperature=10.5),
        dict(start_tokens=z(1, T_(65)), mask=m2(1, T_(65)), temperature=0.7, mask_temperature=0.0, sample_cutoff=0.5,
             _sampling_steps=12),
        dict(start_tokens=z(3, T_(40)), mask=None if not lengths else m3(3, T_(40)), sample_cutoff=-1.0,
             _sampling_steps=1),
        dict(start_tokens=z(1, T_(1)), mask=m3(1, T_(1)), seed=5, temperature=0.7, _sampling_steps=3),
        dict(start_tokens=z(2, T_(64)), mask=m2(2, T_(64)), mask_temperature=0.0, sample_cutoff=0.5,
             _sampling_steps=2),
        dict(start_tokens=z(1, T_(40)), mask=None if not lengths else m2(1, T_(40)), _sampling_steps=12, seed=4),
        dict(start_tokens=z(1, T_(129)), mask=m3(1, T_(129)), seed=6, _sampling_steps=7, sample_cutoff=0.5),
        dict(start_tokens=z(2, T_(40)), mask=m3(2, T_(40)), top_p=0.9, _sampling_steps=7),
        dict(start_tokens=z(1, T_(65)), mask=m2(1, T_(65)), top_p=0.8, seed=3, temperature=0.7, _sampling_steps=2),
        dict(start_tokens=z(1, T_(40)), mask=m3(1, T_(40)), top_p=0.85, _sampling_steps=12, sample_cutoff=-1.0),
        dict(start_tokens=z(2, T_(1)), mask=m3(2, T_(1)), _sampling_steps=1, seed=9, temperature=1.3),
    ]
    for i, c in enumerate(out):
        c["return_signal"] = False
        if adapters and adapters[i % len(adapters)] is not None:
            c["adapter"] = adapters[i % len(adapters)]
    return out


def sequential_and_mixed(model, codec, calls, rng_seed, **kw):
    reseed_globals(rng_seed)
    want = [model.generate(codec, **c) for c in calls]
    want_rng = rng_state()
    reseed_globals(rng_seed)
    got = model.generate_many(codec, calls, mixed_steps=True, **kw)
    return want, want_rng, got, rng_state()


class spy_launches:
    """Records (entry point, B, T, steps per group, rows per group) of every generate launch while installed."""
    NAMES = ("vnb_generate_many", "vnb_generate_many_adapted", "vnb_generate_ragged", "vnb_generate_steps")

    def __init__(self, seen):
        from vampnet_b200 import _lib as L
        self.L, self.real, self.seen = L, L.lib, seen

    def __enter__(self):
        lib, seen = self.real(), self.seen

        class Spy:
            def __getattr__(self, name):
                fn = getattr(lib, name)
                if name not in spy_launches.NAMES:
                    return fn

                def rec(*a):
                    if name == "vnb_generate_steps":
                        n = a[8]
                        seen.append((name, a[3], a[4], tuple(a[5][:n]), tuple(a[7][g].rows for g in range(n))))
                    else:
                        n = a[8]
                        seen.append((name, a[3], a[4], (a[5],) * n, tuple(a[7][g].rows for g in range(n))))
                    return fn(*a)
                return rec
        self.L.lib = lambda: Spy()
        return self

    def __exit__(self, *exc):
        self.L.lib = self.real


@pytest.mark.parametrize("fused", [1, 0])
@pytest.mark.parametrize("tag,cfgd,lora", [("coarse", TINY_COARSE, False), ("c2f", TINY_C2F, False),
                                           ("coarse_lora", TINY_COARSE, True)])
def test_mixed_steps_equal_sequential_calls(tag, cfgd, lora, fused):
    _, _, model, _, codec = build(cfgd, lora=lora)
    prev = set_fused(fused)
    seen = []
    try:
        with spy_launches(seen):
            want, want_rng, got, got_rng = sequential_and_mixed(model, codec, steps_mix(cfgd, seed=31), rng_seed=123)
    finally:
        set_fused(prev)
    assert_all_equal(got, want, tag)
    assert_same_rng(got_rng, want_rng)
    # the batched part: one launch per top-p state, longest calls first
    batched = [s for s in seen if s[0] == "vnb_generate_steps"]
    assert [s[3] for s in batched] == [(12, 12, 7, 7, 3, 2, 1, 1), (12, 7, 2)], batched


@pytest.mark.parametrize("fused", [1, 0])
@pytest.mark.parametrize("tag,cfgd", [("coarse", TINY_COARSE), ("c2f", TINY_C2F)])
def test_mixed_steps_with_adapters_and_lengths(tag, cfgd, fused):
    """Adapters, mixed lengths and mixed steps in the same launches."""
    _, _, model, _, codec = base_with_adapters(cfgd, seed=2)
    prev = set_fused(fused)
    try:
        calls = steps_mix(cfgd, seed=17, adapters=(None, "ft0", "ft1"), lengths=True)
        want, want_rng, got, got_rng = sequential_and_mixed(model, codec, calls, rng_seed=5, mixed_lengths=True)
        calls = steps_mix(cfgd, seed=18, adapters=("ft1", None))
        want2, want_rng2, got2, got_rng2 = sequential_and_mixed(model, codec, calls, rng_seed=6)
    finally:
        set_fused(prev)
    assert_all_equal(got, want, tag + " adapters + lengths")
    assert_same_rng(got_rng, want_rng)
    assert_all_equal(got2, want2, tag + " adapters")
    assert_same_rng(got_rng2, want_rng2)


@pytest.mark.parametrize("lengths", [False, True], ids=["T575", "mixed_lengths"])
def test_full_size_coarse_app_shapes(lengths):
    """The 20-layer d = 1280 coarse model: B = 2 calls of a 10 s chunk (575 frames) with 12, 24, 36 and 48 steps, and
    the same with three remainder lengths mixed in."""
    _, _, model, _, codec = build(FULL_COARSE)
    g = torch.Generator().manual_seed(8)
    calls = []
    for i, (T, steps) in enumerate(zip((575, 502, 271, 133) if lengths else (575,) * 4, (12, 24, 36, 48))):
        z = torch.randint(0, 1024, (2, 4, T), generator=g).cuda()
        mask = (torch.rand(2, 4, T, generator=g) < 0.7).long().cuda()
        calls.append(dict(start_tokens=z, mask=mask, _sampling_steps=steps, return_signal=False,
                          seed=None if i % 3 else 100 + i, temperature=1.0 if i % 2 else 0.8))
    seen = []
    with spy_launches(seen):
        want, want_rng, got, got_rng = sequential_and_mixed(model, codec, calls, rng_seed=9, mixed_lengths=lengths)
    assert [s for s in seen if s[0] == "vnb_generate_steps"] == \
        [("vnb_generate_steps", 8, 575, (48, 36, 24, 12), (2, 2, 2, 2))], seen
    assert_all_equal(got, want, "full coarse")
    assert_same_rng(got_rng, want_rng)


def test_mixed_steps_launch_grouping(monkeypatch):
    """Different steps with the same top-p state are one launch at S = max, longest steps first (stable); top-p on and
    off stay separate launches; a launch still splits where rows x T would pass MANY_MAX_ROWS."""
    from vampnet_b200.modules import transformer as TR
    _, _, model, _, codec = build(TINY_COARSE)
    g = torch.Generator().manual_seed(3)
    spec = [(1, 2, None), (2, 5, None), (1, 5, 0.9), (1, 1, None), (2, 9, None), (1, 3, 0.9), (1, 5, None)]
    calls = [dict(start_tokens=torch.randint(0, 1024, (B, 4, 50), generator=g).cuda(), _sampling_steps=s, top_p=tp,
                  return_signal=False, seed=i) for i, (B, s, tp) in enumerate(spec)]
    seen = []
    with spy_launches(seen):
        model.generate_many(codec, calls, mixed_steps=True)
    assert seen == [("vnb_generate_steps", 7, 50, (9, 5, 5, 2, 1), (2, 2, 1, 1, 1)),
                    ("vnb_generate_steps", 2, 50, (5, 3), (1, 1))], seen
    seen.clear()
    monkeypatch.setattr(TR, "MANY_MAX_ROWS", 200)
    with spy_launches(seen):
        reseed_globals(4)
        got = model.generate_many(codec, calls, mixed_steps=True)
    # list order packs calls 0, 1, 3 (4 rows x 50 = 200); call 4 would make 300: [4, 6] is the next launch; each launch
    # is then ordered longest first
    assert seen == [("vnb_generate_steps", 4, 50, (5, 2, 1), (2, 1, 1)),
                    ("vnb_generate_steps", 3, 50, (9, 5), (2, 1)),
                    ("vnb_generate_steps", 2, 50, (5, 3), (1, 1))], seen
    reseed_globals(4)
    assert_all_equal(got, [model.generate(codec, **c) for c in calls], "split launch")


def test_new_step_counts_on_a_captured_workspace_need_no_capture():
    """The live table and the schedules are written before every replay: a second launch on the same (B, T, S)
    workspace with other step counts in another order replays the captured graph and is still bit-identical."""
    from vampnet_b200 import _lib as L
    _, _, model, _, codec = build(TINY_COARSE)
    g = torch.Generator().manual_seed(6)

    def calls(steps, seeds):
        return [dict(start_tokens=torch.randint(0, 1024, (1, 4, 48), generator=g).cuda(),
                     mask=(torch.rand(1, 4, 48, generator=g) < 0.6).long().cuda(), seed=s, _sampling_steps=n,
                     return_signal=False) for n, s in zip(steps, seeds)]
    model.generate_many(codec, calls([8, 2, 5], [1, None, 2]), mixed_steps=True)
    second = calls([1, 8, 6], [None, 9, 10])
    before = L.lib().vnb_graph_capture_count()
    reseed_globals(77)
    got = model.generate_many(codec, second, mixed_steps=True)
    assert L.lib().vnb_graph_capture_count() == before, "new step counts captured a new graph"
    got_rng = rng_state()
    reseed_globals(77)
    assert_all_equal(got, [model.generate(codec, **c) for c in second], "replay")
    assert_same_rng(got_rng, rng_state())


def test_steps_refusals():
    from vampnet_b200 import _lib as L
    _, _, model, _, codec = build(TINY_COARSE)
    model._ensure_handle(codec)
    B, T = 3, 16
    z = torch.randint(0, 1024, (B, 4, T)).cuda()
    mask = torch.zeros(B, 4, T, dtype=torch.int32).cuda()
    mask[:, :, :4] = 1
    out = torch.empty_like(z)
    keep = []

    def launch(steps, gammas="ok", frames=None, m=mask, top_p=(0.0, 0.0)):
        arr = (L.GenGroup * 2)()
        for gr, rows, n, tp in zip(arr, (1, 2), steps, top_p):
            n_arr = max(n, 1)
            tef = (ctypes.c_float * n_arr)(*([1.0] * n_arr))
            dos = (ctypes.c_int32 * n_arr)(*([1] * n_arr))
            keep.extend([tef, dos])
            gr.rows, gr.temperature, gr.temp_eff, gr.do_sample, gr.seed_lo, gr.seed_hi, gr.top_p = rows, 1.0, tef, dos, 1, 0, tp
        gam = [(ctypes.c_float * max(n, 1))(*([0.5] * max(n, 1))) for n in steps]
        keep.extend(gam)
        ptrs = None
        if gammas is not None:
            ptrs = (ctypes.POINTER(ctypes.c_float) * 2)(*[ctypes.cast(a, ctypes.POINTER(ctypes.c_float)) for a in gam])
            if gammas == "null_entry":
                ptrs[1] = ctypes.POINTER(ctypes.c_float)()
        st = None if steps is None else (ctypes.c_int32 * 2)(*steps)
        fr = None if frames is None else (ctypes.c_int32 * 2)(*frames)
        with torch.cuda.device(model.device):
            L.check(L.lib().vnb_generate_steps(model._handle, L.ptr(z), L.ptr(m), B, T, st, ptrs, arr, 2, fr, None, 0,
                                               L.ptr(out), L.stream_ptr(model.device)))
    launch((5, 2))                       # well formed
    launch((3, 3), m=None)               # equal steps: the plain launch, default mask allowed
    launch((4, 1), frames=(16, 7))       # with lengths
    cases = [
        (lambda: launch((2, 5)), "non-increasing"),
        (lambda: launch((0, 0)), "outside 1..256"),
        (lambda: launch((257, 3)), "outside 1..256"),
        (lambda: launch((3, -1)), "outside 1..256"),
        (lambda: launch((3, 2), gammas=None), "required"),
        (lambda: launch((3, 2), gammas="null_entry"), "lacks its schedules"),
        (lambda: launch((3, 2), frames=(16, 17)), "outside 1..T"),
        (lambda: launch((3, 2), frames=(16, 5), m=None), "needs a mask"),
        (lambda: launch((3, 2), top_p=(0.9, 0.0)), "mix top-p"),
    ]
    for fn, what in cases:
        with pytest.raises(RuntimeError, match=what):
            fn()
    with pytest.raises(RuntimeError, match="required"):
        with torch.cuda.device(model.device):
            L.check(L.lib().vnb_generate_steps(model._handle, L.ptr(z), L.ptr(mask), B, T, None, None, None, 2, None,
                                               None, 0, L.ptr(out), L.stream_ptr(model.device)))
    torch.cuda.synchronize()
    launch((6, 1))  # the library still works after the refusals
    torch.cuda.synchronize()
