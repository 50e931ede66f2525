"""GPU: the CUDA beat tracker (vampnet_b200/beats.py, csrc/beat.cu) against the float64 restatement of librosa 0.10.1's
beat_track in oracle/beat_oracle.py, and the beat-synced mask of Interface.make_beat_mask.

The envelope is computed in fp32, so it is compared within ENV_RTOL of its maximum.  Everything after it runs in
float64, so fed the same envelope (vnb_dbg_beat_from_envelope) the kernels take the oracle's decisions exactly: tempo
and beat frames are compared with ==, on inputs whose smallest relative decision margin the test asserts to be far
above float64 rounding.  End to end, beat frames are compared exactly on signals whose smallest relative margin
exceeds twice ENV_RTOL; the test asserts that margin, so a knife-edge signal fails loudly instead of passing by luck."""
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import beat_oracle as bo

pytestmark = pytest.mark.gpu

SR, HOP = 44100, 512
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
# largest |envelope - oracle| allowed, relative to the envelope's maximum (fp32 FFT, mel, dB and flux against float64)
ENV_RTOL = 1e-5  # measured on an H100: at most 1.7e-6 on these signals
# signals compared end to end; bursts_10's smallest margin (1.5e-5, a DP argmax) is too thin for a cross-precision
# comparison, and its decisions are checked exactly from the oracle's envelope instead
END_TO_END = [s for s in bo.SIGNALS if s != "bursts_10"]


def golden(name):
    return np.load(os.path.join(GOLDEN, f"beat_{name}.npz"))


def _track(y, **kw):
    from vampnet_b200.beats import beat_track
    return beat_track(torch.from_numpy(np.ascontiguousarray(y)).cuda(), SR, HOP, **kw)


def _from_envelope(env, sr=SR, hop=HOP, start_bpm=120.0, tightness=100.0, trim=True):
    """vnb_dbg_beat_from_envelope on a (B, F) float32 envelope: (tempo (B,), [beat frames per row])."""
    from vampnet_b200 import _lib
    L = _lib.lib()
    env = torch.as_tensor(np.ascontiguousarray(env, dtype=np.float32)).reshape(-1, np.shape(env)[-1]).cuda()
    B, F = env.shape
    ws_bytes = ctypes.c_uint64(0)
    _lib.check(L.vnb_beat_workspace_bytes(B, (F - 1) * hop + 1, hop, ctypes.byref(ws_bytes)))
    ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device="cuda")
    tempo = torch.empty(B, dtype=torch.float64, device="cuda")
    beats = torch.empty(B, F, dtype=torch.int32, device="cuda")
    counts = torch.empty(B, dtype=torch.int32, device="cuda")
    _lib.check(L.vnb_dbg_beat_from_envelope(_lib.ptr(env), B, F, sr, hop, start_bpm, tightness, int(trim),
                                            _lib.ptr(ws), ws_bytes.value, _lib.ptr(tempo), _lib.ptr(beats),
                                            _lib.ptr(counts), _lib.stream_ptr()))
    counts = counts.cpu()
    return tempo.cpu().numpy(), [beats[b, :int(counts[b])].cpu().numpy() for b in range(B)]


@pytest.mark.parametrize("name", bo.SIGNALS)
def test_envelope_matches_oracle(name):
    y = bo.test_signal(name)
    want = golden(name)["envelope"]
    got = _track(y).envelope[0].cpu().double().numpy()
    assert got.shape == want.shape == (1 + y.shape[0] // HOP,)
    err = np.abs(got - want).max() / max(want.max(), 1e-30)
    assert err <= ENV_RTOL, f"{name}: relative envelope error {err:.3e}"


@pytest.mark.parametrize("name", bo.SIGNALS)
def test_decisions_from_oracle_envelope_are_exact(name):
    g = golden(name)
    env32 = g["envelope"].astype(np.float32)
    want = bo.beat_track_envelope(env32, SR, HOP)
    assert want["margin"] > 1e-9
    tempo, beats = _from_envelope(env32)
    assert tempo[0] == want["tempo"] == float(g["tempo"])
    assert beats[0].tolist() == want["beats"].tolist() == g["beats"].tolist()


def _random_envelope(seed):
    rng = np.random.default_rng(seed)
    F = int(rng.integers(200, 2600))
    env = rng.exponential(0.3, F) * (rng.random(F) < 0.7)
    period, phase = int(rng.integers(22, 80)), int(rng.integers(0, 20))
    env[phase::period] += rng.uniform(1.0, 4.0, len(env[phase::period]))
    env[:3] = 0.0  # the envelope's left padding
    return env.astype(np.float32)


@pytest.mark.parametrize("seed", range(8))
def test_decisions_on_random_envelopes_are_exact(seed):
    env = _random_envelope(seed)
    want = bo.beat_track_envelope(env, SR, HOP)
    assert want["margin"] > 1e-9, want["margin"]
    tempo, beats = _from_envelope(env)
    assert tempo[0] == want["tempo"]
    assert beats[0].tolist() == want["beats"].tolist()


@pytest.mark.parametrize("kw", [dict(trim=False), dict(start_bpm=90.0, tightness=400.0)])
def test_decisions_with_other_arguments(kw):
    env = _random_envelope(11)
    want = bo.beat_track_envelope(env, SR, HOP, **kw)
    assert want["margin"] > 1e-9
    tempo, beats = _from_envelope(env, **kw)
    assert tempo[0] == want["tempo"] and beats[0].tolist() == want["beats"].tolist()


@pytest.mark.parametrize("name", END_TO_END)
def test_end_to_end_beats_match_oracle(name):
    g = golden(name)
    assert float(g["margin"]) > 2 * ENV_RTOL, f"{name}: oracle decision margin {float(g['margin']):.3e} is too thin"
    r = _track(bo.test_signal(name))
    assert float(r.tempo[0]) == float(g["tempo"])
    assert r.frames[0, :int(r.counts[0])].cpu().numpy().tolist() == g["beats"].tolist()


def test_short_clips():
    for n in (1, 300, 2047, 2600):
        y = (0.3 * np.random.default_rng(n).standard_normal(n)).astype(np.float32)
        want = bo.beat_track(y, SR, HOP)
        r = _track(y)
        assert r.envelope.shape == (1, 1 + n // HOP)
        if want["margin"] > 2 * ENV_RTOL:
            assert float(r.tempo[0]) == want["tempo"]
            assert r.frames[0, :int(r.counts[0])].cpu().numpy().tolist() == want["beats"].tolist()


def test_batch_rows_equal_single_rows():
    ys = np.stack([bo.test_signal("bursts_10", seed=s) for s in range(4)])
    ys[2] *= 0.01  # a quieter row: its own dB maximum
    ys[3] = 0.0    # a silent row: tempo 0, no beats
    many = _track(ys)
    for b in range(4):
        one = _track(ys[b])
        assert torch.equal(many.envelope[b], one.envelope[0])
        assert torch.equal(many.tempo[b], one.tempo[0])
        assert int(many.counts[b]) == int(one.counts[0])
        n = int(one.counts[0])
        assert torch.equal(many.frames[b, :n], one.frames[0, :n])
    assert float(many.tempo[3]) == 0.0 and int(many.counts[3]) == 0


def test_tracker_does_not_synchronise():
    """Every launch of the tracker runs without waiting for the device: torch's sync debug mode turns any
    synchronising torch call into an error.  Only reading the times afterwards synchronises."""
    y = torch.from_numpy(bo.test_signal("bursts_4")).cuda()
    from vampnet_b200.beats import beat_track
    beat_track(y, SR, HOP)  # warm: tables, allocator
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        r = beat_track(y, SR, HOP)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert r.frames[0, :int(r.counts[0])].cpu().numpy().tolist() == golden("bursts_4")["beats"].tolist()


def _interface():
    from vampnet_b200.beats import BeatTracker
    from vampnet_b200.interface import Interface
    stub = types.SimpleNamespace(codec=types.SimpleNamespace(sample_rate=SR, hop_length=768), device="cuda",
                                 c2f=types.SimpleNamespace(n_codebooks=14), coarse=None, beat_tracker=BeatTracker("cuda"))
    stub.s2t = lambda s: Interface.s2t(stub, s)
    return stub


@pytest.mark.parametrize("on_cpu", [False, True])
def test_make_beat_mask_equals_assembly_of_tracker_times(on_cpu):
    from vampnet_b200.audio import AudioSignal
    from vampnet_b200.beats import beat_mask
    from vampnet_b200.interface import Interface
    y = bo.test_signal("bursts_10")
    sig = AudioSignal(torch.from_numpy(np.stack([y, 0.5 * y]))[None], SR)  # stereo: the tracker averages channels
    if not on_cpu:
        sig = sig.to("cuda")
    iface = _interface()
    kw = dict(before_beat_s=0.03, after_beat_s=0.05, dropout=0.3, beat_downsample_factor=2)
    beats, downbeats = iface.beat_tracker.extract_beats(sig)
    assert beats.dtype == np.float64 and downbeats.dtype == np.float64 and downbeats.size == 0
    alone = _track(sig.audio_data[0].float().mean(0).cpu().numpy())
    frames = alone.frames[0, :int(alone.counts[0])].cpu().numpy()
    assert len(frames) > 4 and np.array_equal(beats, bo.frames_to_time(frames, SR, HOP))
    torch.manual_seed(3)
    got = Interface.make_beat_mask(iface, sig, **kw)
    got_state = torch.cuda.get_rng_state()
    torch.manual_seed(3)
    want = beat_mask(beats, downbeats, sig.duration, iface.s2t, 14, "cuda", **kw)
    assert got.is_cuda and got.shape == (1, 14, iface.s2t(sig.duration))
    assert torch.equal(got, want) and torch.equal(got_state, torch.cuda.get_rng_state())
    assert (got == 0).any() and (got == 1).any()


def test_snap_to_beats_trims_to_first_and_last_beat():
    from vampnet_b200.audio import AudioSignal
    from vampnet_b200.interface import Interface
    y = bo.test_signal("bursts_4")
    sig = AudioSignal(torch.from_numpy(y)[None, None].cuda(), SR)
    beats = bo.frames_to_time(golden("bursts_4")["beats"], SR, HOP)
    out = Interface.snap_to_beats(_interface(), sig)
    lo, hi = int(beats[0] * SR), int(beats[-1] * SR)
    assert torch.equal(out.samples[0, 0].cpu(), torch.from_numpy(y[lo:hi]))


def test_make_beat_mask_needs_a_cuda_interface():
    iface = _interface()
    iface.device = "cpu"
    from vampnet_b200.interface import Interface
    with pytest.raises(RuntimeError):
        Interface.make_beat_mask(iface)


@pytest.fixture(scope="module")
def cache(tmp_path_factory):
    from tests.dropin_cache import write_cache
    root = tmp_path_factory.mktemp("cache") / "models" / "vampnet"
    write_cache(root)
    old = os.environ.get("VAMPNET_MODELS_DIR")
    os.environ["VAMPNET_MODELS_DIR"] = str(root)
    for k in [k for k in sys.modules if k == "vampnet" or k.startswith("vampnet.")]:
        del sys.modules[k]
    yield root
    if old is None:
        os.environ.pop("VAMPNET_MODELS_DIR", None)
    else:
        os.environ["VAMPNET_MODELS_DIR"] = old


def test_app_follow_beat_sequence(cache):
    """app.py:196-218 with beat_mask_ms = 50: build_mask, mask_and with the beat mask, codebook_mask, then vamp and
    decode, through the vampnet import names."""
    from vampnet import mask as pmask
    from vampnet.interface import AudioSignal, Interface
    interface = Interface.default(device="cuda")
    # 229 code frames: for some lengths (230 frames, say) s2t(duration) rounds up to one frame more than the codes
    # hold, in the reference as here, and mask_and would then refuse the two shapes
    y = bo.test_signal("bursts_4")[:229 * 768]
    sig = interface._preprocess(AudioSignal(torch.from_numpy(y)[None, None], SR).to("cuda"))
    codes = interface.encode(sig)
    mask = interface.build_mask(codes, sig=sig, periodic_prompt=7, onset_mask_width=0, _dropout=0.0,
                                upper_codebook_mask=3)
    beat = interface.make_beat_mask(sig, after_beat_s=0.05)
    assert beat.shape == codes.shape and (beat == 0).any()
    mask = pmask.codebook_mask(pmask.mask_and(mask, beat), 4)
    z = interface.vamp(codes, mask, return_mask=False, _sampling_steps=3, seed=2, temperature=1.0)
    assert z.shape == codes.shape and not (z == 1024).any()
    keep = mask == 0
    assert torch.equal(z[keep], codes[keep])
    out = interface.decode(z)
    assert out.samples.shape[-1] == codes.shape[-1] * 768 and torch.isfinite(out.samples).all()


def test_refusals():
    from vampnet_b200 import _lib
    from vampnet_b200.beats import beat_track
    y = torch.zeros(4000, device="cuda")
    for bad in (lambda: beat_track(y.double(), SR), lambda: beat_track(y.cpu(), SR), lambda: beat_track(y, SR, 0),
                lambda: beat_track(y, SR, -512), lambda: beat_track(torch.zeros(0, 4000, device="cuda"), SR),
                lambda: beat_track(y, 0), lambda: beat_track(y, SR, start_bpm=0.0),
                lambda: beat_track(y, SR, tightness=-1.0), lambda: beat_track(y, SR, 200000),
                lambda: beat_track(torch.zeros(65536, 8, device="cuda"), SR)):
        with pytest.raises(RuntimeError):
            bad()
    L = _lib.lib()
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    out = [torch.empty(64, dtype=t, device="cuda") for t in (torch.float32, torch.float64, torch.int32, torch.int32)]
    args = lambda B, N, s, h, w=ws, nbytes=ws.numel(): (_lib.ptr(y), B, N, s, h, 120.0, 100.0, 1, _lib.ptr(w),  # noqa
                                                        nbytes, *map(_lib.ptr, out), None)
    assert L.vnb_beat_track(*args(1, 0, SR, HOP)) != 0
    assert L.vnb_beat_track(*args(1, 40, SR, HOP, w=None)) != 0
    assert L.vnb_beat_track(*args(1, 4000, SR, HOP, nbytes=16)) != 0
    assert L.vnb_beat_track(*args(1, 4000, SR, 64)) != 0  # an 8 s window of 5512 frames
    need = ctypes.c_uint64(0)
    assert L.vnb_beat_workspace_bytes(0, 4000, HOP, ctypes.byref(need)) != 0
    assert L.vnb_beat_workspace_bytes(1, 4000, 0, ctypes.byref(need)) != 0
    assert L.vnb_beat_workspace_bytes(1, 4000, HOP, None) != 0
    assert L.vnb_dbg_beat_from_envelope(_lib.ptr(out[0]), 1, 0, SR, HOP, 120.0, 100.0, 1, _lib.ptr(ws), ws.numel(),
                                        *map(_lib.ptr, out[1:]), None) != 0
    assert L.vnb_beat_track(*args(1, 4000, SR, HOP)) == 0  # the same call with good arguments goes through
    torch.cuda.synchronize()
