"""GPU: the CUDA onset detector and onset-prompt mask (vampnet_b200/onset.py, csrc/onset.cu) against the float64
restatement of librosa 0.10's onset_detect in oracle/onset_oracle.py.

The kernels compute in fp32, so the envelope is compared within ENV_TOL.  Onset frames are compared exactly, but only
on signals whose smallest decision margin (oracle) exceeds twice ENV_TOL: a decision compares two envelope-derived
quantities, each within ENV_TOL, so such a decision cannot flip.  The test asserts that margin, so a knife-edge
signal fails loudly instead of passing by luck."""
import types

import numpy as np
import pytest
import torch

from oracle import onset_oracle as oo

pytestmark = pytest.mark.gpu

SR, HOP = 44100, 768
# largest |envelope - oracle| allowed on the normalised [0, 1] envelope (fp32 FFT, mel and dB against float64)
ENV_TOL = 5e-6  # measured on an H100: at most 3.5e-7 on these signals


@pytest.fixture(scope="module")
def oracle():
    return {n: oo.onset_detect(oo.test_signal(n), SR, HOP) for n in oo.SIGNALS}


def _detect(y, **kw):
    from vampnet_b200.onset import onset_detect
    return onset_detect(torch.from_numpy(np.ascontiguousarray(y)).cuda(), SR, HOP, **kw)


@pytest.mark.parametrize("name", oo.SIGNALS)
def test_envelope_matches_oracle(oracle, name):
    got = _detect(oo.test_signal(name))
    want = oracle[name]["envelope"]
    env = got.envelope[0].cpu().double().numpy()
    assert env.shape == want.shape == (oo.n_frames(oo.test_signal(name).shape[0], HOP),)
    err = np.abs(env - want).max()
    assert err <= ENV_TOL, f"{name}: envelope error {err:.3e}"


@pytest.mark.parametrize("name", oo.SIGNALS)
def test_onsets_match_oracle(oracle, name):
    want = oracle[name]
    assert want["margin"] > 2 * ENV_TOL, f"{name}: oracle decision margin {want['margin']:.3e} is too thin to test"
    got = _detect(oo.test_signal(name))
    n = int(got.counts[0])
    assert got.frames[0, :n].cpu().numpy().tolist() == want["onsets"].tolist()


def test_onsets_without_backtrack(oracle):
    y = oo.test_signal("bursts")
    env = oracle["bursts"]["envelope"]
    peaks, margin = oo.peak_pick(env, **oo.peak_params(SR, HOP))
    assert margin > 2 * ENV_TOL
    got = _detect(y, backtrack=False)
    assert got.frames[0, :int(got.counts[0])].cpu().numpy().tolist() == peaks.tolist()


def test_silence_and_dc_edge_cases(oracle):
    assert int(_detect(oo.test_signal("silence")).counts[0]) == 0
    assert int(_detect(oo.test_signal("short")).counts[0]) == 0 == len(oracle["short"]["onsets"])
    # shorter than one hop: a single frame, no onsets
    got = _detect(np.full(300, 0.5, dtype=np.float32))
    assert got.envelope.shape == (1, 1) and int(got.counts[0]) == 0


@pytest.mark.parametrize("name", ["clicks", "bursts", "bursts_441600", "dc"])
@pytest.mark.parametrize("width", [0, 1, 2, 5])
def test_masks_match_oracle(oracle, name, width):
    from vampnet_b200.onset import onset_mask
    y = oo.test_signal(name)
    det = _detect(y)
    T = -(-y.shape[0] // HOP)  # codes frames of the clip
    for shape in [(2, 14, T), (1, 4, T - 3)]:
        z = torch.zeros(shape, dtype=torch.int64, device="cuda")
        got = onset_mask(det, z, width).cpu().numpy()
        want = oo.onset_mask(oracle[name]["onsets"], width, shape)
        assert got.dtype == np.int64 and np.array_equal(got, want), (name, width, shape)


def test_batch_rows_equal_single_rows():
    ys = np.stack([oo.test_signal("bursts_441600", seed=s) for s in range(4)])
    ys[2] *= 0.01  # a quieter row: its own dB maximum and normalisation
    many = _detect(ys)
    for b in range(4):
        one = _detect(ys[b])
        assert torch.equal(many.envelope[b], one.envelope[0])
        assert int(many.counts[b]) == int(one.counts[0])
        n = int(one.counts[0])
        assert torch.equal(many.frames[b, :n], one.frames[0, :n])


def _stub_interface():
    from vampnet_b200.interface import Interface
    stub = types.SimpleNamespace(codec=types.SimpleNamespace(sample_rate=SR, hop_length=HOP))
    stub.s2t = lambda s: Interface.s2t(stub, s)
    return stub


def test_build_mask_equals_oracle_onsets_and_rng(oracle, monkeypatch):
    """build_mask(onset_mask_width=w) on a CUDA signal = the same call with the oracle's onsets put through the
    reference's mask loop; the onset step draws no random numbers, so the RNG states match afterwards."""
    from vampnet_b200 import mask as pmask
    from vampnet_b200.audio import AudioSignal
    from vampnet_b200.interface import Interface
    y = oo.test_signal("bursts_441600")
    sig = AudioSignal(torch.from_numpy(y)[None, None].cuda(), SR)
    T = -(-y.shape[0] // HOP)
    z = torch.randint(0, 1024, (2, 14, T), generator=torch.Generator().manual_seed(0)).cuda()
    stub = _stub_interface()
    kw = dict(rand_mask_intensity=0.8, prefix_s=0.5, periodic_prompt=5, onset_mask_width=3, _dropout=0.1,
              upper_codebook_mask=4, ncc=1)

    def run():
        torch.manual_seed(7)
        np.random.seed(7)
        m = Interface.build_mask(stub, z, sig=sig, **kw)
        return m.cpu(), torch.get_rng_state(), torch.cuda.get_rng_state(), np.random.get_state()[1].copy()

    got = run()
    want_onsets = oracle["bursts_441600"]["onsets"]
    monkeypatch.setattr(pmask, "onset_mask", lambda s, zz, iface, width=1: torch.from_numpy(
        oo.onset_mask(want_onsets, width, tuple(zz.shape))).to(zz.device))
    want = run()
    assert torch.equal(got[0], want[0])
    assert torch.equal(got[1], want[1]) and torch.equal(got[2], want[2]) and np.array_equal(got[3], want[3])
    assert (got[0] == 0).any() and (got[0] == 1).any()


def test_onset_step_of_build_mask_does_not_synchronise():
    """The onset layer of build_mask, detection and mask kernels included, runs without waiting for the device:
    torch's sync debug mode turns any synchronising torch call inside it into an error."""
    from vampnet_b200 import mask as pmask
    from vampnet_b200.audio import AudioSignal
    from vampnet_b200.interface import Interface
    y = oo.test_signal("bursts_441600")
    sig = AudioSignal(torch.from_numpy(y)[None, None].cuda(), SR)
    z = torch.zeros(1, 14, -(-y.shape[0] // HOP), dtype=torch.int64, device="cuda")
    stub = _stub_interface()
    Interface.build_mask(stub, z, sig=sig, onset_mask_width=2)  # warm: tables, allocator
    torch.cuda.synchronize()
    orig, seen = pmask.onset_mask, []

    def armed(*a, **k):
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = orig(*a, **k)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        seen.append(out)
        return out

    pmask.onset_mask = armed
    try:
        mask = Interface.build_mask(stub, z, sig=sig, onset_mask_width=2)
    finally:
        pmask.onset_mask = orig
    assert len(seen) == 1 and mask.shape == z.shape and (seen[0] == 0).any()


def test_refusals():
    from vampnet_b200.onset import onset_detect, onset_mask
    y = torch.zeros(4000, device="cuda")
    with pytest.raises(RuntimeError):
        onset_detect(y.double(), SR, HOP)
    with pytest.raises(RuntimeError):
        onset_detect(y.cpu(), SR, HOP)
    with pytest.raises(RuntimeError):
        onset_detect(y, SR, 0)
    with pytest.raises(RuntimeError):
        onset_detect(y, SR, -768)
    with pytest.raises(RuntimeError):
        onset_detect(torch.zeros(0, 4000, device="cuda"), SR, HOP)
    with pytest.raises(RuntimeError):
        onset_detect(y, 0, HOP)
    det = onset_detect(torch.zeros(3, 4000, device="cuda"), SR, HOP)
    with pytest.raises(RuntimeError):  # three onset rows for a batch of two
        onset_mask(det, torch.zeros(2, 4, 6, dtype=torch.int64, device="cuda"), 1)
