"""CPU: the experiment script's registry (vampnet_b200.experiment), the CoarseCond mask against the ORIGINAL project's
vampnet/mask.py (tests/golden/reference_experiment_masks.npz, written by oracle/gen_experiment_golden.py), the excerpt
rule, the refusal of unreadable --ext values and the sampling_steps -> _sampling_steps mapping."""
import os
import random
import types
import wave

import numpy as np
import pytest
import torch

from oracle.gen_experiment_golden import CASES, codes
from vampnet_b200 import experiment as ex
from vampnet_b200.audio import AudioSignal


def test_registry_names_and_order():
    assert list(ex.EXP_REGISTRY) == ["gen-compression", "sampling-steps", "musical-sampling"]
    assert list(ex.EXP_REGISTRY["gen-compression"]) == [
        "baseline", "reconstructed", "coarse2fine", "1_codebooks_downsampled_1x", "4_codebooks_downsampled_4x",
        "4_codebooks_downsampled_16x", "4_codebooks_downsampled_32x", "token_noise_0.25", "token_noise_0.5",
        "token_noise_0.75"]
    assert list(ex.EXP_REGISTRY["sampling-steps"]) == [f"steps_{n}" for n in (1, 4, 12, 36, 64, 72)]
    assert list(ex.EXP_REGISTRY["musical-sampling"]) == ["beat_mask_0.075", "inpaint_0.5", "inpaint_1.0"]
    with pytest.raises(ValueError, match="Unknown exp_type"):
        ex.conditions("codec")


def test_plans_follow_the_conditions():
    """What run_experiment runs per condition: stages, generate arguments and codes."""
    gc = ex.EXP_REGISTRY["gen-compression"]
    assert gc["baseline"].plan is None
    assert gc["reconstructed"].plan.mask is None and not gc["reconstructed"].plan.fine
    assert gc["coarse2fine"].plan.mask is None and gc["coarse2fine"].plan.fine
    iface = types.SimpleNamespace(c2f=types.SimpleNamespace(n_conditioning_codebooks=4))
    assert gc["coarse2fine"].plan.codes(torch.zeros(1, 14, 5), iface).shape == (1, 4, 5)
    for n, x in ((1, 1), (4, 4), (4, 16), (4, 32)):
        p = gc[f"{n}_codebooks_downsampled_{x}x"].plan
        assert p.mask is not None and p.coarse == {} and p.fine
    for r in (0.25, 0.5, 0.75):
        p = gc[f"token_noise_{r}"].plan
        assert p.coarse == {"_sampling_steps": 1} and not p.fine
    for name, p in ((k, c.plan) for k, c in ex.EXP_REGISTRY["musical-sampling"].items()):
        assert p.coarse == {} and p.fine, name


def test_sampling_steps_is_generates_private_argument():
    assert ex.generate_kwargs(sampling_steps=4) == {"_sampling_steps": 4}
    assert ex.generate_kwargs(temperature=0.5) == {"temperature": 0.5}
    for n in (1, 4, 12, 36, 64, 72):
        p = ex.EXP_REGISTRY["sampling-steps"][f"steps_{n}"].plan
        assert p.coarse == {"_sampling_steps": n} and p.fine


def test_coarse_cond_mask_matches_reference():
    """CoarseCond's codebook_unmask is discarded by the periodic_mask after it (a fresh full mask): the mask, and the
    torch CPU generator's position afterwards, are the reference's."""
    golden = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_experiment_masks.npz"))
    for c, (kind, n, x, T, seed) in enumerate(CASES):
        z = codes(T)
        torch.manual_seed(seed)
        if kind == "coarse_cond":
            got = ex.EXP_REGISTRY["gen-compression"][f"{n}_codebooks_downsampled_{x}x"].mask(z)
        else:
            got = ex.EXP_REGISTRY["sampling-steps"]["steps_4"].plan.mask(None, z, None)
        nxt = torch.rand(4)
        assert got.dtype == torch.long
        assert torch.equal(got, torch.from_numpy(golden[f"mask{c}"]).long()), f"case {c}"
        assert torch.equal(nxt, torch.from_numpy(golden[f"next{c}"])), f"case {c}: RNG position"
        if kind == "coarse_cond":  # the conditioning codebooks are masked like every other codebook
            assert torch.equal(got[:, :n], got[:, n:n + n])


def test_coarse_cond_mask_matches_live_reference():
    from oracle import ref_shims
    if not ref_shims.available():
        pytest.skip("no checkout of the original project (VAMPNET_REFERENCE_ROOT)")
    _, rm, _ = ref_shims.load_reference()
    try:
        for n, x in ((1, 1), (4, 4), (4, 16), (4, 32)):
            z = codes(101)
            torch.manual_seed(5)
            want = rm.periodic_mask(rm.codebook_unmask(rm.full_mask(z), n), x)
            torch.manual_seed(5)
            assert torch.equal(ex.EXP_REGISTRY["gen-compression"][f"{n}_codebooks_downsampled_{x}x"].mask(z), want)
    finally:
        ref_shims.uninstall()


# ------------------------------------------------------------------------------------------------ excerpts
def _write_wav(path, data, sr):
    data = np.atleast_2d(data)
    pcm = (np.clip(data, -1, 1).T * 32767).astype("<i2")
    with wave.open(str(path), "wb") as w:
        w.setnchannels(data.shape[0])
        w.setsampwidth(2)
        w.setframerate(sr)
        w.writeframes(pcm.tobytes())


@pytest.fixture()
def sources(tmp_path):
    g = np.random.default_rng(0)
    d = tmp_path / "src"
    (d / "sub").mkdir(parents=True)
    quiet_then_loud = np.concatenate([np.zeros(16000), 0.3 * g.standard_normal(16000)])
    _write_wav(d / "a.wav", quiet_then_loud, 8000)
    _write_wav(d / "sub" / "b.wav", 0.2 * g.standard_normal((2, 40000)), 16000)    # stereo, resampled
    _write_wav(d / "c.wav", 0.3 * g.standard_normal(1500), 8000)                    # shorter than an excerpt
    _write_wav(d / "d.wav", np.zeros(20000), 8000)                                  # silent: no candidate passes
    (d / "e.mp3").write_bytes(b"not read")
    single = tmp_path / "f.wav"
    _write_wav(single, 0.1 * g.standard_normal(30000), 8000)
    return [str(d), str(single)]


def rng_state():
    return random.getstate(), np.random.get_state()[1].copy(), torch.get_rng_state()


def test_find_files_sorted_wav_only(sources):
    files = ex.find_files(sources, [".wav"])
    assert [f.name for f in files] == ["f.wav", "a.wav", "c.wav", "d.wav", "b.wav"]
    assert files == sorted(files, key=str)


def test_non_wav_ext_is_refused(sources):
    with pytest.raises(ValueError, match="only .wav"):
        ex.find_files(sources, [".mp3"])
    with pytest.raises(ValueError, match="only .wav"):
        ex.find_files(sources, [".wav", ".flac"])
    with pytest.raises(ValueError, match="only .wav"):  # before any model is loaded
        ex.main(["--sources", *sources, "--ext", ".mp3"])


def test_excerpt_rule(sources):
    files = ex.find_files(sources)
    dur, sr, seed = 0.5, 8000, 3
    idx = list(range(12))
    torch.manual_seed(1)
    np.random.seed(1)
    random.seed(1)
    before = rng_state()
    whole = ex.load_excerpts(files, idx, dur, sr, seed, device="cpu")
    after = rng_state()
    assert before[0] == after[0] and np.array_equal(before[1], after[1]) and torch.equal(before[2], after[2])
    again = ex.load_excerpts(files, idx, dur, sr, seed, device="cpu")
    blocks = [s for lo in range(0, 12, 5) for s in ex.load_excerpts(files, idx[lo:lo + 5], dur, sr, seed, device="cpu")]
    one = [ex.load_excerpts(files, [i], dur, sr, seed, device="cpu")[0] for i in reversed(idx)][::-1]
    for k, s in enumerate(whole):
        assert s.audio_data.shape == (1, 1, 4000) and s.sample_rate == sr
        for other in (again, blocks, one):
            assert torch.equal(s.audio_data, other[k].audio_data), f"excerpt {k}"

    # the rule, restated per excerpt
    order = list(files)
    np.random.RandomState(seed).shuffle(order)
    for i in idx:
        data, fsr = ex._read_wav(str(order[i % len(order)]))
        n_in = int(np.ceil(dur * fsr))
        spare = data.shape[-1] - n_in
        offs = np.random.RandomState(i).randint(0, spare + 1, size=8) if spare > 0 else [0]
        w = np.zeros((len(offs), data.shape[0], n_in), np.float32)
        for k, o in enumerate(offs):
            piece = data[:, o:o + n_in]
            w[k, :, :piece.shape[-1]] = piece
        cands = AudioSignal(torch.from_numpy(w), fsr).to_mono().resample(sr).audio_data[..., :4000]
        cands = torch.nn.functional.pad(cands, (0, 4000 - cands.shape[-1]))
        loud = [AudioSignal(c[None], sr).loudness().item() for c in cands]
        pick = next((k for k, v in enumerate(loud) if v > ex.LOUDNESS_CUTOFF), len(loud) - 1)
        assert torch.equal(whole[i].audio_data, cands[pick:pick + 1]), f"excerpt {i}"
        name = order[i % len(order)].name
        if name == "c.wav":   # short: one candidate, zero-padded at the end
            assert len(offs) == 1 and (whole[i].audio_data[..., 1500:] == 0).all()
        if name == "d.wav":   # silent: the last candidate
            assert pick == 7
        if name == "a.wav":   # the quiet half is skipped when a candidate in the loud half was drawn
            assert loud[pick] > ex.LOUDNESS_CUTOFF


def test_default_block_size_at_the_shipped_shapes():
    iface = types.SimpleNamespace(coarse=types.SimpleNamespace(chunk_size_s=10),
                                  codec=types.SimpleNamespace(sample_rate=44100, hop_length=768))
    iface.s2t = lambda s: int(np.ceil(s * 44100 / 768))
    assert ex.excerpt_samples(iface) == 441000
    assert ex.default_block_size(iface) == 32  # 32 x 441 600 samples fill one encoder launch
