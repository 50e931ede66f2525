"""GPU: the experiment script's batched runner (vampnet_b200.experiment.run_experiment) equals its sequential condition
functions run in the reference's order, bit for bit, with the same random / numpy / torch (CPU and CUDA) RNG states
afterwards, for every registry, on excerpts of different lengths (several coarse chunks, padded fine-stage chunks) and
at every block size; a block is one encode launch group, one coarse and one fine generate_many and one decode group;
and the CLI's resume rule and its output layout, scored by python -m vampnet_b200.eval."""
import csv
import random
import wave

import numpy as np
import pytest
import torch

from tests.test_gpu_interface import iface  # noqa: F401  (module fixture: tiny coarse / c2f / codec)
from vampnet_b200 import experiment as ex
from vampnet_b200.audio import AudioSignal

pytestmark = pytest.mark.gpu

# coarse chunks of 35 frames (0.6 s), fine-stage chunks of 15 (0.25 s), hop 768 at 44.1 kHz
SECONDS = (1.3, 0.45, 0.9, 2.1)


def excerpts(seconds=SECONDS, seed=0):
    """Noise under a click every half second (so the beat tracker finds beats), one clip per duration."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for s in seconds:
        n = int(s * 44100)
        x = 0.05 * torch.randn(n, generator=g)
        x[::22050] += 0.9
        out.append(AudioSignal(x[None, None].cuda(), 44100))
    return out


def reseed(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def rng_state():
    return (random.getstate(), np.random.get_state()[1].copy(), torch.get_rng_state(), torch.cuda.get_rng_state())


def assert_rng_equal(a, b):
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and torch.equal(a[2], b[2]) and torch.equal(a[3], b[3])


def sequential(iface, sigs, exp_type):  # noqa: F811
    conds = ex.conditions(exp_type)
    out = {name: [] for name in conds}
    for sig in sigs:
        for name, cond in conds.items():
            out[name].append(cond(sig, iface))
    return out


def assert_same(got, want):
    assert list(got) == list(want)
    for name in want:
        assert len(got[name]) == len(want[name])
        for k, (a, b) in enumerate(zip(got[name], want[name])):
            assert a.sample_rate == b.sample_rate and a.audio_data.shape == b.audio_data.shape, f"{name}[{k}]"
            assert torch.equal(a.audio_data, b.audio_data), f"{name}[{k}] differs"


@pytest.mark.parametrize("exp_type", list(ex.EXP_REGISTRY))
def test_runner_equals_sequential_conditions(iface, exp_type):  # noqa: F811
    reseed(7)
    want = sequential(iface, excerpts(), exp_type)
    want_rng = rng_state()
    reseed(7)
    got = ex.run_experiment(iface, excerpts(), exp_type)
    assert_rng_equal(rng_state(), want_rng)
    assert_same(got, want)


def test_block_size_does_not_change_outputs(iface):  # noqa: F811
    outs = []
    for bs in (1, 2, len(SECONDS)):
        reseed(3)
        outs.append((ex.run_experiment(iface, excerpts(seed=1), "gen-compression", block_size=bs), rng_state()))
    for got, rng in outs[1:]:
        assert_same(got, outs[0][0])
        assert_rng_equal(rng, outs[0][1])


class Spy:
    """Counts calls of the named methods of one object (instance attributes shadow the class's) and the generate
    launches made through vampnet_b200._lib."""
    GENERATE = ("vnb_generate_many", "vnb_generate_many_adapted", "vnb_generate_ragged", "vnb_generate_steps",
                "vnb_generate_mixed_top_p")

    def __init__(self, monkeypatch):
        from vampnet_b200 import _lib as L
        self.mp, self.count, self.args, self.launches = monkeypatch, {}, {}, []
        real = L.lib
        spy = self

        class Lib:
            def __getattr__(self, name):
                fn = getattr(real(), name)
                if name not in Spy.GENERATE:
                    return fn

                def counted(*a):
                    spy.launches.append((a[0].value, a[3], a[4]))  # handle, B, T
                    return fn(*a)
                return counted
        monkeypatch.setattr(L, "lib", lambda: Lib())

    def watch(self, obj, tag, name):
        fn = getattr(obj, name)
        key = f"{tag}.{name}"
        self.count[key], self.args[key] = 0, []

        def counted(*a, **k):
            self.count[key] += 1
            self.args[key].append(a)
            return fn(*a, **k)
        self.mp.setattr(obj, name, counted)


def planned_launches(calls, max_rows):
    """The launches generate_many(mixed_lengths, mixed_steps, mixed_top_p) makes of `calls`: longest T first, split
    where rows x the launch's T would pass max_rows."""
    n, open_, rows, T = 0, False, 0, 0
    for t, b in sorted(((c["start_tokens"].shape[-1], c["start_tokens"].shape[0]) for c in calls), key=lambda x: -x[0]):
        if open_ and (rows + b) * T > max_rows:
            open_, rows = False, 0
        if not open_:
            n, open_, T = n + 1, True, t
        rows += b
    return n


@pytest.mark.parametrize("max_rows", [None, 150])
def test_launches_per_block(iface, monkeypatch, max_rows):  # noqa: F811
    from vampnet_b200.codec import plan_launches
    from vampnet_b200.modules import transformer as TR
    if max_rows is not None:  # a limit the tiny chunks reach: each stage then splits, only there
        monkeypatch.setattr(TR, "MANY_MAX_ROWS", max_rows)
    limit = TR.MANY_MAX_ROWS
    spy = Spy(monkeypatch)
    for obj, tag, names in ((iface.codec, "codec", ("encode_many", "decode_many", "_encode_launch", "_decode_launch",
                                                    "encode", "decode")),
                            (iface.coarse, "coarse", ("generate_many", "generate")),
                            (iface.c2f, "c2f", ("generate_many", "generate"))):
        for name in names:
            spy.watch(obj, tag, name)
    sigs = excerpts()
    ex.run_experiment(iface, sigs, "gen-compression", block_size=2)
    blocks, conds = 2, len(ex.EXP_REGISTRY["gen-compression"])
    c = spy.count
    assert c["codec.encode_many"] == blocks and c["codec.decode_many"] == blocks
    assert c["codec.encode"] == c["codec.decode"] == 0
    assert c["coarse.generate_many"] == blocks and c["c2f.generate_many"] == blocks
    assert c["coarse.generate"] == c["c2f.generate"] == 0
    hop = iface.codec.hop_length
    padded = [-(-s.signal_length // hop) * hop for s in sigs]
    assert c["codec._encode_launch"] == sum(len(plan_launches(padded[lo:lo + 2])) for lo in (0, 2))
    # every decode of a block (conditions other than the baseline) in one decode_many
    assert [len(a[0]) for a in spy.args["codec.decode_many"]] == [2 * (conds - 1)] * blocks
    assert c["codec._decode_launch"] == sum(len(plan_launches([z.shape[-1] * hop for z in a[0]]))
                                            for a in spy.args["codec.decode_many"])
    for tag, model in (("coarse", iface.coarse), ("c2f", iface.c2f)):
        want = sum(planned_launches(a[1], limit) for a in spy.args[f"{tag}.generate_many"])
        got = [x for x in spy.launches if x[0] == model._handle.value]
        assert len(got) == want, (tag, got)
        assert all(B * T <= limit for _, B, T in got)
    if max_rows is None:  # the tiny block fits: one launch per stage per block, not one per condition
        assert c["codec._encode_launch"] == blocks
        assert len([x for x in spy.launches if x[0] == iface.coarse._handle.value]) == blocks
        assert len([x for x in spy.launches if x[0] == iface.c2f._handle.value]) == blocks


# ------------------------------------------------------------------------------------------------ CLI
def _write_wav(path, x, sr=44100):
    pcm = (np.clip(x, -1, 1) * 32767).astype("<i2")
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(sr)
        w.writeframes(pcm.tobytes())


def _snapshot(root):
    return {str(p.relative_to(root)): (p.read_bytes(), p.stat().st_mtime_ns) for p in sorted(root.rglob("*.wav"))}


def test_cli_end_to_end(iface, tmp_path):  # noqa: F811
    from vampnet_b200 import eval as ev
    g = np.random.default_rng(0)
    src = tmp_path / "src"
    src.mkdir()
    for k, secs in enumerate((4.0, 3.2, 1.5)):
        x = 0.05 * g.standard_normal(int(secs * 44100))
        x[::22050] += 0.9
        _write_wav(src / f"{k}.wav", x)
    out = tmp_path / "samples"
    old = iface.coarse.chunk_size_s
    iface.set_chunk_size(2.5)  # excerpts long enough for eval's inpaint_1.0 trim
    try:
        n = 5
        gc, ms = ex.EXP_REGISTRY["gen-compression"], ex.EXP_REGISTRY["musical-sampling"]
        assert sorted(ex.experiment(iface, [src], out, max_excerpts=n, exp_type="gen-compression", block_size=2)) \
            == list(range(n))
        assert sorted(ex.experiment(iface, [src], out, max_excerpts=n, exp_type="musical-sampling")) == list(range(n))
        assert sorted(d.name for d in out.iterdir()) == sorted([*gc, *ms])
        for name in [*gc, *ms]:
            assert sorted(p.name for p in (out / name).iterdir()) == [f"{i}.wav" for i in range(n)]
        before = _snapshot(out)
        assert ex.experiment(iface, [src], out, max_excerpts=n, exp_type="gen-compression") == []
        assert ex.experiment(iface, [src], out, max_excerpts=n, exp_type="musical-sampling") == []
        assert _snapshot(out) == before

        # one file gone: only its excerpt is redone, as the sequential loop under the same skip pattern redoes it
        (out / "token_noise_0.5" / "3.wav").unlink()
        assert ex.experiment(iface, [src], out, max_excerpts=n, exp_type="gen-compression") == [3]
        after = _snapshot(out)
        for key, (data, mtime) in after.items():
            if not key.endswith("/3.wav") or key.split("/")[0] not in gc:
                assert (data, mtime) == before[key], key
        ex.seed_all(0)
        idx = list(range(n))
        random.shuffle(idx)
        sig = ex.load_excerpts(ex.find_files([src]), [3], 2.5, 44100, 0, "cuda")[0]
        for name, cond in gc.items():
            ref = tmp_path / "ref.wav"
            cond(sig, iface).cpu().write(ref)
            assert ref.read_bytes() == after[f"{name}/3.wav"][0], name
    finally:
        iface.set_chunk_size(old)

    ev.main(["--exp_dir", str(out)])
    with open(out / "stats-mel.csv") as f:
        rows = list(csv.DictReader(f))
    assert sorted(r["condition"] for r in rows) == sorted(k for k in [*gc, *ms] if k != "baseline")
    assert all(int(r["count"]) == n and np.isfinite(float(r["mean"])) for r in rows)
