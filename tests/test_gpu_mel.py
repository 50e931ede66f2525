"""GPU: MelSpectrogramLoss, AudioSignal.mel_spectrogram and the eval CLI (vampnet_b200.metrics, vampnet_b200.eval)
against oracle/mel_oracle.py in float64 and its goldens: 10 s signals, several items, seven scales, CPU signals, no
host sync, and an experiment directory scored end to end."""
import csv

import numpy as np
import pytest
import torch

from oracle import gen_mel_golden as gm
from oracle import mel_oracle as mo
from vampnet_b200.audio import AudioSignal
from vampnet_b200.metrics import MelSpectrogramLoss

pytestmark = pytest.mark.gpu

LOSS_TOL = 1e-6  # relative to the float64 oracle


def sig(a, sr, device="cuda"):
    return AudioSignal(torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device), sr)


def loss_for(scales):
    m, lo, hi, w = zip(*scales)
    return MelSpectrogramLoss(n_mels=list(m), window_lengths=list(w), mel_fmin=list(lo), mel_fmax=list(hi))


def test_default_loss_on_10s_matches_oracle():
    sr = 44100
    x, y = mo.test_pair(10 * sr, sr, seed=1)
    got = MelSpectrogramLoss()(sig(x[None], sr), sig(y[None], sr))
    assert got.dtype == torch.float32 and got.shape == () and got.device.type == "cuda"
    want, _ = mo.mel_loss(x[None], y[None], sr)
    assert abs(got.item() - want) <= LOSS_TOL * want, (got.item(), want)


@pytest.mark.parametrize("name", list(gm.CASES))
def test_goldens(name):
    g = np.load(f"{gm.OUT}/{name}.npz")
    sr = int(g["sr"])
    scales = [(int(m), lo, hi, int(w)) for m, lo, hi, w in g["scales"]]
    fn = loss_for(scales)
    x, y = sig(g["x"], sr), sig(g["y"], sr)
    got = fn(x, y).item()
    assert abs(got - float(g["loss"])) <= LOSS_TOL * float(g["loss"])
    items = fn.per_item(x, y).cpu().numpy().astype(np.float64)
    assert np.all(np.abs(items - g["item_loss"]) <= LOSS_TOL * g["item_loss"])
    m, lo, hi, w = scales[0]
    spec = x.mel_spectrogram(m, lo, hi, w, w // 4).cpu().numpy()
    ref = g["spec"]
    assert spec.shape == ref.shape
    frame_max = ref.max(axis=2, keepdims=True)
    silent = np.broadcast_to(frame_max == 0, ref.shape)  # the signal's silent start: exactly 0 on both sides
    assert (spec[silent] == 0).all()
    assert (np.abs(spec - ref)[~silent] / np.broadcast_to(frame_max, ref.shape)[~silent]).max() <= 1e-6


def test_equal_signals_give_zero_and_swapping_is_exact():
    sr = 22050
    x, y = mo.test_pair(3 * sr, sr, seed=2, channels=2)
    fn = MelSpectrogramLoss()
    assert fn(sig(x[None], sr), sig(x[None], sr)).item() == 0.0
    a, b = fn(sig(x[None], sr), sig(y[None], sr)), fn(sig(y[None], sr), sig(x[None], sr))
    assert a.item() == b.item() and a.item() > 0


def test_batch_is_mean_of_items_and_items_equal_alone():
    sr, B = 16000, 4
    pairs = [mo.test_pair(2 * sr, sr, seed=10 + b) for b in range(B)]
    x = np.stack([p[0] for p in pairs])
    y = np.stack([p[1] for p in pairs])
    fn = MelSpectrogramLoss()
    total = fn(sig(x, sr), sig(y, sr)).item()
    items = fn.per_item(sig(x, sr), sig(y, sr))
    assert items.shape == (B,) and items.dtype == torch.float32
    mean = float(items.double().mean())
    assert abs(total - mean) <= 2 * np.finfo(np.float32).eps * total
    for b in range(B):
        alone = fn.per_item(sig(x[b:b + 1], sr), sig(y[b:b + 1], sr))
        assert alone.item() == items[b].item()
        assert fn(sig(x[b:b + 1], sr), sig(y[b:b + 1], sr)).item() == items[b].item()
    want_total, want_items = mo.mel_loss(x, y, sr)
    assert abs(total - want_total) <= LOSS_TOL * want_total
    assert np.all(np.abs(items.cpu().numpy() - want_items) <= LOSS_TOL * want_items)


def test_seven_scales_on_10s():
    sr = 48000
    x, y = mo.test_pair(10 * sr, sr, seed=4)
    got = loss_for(mo.SEVEN_SCALES)(sig(x[None], sr), sig(y[None], sr)).item()
    want, _ = mo.mel_loss(x[None], y[None], sr, mo.SEVEN_SCALES)
    assert abs(got - want) <= LOSS_TOL * want, (got, want)


def test_cpu_signals_round_trip():
    sr = 16000
    x, y = mo.test_pair(sr, sr, seed=5)
    fn = MelSpectrogramLoss()
    on_cpu = fn(sig(x[None], sr, "cpu"), sig(y[None], sr, "cpu"))
    assert on_cpu.device.type == "cpu"
    assert on_cpu.item() == fn(sig(x[None], sr), sig(y[None], sr)).item()
    s = sig(x[None], sr, "cpu")
    m = s.mel_spectrogram()
    assert m.device.type == "cpu" and m.shape == (1, 1, 80, 1 + sr // 128)  # 16 kHz: window 512, hop 128
    assert torch.equal(m, sig(x[None], sr).mel_spectrogram().cpu())


def test_no_host_sync():
    sr = 44100
    x, y = mo.test_pair(2 * sr, sr, seed=6)
    xs, ys = sig(np.stack([x, x]), sr), sig(np.stack([y, x]), sr)
    fn = MelSpectrogramLoss()
    fn(xs, ys)  # the first call per configuration builds and uploads the tables
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = fn(xs, ys)
        items = fn.per_item(xs, ys)
        spec = xs.mel_spectrogram(150, 0.0, None, 2048, 512)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert loss.item() > 0 and items[1].item() == 0.0 and spec.shape == (2, 1, 150, 1 + 2 * sr // 512)


def test_mismatched_signals_are_refused():
    fn = MelSpectrogramLoss()
    a = sig(np.zeros((1, 1, 4000)), 16000)
    with pytest.raises(ValueError):
        fn(a, sig(np.zeros((1, 1, 4001)), 16000))
    with pytest.raises(ValueError):
        fn(a, sig(np.zeros((1, 1, 4000)), 22050))
    with pytest.raises(RuntimeError):  # N <= 2048 // 2 at the default first scale
        fn(sig(np.zeros((1, 1, 1024)), 44100), sig(np.zeros((1, 1, 1024)), 44100))


def test_eval_cli_end_to_end(tmp_path):
    from vampnet_b200 import eval as ev
    sr, n = 16000, 2 * 16000
    for d in ("baseline", "plain", "inpaint_0.5"):
        (tmp_path / d).mkdir()
    for i in range(3):
        x, y = mo.test_pair(n, sr, seed=20 + i)
        sig(x[None], sr, "cpu").write(tmp_path / "baseline" / f"{i}.wav")
        sig(0.5 * x[None] + 0.5 * y[None], sr, "cpu").write(tmp_path / "plain" / f"{i}.wav")
        sig(y[None], sr, "cpu").write(tmp_path / "inpaint_0.5" / f"{i}.wav")
    ev.main(["--exp_dir", str(tmp_path)])
    with open(tmp_path / "metrics-all.csv") as f:
        rows = list(csv.reader(f))[1:]
    assert [(r[1], r[2]) for r in rows] == [("inpaint_0.5", s) for s in "012"] + [("plain", s) for s in "012"]
    for mel, cond, stem in rows:
        b = AudioSignal(tmp_path / "baseline" / f"{stem}.wav").audio_data.numpy()
        c = AudioSignal(tmp_path / cond / f"{stem}.wav").audio_data.numpy()
        if cond.startswith("inpaint"):
            k = int(0.5 * sr)
            b, c = b[..., k:-k], c[..., k:-k]
        want, _ = mo.mel_loss(b, c, sr)
        assert abs(float(mel) - want) <= LOSS_TOL * want
    with open(tmp_path / "stats-mel.csv") as f:
        stats = list(csv.reader(f))
    assert stats[0] == ["condition", "mean", "count", "std"] and [r[0] for r in stats[1:]] == ["inpaint_0.5", "plain"]
    for r in stats[1:]:
        v = np.array([float(m) for m, c, _ in rows if c == r[0]])
        assert float(r[1]) == v.mean() and r[2] == "3" and float(r[3]) == np.std(v, ddof=1)
