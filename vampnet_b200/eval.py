"""Score an experiment directory's conditions against its baseline by multi-scale mel distance, on the GPU:

    python -m vampnet_b200.eval --exp_dir D [--baseline_key baseline] [--audio_ext .wav] [--vggish_ckpt PATH]

The reference's scripts/exp/eval.py restated (DESIGN.md §13, §14).  D holds one directory of audio files per
condition, named by integer stems (0.wav, 1.wav, ...), as the reference's scripts/exp/experiment.py writes them.  Every
condition other than the baseline is scored file by file against the baseline with MelSpectrogramLoss(), and two CSV
files are written into D: metrics-all.csv (mel,condition,file) and stats-mel.csv (condition,mean,count,std, std with
ddof 1).  With --vggish_ckpt (torchvggish's checkpoint), each condition directory is also scored against the baseline
directory by Fréchet audio distance (vampnet_b200.fad, every file of both directories), metrics-all.csv gets the column
(mel,frechet,condition,file) and stats-frechet.csv is written the same way.
"""
from __future__ import annotations

import argparse
import csv
import math
from pathlib import Path

import numpy as np
import torch

from .audio import AudioSignal


def _stem_key(path: Path) -> int:
    return int(path.stem)


def _pairs(exp_dir: Path, baseline_key: str, audio_ext: str):
    """[(condition, [(baseline file, condition file), ...])] with conditions sorted by name and each condition's list
    cut to the shorter of the two directories.  Raises ValueError when a pair's stems differ."""
    if not exp_dir.is_dir():
        raise ValueError(f"exp_dir {exp_dir} does not exist")
    conditions = sorted(d.name for d in exp_dir.iterdir() if d.is_dir())
    if baseline_key not in conditions:
        raise ValueError(f"baseline_key {baseline_key} not found in {exp_dir}")
    conditions.remove(baseline_key)
    baseline = sorted((exp_dir / baseline_key).glob(f"*{audio_ext}"), key=_stem_key)
    out = []
    for cond in conditions:
        files = sorted((exp_dir / cond).glob(f"*{audio_ext}"), key=_stem_key)
        n = min(len(baseline), len(files))
        for b, c in zip(baseline[:n], files[:n]):
            if b.stem != c.stem:
                raise ValueError(f"baseline file {b} and condition file {c} do not match")
        out.append((cond, list(zip(baseline[:n], files[:n]))))
    return out


def _load_pair(cond: str, base_file: Path, cond_file: Path):
    """The two signals as the reference prepares them: the condition resampled to the baseline's rate and truncated to
    its length; for an inpaint_<s> condition, int(s * sr) samples trimmed from both ends of both."""
    base = AudioSignal(base_file)
    sig = AudioSignal(cond_file)
    sig.resample(base.sample_rate)
    sig.truncate_samples(base.signal_length)
    if "inpaint" in cond:
        ctx = int(float(cond.split("_")[-1]) * base.sample_rate)
        sig.trim(ctx, ctx)
        base.trim(ctx, ctx)
    return base, sig


def _write_stats(path, rows, col):
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["condition", "mean", "count", "std"])
        for cond in sorted({r[-2] for r in rows}):
            v = np.array([r[col] for r in rows if r[-2] == cond], dtype=np.float64)
            std = float(np.std(v, ddof=1)) if v.size > 1 else math.nan
            w.writerow([cond, repr(float(v.mean())), v.size, "" if math.isnan(std) else repr(std)])


def evaluate(exp_dir, baseline_key: str = "baseline", audio_ext: str = ".wav", loss=None, fad=None):
    """Scores every condition; returns the rows of metrics-all.csv as (mel, condition, file) and writes both CSVs.
    loss(x, y) takes two batched AudioSignals and returns one value per item; the default is
    MelSpectrogramLoss().per_item.  The pairs of one condition that share a shape and rate are scored in one call.
    With fad (a vampnet_b200.fad.FrechetAudioDistance) the rows are (mel, frechet, condition, file), frechet the
    distance between the condition's directory and the baseline's (whose embeddings are computed once), and
    stats-frechet.csv is written too."""
    exp_dir = Path(exp_dir)
    if loss is None:
        from .metrics import MelSpectrogramLoss
        loss = MelSpectrogramLoss().per_item
    rows = []
    base_moments = fad.dir_moments(exp_dir / baseline_key, audio_ext) if fad is not None else None
    for cond, pairs in _pairs(exp_dir, baseline_key, audio_ext):
        loaded = [_load_pair(cond, b, c) for b, c in pairs]
        groups = {}
        for i, (b, c) in enumerate(loaded):
            if tuple(b.audio_data.shape) != tuple(c.audio_data.shape):
                raise ValueError(f"{cond}/{pairs[i][1].name}: shape {tuple(c.audio_data.shape)} after resampling and "
                                 f"truncation differs from the baseline's {tuple(b.audio_data.shape)}")
            groups.setdefault((tuple(b.audio_data.shape), b.sample_rate), []).append(i)
        mel = [0.0] * len(loaded)
        for (_, sr), idx in groups.items():
            x = AudioSignal(torch.cat([loaded[i][0].audio_data for i in idx]), sr)
            y = AudioSignal(torch.cat([loaded[i][1].audio_data for i in idx]), sr)
            for i, v in zip(idx, torch.as_tensor(loss(x, y)).reshape(-1).tolist()):
                mel[i] = float(v)
        if fad is None:
            rows.extend((mel[i], cond, pairs[i][0].stem) for i in range(len(loaded)))
        else:
            frechet = fad.score_moments(base_moments, fad.dir_moments(exp_dir / cond, audio_ext))
            rows.extend((mel[i], frechet, cond, pairs[i][0].stem) for i in range(len(loaded)))
    with open(exp_dir / "metrics-all.csv", "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["mel", "condition", "file"] if fad is None else ["mel", "frechet", "condition", "file"])
        w.writerows([repr(v) for v in r[:-2]] + list(r[-2:]) for r in rows)
    _write_stats(exp_dir / "stats-mel.csv", rows, 0)
    if fad is not None:
        _write_stats(exp_dir / "stats-frechet.csv", rows, 1)
    return rows


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--exp_dir", required=True)
    ap.add_argument("--baseline_key", default="baseline")
    ap.add_argument("--audio_ext", default=".wav")
    ap.add_argument("--vggish_ckpt", default=None, help="torchvggish checkpoint: also score by Fréchet audio distance")
    a = ap.parse_args(argv)
    fad = None
    if a.vggish_ckpt is not None:
        from .fad import FrechetAudioDistance
        fad = FrechetAudioDistance(a.vggish_ckpt, use_pca=False, use_activation=False)
    rows = evaluate(a.exp_dir, a.baseline_key, a.audio_ext, fad=fad)
    d = Path(a.exp_dir)
    stats = f"{d / 'stats-mel.csv'}" + ("" if fad is None else f" and {d / 'stats-frechet.csv'}")
    print(f"scored {len(rows)} files in {len({r[-2] for r in rows})} conditions; wrote {d / 'metrics-all.csv'} and {stats}")


if __name__ == "__main__":
    main()
