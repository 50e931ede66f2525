"""Write the sample conditions of an experiment, one directory of WAVs per condition, on the GPU:

    python -m vampnet_b200.experiment --sources DIR_OR_FILE [...] [--output_dir ./samples] [--max_excerpts 2000]
        [--exp_type gen-compression] [--seed 0] [--ext .wav] [--coarse_ckpt P --coarse2fine_ckpt P --codec_ckpt P]

The reference's scripts/exp/experiment.py restated (DESIGN.md §15).  Every excerpt i is put through every condition of
EXP_REGISTRY[exp_type] and written as <output_dir>/<condition>/<i>.wav, the layout python -m vampnet_b200.eval scores.
sampling-steps and musical-sampling write no baseline directory, as in the reference: score them by running
gen-compression into the same output directory first.

The condition functions below are the sequential path, each a line-for-line restatement of the reference's.  The CLI
runs run_experiment instead, which gives the same audio bit for bit and leaves the random, numpy and torch RNGs where
the sequential calls leave them, while it encodes, generates and decodes a block of excerpts with a handful of
launches: one encode_many, one coarse and one fine generate_many over every condition of every excerpt, one decode_many.
"""
from __future__ import annotations

import argparse
import math
import random
from pathlib import Path
from typing import Callable, NamedTuple, Optional

import numpy as np
import torch

from . import mask as pmask
from .audio import AudioSignal, _read_wav
from .codec import CODEC_MANY_MAX_SAMPLES
from .modules.transformer import MANY_MAX_ROWS


def generate_kwargs(**kwargs) -> dict:
    """The generate() keyword arguments the reference script means: it passes sampling_steps=, which generate() names
    _sampling_steps= (as written the script raises TypeError there)."""
    if "sampling_steps" in kwargs:
        kwargs["_sampling_steps"] = kwargs.pop("sampling_steps")
    return kwargs


class Plan(NamedTuple):
    """How run_experiment runs a condition on an excerpt's codes z.  codes(z, interface): the codes the condition
    starts from; mask(sig, z, interface): its coarse mask, with every random draw the condition makes (None: no coarse
    stage); coarse: the coarse stage's generate() keyword arguments; fine: whether coarse_to_fine follows (with
    generate()'s defaults).  The result is decoded."""
    codes: Callable = lambda z, interface: z
    mask: Optional[Callable] = None
    coarse: dict = {}
    fine: bool = False


# ------------------------------------------------------------------------------------------------ conditions
def baseline(sig, interface):
    """The excerpt as the codec sees it (the reference calls interface.preprocess, which is _preprocess)."""
    return interface._preprocess(sig)


baseline.plan = None  # no codes: run_experiment calls the function itself


def reconstructed(sig, interface):
    return interface.decode(interface.encode(sig))


reconstructed.plan = Plan()


def coarse2fine(sig, interface):
    z = interface.encode(sig)
    z = z[:, :interface.c2f.n_conditioning_codebooks, :]
    z = interface.coarse_to_fine(z)
    return interface.decode(z)


coarse2fine.plan = Plan(codes=lambda z, interface: z[:, :interface.c2f.n_conditioning_codebooks, :], fine=True)


class CoarseCond:
    def __init__(self, num_conditioning_codebooks, downsample_factor):
        self.num_conditioning_codebooks = num_conditioning_codebooks
        self.downsample_factor = downsample_factor
        self.plan = Plan(mask=lambda sig, z, interface: self.mask(z), fine=True)

    def mask(self, z):
        """As the reference builds it: periodic_mask(mask, x) starts from a fresh full mask of mask's shape, so the
        codebook_unmask before it has no effect and the mask is periodic_mask(z, x) over every codebook."""
        mask = pmask.full_mask(z)
        mask = pmask.codebook_unmask(mask, self.num_conditioning_codebooks)
        return pmask.periodic_mask(mask, self.downsample_factor)

    def __call__(self, sig, interface):
        z = interface.encode(sig)
        mask = self.mask(z)
        zv = interface.coarse_vamp(z, mask)
        zv = interface.coarse_to_fine(zv)
        return interface.decode(zv)


def mask_ratio_1_step(ratio=1.0):
    def wrapper(sig, interface):
        z = interface.encode(sig)
        mask = pmask.linear_random(z, ratio)
        zv = interface.coarse_vamp(z, mask, **generate_kwargs(sampling_steps=1))
        return interface.decode(zv)
    wrapper.plan = Plan(mask=lambda sig, z, interface: pmask.linear_random(z, ratio),
                        coarse=generate_kwargs(sampling_steps=1))
    return wrapper


def num_sampling_steps(num_steps=1):
    def wrapper(sig, interface):
        z = interface.encode(sig)
        mask = pmask.periodic_mask(z, 16)
        zv = interface.coarse_vamp(z, mask, **generate_kwargs(sampling_steps=num_steps))
        zv = interface.coarse_to_fine(zv)
        return interface.decode(zv)
    wrapper.plan = Plan(mask=lambda sig, z, interface: pmask.periodic_mask(z, 16),
                        coarse=generate_kwargs(sampling_steps=num_steps), fine=True)
    return wrapper


def _beat_mask(ctx_time, sig, interface):
    return interface.make_beat_mask(sig, before_beat_s=ctx_time / 2, after_beat_s=ctx_time / 2, invert=True)


def beat_mask(ctx_time):
    """Beats from interface.beat_tracker: the librosa-style tracker of DESIGN.md §10, not the reference's WaveBeat."""
    def wrapper(sig, interface):
        mask = _beat_mask(ctx_time, sig, interface)
        z = interface.encode(sig)
        zv = interface.coarse_vamp(z, mask)
        zv = interface.coarse_to_fine(zv)
        return interface.decode(zv)
    wrapper.plan = Plan(mask=lambda sig, z, interface: _beat_mask(ctx_time, sig, interface), fine=True)
    return wrapper


def _inpaint_mask(ctx_time, z, interface):
    return pmask.inpaint(z, interface.s2t(ctx_time), interface.s2t(ctx_time))


def inpaint(ctx_time):
    def wrapper(sig, interface):
        z = interface.encode(sig)
        mask = _inpaint_mask(ctx_time, z, interface)
        zv = interface.coarse_vamp(z, mask)
        zv = interface.coarse_to_fine(zv)
        return interface.decode(zv)
    wrapper.plan = Plan(mask=lambda sig, z, interface: _inpaint_mask(ctx_time, z, interface), fine=True)
    return wrapper


# the reference's opus and token_noise conditions are in no registry and are left out
EXP_REGISTRY = {}
EXP_REGISTRY["gen-compression"] = {
    "baseline": baseline,
    "reconstructed": reconstructed,
    "coarse2fine": coarse2fine,
    **{f"{n}_codebooks_downsampled_{x}x": CoarseCond(num_conditioning_codebooks=n, downsample_factor=x)
       for (n, x) in ((1, 1), (4, 4), (4, 16), (4, 32))},
    **{f"token_noise_{x}": mask_ratio_1_step(ratio=x) for x in [0.25, 0.5, 0.75]},
}
EXP_REGISTRY["sampling-steps"] = {f"steps_{n}": num_sampling_steps(n) for n in [1, 4, 12, 36, 64, 72]}
EXP_REGISTRY["musical-sampling"] = {
    **{f"beat_mask_{t}": beat_mask(t) for t in [0.075]},
    **{f"inpaint_{t}": inpaint(t) for t in [0.5, 1.0]},
}


def conditions(exp_type: str) -> dict:
    if exp_type not in EXP_REGISTRY:
        raise ValueError(f"Unknown exp_type {exp_type}; one of {sorted(EXP_REGISTRY)}")
    return EXP_REGISTRY[exp_type]


# ------------------------------------------------------------------------------------------------ batched runner
def excerpt_samples(interface) -> int:
    """Samples of one excerpt: coarse.chunk_size_s seconds at the codec's rate."""
    return int(interface.coarse.chunk_size_s * interface.codec.sample_rate)


def default_block_size(interface) -> int:
    """Excerpts per block: as many as one encoder launch holds (CODEC_MANY_MAX_SAMPLES) and as many as one generate
    launch holds one coarse chunk each (MANY_MAX_ROWS): 32 for 10 s excerpts at 44.1 kHz."""
    hop = interface.codec.hop_length
    padded = math.ceil(excerpt_samples(interface) / hop) * hop
    return max(1, min(CODEC_MANY_MAX_SAMPLES // padded, MANY_MAX_ROWS // interface.s2t(interface.coarse.chunk_size_s)))


def run_experiment(interface, excerpts: list, exp_type: str, block_size: int = None) -> dict:
    """{condition: [AudioSignal per excerpt]} for every condition of EXP_REGISTRY[exp_type], equal bit for bit to
    [cond(sig, interface) for sig in excerpts for cond in the registry's conditions] run in that order, and leaving the
    random, numpy and torch (CPU and CUDA) RNG states as those calls leave them.  Excerpts are moved to the Interface's
    device first (in place, as encode moves them).  block_size: excerpts per block (default_block_size when None); the
    results do not depend on it.

    Per block, a prepare phase walks the excerpts and, for each, the conditions in registry order, building each
    condition's mask and drawing the Philox keys of its coarse and fine chunks: the draws the sequential calls make, in
    their order.  Then the launches: one encode_many for the block, every condition's coarse chunks as one
    generate_many(mixed_lengths, mixed_steps, mixed_top_p), every fine-stage chunk as one more, one decode_many."""
    conds = conditions(exp_type)
    block_size = default_block_size(interface) if block_size is None else int(block_size)
    if block_size < 1:
        raise ValueError(f"run_experiment: block_size must be >= 1, got {block_size}")
    excerpts = [s.to(interface.device) for s in excerpts]
    out = {name: [] for name in conds}
    for lo in range(0, len(excerpts), block_size):
        for name, sigs in _run_block(interface, excerpts[lo:lo + block_size], conds).items():
            out[name] += sigs
    return out


def _run_block(interface, excerpts: list, conds: dict) -> dict:
    codes = interface.encode_many(excerpts)  # deterministic: one encode serves every condition
    reqs, out = [], {name: [None] * len(excerpts) for name in conds}
    for k, (sig, z) in enumerate(zip(excerpts, codes)):
        for name, cond in conds.items():
            if cond.plan is None:
                out[name][k] = cond(sig, interface)
                continue
            p = cond.plan
            zc = p.codes(z, interface)
            mask = p.mask(sig, zc, interface) if p.mask is not None else None
            q = interface._vamp_request(zc, mask, 0 if mask is None else 1, p.coarse, fine={} if p.fine else None)
            reqs.append((name, k, q))
    interface._run_vamp_requests([q for _, _, q in reqs], dict(mixed_lengths=True, mixed_steps=True, mixed_top_p=True))
    if reqs:
        for (name, k, _), sig in zip(reqs, interface.decode_many([q["zv"] for _, _, q in reqs])):
            out[name][k] = sig
    return out


# ------------------------------------------------------------------------------------------------ excerpts
LOUDNESS_CUTOFF = -40.0  # LUFS; audiotools' default salient-excerpt cutoff, as taken here (unchecked against it)
N_CANDIDATES = 8


def find_files(sources, ext=(".wav",)) -> list:
    """The sorted files with one of the extensions `ext` under `sources` (files or directories, searched recursively).
    Only WAV can be read here; any other extension raises ValueError."""
    ext = [ext] if isinstance(ext, str) else list(ext)
    bad = [e for e in ext if e.lower() != ".wav"]
    if bad:
        raise ValueError(f"--ext {' '.join(bad)}: only .wav files can be read (no MP3 or FLAC decoder here); convert the "
                         f"sources to WAV and pass --ext .wav")
    files = set()
    for s in sources:
        p = Path(s)
        if p.is_dir():
            files.update(f for f in p.rglob("*") if f.is_file() and f.suffix.lower() == ".wav")
        elif p.is_file() and p.suffix.lower() == ".wav":
            files.add(p)
    return sorted(files, key=str)


def load_excerpts(files: list, indices: list, duration: float, sample_rate: int, seed: int, device="cuda") -> list:
    """The excerpts `indices` (one mono AudioSignal of int(duration * sample_rate) samples each, on `device`).

    Excerpt i is taken from file i % len(files) of `files` shuffled once with np.random.RandomState(seed).  Its
    candidate offsets, up to N_CANDIDATES, are drawn by np.random.RandomState(i) uniformly over the file's whole
    windows (one candidate at offset 0 when the file is no longer than the excerpt; a short file is zero-padded at the
    end).  Each candidate is averaged to mono and resampled to sample_rate, and the excerpt is the first candidate
    louder than LOUDNESS_CUTOFF, or the last if none is; the loudness of every candidate of the call is measured in one
    batched AudioSignal.loudness.  The global RNGs are not touched."""
    if not files:
        raise ValueError("load_excerpts: no source files")
    order = list(files)
    np.random.RandomState(seed).shuffle(order)
    n_out = int(duration * sample_rate)
    cands = []
    for i in indices:
        data, sr = _read_wav(str(order[i % len(order)]))
        n_in = int(math.ceil(duration * sr))
        spare = data.shape[-1] - n_in
        offsets = np.random.RandomState(i).randint(0, spare + 1, size=N_CANDIDATES) if spare > 0 else [0]
        windows = np.zeros((len(offsets), data.shape[0], n_in), dtype=np.float32)
        for c, o in enumerate(offsets):
            piece = data[:, int(o):int(o) + n_in]
            windows[c, :, :piece.shape[-1]] = piece
        sig = AudioSignal(torch.from_numpy(windows), sr).to(device).to_mono().resample(sample_rate)
        x = sig.audio_data[..., :n_out]
        cands.append(torch.nn.functional.pad(x, (0, n_out - x.shape[-1])))
    loud = AudioSignal(torch.cat(cands), sample_rate).loudness().cpu().tolist() if cands else []
    out, at = [], 0
    for x in cands:
        mine = loud[at:at + x.shape[0]]
        at += x.shape[0]
        pick = next((c for c, v in enumerate(mine) if v > LOUDNESS_CUTOFF), len(mine) - 1)
        out.append(AudioSignal(x[pick:pick + 1].clone(), sample_rate))
    return out


# ------------------------------------------------------------------------------------------------ CLI
def seed_all(seed: int):
    """What audiotools' util.seed does."""
    torch.manual_seed(seed)
    np.random.seed(seed)
    random.seed(seed)


def experiment(interface, sources, output_dir="./samples", max_excerpts: int = 2000,
               exp_type: str = "gen-compression", seed: int = 0, ext=(".wav",), block_size: int = None) -> list:
    """The reference's main(): seed, shuffle the excerpt indices with `random`, skip every excerpt whose files all exist
    (a skipped excerpt draws nothing), and write each other excerpt's conditions as <output_dir>/<condition>/<i>.wav.
    Runs the excerpts in blocks through run_experiment; returns the indices written, in order."""
    conds = conditions(exp_type)
    files = find_files(sources, ext)
    if not files:
        raise ValueError(f"no .wav files under {' '.join(map(str, sources))}")
    output_dir = Path(output_dir)
    output_dir.mkdir(exist_ok=True, parents=True)
    seed_all(seed)
    indices = list(range(max_excerpts))
    random.shuffle(indices)
    todo = [i for i in indices if not all((output_dir / name / f"{i}.wav").exists() for name in conds)]
    block_size = default_block_size(interface) if block_size is None else int(block_size)
    duration, sr = interface.coarse.chunk_size_s, interface.codec.sample_rate
    for lo in range(0, len(todo), block_size):
        block = todo[lo:lo + block_size]
        excerpts = load_excerpts(files, block, duration, sr, seed, interface.device)
        results = run_experiment(interface, excerpts, exp_type, block_size=len(block))
        for name, sigs in results.items():
            o_dir = output_dir / name
            o_dir.mkdir(exist_ok=True, parents=True)
            for i, sig in zip(block, sigs):
                sig.cpu().write(o_dir / f"{i}.wav")
    return todo


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sources", nargs="+", required=True, help="audio files or directories")
    ap.add_argument("--output_dir", default="./samples")
    ap.add_argument("--max_excerpts", type=int, default=2000)
    ap.add_argument("--exp_type", default="gen-compression", choices=list(EXP_REGISTRY))
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--ext", nargs="+", default=[".wav"], help="file extensions to read (only .wav is supported)")
    ap.add_argument("--coarse_ckpt", "--Interface.coarse_ckpt", dest="coarse_ckpt", default=None)
    ap.add_argument("--coarse2fine_ckpt", "--Interface.coarse2fine_ckpt", dest="coarse2fine_ckpt", default=None)
    ap.add_argument("--codec_ckpt", "--Interface.codec_ckpt", dest="codec_ckpt", default=None)
    ap.add_argument("--device", default="cuda")
    a = ap.parse_args(argv)
    find_files(a.sources, a.ext)  # refuse an unreadable --ext before loading any model
    from .interface import Interface
    ckpts = dict(coarse_ckpt=a.coarse_ckpt, coarse2fine_ckpt=a.coarse2fine_ckpt, codec_ckpt=a.codec_ckpt)
    if all(v is None for v in ckpts.values()):
        interface = Interface.default(device=a.device)
    else:
        models = Interface.models_dir()
        defaults = dict(coarse_ckpt=models / "coarse.pth", coarse2fine_ckpt=models / "c2f.pth",
                        codec_ckpt=models / "codec.pth")
        interface = Interface(**{k: v if v is not None else defaults[k] for k, v in ckpts.items()}, device=a.device)
    done = experiment(interface, a.sources, a.output_dir, a.max_excerpts, a.exp_type, a.seed, a.ext)
    print(f"wrote {len(done)} excerpts x {len(EXP_REGISTRY[a.exp_type])} conditions under {a.output_dir}")


if __name__ == "__main__":
    main()
