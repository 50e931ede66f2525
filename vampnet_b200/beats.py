"""Beat tracking on the GPU and the beat-synced mask.

The reference takes its beat times from WaveBeat (vampnet/beats.py:203-223), a separate network whose package is not
available here.  ``beat_track`` restates librosa 0.10.1's classical tracker, ``beat.beat_track(y, sr, hop_length=H)``,
as CUDA kernels (csrc/beat.cu): onset strength, tempo and the dynamic programme all stay on the device and nothing
synchronises.  Its beat times differ from WaveBeat's, and it estimates no downbeats.  ``beat_mask`` builds the mask
from beat times exactly as the reference's ``Interface.make_beat_mask`` does (interface.py:241-322), random draws
included.  DESIGN.md §10 has the numerics.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch

from . import _lib
from .onset import as_rows


class Beats(NamedTuple):
    """Device tensors.  Row b's beat frames are ``frames[b, :counts[b]]``, in increasing order."""
    frames: torch.Tensor    # (B, F) int32, F = 1 + N // hop_length
    counts: torch.Tensor    # (B,) int32
    tempo: torch.Tensor     # (B,) float64 BPM, 0 where the onset envelope is all zero
    envelope: torch.Tensor  # (B, F) float32 onset strength (median over the mel bands)


def beat_track(samples: torch.Tensor, sample_rate: int, hop_length: int = 512, start_bpm: float = 120.0,
               tightness: float = 100.0, trim: bool = True) -> Beats:
    """Beats of every row of ``samples`` ((N,) or (B, N) float32 on a CUDA device), each row analysed on its own."""
    samples = as_rows(samples, "beat_track")
    B, N = samples.shape
    L = _lib.lib()
    hop = int(hop_length)
    F = 1 + N // hop if hop > 0 else 1
    dev = samples.device
    # out-of-range shapes go straight to vnb_beat_track, which names them
    workspace, ws_bytes = (_lib.workspace(dev, L.vnb_beat_workspace_bytes, B, N, hop) if B > 0 and N > 0 and hop > 0
                           else (None, 0))
    with torch.cuda.device(dev):
        frames = torch.empty(max(B, 1), F, dtype=torch.int32, device=dev)
        counts = torch.empty(max(B, 1), dtype=torch.int32, device=dev)
        tempo = torch.empty(max(B, 1), dtype=torch.float64, device=dev)
        envelope = torch.empty(max(B, 1), F, dtype=torch.float32, device=dev)
        _lib.check(L.vnb_beat_track(_lib.ptr(samples), B, N, int(sample_rate), hop, float(start_bpm), float(tightness),
                                    int(bool(trim)), _lib.ptr(workspace), ws_bytes, _lib.ptr(envelope),
                                    _lib.ptr(tempo), _lib.ptr(frames), _lib.ptr(counts), _lib.stream_ptr(dev)))
    return Beats(frames, counts, tempo, envelope)


def frames_to_time(frames, sample_rate: int, hop_length: int) -> np.ndarray:
    """librosa's frames_to_time: frames * hop / sr in float64."""
    return np.asarray(frames, dtype=np.int64) * int(hop_length) / float(sample_rate)


class BeatTracker:
    """The reference's tracker protocol (vampnet/beats.py: ``extract_beats(signal) -> (beat_times, downbeat_times)``,
    seconds as float64 numpy arrays) over ``beat_track``.  It reads ``samples[0]`` averaged over channels at the
    signal's own rate, on ``device`` (a CPU signal is copied there).  It estimates no downbeats: the second array is
    always empty."""

    def __init__(self, device="cuda", hop_length: int = 512):
        self.device = device
        self.hop_length = hop_length

    def extract_beats(self, signal):
        if signal.batch_size != 1:
            raise ValueError(f"extract_beats: one signal at a time (batch size 1), got {signal.batch_size}")
        y = signal.audio_data[0].float().mean(0).to(self.device)
        r = beat_track(y, signal.sample_rate, self.hop_length)
        frames = r.frames[0, :int(r.counts[0])].cpu().numpy()  # the one synchronisation: the host needs the times
        return frames_to_time(frames, signal.sample_rate, self.hop_length), np.zeros(0, dtype=np.float64)


def beat_mask(beats, downbeats, duration: float, s2t, n_codebooks: int, device, before_beat_s: float = 0.0,
              after_beat_s: float = 0.02, mask_downbeats: bool = True, mask_upbeats: bool = True,
              downbeat_downsample_factor: int = None, beat_downsample_factor: int = None, dropout: float = 0.0,
              invert: bool = True) -> torch.Tensor:
    """The reference's Interface.make_beat_mask after its extract_beats call (interface.py:258-322), line for line:
    beat and downbeat times in seconds (numpy arrays), the clip's duration, the Interface's s2t.  One torch.bernoulli
    draw per window on `device`, upbeats first, so the torch RNG ends where the reference leaves it."""
    beats_z, downbeats_z = s2t(beats), s2t(downbeats)
    beats_z = torch.tensor(beats_z)[~torch.isin(torch.tensor(beats_z), torch.tensor(downbeats_z))]
    beats_z = beats_z.tolist()
    downbeats_z = downbeats_z.tolist()
    seq_len = s2t(duration)
    mask = torch.zeros(seq_len, device=device)
    mask_b4 = s2t(before_beat_s)
    mask_after = s2t(after_beat_s)
    if beat_downsample_factor is not None:
        if beat_downsample_factor < 1:
            raise ValueError("mask_beat_downsample_factor must be >= 1 or None")
    else:
        beat_downsample_factor = 1
    if downbeat_downsample_factor is not None:
        if downbeat_downsample_factor < 1:
            raise ValueError("mask_beat_downsample_factor must be >= 1 or None")
    else:
        downbeat_downsample_factor = 1
    beats_z = beats_z[::beat_downsample_factor]
    downbeats_z = downbeats_z[::downbeat_downsample_factor]
    windows = (beats_z if mask_upbeats else []) + (downbeats_z if mask_downbeats else [])
    for idx in windows:
        lo, hi = int(idx - mask_b4), int(idx + mask_after)
        m = torch.ones(mask[lo:hi].shape[0], device=device)
        m = m * torch.bernoulli(m * (1 - dropout)).long()
        mask[lo:hi] = m
    mask = mask.clamp(0, 1)
    if invert:
        mask = 1 - mask
    return mask[None, None, :].bool().long().repeat(1, n_codebooks, 1)
