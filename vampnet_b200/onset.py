"""Onset detection on the GPU: librosa 0.10's ``onset.onset_detect(y, sr, hop_length=H, backtrack=True)`` (the detector
behind the reference's ``mask.onset_mask``, vampnet/mask.py:203-226, and the app's ``onsets()`` helper, app.py:69-78)
restated as CUDA kernels (csrc/onset.cu).  Everything stays on the device and nothing synchronises, so an onset prompt
can be built in the middle of a request without a host round trip.  DESIGN.md §9 has the numerics.
"""
from __future__ import annotations

from typing import NamedTuple

import torch

from . import _lib


class Onsets(NamedTuple):
    """Device tensors.  Row b's onset frames are ``frames[b, :counts[b]]``, in increasing order."""
    frames: torch.Tensor    # (B, F) int32, F = 1 + N // hop_length
    counts: torch.Tensor    # (B,) int32
    envelope: torch.Tensor  # (B, F) float32, the normalised onset strength the peaks were picked from


def n_frames(n_samples: int, hop_length: int) -> int:
    return 1 + n_samples // hop_length


def as_rows(samples: torch.Tensor, who: str) -> torch.Tensor:
    """``samples`` ((N,) or (B, N) float32 on a CUDA device) as a contiguous (B, N) tensor; RuntimeError otherwise."""
    if not torch.is_tensor(samples) or samples.dtype != torch.float32:
        raise RuntimeError(f"{who}: samples must be a float32 tensor, got {getattr(samples, 'dtype', type(samples))}")
    if samples.device.type != "cuda":
        raise RuntimeError(f"{who}: samples must be on a CUDA device, got {samples.device}")
    if samples.ndim == 1:
        samples = samples[None]
    if samples.ndim != 2:
        raise RuntimeError(f"{who}: samples must be (N,) or (B, N), got {tuple(samples.shape)}")
    return samples.contiguous()


def onset_detect(samples: torch.Tensor, sample_rate: int, hop_length: int, backtrack: bool = True) -> Onsets:
    """Onsets of every row of ``samples`` ((N,) or (B, N) float32 on a CUDA device), each row analysed on its own.
    With ``backtrack`` each onset moves to the preceding local minimum of the envelope, as librosa's does."""
    samples = as_rows(samples, "onset_detect")
    B, N = samples.shape
    L = _lib.lib()
    hop = int(hop_length)
    F = n_frames(N, hop) if hop > 0 else 1
    dev = samples.device
    # out-of-range shapes go straight to vnb_onset_detect, which names them
    workspace, ws_bytes = (_lib.workspace(dev, L.vnb_onset_workspace_bytes, B, N, hop) if B > 0 and N > 0 and hop > 0
                           else (None, 0))
    with torch.cuda.device(dev):
        frames = torch.empty(max(B, 1), F, dtype=torch.int32, device=dev)
        counts = torch.empty(max(B, 1), dtype=torch.int32, device=dev)
        envelope = torch.empty(max(B, 1), F, dtype=torch.float32, device=dev)
        _lib.check(L.vnb_onset_detect(_lib.ptr(samples), B, N, int(sample_rate), hop, int(bool(backtrack)),
                                      _lib.ptr(workspace), ws_bytes, _lib.ptr(envelope), _lib.ptr(frames),
                                      _lib.ptr(counts), _lib.stream_ptr(dev)))
    return Onsets(frames, counts, envelope)


def onset_mask(onsets: Onsets, z: torch.Tensor, width: int) -> torch.Tensor:
    """``ones_like(z)`` with ``mask[:, :, idx - width:idx + width] = 0`` for every onset (reference mask.py:222-225,
    Python slice semantics included).  One onset row applies to every row of z; B rows apply row by row."""
    if z.ndim != 3:
        raise RuntimeError(f"onset_mask: z must be (batch, n_codebooks, seq), got {tuple(z.shape)}")
    if z.device != onsets.frames.device:
        raise RuntimeError(f"onset_mask: z is on {z.device}, the onsets on {onsets.frames.device}")
    B, Cb, T = z.shape
    mask = torch.empty(B, Cb, T, dtype=torch.int64, device=z.device)
    if mask.numel():
        with torch.cuda.device(z.device):
            _lib.check(_lib.lib().vnb_onset_mask(_lib.ptr(onsets.frames), _lib.ptr(onsets.counts),
                                                 onsets.frames.shape[0], onsets.frames.shape[1], int(width),
                                                 _lib.ptr(mask), B, Cb, T, _lib.stream_ptr(z.device)))
    return mask if z.dtype == torch.int64 else mask.to(z.dtype)
