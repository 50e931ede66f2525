"""Pitch shift on the GPU: torch_pitch_shift 1.2's ``pitch_shift`` and ``get_fast_shifts``.

The app shifts its preprocessed signal with ``torch_pitch_shift.pitch_shift`` before encoding (app.py:59-66,
183-184).  That package composes torch.stft, torchaudio's phase vocoder, torch.istft and torchaudio's sinc resampler,
and its resampler materialises a (new_freq / g) x (orig_freq / g) filter table, gigabytes for half of the app's
semitone slider.  Here the same composition runs as CUDA kernels (csrc/pitch.cu) in float64 between fp32 ends, and
the resampler evaluates only each output's nonzero taps.  DESIGN.md §11 has the definition and the numerics.
"""
from __future__ import annotations

from fractions import Fraction
from itertools import product

import torch

from . import _lib


def shift_params(shift, sample_rate: int, bins_per_octave: int = 12, n_fft: int = 0, hop_length: int = 0):
    """(n_fft, hop, new_freq, rate) exactly as torch_pitch_shift derives them: a Fraction is the frequency ratio
    itself, anything else is a shift in bins of ``bins_per_octave`` per octave."""
    n_fft = int(n_fft) or int(sample_rate) // 64
    hop = int(hop_length) or n_fft // 32
    ratio = shift if isinstance(shift, Fraction) else 2.0 ** (float(shift) / bins_per_octave)
    return n_fft, hop, int(sample_rate / ratio), float(1 / ratio)


def pitch_shift(input: torch.Tensor, shift, sample_rate: int, bins_per_octave: int = 12, n_fft: int = 0,
                hop_length: int = 0) -> torch.Tensor:
    """Shift the pitch of ``input`` ((B, C, N) float32) by ``shift`` bins, or by the ratio of a Fraction shift, keeping
    its length.  Each of the B * C rows is shifted on its own.  A CUDA input returns without a host sync; a CPU input
    is copied to the current CUDA device, shifted there and copied back."""
    if not torch.is_tensor(input) or input.dtype != torch.float32:
        raise RuntimeError(f"pitch_shift: input must be a float32 tensor, got {getattr(input, 'dtype', type(input))}")
    if input.ndim != 3:
        raise RuntimeError(f"pitch_shift: input must be (batch, channels, samples), got {tuple(input.shape)}")
    if input.device.type != "cuda":
        if not torch.cuda.is_available():
            raise RuntimeError("pitch_shift: no CUDA device; vampnet_b200 runs its kernels on the GPU only")
        out = pitch_shift(input.to(f"cuda:{torch.cuda.current_device()}"), shift, sample_rate, bins_per_octave, n_fft,
                          hop_length)
        return out.to(input.device)
    B, Ch, N = input.shape
    n_fft, hop, new_freq, rate = shift_params(shift, sample_rate, bins_per_octave, n_fft, hop_length)
    x = input.reshape(B * Ch, N).contiguous()
    L = _lib.lib()
    args = (B * Ch, N, int(sample_rate), new_freq, n_fft, hop, rate)
    dev = input.device
    workspace, ws_bytes = _lib.workspace(dev, L.vnb_pitch_workspace_bytes, *args)
    with torch.cuda.device(dev):
        out = torch.empty_like(x)
        _lib.check(L.vnb_pitch_shift(_lib.ptr(x), *args, _lib.ptr(workspace), ws_bytes, _lib.ptr(out),
                                     _lib.stream_ptr(dev)))
    return out.reshape(B, Ch, N)


def get_fast_shifts(sample_rate: int, condition=lambda x: x >= 0.5 and x <= 2 and x != 1) -> list:
    """The ratios i / j (Fractions) that ``condition`` accepts, where i and j are products of non-empty sub-multisets
    of the prime factors of ``sample_rate``: the shifts whose resampler tables stay small.  Sorted."""
    n, factors, p = int(sample_rate), [], 2
    while p * p <= n:
        while n % p == 0:
            factors.append(p)
            n //= p
        p += 1
    if n > 1:
        factors.append(n)
    products = set()
    for keep in product((0, 1), repeat=len(factors)):
        if not any(keep):
            continue
        v = 1
        for k, f in zip(keep, factors):
            v *= f if k else 1
        products.add(v)
    return sorted({Fraction(i, j) for i in products for j in products if condition(Fraction(i, j))})


def time_steps(F: int, rate: float, device="cuda") -> torch.Tensor:
    """The vocoder's time steps for F frames as the kernels compute them (test hook)."""
    n = int(torch.arange(0, F, rate, dtype=torch.float64).numel())
    out = torch.empty(n, dtype=torch.float32, device=device)
    with torch.cuda.device(out.device):
        _lib.check(_lib.lib().vnb_dbg_pitch_time_steps(float(rate), n, _lib.ptr(out), _lib.stream_ptr(out.device)))
    return out
