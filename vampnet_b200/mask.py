"""Mask algebra used by Interface.build_mask — same function names, argument meaning and results as the
reference's vampnet/mask.py (cited per function), written as vectorised tensor ops that run on whatever
device the codes live on (the reference's periodic_mask is an O(B*T) Python loop with one
torch.bernoulli per frame, mask.py:111-125).

Where the reference consumes the global torch RNG we consume it in the same order with the same calls,
so a caller that seeds torch gets the same masks from either implementation.
"""
from __future__ import annotations

import torch


def _scalar_to_batch(x, batch_size):
    return torch.tensor(x).repeat(batch_size)  # reference util.py:6-7


def _gamma(r):
    """Cosine schedule (mask.py:8-9)."""
    return (r * torch.pi / 2).cos().clamp(1e-10, 1.0)


def _invgamma(y):
    if not torch.is_tensor(y):
        y = torch.tensor(y)[None]
    return 2 * y.acos() / torch.pi


def full_mask(x: torch.Tensor):
    assert x.ndim == 3, "x must be (batch, n_codebooks, seq)"
    return torch.ones_like(x).long()


def empty_mask(x: torch.Tensor):
    assert x.ndim == 3, "x must be (batch, n_codebooks, seq)"
    return torch.zeros_like(x).long()


def apply_mask(x: torch.Tensor, mask: torch.Tensor, mask_token: int, check: bool = True):
    """x*(1-m) + token*m (mask.py:24-38).  The reference checks binariness with two host syncs; one here.
    check=False skips that device->host round trip: the Interface validates a mask ONCE per call and then slices it,
    so the chunk loops run without synchronising (SURVEY.md 8f row f-2)."""
    assert mask.ndim == 3, f"mask must be (batch, n_codebooks, seq), but got {mask.ndim}"
    assert mask.shape == x.shape, f"mask must be same shape as x, but got {mask.shape} and {x.shape}"
    assert mask.dtype == torch.long, f"mask must be long dtype, but got {mask.dtype}"
    if check:
        assert bool(((mask == 0) | (mask == 1)).all()), "mask must be binary"
    return torch.where(mask.bool(), torch.full_like(x, mask_token), x), mask


def random(x: torch.Tensor, r: torch.Tensor):
    """Bernoulli(gamma(r)) per element (mask.py:40-54)."""
    assert x.ndim == 3, "x must be (batch, n_codebooks, seq)"
    if not isinstance(r, torch.Tensor):
        r = _scalar_to_batch(r, x.shape[0]).to(x.device)
    probs = torch.ones_like(x) * _gamma(r)[:, None, None]
    return torch.bernoulli(probs).round().long()


def linear_random(x: torch.Tensor, r):
    """Bernoulli(r) per element (mask.py:56-73)."""
    assert x.ndim == 3, "x must be (batch, n_codebooks, seq)"
    if not isinstance(r, torch.Tensor):
        r = _scalar_to_batch(r, x.shape[0]).to(x.device).float()
        r = r[:, None, None]
    probs = torch.ones_like(x).float().expand(x.shape[0], x.shape[1], -1) * r
    return torch.bernoulli(probs).round().long()


def inpaint(x: torch.Tensor, n_prefix, n_suffix):
    """Unmask a prefix and/or suffix of frames (mask.py:75-99)."""
    assert n_prefix is not None and n_suffix is not None
    B, _, T = x.shape
    mask = full_mask(x)
    t = torch.arange(T, device=x.device)[None, None, :]

    def per_batch(n):
        if not isinstance(n, torch.Tensor):
            n = _scalar_to_batch(n, B)
        return n.to(x.device).long().view(B, 1, 1)

    if torch.as_tensor(n_prefix).max() > 0:
        mask = torch.where(t < per_batch(n_prefix), torch.zeros_like(mask), mask)
    if torch.as_tensor(n_suffix).max() > 0:
        ns = per_batch(n_suffix)
        mask = torch.where((t >= T - ns) & (ns > 0), torch.zeros_like(mask), mask)
    return mask


def periodic_mask(x: torch.Tensor, period, width: int = 1, random_roll=False):
    """Zero `width` frames around every multiple of `period` (mask.py:101-131)."""
    mask = full_mask(x)
    if isinstance(period, int) and period == 0:
        return mask
    B, _, T = x.shape
    if not isinstance(period, torch.Tensor):
        period = _scalar_to_batch(period, B)
    t = torch.arange(T, device=x.device)
    for i, factor in enumerate(period.tolist()):
        if factor == 0:
            continue
        centres = torch.arange(0, T, factor, device=x.device)  # j with j % factor == 0
        lo = (centres - width // 2).clamp(min=0)
        hi = (centres + width // 2).clamp(max=T - 1) + 1
        hit = ((t[None, :] >= lo[:, None]) & (t[None, :] < hi[:, None])).any(0)
        mask[i, :, hit] = 0
        # keep the global RNG stream aligned with the reference, which draws bernoulli(ones(n)) per hit
        for l, h in zip(lo.tolist(), hi.tolist()):
            torch.bernoulli(torch.ones(h - l))
    if random_roll:
        offset = torch.randint(0, int(period[0]), (1,))
        mask = torch.roll(mask, offset.item(), dims=-1)
    return mask


def codebook_unmask(mask: torch.Tensor, n_conditioning_codebooks: int):
    """mask.py:133-142."""
    if n_conditioning_codebooks is None:
        return mask
    mask = mask.clone()
    mask[:, :n_conditioning_codebooks, :] = 0
    return mask


def codebook_mask(mask: torch.Tensor, val1: int, val2: int = None):
    """Mask every codebook >= val1 (mask.py:144-153)."""
    mask = mask.clone()
    mask[:, val1:, :] = 1
    return mask


def mask_and(mask1: torch.Tensor, mask2: torch.Tensor):
    assert mask1.shape == mask2.shape, "masks must be same shape"
    return torch.min(mask1, mask2)


def dropout(mask: torch.Tensor, p: float):
    """Re-mask int(T*p) random frames (mask.py:162-173)."""
    tsteps = mask.shape[-1]
    idxs = torch.randint(0, tsteps, (int(tsteps * p),))
    mask = mask.clone()
    mask[:, :, idxs.to(mask.device)] = 1
    return mask.long()


def mask_or(mask1: torch.Tensor, mask2: torch.Tensor):
    assert mask1.shape == mask2.shape, f"masks must be same shape, but got {mask1.shape} and {mask2.shape}"
    assert mask1.max() <= 1 and mask2.max() <= 1 and mask1.min() >= 0 and mask2.min() >= 0, "masks must be binary"
    return (mask1 + mask2).clamp(0, 1)


def time_stretch_mask(x: torch.Tensor, stretch_factor: int):
    """mask.py:188-201."""
    assert stretch_factor >= 1, "stretch factor must be >= 1"
    c_seq_len = x.shape[-1]
    x = x.repeat_interleave(stretch_factor, dim=-1)[:, :, :c_seq_len]
    return periodic_mask(x, stretch_factor, width=1)


def onset_mask(sig, z: torch.Tensor, interface, width: int = 1):
    """mask.py:203-226.  A signal on a CUDA device takes the CUDA detector (vampnet_b200/onset.py: librosa 0.10's
    onset_detect restated, no host sync); a CPU signal calls librosa's detector as the reference does.  Either way only
    samples[0][0] is analysed and its onsets apply to every row of z."""
    if sig.samples.is_cuda:
        from . import onset
        det = onset.onset_detect(sig.samples[0][0].detach().float(), sig.sample_rate, interface.codec.hop_length,
                                 backtrack=True)
        if z.device != det.frames.device:  # codes held elsewhere: build the mask next to the onsets, then move it
            return onset.onset_mask(det, z.to(det.frames.device), width).to(z.device)
        return onset.onset_mask(det, z, width)
    try:
        import librosa
    except ImportError as e:  # pragma: no cover
        raise ImportError("onset_mask needs librosa (optional dependency, not part of the CUDA hot path)") from e
    idxs = librosa.onset.onset_detect(y=sig.samples[0][0].detach().cpu().numpy(), sr=sig.sample_rate,
                                      hop_length=interface.codec.hop_length, backtrack=True)
    mask = torch.ones_like(z)
    for idx in idxs:
        mask[:, :, idx - width:idx + width] = 0
    return mask
