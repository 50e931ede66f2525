"""Validation metrics of the reference's training script (scripts/exp/train.py:155-213, 327-371) from a forward's
logits: the label-smoothed cross-entropy over the masked tokens and top-1 / top-25 accuracy split by mask ratio and by
masked / unmasked position, computed by the kernels of csrc/validate.cu (DESIGN.md §12).  VampNet.validate is the
user-facing entry; xent_metrics is the launch it makes.

The evaluation script's audio metric, audiotools' multi-scale MelSpectrogramLoss, and the mel spectrogram under it,
computed by the kernels of csrc/mel.cu (DESIGN.md §13); vampnet_b200.eval scores experiment directories with it."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

# the reference's output keys, in its order (train.py:366, 182-213); also the order of the kernel's 9 outputs
KEYS = ("loss",) + tuple(f"accuracy-{s}-{e}/top{k}/{sel}" for s, e in ((0, 0.5), (0.5, 1.0)) for k in (1, 25)
                         for sel in ("unmasked", "masked"))


def xent_metrics(logits: torch.Tensor, z: torch.Tensor, mask: torch.Tensor, r: torch.Tensor, n_conditioning_codebooks: int,
                 label_smoothing: float = 0.1, return_ambiguous: bool = False):
    """logits (B, S, V) fp32, z and mask (B, C, T) int64, r (B,): all on one CUDA device; S = T * (C - ncc).
    Returns the 9 metrics in KEYS order as an fp32 (9,) tensor on that device without synchronising, and with
    return_ambiguous also the int32 (9,) counts of rows whose top-k decision is a tie at the k-th place."""
    B, C_, T = z.shape
    ncc = int(n_conditioning_codebooks)
    V = logits.shape[-1]
    dev = logits.device
    if logits.dtype != torch.float32 or tuple(logits.shape) != (B, T * (C_ - ncc), V):
        raise ValueError(f"xent_metrics: logits must be fp32 (B, T * (C - ncc), V) = ({B}, {T * (C_ - ncc)}, V), got "
                         f"{logits.dtype} {tuple(logits.shape)}")
    if tuple(mask.shape) != (B, C_, T):
        raise ValueError(f"xent_metrics: mask {tuple(mask.shape)} must have z's shape {(B, C_, T)}")
    logits = logits.contiguous()
    z = z.to(dev, torch.int64).contiguous()
    mask = mask.to(dev, torch.int64).contiguous()
    r = r.to(dev, torch.float64).contiguous()
    L = _lib.lib()
    ws, ws_bytes = _lib.workspace(dev, L.vnb_xent_metrics_workspace_bytes, B, T * (C_ - ncc))
    out = torch.empty(len(KEYS), dtype=torch.float32, device=dev)
    amb = torch.empty(len(KEYS), dtype=torch.int32, device=dev) if return_ambiguous else None
    with torch.cuda.device(dev):
        _lib.check(L.vnb_xent_metrics(_lib.ptr(logits), _lib.ptr(z), _lib.ptr(mask), _lib.ptr(r), B, C_, T, ncc, V,
                                      float(label_smoothing), _lib.ptr(ws), ws_bytes, _lib.ptr(out),
                                      _lib.ptr(amb) if amb is not None else None, _lib.stream_ptr(dev)))
    return (out, amb) if return_ambiguous else out


# ---------------------------------------------------------------------------------------------------- mel distance
MEL_MIN_NFFT, MEL_MAX_NFFT = 32, 4096  # csrc/mel.cu: power-of-two transforms in this range


def default_stft(sample_rate: int):
    """audiotools' default (window_length, hop_length) for a sample rate: 2 ** ceil(log2(0.032 sr)) and a quarter."""
    w = int(2 ** np.ceil(np.log2(0.032 * sample_rate)))
    return w, w // 4


def _check_window(window_length: int, window_type):
    if window_type not in (None, "hann"):
        raise ValueError(f"window_type {window_type!r}: only the periodic Hann window (None or 'hann') is supported")
    w = int(window_length)
    if w < MEL_MIN_NFFT or w > MEL_MAX_NFFT or w & (w - 1):
        raise ValueError(f"window_length {w}: a power of two in {MEL_MIN_NFFT}..{MEL_MAX_NFFT} is supported")
    return w


def _scale(sample_rate, n_mels, mel_fmin, mel_fmax, window_length, hop_length):
    fmax = float(sample_rate) / 2 if mel_fmax is None else float(mel_fmax)
    return _lib.MelScale(int(window_length), int(hop_length), int(n_mels), float(mel_fmin), fmax)


def _on_cuda(t: torch.Tensor, who: str) -> torch.Tensor:
    """t as contiguous fp32 on a CUDA device: its own, or the current one for a CPU tensor."""
    if t.device.type != "cuda":
        if not torch.cuda.is_available():
            raise RuntimeError(f"{who}: no CUDA device; vampnet_b200 runs its kernels on the GPU only")
        t = t.to(f"cuda:{torch.cuda.current_device()}")
    return t.float().contiguous()


def mel_spectrogram(samples: torch.Tensor, sample_rate: int, n_mels: int = 80, mel_fmin: float = 0.0,
                    mel_fmax: float = None, window_length: int = None, hop_length: int = None,
                    window_type: str = None) -> torch.Tensor:
    """audiotools' AudioSignal.mel_spectrogram of (B, C, N) samples: (B, C, n_mels, 1 + N // hop) fp32 on the samples'
    device, without a host sync on a CUDA input.  A CPU input is copied to the current CUDA device and back."""
    w0, h0 = default_stft(sample_rate)
    w = _check_window(w0 if window_length is None else window_length, window_type)
    hop = h0 if hop_length is None else int(hop_length)
    B, Ch, N = samples.shape
    x = _on_cuda(samples, "mel_spectrogram")
    sc = _scale(sample_rate, n_mels, mel_fmin, mel_fmax, w, hop)
    dev = x.device
    out = torch.empty((B, Ch, int(n_mels), 1 + N // max(hop, 1)), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().vnb_mel_spectrogram(_lib.ptr(x), B * Ch, N, int(sample_rate), C.byref(sc), _lib.ptr(out),
                                                  _lib.stream_ptr(dev)))
    return out.to(samples.device)


class MelSpectrogramLoss(torch.nn.Module):
    """audiotools.metrics.spectral.MelSpectrogramLoss, forward only (DESIGN.md §13): for each scale (n_mels, fmin,
    fmax, window w, hop w // 4), log_weight * L1(log10(clamp(X, eps) ** pow), log10(clamp(Y, eps) ** pow)) +
    mag_weight * L1(X, Y) of the two signals' mel spectrograms, summed over scales.  ``weight`` is stored for training
    loops and not applied, as in audiotools.  Supported: loss_fn an nn.L1Loss with reduction "mean", match_stride
    False, window_type None or "hann", window lengths that are powers of two in 32..4096; anything else raises
    ValueError."""

    def __init__(self, n_mels=[150, 80], window_lengths=[2048, 512], loss_fn=torch.nn.L1Loss(),
                 clamp_eps: float = 1e-5, mag_weight: float = 1.0, log_weight: float = 1.0, pow: float = 2.0,
                 weight: float = 1.0, match_stride: bool = False, mel_fmin=[0.0, 0.0], mel_fmax=[None, None],
                 window_type: str = None):
        super().__init__()
        if not isinstance(loss_fn, torch.nn.L1Loss) or loss_fn.reduction != "mean":
            raise ValueError("MelSpectrogramLoss: only loss_fn = nn.L1Loss(reduction='mean') is supported")
        if match_stride:
            raise ValueError("MelSpectrogramLoss: match_stride=True is not supported")
        if not (len(n_mels) == len(window_lengths) == len(mel_fmin) == len(mel_fmax)):
            raise ValueError("MelSpectrogramLoss: n_mels, window_lengths, mel_fmin and mel_fmax must have one entry "
                             "per scale")
        self.window_lengths = [_check_window(w, window_type) for w in window_lengths]
        self.n_mels, self.mel_fmin, self.mel_fmax = list(n_mels), list(mel_fmin), list(mel_fmax)
        self.loss_fn, self.clamp_eps, self.mag_weight, self.log_weight = loss_fn, clamp_eps, mag_weight, log_weight
        self.pow, self.weight, self.match_stride, self.window_type = pow, weight, match_stride, window_type

    def _launch(self, x, y, per_item: bool):
        if x.sample_rate != y.sample_rate or tuple(x.audio_data.shape) != tuple(y.audio_data.shape):
            raise ValueError(f"MelSpectrogramLoss: signals differ: {tuple(x.audio_data.shape)} at {x.sample_rate} Hz "
                             f"and {tuple(y.audio_data.shape)} at {y.sample_rate} Hz")
        home = x.audio_data.device
        xs = _on_cuda(x.audio_data, "MelSpectrogramLoss")
        dev = xs.device
        ys = y.audio_data.to(dev).float().contiguous()
        B, Ch, N = xs.shape
        sr = int(x.sample_rate)
        n = len(self.n_mels)
        scales = (_lib.MelScale * n)(*[_scale(sr, m, lo, hi, w, w // 4) for m, lo, hi, w in
                                       zip(self.n_mels, self.mel_fmin, self.mel_fmax, self.window_lengths)])
        L = _lib.lib()
        ws, ws_bytes = _lib.workspace(dev, L.vnb_mel_workspace_bytes, B, Ch, N, sr, scales, n)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        items = torch.empty(B, dtype=torch.float32, device=dev) if per_item else None
        with torch.cuda.device(dev):
            _lib.check(L.vnb_mel_loss(_lib.ptr(xs), _lib.ptr(ys), B, Ch, N, sr, scales, n, float(self.clamp_eps),
                                      float(self.pow), float(self.log_weight), float(self.mag_weight), _lib.ptr(ws),
                                      ws_bytes, _lib.ptr(loss), _lib.ptr(items), _lib.stream_ptr(dev)))
        return (items if per_item else loss).to(home)

    def forward(self, x, y) -> torch.Tensor:
        """x, y: AudioSignals of the same (B, C, N) shape and sample rate.  A 0-d fp32 tensor on x's device, returned
        without a host sync for CUDA signals."""
        return self._launch(x, y, per_item=False)

    def per_item(self, x, y) -> torch.Tensor:
        """The loss of each batch item on its own, (B,) fp32: item b equals forward() of item b alone, bit for bit,
        and forward() is their mean up to fp32 rounding."""
        return self._launch(x, y, per_item=True)
