"""AudioSignal — the subset of ``audiotools.AudioSignal`` the hot path touches (reference
vampnet/interface.py:206-224, transformer.py:670-675, app.py:175-178, 247-248): a (batch, channels, samples)
float tensor + sample rate with resample / to_mono / BS.1770 loudness normalise / peak clamp, all as torch
ops on the signal's own device (SURVEY.md §8f row f-3).  ``descript-audiotools`` itself is a third-party,
unpinned dependency that is not present here, so numerical parity with it is unpinned.
"""
from __future__ import annotations

import math
import wave
from pathlib import Path

import numpy as np
import torch


class AudioSignal:
    def __init__(self, audio_path_or_array, sample_rate: int = None, device=None):
        if isinstance(audio_path_or_array, (str, Path)):
            data, sr = _read_wav(str(audio_path_or_array))
            audio, sample_rate = torch.from_numpy(data), sr if sample_rate is None else sample_rate
        elif isinstance(audio_path_or_array, np.ndarray):
            audio = torch.from_numpy(audio_path_or_array)
        elif torch.is_tensor(audio_path_or_array):
            audio = audio_path_or_array
        else:
            raise ValueError("audio_path_or_array must be a path, a numpy array or a torch tensor")
        assert sample_rate is not None, "sample_rate is required for array input"
        if audio.ndim == 1:
            audio = audio[None, None, :]
        elif audio.ndim == 2:
            audio = audio[None]
        assert audio.ndim == 3, "audio must be (batch, channels, samples)"
        self.audio_data = audio.float() if not audio.is_floating_point() else audio
        self.sample_rate = int(sample_rate)
        if device is not None:
            self.to(device)

    # ---- views -----------------------------------------------------------------------------
    @property
    def samples(self):
        return self.audio_data

    @samples.setter
    def samples(self, v):
        self.audio_data = v

    @property
    def device(self):
        return self.audio_data.device

    @property
    def batch_size(self):
        return self.audio_data.shape[0]

    @property
    def num_channels(self):
        return self.audio_data.shape[1]

    @property
    def signal_length(self):
        return self.audio_data.shape[-1]

    length = signal_length

    @property
    def duration(self):
        return self.signal_length / self.sample_rate

    signal_duration = duration

    def clone(self):
        return AudioSignal(self.audio_data.clone(), self.sample_rate)

    def to(self, device):
        self.audio_data = self.audio_data.to(device)
        return self

    def cpu(self):
        return self.to("cpu")

    def cuda(self):
        return self.to("cuda")

    def detach(self):
        self.audio_data = self.audio_data.detach()
        return self

    def numpy(self):
        return self.audio_data.detach().cpu().numpy()

    # ---- transforms --------------------------------------------------------------------------
    def to_mono(self):
        self.audio_data = self.audio_data.mean(1, keepdim=True)
        return self

    def trim(self, before: int, after: int):
        """Drop `before` samples at the start and `after` at the end, in place (audiotools' trim: after == 0 keeps the
        end, a negative count is a Python slice bound)."""
        if after == 0:
            self.audio_data = self.audio_data[..., before:]
        else:
            self.audio_data = self.audio_data[..., before:-after]
        return self

    def truncate_samples(self, length_in_samples: int):
        """Keep the first `length_in_samples` samples, in place (audiotools' truncate_samples)."""
        self.audio_data = self.audio_data[..., :int(length_in_samples)]
        return self

    def mel_spectrogram(self, n_mels: int = 80, mel_fmin: float = 0.0, mel_fmax: float = None,
                        window_length: int = None, hop_length: int = None, window_type: str = None):
        """(batch, channels, n_mels, frames) fp32 magnitude mel spectrogram, audiotools' definition, computed on the
        GPU (vampnet_b200.metrics.mel_spectrogram, DESIGN.md §13)."""
        from .metrics import mel_spectrogram
        return mel_spectrogram(self.audio_data, self.sample_rate, n_mels, mel_fmin, mel_fmax, window_length,
                               hop_length, window_type)

    def resample(self, sample_rate: int):
        """Band-limited (Kaiser-windowed sinc) polyphase resampling as one strided conv."""
        sample_rate = int(sample_rate)
        if sample_rate == self.sample_rate:
            return self
        g = math.gcd(sample_rate, self.sample_rate)
        up, down = sample_rate // g, self.sample_rate // g
        x = self.audio_data
        B, Cn, N = x.shape
        zeros = 24
        cutoff = 0.5 * 0.945 / max(up, down)  # cycles/sample at the up-sampled rate: 94.5 % of the lower Nyquist
        half = zeros * max(up, down)
        t = torch.arange(-half, half + 1, device=x.device, dtype=torch.float64)
        h = 2 * cutoff * torch.sinc(2 * cutoff * t) * torch.kaiser_window(2 * half + 1, periodic=False, beta=8.6,
                                                                         dtype=torch.float64, device=x.device)
        h = (h * up).float()
        xu = torch.zeros(B * Cn, 1, N * up, device=x.device)
        xu[:, 0, ::up] = x.reshape(B * Cn, N)
        y = torch.nn.functional.conv1d(xu, h.flip(0)[None, None], padding=half, stride=down)
        n_out = int(math.ceil(N * up / down))
        self.audio_data = y[..., :n_out].reshape(B, Cn, -1)
        self.sample_rate = sample_rate
        return self

    def loudness(self, block_size: float = 0.400):
        """Integrated loudness in LUFS, ITU-R BS.1770-4: K-weighting, 400 ms blocks with 75 % overlap,
        absolute (-70 LUFS) and relative (-10 LU) gating.  Returns a (batch,) tensor."""
        x = self.audio_data
        B, Cn, N = x.shape
        min_len = int(block_size * self.sample_rate)
        if N < min_len:
            x = torch.nn.functional.pad(x, (0, min_len - N))
            N = min_len
        xw = _k_weight(x, self.sample_rate)
        blk = int(block_size * self.sample_rate)
        hop = int(blk * 0.25)
        frames = xw.unfold(-1, blk, hop)  # (B, C, nblocks, blk)
        z = frames.pow(2).mean(-1)  # mean square per block and channel
        G = torch.ones(Cn, device=x.device)
        if Cn >= 4:
            G[3:] = 1.41
        zsum = (z * G[None, :, None]).sum(1)  # (B, nblocks)
        lj = -0.691 + 10 * torch.log10(zsum.clamp_min(1e-12))
        # two-stage gating, batched (no per-item loop, no host synchronisation): absolute gate at -70 LUFS, then the
        # relative gate 10 LU below the mean of the blocks that passed it; items with no block left report -70
        def gated_mean(keep):
            n = keep.sum(1)
            return (zsum * keep).sum(1) / n.clamp_min(1), n
        keep = lj > -70.0
        m1, n1 = gated_mean(keep)
        rel = -0.691 + 10 * torch.log10(m1.clamp_min(1e-12)) - 10.0
        keep2 = keep & (lj > rel[:, None])
        m2, n2 = gated_mean(keep2)
        out = -0.691 + 10 * torch.log10(m2.clamp_min(1e-12))
        floor = torch.full_like(out, -70.0)
        return torch.where((n1 > 0) & (n2 > 0), out, floor).clamp_min(-70.0)

    def normalize(self, db=-24.0):
        """Scale to the target integrated loudness: a number, or a tensor broadcast over the batch (app.py:248 passes
        the input's measured loudness, one value, to a batch of generated variations)."""
        ref = self.loudness()
        target = torch.as_tensor(db, dtype=ref.dtype, device=ref.device).reshape(-1)
        gain = torch.exp((target - ref) * math.log(10.0) / 20.0)
        self.audio_data = self.audio_data * gain[:, None, None]
        return self

    def ensure_max_of_audio(self, max_val: float = 1.0):
        peak = self.audio_data.abs().amax(dim=(1, 2), keepdim=True)
        scale = torch.where(peak > max_val, max_val / peak.clamp_min(1e-12), torch.ones_like(peak))
        self.audio_data = self.audio_data * scale
        return self

    def write(self, path):
        data = self.audio_data[0].detach().cpu().clamp(-1, 1).numpy()
        pcm = (data.T * 32767.0).astype("<i2")
        with wave.open(str(path), "wb") as w:
            w.setnchannels(data.shape[0])
            w.setsampwidth(2)
            w.setframerate(self.sample_rate)
            w.writeframes(pcm.tobytes())
        return self

    def __repr__(self):
        return f"AudioSignal(shape={tuple(self.audio_data.shape)}, sample_rate={self.sample_rate}, device={self.device})"


def _read_wav(path):
    with wave.open(path, "rb") as w:
        n, ch, sw, sr = w.getnframes(), w.getnchannels(), w.getsampwidth(), w.getframerate()
        raw = w.readframes(n)
    if sw == 2:
        a = np.frombuffer(raw, dtype="<i2").astype(np.float32) / 32768.0
    elif sw == 4:
        a = np.frombuffer(raw, dtype="<i4").astype(np.float32) / 2147483648.0
    elif sw == 1:
        a = (np.frombuffer(raw, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
    else:
        raise ValueError(f"unsupported sample width {sw}")
    return a.reshape(-1, ch).T.copy(), sr


def _biquad_response(b, a, w):
    e1, e2 = torch.exp(-1j * w), torch.exp(-2j * w)
    return (b[0] + b[1] * e1 + b[2] * e2) / (a[0] + a[1] * e1 + a[2] * e2)


def _k_weight(x, sr):
    """BS.1770 K-weighting (high-shelf pre-filter + RLB high-pass) applied in the frequency domain."""
    N = x.shape[-1]
    nfft = 1 << (N + 4096 - 1).bit_length()
    w = torch.arange(nfft // 2 + 1, device=x.device, dtype=torch.float64) * (2 * math.pi / nfft)
    # Stage 1, shelving pre-filter, and stage 2, RLB high-pass: the BS.1770 48 kHz biquads re-derived for any
    # sample rate through the bilinear-transform parameters (f0, G, Q) that reproduce the standard's table.
    f0, G, Q = 1681.974450955533, 3.999843853973347, 0.7071752369554196
    K = math.tan(math.pi * f0 / sr)
    Vh = 10.0 ** (G / 20.0)
    Vb = Vh ** 0.4996667741545416
    a0 = 1.0 + K / Q + K * K
    b1 = [(Vh + Vb * K / Q + K * K) / a0, 2.0 * (K * K - Vh) / a0, (Vh - Vb * K / Q + K * K) / a0]
    a1 = [1.0, 2.0 * (K * K - 1.0) / a0, (1.0 - K / Q + K * K) / a0]
    f0, Q = 38.13547087602444, 0.5003270373238773
    K = math.tan(math.pi * f0 / sr)
    a0 = 1.0 + K / Q + K * K
    b2 = [1.0, -2.0, 1.0]
    a2 = [1.0, 2.0 * (K * K - 1.0) / a0, (1.0 - K / Q + K * K) / a0]
    H = (_biquad_response(b1, a1, w) * _biquad_response(b2, a2, w)).to(torch.complex64)
    X = torch.fft.rfft(x.float(), n=nfft)
    return torch.fft.irfft(X * H, n=nfft)[..., :N]
