"""Float64 restatement of the Fréchet audio distance of the evaluation script (frechet_audio_distance with torchvggish's
VGGish, use_pca=False, use_activation=False), from the published definitions (DESIGN.md §14):

* the log-mel examples of Google's vggish_input.waveform_to_examples / mel_features.py at 16 kHz (window 400, hop 160,
  FFT 512, periodic Hann, |rfft| on the 64-band HTK matrix over 125..7500 Hz, log(mel + 0.01), 96-frame examples);
* torchvggish's VGG: six 3x3 convolutions with ReLU and four 2x2 max-pools, the (N, H, W, C) flatten, three fully
  connected layers without the last ReLU;
* frechet_audio_distance's moments (np.mean, np.cov) and calculate_frechet_distance (scipy.linalg.sqrtm).

Parity with the frechet_audio_distance package and the real checkpoint is unpinned: neither is used by the tests.  The
tests use seeded random weights (random_state_dict) with Kaiming-scaled draws, so activations stay in range."""
from __future__ import annotations

import numpy as np
import torch

SR, WIN, HOP, NFFT, NMELS, EXF = 16000, 400, 160, 512, 64, 96
FMIN, FMAX = 125.0, 7500.0
CONVS = {0: (1, 64), 3: (64, 128), 6: (128, 256), 8: (256, 256), 11: (256, 512), 13: (512, 512)}
FCS = {0: (512 * 4 * 6, 4096), 2: (4096, 4096), 4: (4096, 128)}
LAYERS = [64, "M", 128, "M", 256, 256, "M", 512, 512, "M"]  # torchvggish's make_layers


def hz_to_mel(f):
    return 1127.0 * np.log(1.0 + np.asarray(f, np.float64) / 700.0)


def htk_matrix(num_mel_bins=NMELS, num_spectrogram_bins=NFFT // 2 + 1, sr=SR, lower=FMIN, upper=FMAX):
    """mel_features.spectrogram_to_mel_matrix: (257, 64) float64."""
    bins_mel = hz_to_mel(np.linspace(0.0, sr / 2.0, num_spectrogram_bins))
    edges = np.linspace(hz_to_mel(lower), hz_to_mel(upper), num_mel_bins + 2)
    m = np.empty((num_spectrogram_bins, num_mel_bins))
    for i in range(num_mel_bins):
        lo, c, hi = edges[i:i + 3]
        m[:, i] = np.maximum(0.0, np.minimum((bins_mel - lo) / (c - lo), (hi - bins_mel) / (hi - c)))
    m[0, :] = 0.0
    return m


def num_examples(n):
    if n < WIN:
        return 0
    f = 1 + (n - WIN) // HOP
    return 0 if f < EXF else 1 + (f - EXF) // EXF


def examples(x):
    """x (N,) at 16 kHz -> (n_ex, 96, 64) float32 log-mel examples (computed in float64, rounded once)."""
    x = np.asarray(x, np.float64)
    n_ex = num_examples(len(x))
    if n_ex == 0:
        return np.zeros((0, EXF, NMELS), np.float32)
    F = 1 + (len(x) - WIN) // HOP
    idx = np.arange(F)[:, None] * HOP + np.arange(WIN)[None, :]
    win = 0.5 - 0.5 * np.cos(2 * np.pi / WIN * np.arange(WIN))
    mag = np.abs(np.fft.rfft(x[idx] * win, NFFT))
    logmel = np.log(mag @ htk_matrix() + 0.01)
    return logmel[:n_ex * EXF].reshape(n_ex, EXF, NMELS).astype(np.float32)


def random_state_dict(seed, pproc=False):
    """torchvggish-shaped fp32 weights from torch.Generator draws: normal * sqrt(2 / fan_in) weights (Kaiming), so the
    activations stay in range through the ReLU layers, and biases uniform in [-0.1, 0.1)."""
    g = torch.Generator().manual_seed(int(seed))
    sd = {}
    for i, (ci, co) in CONVS.items():
        fan = 9 * ci
        sd[f"features.{i}.weight"] = torch.randn(co, ci, 3, 3, generator=g) * (2.0 / fan) ** 0.5
        sd[f"features.{i}.bias"] = (torch.rand(co, generator=g) - 0.5) * 0.2
    for i, (k, n) in FCS.items():
        sd[f"embeddings.{i}.weight"] = torch.randn(n, k, generator=g) * (2.0 / k) ** 0.5
        sd[f"embeddings.{i}.bias"] = (torch.rand(n, generator=g) - 0.5) * 0.2
    if pproc:  # the checkpoint's PCA tensors, which use_pca=False ignores
        sd["pproc._pca_matrix"] = torch.randn(128, 128, generator=g)
        sd["pproc._pca_means"] = torch.randn(128, 1, generator=g)
    return sd


def _conv3x3(x, w, b):
    """x (n, H, W, Cin), w (Cout, Cin, 3, 3) -> (n, H, W, Cout), zero padding 1, float64."""
    n, H, W, ci = x.shape
    xp = np.zeros((n, H + 2, W + 2, ci))
    xp[:, 1:-1, 1:-1] = x
    cols = np.stack([xp[:, dh:dh + H, dw:dw + W] for dh in range(3) for dw in range(3)], axis=3)  # (n,H,W,9,Cin)
    wm = np.asarray(w, np.float64).transpose(2, 3, 1, 0).reshape(9 * ci, -1)
    return cols.reshape(n * H * W, 9 * ci) @ wm + np.asarray(b, np.float64)


def _pool(x):
    n, H, W, c = x.shape
    return x.reshape(n, H // 2, 2, W // 2, 2, c).max(axis=(2, 4))


def layer(x, sd, kind, idx):
    """One layer in float64 on NHWC input: ("conv", i) relu(conv), ("pool",) 2x2 max, ("fc", i) x W^T + b."""
    if kind == "conv":
        n, H, W, _ = x.shape
        return np.maximum(_conv3x3(x, sd[f"features.{idx}.weight"], sd[f"features.{idx}.bias"]).reshape(n, H, W, -1), 0.0)
    if kind == "pool":
        return _pool(x)
    return x @ np.asarray(sd[f"embeddings.{idx}.weight"], np.float64).T + np.asarray(sd[f"embeddings.{idx}.bias"], np.float64)


def embed(ex, sd):
    """ex (n, 96, 64) -> (n, 128) float64 embeddings of VGG(features, embeddings) without the final ReLU."""
    sd = {k: v.double().numpy() if isinstance(v, torch.Tensor) else np.asarray(v, np.float64) for k, v in sd.items()}
    x = np.asarray(ex, np.float64)[..., None]
    i = 0
    for v in LAYERS:
        if v == "M":
            x = layer(x, sd, "pool", None)
            i += 1
        else:
            x = layer(x, sd, "conv", i)
            i += 2
    x = x.reshape(x.shape[0], -1)  # NHWC flatten
    x = np.maximum(layer(x, sd, "fc", 0), 0.0)
    x = np.maximum(layer(x, sd, "fc", 2), 0.0)
    return layer(x, sd, "fc", 4)


def stats(emb):
    emb = np.asarray(emb, np.float64)
    return emb.mean(axis=0), np.cov(emb, rowvar=False)


def _sqrtm(a):
    """scipy.linalg.sqrtm(a, disp=False)'s matrix; scipy releases without the disp argument return it alone."""
    from scipy import linalg
    try:
        return linalg.sqrtm(a, disp=False)[0]
    except TypeError:
        return linalg.sqrtm(a)


def frechet_distance(mu1, sigma1, mu2, sigma2, eps=1e-6):
    """calculate_frechet_distance of frechet_audio_distance, float64."""
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    sigma1, sigma2 = np.atleast_2d(sigma1), np.atleast_2d(sigma2)
    diff = mu1 - mu2
    covmean = _sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = _sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError(f"Imaginary component {np.max(np.abs(covmean.imag))}")
        covmean = covmean.real
    return float(diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean))


def test_signal(n, seed, sr=SR):
    """A tone pair with noise at sr, float32 in [-1, 1]."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    f1, f2 = rng.uniform(100, 3000, 2)
    x = 0.4 * np.sin(2 * np.pi * f1 * t) + 0.2 * np.sin(2 * np.pi * f2 * t + rng.uniform(0, 6)) + 0.05 * rng.standard_normal(n)
    return x.astype(np.float32)


def torch_module(sd):
    """torchvggish's VGG layer list as a float64 torch.nn module with the transpose / flatten of VGG.forward and
    without the final ReLU; loads sd strictly."""
    import torch.nn as nn

    layers, cin = [], 1
    for v in LAYERS:
        if v == "M":
            layers.append(nn.MaxPool2d(2, 2))
        else:
            layers += [nn.Conv2d(cin, v, 3, padding=1), nn.ReLU(inplace=True)]
            cin = v

    class VGG(nn.Module):
        def __init__(self):
            super().__init__()
            self.features = nn.Sequential(*layers)
            self.embeddings = nn.Sequential(nn.Linear(512 * 4 * 6, 4096), nn.ReLU(True), nn.Linear(4096, 4096),
                                            nn.ReLU(True), nn.Linear(4096, 128))

        def forward(self, x):
            x = self.features(x)
            x = torch.transpose(x, 1, 3)
            x = torch.transpose(x, 1, 2)
            x = x.contiguous().view(x.size(0), -1)
            return self.embeddings(x)

    m = VGG().double()
    m.load_state_dict({k: v for k, v in sd.items() if not k.startswith("pproc.")}, strict=True)
    return m
