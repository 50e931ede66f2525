"""The evaluation script's Fréchet audio distance: frechet_audio_distance's FrechetAudioDistance(use_pca=False,
use_activation=False) with torchvggish's VGGish, restated on the GPU (DESIGN.md §14).  The log-mel frontend, the
network and the embedding moments run in the kernels of csrc/mel.cu, csrc/conv_wgmma.cu and csrc/fad.cu without a host
sync; the 128 x 128 matrix square root of the distance runs in scipy.linalg.sqrtm on the host in float64, as in the
reference.  The real weights are torchvggish's checkpoint (vggish-10086976.pth), which the package downloads on first
use; parity with the package itself is unpinned."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np
import torch

from . import _lib

SAMPLE_RATE = 16000
EX_FRAMES, N_MELS, EMB_DIM = 96, 64, 128
MIN_SAMPLES = 15600  # the shortest signal that gives one example
MAX_BATCH = 512      # examples per embed launch (the workspace is 786 KB per example)

# torchvggish's VGG: features (index: Cin, Cout) and embeddings (index: K, N), in state-dict order
CONVS = {0: (1, 64), 3: (64, 128), 6: (128, 256), 8: (256, 256), 11: (256, 512), 13: (512, 512)}
FCS = {0: (512 * 4 * 6, 4096), 2: (4096, 4096), 4: (4096, EMB_DIM)}


def expected_shapes():
    """{state-dict key: shape} of the tensors VGGish.load reads."""
    shapes = {}
    for i, (ci, co) in CONVS.items():
        shapes[f"features.{i}.weight"] = (co, ci, 3, 3)
        shapes[f"features.{i}.bias"] = (co,)
    for i, (k, n) in FCS.items():
        shapes[f"embeddings.{i}.weight"] = (n, k)
        shapes[f"embeddings.{i}.bias"] = (n,)
    return shapes


def num_examples(n_samples: int) -> int:
    """vggish_input's example count for n_samples at 16 kHz: 1 + (F - 96) // 96 with F = 1 + (n - 400) // 160."""
    if n_samples < 400:
        return 0
    f = 1 + (n_samples - 400) // 160
    return 0 if f < EX_FRAMES else 1 + (f - EX_FRAMES) // EX_FRAMES


def _split(w: torch.Tensor):
    """fp32 -> (hi, lo) bf16 with w = hi + lo to 16 mantissa bits, the kernels' split operands."""
    hi = w.to(torch.bfloat16)
    lo = (w - hi.float()).to(torch.bfloat16)
    return hi.contiguous(), lo.contiguous()


class VGGish:
    """torchvggish's VGG (features + embeddings, without the final ReLU and without PCA) on the GPU.  The weights are
    packed once into the layouts the kernels read: 3x3 kernels as (Cout, 3, 3, Cin), the first fully connected layer's
    columns in NHWC order (torchvggish's flatten order already), all but the first layer split into bf16 hi/lo."""

    def __init__(self, state_dict, device=None):
        sd = {k: v for k, v in state_dict.items() if not k.startswith("pproc.")}
        want = expected_shapes()
        missing = sorted(set(want) - set(sd))
        if missing:
            raise ValueError(f"VGGish: missing keys {missing}")
        for k, shape in want.items():
            if tuple(sd[k].shape) != shape:
                raise ValueError(f"VGGish: {k} has shape {tuple(sd[k].shape)}, expected {shape}")
        extra = sorted(set(sd) - set(want))
        if extra:
            raise ValueError(f"VGGish: unexpected keys {extra}")
        if device is None:
            if not torch.cuda.is_available():
                raise RuntimeError("VGGish: no CUDA device; vampnet_b200 runs its kernels on the GPU only")
            device = f"cuda:{torch.cuda.current_device()}"
        self.device = torch.device(device)
        f = lambda k: sd[k].detach().to(self.device, torch.float32).contiguous()  # noqa: E731
        keep = []
        w = _lib.VggishWeights()
        w1, b1 = f("features.0.weight").reshape(64, 9).contiguous(), f("features.0.bias")
        keep += [w1, b1]
        w.w1, w.b1 = w1.data_ptr(), b1.data_ptr()
        for l, i in enumerate((3, 6, 8, 11, 13)):
            co, ci = CONVS[i][1], CONVS[i][0]
            hi, lo = _split(f(f"features.{i}.weight").permute(0, 2, 3, 1).reshape(co, 9 * ci))
            b = f(f"features.{i}.bias")
            keep += [hi, lo, b]
            w.conv_hi[l], w.conv_lo[l], w.conv_b[l] = hi.data_ptr(), lo.data_ptr(), b.data_ptr()
        for l, i in enumerate((0, 2, 4)):
            hi, lo = _split(f(f"embeddings.{i}.weight"))
            b = f(f"embeddings.{i}.bias")
            keep += [hi, lo, b]
            w.fc_hi[l], w.fc_lo[l], w.fc_b[l] = hi.data_ptr(), lo.data_ptr(), b.data_ptr()
        self._keep = keep
        self._handle = C.c_void_p()
        self._L = _lib.lib()
        _lib.check(self._L.vnb_vggish_create(C.byref(w), C.byref(self._handle)))

    @classmethod
    def load(cls, path, device=None) -> "VGGish":
        """From a torchvggish checkpoint (a state dict; its pproc.* PCA tensors are ignored).  Missing keys, unexpected
        keys and wrong shapes raise ValueError."""
        sd = torch.load(path, map_location="cpu", weights_only=True)
        if not isinstance(sd, dict):
            raise ValueError(f"VGGish.load: {path} does not hold a state dict")
        return cls(sd, device)

    def __del__(self):
        h = getattr(self, "_handle", None)
        if h is not None and h.value:
            self._L.vnb_vggish_destroy(h)
            self._handle = None

    def examples(self, samples: torch.Tensor) -> torch.Tensor:
        """samples (N,) or (rows, N) at 16 kHz -> (rows * num_examples(N), 96, 64) fp32 log-mel examples on the device.
        N < 15600 gives an empty (0, 96, 64) tensor."""
        x = samples.to(self.device, torch.float32).reshape(-1, samples.shape[-1]).contiguous()
        rows, n = x.shape
        n_ex = num_examples(n)
        out = torch.empty((rows * n_ex, EX_FRAMES, N_MELS), dtype=torch.float32, device=self.device)
        if n_ex == 0 or rows == 0:
            return out
        with torch.cuda.device(self.device):
            _lib.check(self._L.vnb_vggish_frontend(_lib.ptr(x), rows, n, _lib.ptr(out), _lib.stream_ptr(self.device)))
        return out

    def embed(self, examples: torch.Tensor) -> torch.Tensor:
        """examples (n, 96, 64) fp32 -> (n, 128) fp32 embeddings on the device; each row depends on its example only."""
        x = examples.to(self.device, torch.float32).contiguous()
        if x.dim() != 3 or tuple(x.shape[1:]) != (EX_FRAMES, N_MELS):
            raise ValueError(f"VGGish.embed: examples must be (n, 96, 64), got {tuple(x.shape)}")
        out = torch.empty((x.shape[0], EMB_DIM), dtype=torch.float32, device=self.device)
        n_total = x.shape[0]
        if n_total == 0:
            return out
        nb = min(MAX_BATCH, n_total)
        ws, ws_bytes = _lib.workspace(self.device, self._L.vnb_vggish_workspace_bytes, nb)
        with torch.cuda.device(self.device):
            for s in range(0, n_total, nb):
                k = min(nb, n_total - s)
                _lib.check(self._L.vnb_vggish_embed(self._handle, _lib.ptr(x[s:s + k]), k, _lib.ptr(ws), ws_bytes,
                                                    _lib.ptr(out[s:s + k]), _lib.stream_ptr(self.device)))
        return out


def moments(embeddings: torch.Tensor):
    """(mu (128,), sigma (128, 128)) float64 on the device: np.mean(axis=0) and np.cov(rowvar=False) with every sum in
    row order.  Fewer than two embeddings raise ValueError."""
    e = embeddings.float().contiguous()
    if e.dim() != 2 or e.shape[1] != EMB_DIM:
        raise ValueError(f"moments: embeddings must be (M, 128), got {tuple(e.shape)}")
    if e.shape[0] < 2:
        raise ValueError(f"moments: need at least two embeddings, got {e.shape[0]}")
    if e.device.type != "cuda":
        raise ValueError("moments: embeddings must be on a CUDA device")
    mu = torch.empty(EMB_DIM, dtype=torch.float64, device=e.device)
    sigma = torch.empty((EMB_DIM, EMB_DIM), dtype=torch.float64, device=e.device)
    with torch.cuda.device(e.device):
        _lib.check(_lib.lib().vnb_fad_moments(_lib.ptr(e), e.shape[0], _lib.ptr(mu), _lib.ptr(sigma),
                                              _lib.stream_ptr(e.device)))
    return mu, sigma


def _sqrtm(a):
    """scipy.linalg.sqrtm(a, disp=False)'s matrix; scipy releases without the disp argument return it alone."""
    from scipy import linalg
    try:
        return linalg.sqrtm(a, disp=False)[0]
    except TypeError:
        return linalg.sqrtm(a)


def frechet_distance(mu1, sigma1, mu2, sigma2, eps: float = 1e-6) -> float:
    """frechet_audio_distance's calculate_frechet_distance in float64 on the host: |mu1 - mu2|^2 + tr(s1) + tr(s2) -
    2 tr(sqrtm(s1 s2)); eps I is added to both covariances when sqrtm's result is not finite, and a result with an
    imaginary part that is not ~0 (atol 1e-3 on the diagonal) raises ValueError."""
    mu1, mu2 = np.atleast_1d(np.asarray(mu1, np.float64)), np.atleast_1d(np.asarray(mu2, np.float64))
    sigma1, sigma2 = np.atleast_2d(np.asarray(sigma1, np.float64)), np.atleast_2d(np.asarray(sigma2, np.float64))
    if mu1.shape != mu2.shape or sigma1.shape != sigma2.shape:
        raise ValueError("frechet_distance: the two sets' moments differ in shape")
    diff = mu1 - mu2
    covmean = _sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = _sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError(f"frechet_distance: imaginary component {np.max(np.abs(covmean.imag))}")
        covmean = covmean.real
    return float(diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean))


def _load_16k_mono(path, device):
    from .audio import AudioSignal
    sig = AudioSignal(path)
    sig.audio_data = sig.audio_data.to(device)
    sig.to_mono().resample(SAMPLE_RATE)
    return sig.audio_data.reshape(-1)


class FrechetAudioDistance:
    """frechet_audio_distance.FrechetAudioDistance(model_name="vggish", use_pca=False, use_activation=False) on the GPU.
    ckpt: a torchvggish checkpoint path, a state dict or a VGGish.  Other values of use_pca and use_activation raise
    ValueError (the evaluation script uses neither)."""

    def __init__(self, ckpt, use_pca: bool = False, use_activation: bool = False, device=None):
        if use_pca:
            raise ValueError("FrechetAudioDistance: use_pca=True (PCA postprocessing) is not supported")
        if use_activation:
            raise ValueError("FrechetAudioDistance: use_activation=True is not supported")
        if isinstance(ckpt, VGGish):
            self.model = ckpt
        elif isinstance(ckpt, dict):
            self.model = VGGish(ckpt, device)
        else:
            self.model = VGGish.load(ckpt, device)

    def embeddings(self, signals) -> torch.Tensor:
        """signals: 1-D 16 kHz mono tensors -> the embeddings of all their examples, stacked in order, (n, 128) fp32
        on the device.  A signal shorter than 15600 samples contributes none."""
        ex = [self.model.examples(s.reshape(-1)) for s in signals]
        ex = [e for e in ex if e.shape[0]]
        if not ex:
            return torch.empty((0, EMB_DIM), dtype=torch.float32, device=self.model.device)
        return self.model.embed(torch.cat(ex))

    def dir_embeddings(self, directory, audio_ext: str = ".wav") -> torch.Tensor:
        """The embeddings of every file of a directory with the extension (sorted by name), each averaged to mono and
        resampled to 16 kHz."""
        files = sorted(Path(directory).glob(f"*{audio_ext}"))
        return self.embeddings([_load_16k_mono(f, self.model.device) for f in files])

    def dir_moments(self, directory, audio_ext: str = ".wav"):
        """(mu, sigma) float64 of a directory's embeddings, on the device."""
        return moments(self.dir_embeddings(directory, audio_ext))

    @staticmethod
    def score_moments(m1, m2) -> float:
        """The distance between two (mu, sigma) pairs (device or host), through frechet_distance."""
        to_np = lambda t: t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)  # noqa: E731
        return frechet_distance(to_np(m1[0]), to_np(m1[1]), to_np(m2[0]), to_np(m2[1]))

    def score(self, background_dir, eval_dir, audio_ext: str = ".wav") -> float:
        """frechet.score(background_dir, eval_dir): the distance between the two directories' embedding sets."""
        return self.score_moments(self.dir_moments(background_dir, audio_ext), self.dir_moments(eval_dir, audio_ext))
