"""TEST INFRASTRUCTURE — CPU oracle for the codec rows of the hot path (SURVEY.md §8a D1-D3, A20, A21).

The reference's codec is ``lac.model.lac.LAC`` (``lac @ git+https://github.com/hugofloresgarcia/lac.git``,
unpinned git HEAD, reference requirements.txt:6 / setup.py:31), a Descript-Audio-Codec fork that is NOT under
the original project's checkout and not installed here.  Its arithmetic is therefore restated from the published DAC
architecture as implemented by the in-image ``transformers.models.dac.modeling_dac`` (same family; line
numbers below refer to that file), and anchored on the reference's own call sites:
  codec.preprocess / codec.encode(...)["codes"]          interface.py:215, 223
  codec.quantizer.from_latents(latents)[0], codec.decode  transformer.py:671-675
  codec.quantizer.quantizers[i].codebook.weight           layers.py:145
  codec.sample_rate, codec.hop_length                     interface.py:179, 189
PARITY UNPINNED against lac itself (no source, no checkpoints, no reference tests at this boundary);
pinned against the HF DacModel stand-in by tests/test_dac_oracle.py.

Plain functional torch over a flat dict of tensors (make_codec_weights); fp32 everywhere.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F


@dataclass
class CodecConfig:
    encoder_dim: int = 64
    encoder_rates: Tuple[int, ...] = (2, 4, 8, 12)     # hop 768 (SURVEY.md §0.9)
    decoder_dim: int = 1536
    n_codebooks: int = 14
    codebook_size: int = 1024
    codebook_dim: int = 8
    sample_rate: int = 44100

    @property
    def decoder_rates(self):
        return tuple(reversed(self.encoder_rates))

    @property
    def latent_dim(self):
        return self.encoder_dim * 2 ** len(self.encoder_rates)

    @property
    def hop_length(self):
        return int(math.prod(self.encoder_rates))


def make_codec_weights(cfg: CodecConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded synthetic weights with unit-ish gain per layer so that a random-init stack neither dies nor
    explodes (weight norm is considered already folded: these are effective conv weights)."""
    g = torch.Generator().manual_seed(seed)
    w: Dict[str, torch.Tensor] = {}

    def conv(name, cout, cin, k, gain=1.0):
        w[name + ".weight"] = torch.randn(cout, cin, k, generator=g) * (gain / math.sqrt(cin * k))
        w[name + ".bias"] = torch.randn(cout, generator=g) * 0.02

    def convt(name, cin, cout, k, stride):
        w[name + ".weight"] = torch.randn(cin, cout, k, generator=g) * (1.0 / math.sqrt(cin * k / stride))
        w[name + ".bias"] = torch.randn(cout, generator=g) * 0.02

    def snake(name, c):
        w[name + ".alpha"] = 0.5 + torch.rand(c, generator=g)

    def res_unit(name, c):
        snake(name + ".snake1", c)
        conv(name + ".conv1", c, c, 7, gain=0.5)
        snake(name + ".snake2", c)
        conv(name + ".conv2", c, c, 1, gain=0.5)

    d = cfg.encoder_dim
    conv("encoder.conv1", d, 1, 7)
    for i, s in enumerate(cfg.encoder_rates):
        for r in range(3):
            res_unit(f"encoder.block.{i}.res_unit{r + 1}", d)
        snake(f"encoder.block.{i}.snake1", d)
        conv(f"encoder.block.{i}.conv1", 2 * d, d, 2 * s)
        d *= 2
    snake("encoder.snake1", d)
    conv("encoder.conv2", cfg.latent_dim, d, 3)
    for i in range(cfg.n_codebooks):
        conv(f"quantizer.quantizers.{i}.in_proj", cfg.codebook_dim, cfg.latent_dim, 1)
        conv(f"quantizer.quantizers.{i}.out_proj", cfg.latent_dim, cfg.codebook_dim, 1, gain=1.0 / math.sqrt(cfg.n_codebooks))
        w[f"quantizer.quantizers.{i}.codebook.weight"] = torch.randn(cfg.codebook_size, cfg.codebook_dim, generator=g)
    c = cfg.decoder_dim
    conv("decoder.conv1", c, cfg.latent_dim, 7)
    for i, s in enumerate(cfg.decoder_rates):
        snake(f"decoder.block.{i}.snake1", c)
        convt(f"decoder.block.{i}.conv_t1", c, c // 2, 2 * s, s)
        for r in range(3):
            res_unit(f"decoder.block.{i}.res_unit{r + 1}", c // 2)
        c //= 2
    snake("decoder.snake1", c)
    conv("decoder.conv2", 1, c, 7, gain=0.4)  # keeps the tanh out of saturation so parity tests stay sensitive
    return w


# ----------------------------------------------------------------------------------------------------
def snake(x, alpha):
    """Snake1d (modeling_dac.py:85-99): x + sin^2(alpha x) / (alpha + 1e-9), alpha per channel."""
    a = alpha.view(1, -1, 1)
    return x + (a + 1e-9).reciprocal() * torch.sin(a * x).pow(2)


def res_unit(x, w, name, dilation):
    """DacResidualUnit (modeling_dac.py:179-214): y = x + conv1x1(snake(conv7_dilated(snake(x))))."""
    pad = ((7 - 1) * dilation) // 2
    y = F.conv1d(snake(x, w[name + ".snake1.alpha"]), w[name + ".conv1.weight"], w[name + ".conv1.bias"],
                 dilation=dilation, padding=pad)
    y = F.conv1d(snake(y, w[name + ".snake2.alpha"]), w[name + ".conv2.weight"], w[name + ".conv2.bias"])
    return x + y


def encoder(x, w, cfg: CodecConfig):
    """DacEncoder (modeling_dac.py:442-473) with DacEncoderBlock (:217-237). x: (B,1,N) -> (B, latent, N/hop)."""
    h = F.conv1d(x, w["encoder.conv1.weight"], w["encoder.conv1.bias"], padding=3)
    for i, s in enumerate(cfg.encoder_rates):
        p = f"encoder.block.{i}"
        for r, dil in enumerate((1, 3, 9)):
            h = res_unit(h, w, f"{p}.res_unit{r + 1}", dil)
        h = F.conv1d(snake(h, w[p + ".snake1.alpha"]), w[p + ".conv1.weight"], w[p + ".conv1.bias"], stride=s,
                     padding=math.ceil(s / 2))
    h = snake(h, w["encoder.snake1.alpha"])
    return F.conv1d(h, w["encoder.conv2.weight"], w["encoder.conv2.bias"], padding=1)


def decoder(z, w, cfg: CodecConfig):
    """DacDecoder (modeling_dac.py:405-439) with DacDecoderBlock (:240-268). z: (B, latent, T) -> (B,1,T*hop)."""
    h = F.conv1d(z, w["decoder.conv1.weight"], w["decoder.conv1.bias"], padding=3)
    for i, s in enumerate(cfg.decoder_rates):
        p = f"decoder.block.{i}"
        h = F.conv_transpose1d(snake(h, w[p + ".snake1.alpha"]), w[p + ".conv_t1.weight"], w[p + ".conv_t1.bias"],
                               stride=s, padding=math.ceil(s / 2))
        for r, dil in enumerate((1, 3, 9)):
            h = res_unit(h, w, f"{p}.res_unit{r + 1}", dil)
    h = snake(h, w["decoder.snake1.alpha"])
    return torch.tanh(F.conv1d(h, w["decoder.conv2.weight"], w["decoder.conv2.bias"], padding=3))


def vq_nearest(e, codebook):
    """DacVectorQuantize.decode_latents (modeling_dac.py:152-169): e (B, 8, T) -> (codes (B,T), vectors (B,8,T)).
    Both sides L2-normalised; the score keeps the stand-in's exact (sign-quirky) expression."""
    B, D, T = e.shape
    enc = F.normalize(e.permute(0, 2, 1).reshape(B * T, D))
    cb = F.normalize(codebook)
    dist = -(enc.pow(2).sum(1, keepdim=True) - 2 * enc @ cb.t()) + cb.pow(2).sum(1, keepdim=True).t()
    idx = dist.max(1)[1].reshape(B, T)
    return idx, codebook[idx].transpose(1, 2)


def rvq_encode(z, w, cfg: CodecConfig):
    """DacResidualVectorQuantizer.forward in eval mode (modeling_dac.py:282-342).
    Returns (z_q (B,latent,T), codes (B,n_codebooks,T), latents (B,n_codebooks*8,T))."""
    zq = torch.zeros_like(z)
    res = z
    codes, lats = [], []
    for i in range(cfg.n_codebooks):
        p = f"quantizer.quantizers.{i}"
        e = F.conv1d(res, w[p + ".in_proj.weight"], w[p + ".in_proj.bias"])
        idx, q = vq_nearest(e, w[p + ".codebook.weight"])
        qi = F.conv1d(q, w[p + ".out_proj.weight"], w[p + ".out_proj.bias"])
        zq = zq + qi
        res = res - qi
        codes.append(idx)
        lats.append(e)
    return zq, torch.stack(codes, 1), torch.cat(lats, 1)


def rvq_from_codes(codes, w, cfg: CodecConfig):
    """from_codes (modeling_dac.py:344-368)."""
    zq = 0.0
    for i in range(codes.shape[1]):
        p = f"quantizer.quantizers.{i}"
        q = w[p + ".codebook.weight"][codes[:, i, :]].transpose(1, 2)
        zq = zq + F.conv1d(q, w[p + ".out_proj.weight"], w[p + ".out_proj.bias"])
    return zq


def rvq_from_latents(latents, w, cfg: CodecConfig):
    """from_latents (modeling_dac.py:370-402): re-quantise each 8-d chunk, out_proj, sum.  This is what
    VampNet.decode calls (reference transformer.py:672)."""
    D = cfg.codebook_dim
    n = latents.shape[1] // D
    zq = 0.0
    qs = []
    for i in range(n):
        p = f"quantizer.quantizers.{i}"
        chunk = latents[:, i * D:(i + 1) * D, :]
        _, q = vq_nearest(chunk, w[p + ".codebook.weight"])
        qs.append(q)
        zq = zq + F.conv1d(chunk + (q - chunk), w[p + ".out_proj.weight"], w[p + ".out_proj.bias"])
    return zq, torch.cat(qs, 1)


def preprocess(x, cfg: CodecConfig):
    """Right-pad to a whole number of hops (descript DAC.preprocess; reference interface.py:215)."""
    n = x.shape[-1]
    pad = math.ceil(n / cfg.hop_length) * cfg.hop_length - n
    return F.pad(x, (0, pad)), n


def encode(x, w, cfg: CodecConfig):
    """codec.encode(samples, sr)["codes"] (reference interface.py:223)."""
    z = encoder(x, w, cfg)
    zq, codes, lat = rvq_encode(z, w, cfg)
    return dict(z=zq, codes=codes, latents=lat)


def decode(zq, w, cfg: CodecConfig):
    """codec.decode(z)["audio"] (reference transformer.py:671-675)."""
    return dict(audio=decoder(zq, w, cfg))


# ----------------------------------------------------------------------------------------------------
def to_hf_state_dict(w: Dict[str, torch.Tensor], cfg: CodecConfig) -> Dict[str, torch.Tensor]:
    """Map the flat oracle weights onto transformers.DacModel parameter names (for the stand-in pin)."""
    sd = {}
    for k, v in w.items():
        if k.endswith(".alpha"):
            sd[k] = v.view(1, -1, 1)
        elif ".codebook.weight" in k:
            sd[k] = v
        else:
            sd[k] = v
    return sd
