"""CPU: the codec ingests checkpoints written in the descript-audio-codec / ``lac`` module layout — the layout of the
file the reference's Interface actually loads (``lac.model.lac.LAC``, reference interface.py:16, 70).

``lac`` itself is absent from the original project's checkout and from the image, so the module tree below is a TEST-LOCAL
restatement of the published DAC module structure (nn.Sequential stacks of weight-normed convs and Snake1d with a
(1, C, 1) alpha).  It is built with torch's own ``nn.Sequential`` / ``weight_norm`` so that the state_dict KEY NAMES
are produced by torch, not typed by hand, and its forward pass (plain torch, CPU) pins the remapped weights
numerically against oracle/dac_oracle.py.
"""
import math

import pytest
import torch
import torch.nn as nn
from torch.nn.utils import weight_norm

from oracle import dac_oracle as do

CFG = do.CodecConfig(encoder_dim=16, decoder_dim=128, n_codebooks=5)


class Snake1d(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.alpha = nn.Parameter(torch.ones(1, c, 1))

    def forward(self, x):
        return x + (self.alpha + 1e-9).reciprocal() * torch.sin(self.alpha * x).pow(2)


def WNConv1d(*a, **k):
    return weight_norm(nn.Conv1d(*a, **k))


def WNConvTranspose1d(*a, **k):
    return weight_norm(nn.ConvTranspose1d(*a, **k))


class ResidualUnit(nn.Module):
    def __init__(self, dim, dilation):
        super().__init__()
        pad = ((7 - 1) * dilation) // 2
        self.block = nn.Sequential(Snake1d(dim), WNConv1d(dim, dim, kernel_size=7, dilation=dilation, padding=pad),
                                   Snake1d(dim), WNConv1d(dim, dim, kernel_size=1))

    def forward(self, x):
        return x + self.block(x)


class EncoderBlock(nn.Module):
    def __init__(self, dim, stride):
        super().__init__()
        self.block = nn.Sequential(ResidualUnit(dim // 2, 1), ResidualUnit(dim // 2, 3), ResidualUnit(dim // 2, 9),
                                   Snake1d(dim // 2),
                                   WNConv1d(dim // 2, dim, kernel_size=2 * stride, stride=stride,
                                            padding=math.ceil(stride / 2)))

    def forward(self, x):
        return self.block(x)


class Encoder(nn.Module):
    def __init__(self, d_model, strides, d_latent):
        super().__init__()
        blocks = [WNConv1d(1, d_model, kernel_size=7, padding=3)]
        for s in strides:
            d_model *= 2
            blocks.append(EncoderBlock(d_model, s))
        blocks += [Snake1d(d_model), WNConv1d(d_model, d_latent, kernel_size=3, padding=1)]
        self.block = nn.Sequential(*blocks)

    def forward(self, x):
        return self.block(x)


class DecoderBlock(nn.Module):
    def __init__(self, cin, cout, stride):
        super().__init__()
        self.block = nn.Sequential(Snake1d(cin),
                                   WNConvTranspose1d(cin, cout, kernel_size=2 * stride, stride=stride,
                                                     padding=math.ceil(stride / 2)),
                                   ResidualUnit(cout, 1), ResidualUnit(cout, 3), ResidualUnit(cout, 9))

    def forward(self, x):
        return self.block(x)


class Decoder(nn.Module):
    def __init__(self, cin, channels, rates):
        super().__init__()
        layers = [WNConv1d(cin, channels, kernel_size=7, padding=3)]
        for i, s in enumerate(rates):
            layers.append(DecoderBlock(channels // 2 ** i, channels // 2 ** (i + 1), s))
        out = channels // 2 ** len(rates)
        layers += [Snake1d(out), WNConv1d(out, 1, kernel_size=7, padding=3), nn.Tanh()]
        self.model = nn.Sequential(*layers)

    def forward(self, x):
        return self.model(x)


class VQ(nn.Module):
    def __init__(self, latent, size, dim):
        super().__init__()
        self.in_proj = WNConv1d(latent, dim, kernel_size=1)
        self.out_proj = WNConv1d(dim, latent, kernel_size=1)
        self.codebook = nn.Embedding(size, dim)


class RVQ(nn.Module):
    def __init__(self, latent, n, size, dim):
        super().__init__()
        self.quantizers = nn.ModuleList([VQ(latent, size, dim) for _ in range(n)])


class DescriptLayoutCodec(nn.Module):
    def __init__(self, cfg: do.CodecConfig):
        super().__init__()
        self.encoder = Encoder(cfg.encoder_dim, cfg.encoder_rates, cfg.latent_dim)
        self.quantizer = RVQ(cfg.latent_dim, cfg.n_codebooks, cfg.codebook_size, cfg.codebook_dim)
        self.decoder = Decoder(cfg.latent_dim, cfg.decoder_dim, cfg.decoder_rates)


@pytest.fixture(scope="module")
def lac_ckpt(tmp_path_factory):
    torch.manual_seed(0)
    m = DescriptLayoutCodec(CFG).eval()
    with torch.no_grad():  # non-trivial alphas / gains so that every tensor matters
        for n, p in m.named_parameters():
            if n.endswith("alpha"):
                p.copy_(0.5 + torch.rand_like(p))
            elif n.endswith("weight_g"):
                p.mul_(0.6 + 0.3 * torch.rand_like(p))
    path = tmp_path_factory.mktemp("lac") / "codec.pth"
    kwargs = dict(encoder_dim=CFG.encoder_dim, encoder_rates=list(CFG.encoder_rates), decoder_dim=CFG.decoder_dim,
                  decoder_rates=list(CFG.decoder_rates), n_codebooks=CFG.n_codebooks, codebook_size=CFG.codebook_size,
                  codebook_dim=CFG.codebook_dim, sample_rate=CFG.sample_rate,
                  quantizer_dropout=0.5)  # training-only argument the product must ignore
    torch.save({"state_dict": m.state_dict(), "metadata": {"kwargs": kwargs}}, path)
    return m, path


def test_key_names_are_the_descript_layout(lac_ckpt):
    m, _ = lac_ckpt
    keys = set(m.state_dict())
    n = len(CFG.encoder_rates)
    for k in ("encoder.block.0.weight_v", "encoder.block.1.block.0.block.0.alpha", "encoder.block.1.block.0.block.1.weight_g",
              "encoder.block.1.block.3.alpha", "encoder.block.1.block.4.bias", f"encoder.block.{n + 1}.alpha",
              f"encoder.block.{n + 2}.weight_v", "decoder.model.0.weight_g", "decoder.model.1.block.0.alpha",
              "decoder.model.1.block.1.weight_v", "decoder.model.1.block.4.block.3.bias", f"decoder.model.{n + 1}.alpha",
              f"decoder.model.{n + 2}.weight_v", "quantizer.quantizers.0.in_proj.weight_v",
              "quantizer.quantizers.4.codebook.weight"):
        assert k in keys, k


def test_load_lac_layout_checkpoint_and_match_torch_forward(lac_ckpt):
    from vampnet_b200.codec import DAC, _layout
    m, path = lac_ckpt
    codec = DAC.load(path, precision="fp32")  # 16-channel test codec: narrower than the tensor-core path allows
    assert codec.hop_length == CFG.hop_length and codec.n_codebooks == CFG.n_codebooks
    own = _layout(codec._cfg)
    w = {k: codec.params.get(k).detach().clone() for k in own}
    x = torch.randn(2, 1, CFG.hop_length * 3, generator=torch.Generator().manual_seed(1)) * 0.3
    with torch.no_grad():
        z_ref = m.encoder(x)
        z = do.encoder(x, w, CFG)
        assert (z - z_ref).abs().max() < 2e-5 * max(1.0, z_ref.abs().max().item())
        audio_ref = m.decoder(z_ref)
        audio = do.decoder(z_ref, w, CFG)
        assert (audio - audio_ref).abs().max() < 2e-5
        # quantizer tensors: folded weight-norm 1x1 convs and the raw codebooks
        for i, q in enumerate(m.quantizer.quantizers):
            e_ref = q.in_proj(z_ref)
            e = torch.nn.functional.conv1d(z_ref, w[f"quantizer.quantizers.{i}.in_proj.weight"],
                                           w[f"quantizer.quantizers.{i}.in_proj.bias"])
            assert (e - e_ref).abs().max() < 1e-5
            assert torch.equal(w[f"quantizer.quantizers.{i}.codebook.weight"], q.codebook.weight)
            cb = q.codebook.weight.t()[None]  # (1, dim, size): push the whole codebook through out_proj
            o = torch.nn.functional.conv1d(cb, w[f"quantizer.quantizers.{i}.out_proj.weight"],
                                           w[f"quantizer.quantizers.{i}.out_proj.bias"])
            assert (o - q.out_proj(cb)).abs().max() < 1e-5


def test_new_style_parametrization_names_and_flat_names_pass_through(lac_ckpt):
    from vampnet_b200.codec import DAC, remap_descript_keys, _layout
    m, _ = lac_ckpt
    sd = m.state_dict()
    n = len(CFG.encoder_rates)
    new_style = {}
    for k, v in sd.items():
        k = k.replace(".weight_g", ".parametrizations.weight.original0").replace(".weight_v", ".parametrizations.weight.original1")
        new_style[k] = v
    a, b = remap_descript_keys(sd, n), remap_descript_keys(new_style, n)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    folded = set(k.replace("weight_g", "weight").replace("weight_v", "weight") for k in a)
    assert folded == set(_layout(DAC(encoder_dim=CFG.encoder_dim, decoder_dim=CFG.decoder_dim,
                                     n_codebooks=CFG.n_codebooks, precision="fp32")._cfg))
    # idempotent on the flat (HF) layout
    again = remap_descript_keys(a, n)
    assert again.keys() == a.keys()


def test_unknown_stage_is_an_error():
    from vampnet_b200.codec import remap_descript_keys
    with pytest.raises(KeyError):
        remap_descript_keys({"encoder.block.9.weight_v": torch.zeros(1)}, 4)
