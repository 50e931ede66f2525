"""GPU: the codec kernels (vnb_codec_conv1d / vnb_codec_rvq through vampnet_b200.codec.DAC) against the CPU
codec oracle on the same seeded weights and inputs.  fp32 on both sides; tolerance 2e-4 abs on activations of
O(1) (accumulation order, sinf/tanhf vs libm), codes bit-exact except proven near-ties."""
import numpy as np
import pytest
import torch

from oracle import dac_oracle as do

pytestmark = pytest.mark.gpu


PRECISIONS = ["tc", "fp32"]  # wgmma split-bf16 convolutions (default) and the fp32 CUDA-core kernels


def build(cfg, seed=0, precision="tc"):
    from vampnet_b200.codec import DAC
    w = do.make_codec_weights(cfg, seed=seed)
    m = DAC(encoder_dim=cfg.encoder_dim, encoder_rates=cfg.encoder_rates, decoder_dim=cfg.decoder_dim,
            n_codebooks=cfg.n_codebooks, codebook_size=cfg.codebook_size, codebook_dim=cfg.codebook_dim,
            sample_rate=cfg.sample_rate, precision=precision)
    m.load_flat(w)
    return w, m.to("cuda")


SMALL = do.CodecConfig(encoder_dim=32, decoder_dim=512)  # every width a multiple of 32 (tensor-core tiles)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_encoder_and_rvq_encode_small(precision):
    w, m = build(SMALL, precision=precision)
    x = torch.randn(2, 1, 768 * 9 + 100, generator=torch.Generator().manual_seed(1)) * 0.3
    xp, n = do.preprocess(x, SMALL)
    xg, n2 = m.preprocess(x.cuda(), SMALL.sample_rate)
    assert n == n2 and torch.equal(xp, xg.cpu())
    ref = do.encode(xp, w, SMALL)
    got = m.encode(xg, SMALL.sample_rate)
    z_ref = do.encoder(xp, w, SMALL)
    # codes: identical unless the oracle's own top-2 margin is a rounding-level near-tie
    mism = (got["codes"].cpu() != ref["codes"])
    print("encode: code mismatch fraction", mism.float().mean().item())
    assert mism.float().mean() < 0.01
    ok = ~mism.any(dim=1)  # frames where all levels agree -> zq must agree closely
    assert (got["z"].cpu() - ref["z"]).abs().permute(0, 2, 1)[ok].max() < 2e-4
    assert (got["latents"].cpu()[:, :8] - ref["latents"][:, :8]).abs().max() < 2e-4  # level 0 sees the same residual


@pytest.mark.parametrize("precision", PRECISIONS)
def test_decoder_small(precision):
    w, m = build(SMALL, precision=precision)
    zq = torch.randn(2, SMALL.latent_dim, 7, generator=torch.Generator().manual_seed(3))
    ref = do.decode(zq, w, SMALL)["audio"]
    got = m.decode(zq.cuda())["audio"].cpu()
    assert got.shape == ref.shape == (2, 1, 7 * 768)
    err = (got - ref).abs()
    print("decode: max err", err.max().item(), "mean", err.mean().item(), "ref absmean", ref.abs().mean().item())
    assert err.max() < 2e-4


def test_from_latents_and_from_codes():
    w, m = build(SMALL)
    g = torch.Generator().manual_seed(4)
    codes = torch.randint(0, 1024, (2, 14, 11), generator=g)
    ref = do.rvq_from_codes(codes, w, SMALL)
    got = m.quantizer.from_codes(codes.cuda())[0].cpu()
    assert (got - ref).abs().max() < 1e-5
    lat = torch.cat([w[f"quantizer.quantizers.{i}.codebook.weight"][codes[:, i]].transpose(1, 2) for i in range(14)], 1)
    ref2 = do.rvq_from_latents(lat, w, SMALL)[0]
    got2 = m.quantizer.from_latents(lat.cuda())[0].cpu()
    assert (got2 - ref2).abs().max() < 1e-5
    # partial depth (coarse only: 4 codebooks), as VampNet.decode may be called with fewer codebooks
    got3 = m.quantizer.from_latents(lat[:, :32].cuda())[0].cpu()
    assert (got3 - do.rvq_from_latents(lat[:, :32], w, SMALL)[0]).abs().max() < 1e-5
    assert torch.equal(m.quantizer.quantizers[3].codebook.weight.cpu(), w["quantizer.quantizers.3.codebook.weight"])


@pytest.mark.parametrize("precision", PRECISIONS)
def test_full_size_layers(precision):
    """The real widths (64..1024 encoder, 1536..96 decoder) on a short clip."""
    cfg = do.CodecConfig()
    w, m = build(cfg, precision=precision)
    x = torch.randn(1, 1, 768 * 3, generator=torch.Generator().manual_seed(5)) * 0.3
    z_ref = do.encoder(x, w, cfg)
    enc = m.encode(x.cuda())
    ref = do.encode(x, w, cfg)
    mism = (enc["codes"].cpu() != ref["codes"]).float().mean().item()
    print("full-size encode code mismatch", mism)
    assert mism < 0.02
    audio_ref = do.decode(ref["z"], w, cfg)["audio"]
    audio = m.decode(ref["z"].cuda())["audio"].cpu()
    err = (audio - audio_ref).abs()
    print("full-size decode: max err", err.max().item(), "ref absmean", audio_ref.abs().mean().item())
    assert err.max() < 5e-4


def test_cpu_codec_raises():
    from vampnet_b200.codec import DAC
    m = DAC(encoder_dim=32, decoder_dim=512)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.encode(torch.zeros(1, 1, 768))
