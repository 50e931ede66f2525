"""GPU: DAC.encode_many / decode_many and Interface.encode_many / decode_many against the per-entry calls, bit for bit
(codes, the int32 view of z, latents and audio), on the reduced-width (SMALL), the full-size and the odd-rate codec; with
entries of several rows, a mix past CODEC_MANY_MAX_SAMPLES that splits into launches, equal lengths (which must also
equal one batched encode), no host synchronisation, and the refusals."""
import pytest
import torch

from oracle import dac_oracle as do
from tests.test_gpu_codec import SMALL, build
from tests.test_gpu_interface import iface  # noqa: F401  (module fixture: tiny coarse / c2f / SMALL codec)

pytestmark = pytest.mark.gpu

HOP = 768
# one hop, 5 s, 10 s (441 000 samples), 17.3 s and 30 s at 44.1 kHz, padded to whole hops as preprocess pads them
CLIPS = [HOP, 220_500, 441_000, 762_930, 1_323_000]


def padded(n):
    return -(-n // HOP) * HOP


def clips(rows, seed):
    """[(B_i, 1, N_i)] on the GPU: one entry per (rows, samples)."""
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(b, 1, padded(n), generator=g) * 0.3).cuda() for b, n in rows]


def assert_encodes_equal(got, want, label):
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a["codes"], b["codes"]), f"{label}: entry {i} codes"
        assert torch.equal(a["z"].contiguous().view(torch.int32), b["z"].contiguous().view(torch.int32)), \
            f"{label}: entry {i} z"
        assert torch.equal(a["latents"].view(torch.int32), b["latents"].view(torch.int32)), f"{label}: entry {i} latents"
        assert a["z"].shape == b["z"].shape and a["z"].stride() == b["z"].stride() and a["length"] == b["length"]


def assert_decodes_equal(got, want, label):
    for i, (a, b) in enumerate(zip(got, want)):
        assert a["audio"].shape == b["audio"].shape, f"{label}: entry {i} shape"
        assert torch.equal(a["audio"].view(torch.int32), b["audio"].view(torch.int32)), f"{label}: entry {i} audio"


@pytest.fixture(scope="module")
def small():
    return build(SMALL)[1]


@pytest.fixture(scope="module")
def full():
    from tools.codec_bits import full_codec
    return full_codec(seed=0)[2]


ROWS = [(1, CLIPS[2]), (2, CLIPS[0]), (1, CLIPS[4]), (2, CLIPS[3]), (1, CLIPS[1])]


@pytest.mark.parametrize("which", ["small", "full"])
def test_encode_many_and_decode_many_equal_per_entry_calls(which, request):
    m = request.getfixturevalue(which)
    audio = clips(ROWS, seed=1)
    want = [m.encode(a) for a in audio]
    got = m.encode_many(audio)
    assert_encodes_equal(got, want, f"{which} encode")
    zs = [w["z"] for w in want]
    assert_decodes_equal(m.decode_many(zs), [m.decode(z) for z in zs], f"{which} decode")


def test_odd_rate_decoder():
    cfg = do.CodecConfig(encoder_dim=32, decoder_dim=256, encoder_rates=(3, 2))
    _, m = build(cfg)
    assert m.decoder_rates == (2, 3) and m.hop_length == 6
    g = torch.Generator().manual_seed(6)
    zs = [torch.randn(b, cfg.latent_dim, t, generator=g).cuda() for b, t in [(1, 5), (2, 300), (1, 1), (1, 129)]]
    got = m.decode_many(zs)
    assert [tuple(o["audio"].shape) for o in got] == [(1, 1, 29), (2, 1, 1799), (1, 1, 5), (1, 1, 773)]
    assert_decodes_equal(got, [m.decode(z) for z in zs], "odd-rate decode")
    audio = [(torch.randn(b, 1, n, generator=g) * 0.3).cuda() for b, n in [(1, 6), (2, 1800), (1, 774)]]
    assert_encodes_equal(m.encode_many(audio), [m.encode(a) for a in audio], "odd-rate encode")


def test_mix_past_the_budget_splits_longest_first(small):
    from vampnet_b200.codec import CODEC_MANY_MAX_SAMPLES
    rows = [(24, CLIPS[2]), (2, CLIPS[4]), (8, CLIPS[1])]
    audio = clips(rows, seed=2)
    assert sum(a.shape[0] * a.shape[-1] for a in audio) > CODEC_MANY_MAX_SAMPLES
    launches = []
    orig = small._encode_launch

    def counted(x, lens):
        launches.append(tuple(x.shape))
        return orig(x, lens)
    small._encode_launch = counted
    try:
        got = small.encode_many(audio)
    finally:
        del small._encode_launch
    # the two 30 s rows lead; 10 rows x 30 s fit the budget, so 8 ten-second rows join them; the rest share a launch
    assert launches == [(10, 1, padded(CLIPS[4])), (24, 1, padded(CLIPS[2]))]
    assert_encodes_equal(got, [small.encode(a) for a in audio], "split encode")


def test_equal_lengths_equal_one_batched_encode(small):
    audio = clips([(1, CLIPS[2]), (2, CLIPS[2]), (1, CLIPS[2])], seed=3)
    got = small.encode_many(audio)
    batched = small.encode(torch.cat(audio))
    one = {k: [] for k in ("codes", "z", "latents")}
    for e in got:
        for k in one:
            one[k].append(e[k])
    assert torch.equal(torch.cat(one["codes"]), batched["codes"])
    assert torch.equal(torch.cat(one["z"]).contiguous().view(torch.int32), batched["z"].contiguous().view(torch.int32))
    assert torch.equal(torch.cat(one["latents"]), batched["latents"])
    zs = [e["z"] for e in got]
    audio_b = small.decode(torch.cat(zs))["audio"]
    assert torch.equal(torch.cat([d["audio"] for d in small.decode_many(zs)]).view(torch.int32),
                       audio_b.view(torch.int32))


def _signals():
    from vampnet_b200.audio import AudioSignal
    g = torch.Generator().manual_seed(4)
    out = []
    for sr, ch, secs, gain in [(44100, 1, 2.0, 0.05), (48000, 2, 1.3, 0.5), (44100, 2, 0.4, 1.5), (48000, 1, 3.1, 0.2)]:
        out.append(AudioSignal(torch.randn(1, ch, int(sr * secs), generator=g) * gain, sr))
    return out


def test_interface_encode_many_and_decode_many(iface):  # noqa: F811
    signals = _signals()
    want = [iface.encode(s) for s in signals]
    got = iface.encode_many(signals)
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    g = torch.Generator().manual_seed(5)
    outs = []
    for codes in want:
        mask = (torch.rand(codes.shape, generator=g) < 0.7).long().cuda()
        outs.append(iface.vamp(codes, mask, batch_size=2, _sampling_steps=2, seed=7))
    dec = iface.decode_many(outs)
    for a, z in zip(dec, outs):
        b = iface.decode(z)
        assert a.sample_rate == b.sample_rate and torch.equal(a.audio_data.view(torch.int32), b.audio_data.view(torch.int32))


def test_no_host_synchronisation(iface):  # noqa: F811
    signals = [s.to("cuda") for s in _signals()]
    codes = iface.encode_many(signals)                                  # warm: weights packed, caches filled
    iface.decode_many(codes)
    samples = [iface._preprocess(s).samples for s in signals]           # encode()'s own preprocessing, unchanged
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        enc = iface.codec.encode_many(samples)
        dec = iface.decode_many(codes)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert len(enc) == len(dec) == len(signals)


def test_refusals_then_still_works(small, iface):  # noqa: F811
    with pytest.raises(ValueError, match="empty list"):
        small.encode_many([])
    with pytest.raises(ValueError, match="empty list"):
        small.decode_many([])
    with pytest.raises(ValueError, match="empty list"):
        iface.encode_many([])
    with pytest.raises(ValueError, match="empty list"):
        iface.decode_many([])
    with pytest.raises(ValueError, match="entry 1"):
        small.encode_many([torch.zeros(1, 1, HOP, device="cuda"), torch.zeros(1, 1, 0, device="cuda")])
    with pytest.raises(ValueError, match="entry 0"):
        small.decode_many([torch.zeros(1, small.latent_dim, 0, device="cuda")])
    with pytest.raises(ValueError, match="different sample rates"):
        small.encode_many([torch.zeros(1, 1, HOP, device="cuda")] * 2, [44100, 48000])
    with pytest.raises(ValueError, match="different latent counts"):
        small.decode_many([torch.zeros(1, small.latent_dim, 2, device="cuda"),
                           torch.zeros(1, small.latent_dim // 2, 2, device="cuda")])
    with pytest.raises(ValueError, match="different codebook counts"):
        iface.decode_many([torch.zeros(1, 14, 3, dtype=torch.long, device="cuda"),
                           torch.zeros(1, 4, 3, dtype=torch.long, device="cuda")])
    audio = clips([(1, CLIPS[1]), (1, CLIPS[0])], seed=8)
    assert_encodes_equal(small.encode_many(audio), [small.encode(a) for a in audio], "after refusals")
