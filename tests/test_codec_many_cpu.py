"""CPU: the host side of DAC.encode_many / decode_many (clips of different lengths in shared codec launches) with the
device launches replaced by stubs: the launch plan (longest first, the split at the sample budget, results mapped back
to list order), the per-rate length tables including odd decoder rates, the decoder input's select, and the
refusals."""
import pytest
import torch

from vampnet_b200 import codec as K


def small():
    return K.DAC(encoder_dim=32, decoder_dim=512)


def test_plan_longest_first_and_budget():
    lengths = [5, 30, 10, 30, 17, 1]
    assert K.plan_launches(lengths, budget=10 ** 9) == [[1, 3, 4, 2, 0, 5]]
    # 2 x 30 = 60 fits, a third row of 30 would not; the next launch starts at 17
    assert K.plan_launches(lengths, budget=60) == [[1, 3], [4, 2, 0], [5]]
    # an item longer than the budget still runs, alone
    assert K.plan_launches([100, 3], budget=50) == [[0], [1]]
    # ties keep list order (stable)
    assert K.plan_launches([4, 4, 4], budget=8) == [[0, 1], [2]]


def test_default_budget_is_config3_encode():
    assert K.CODEC_MANY_MAX_SAMPLES == 32 * 441_600
    assert K.plan_launches([441_600] * 33) == [list(range(32)), [32]]


def test_length_tables():
    assert K.encoder_lengths([768 * 5, 768], (2, 4, 8, 12)) == [[3840, 768], [1920, 384], [480, 96], [60, 12], [5, 1]]
    assert K.decoder_lengths([5, 1], (8, 8, 4, 2)) == [[5, 1], [40, 8], [320, 64], [1280, 256], [2560, 512]]
    # odd rates: ConvTranspose1d(2s, stride s, pad ceil(s/2)) gives T * s - s % 2 rows at every odd layer
    assert K.decoder_lengths([5, 2], (3, 2)) == [[5, 2], [14, 5], [28, 10]]
    assert K.decoder_lengths([4], (3, 3)) == [[4], [11], [32]]


def test_zero_frames_past_is_a_select():
    zc = torch.full((3, 5, 2), float("nan"))
    zc[0, :2] = -0.0
    zc[1, :5] = torch.arange(10.0).view(5, 2) - 4.5
    zc[2, :1] = 7.0
    out = K.zero_frames_past(zc, torch.tensor([2, 5, 1], dtype=torch.int32))
    bits = out.view(torch.int32)
    assert torch.equal(bits[0, :2], zc[0, :2].view(torch.int32))          # -0 kept as -0 (no arithmetic)
    assert (bits[0, 2:] == 0).all() and (bits[2, 1:] == 0).all()          # +0, bit pattern 0, over NaN
    assert torch.equal(out[1], zc[1]) and torch.equal(out[2, :1], zc[2, :1])


def _encode_stub(m, launches):
    def stub(x, lens):
        launches.append((tuple(x.shape), lens.tolist()))
        B, _, N = x.shape
        T = N // m.hop_length
        first = x[:, 0, ::m.hop_length]                                    # (B, T): the first sample of each frame
        z = first.unsqueeze(-1).expand(B, T, m.latent_dim).clone()
        codes = first.round().long().unsqueeze(1).expand(B, m.n_codebooks, T).clone()
        lat = first.unsqueeze(1).expand(B, 8 * m.n_codebooks, T).clone()
        return {"z": z, "codes": codes, "latents": lat}
    return stub


def test_encode_many_maps_back_to_list_order():
    m = small()
    hop = m.hop_length
    launches = []
    m._encode_launch = _encode_stub(m, launches)
    frames = [(2, 3), (1, 7), (2, 1), (1, 7)]                               # (rows, frames) per entry
    audio, ident = [], 0
    for b, t in frames:
        a = torch.zeros(b, 1, t * hop)
        for j in range(b):
            ident += 1
            a[j, 0] = ident                                                 # every row carries its own number
        audio.append(a)
    out = m.encode_many(audio, budget=2 * 7 * hop)
    # longest first: the two 7-frame rows (a third would pass 14 frames of samples), then 3, 3, 1, 1 (4 x 3 <= 14)
    assert [s for s, _ in launches] == [(2, 1, 7 * hop), (4, 1, 3 * hop)]
    assert launches[1][1] == K.encoder_lengths([3 * hop, 3 * hop, hop, hop], m.encoder_rates)
    ident = 0
    for (b, t), a, o in zip(frames, audio, out):
        assert o["codes"].shape == (b, m.n_codebooks, t) and o["z"].shape == (b, m.latent_dim, t)
        assert o["latents"].shape == (b, 8 * m.n_codebooks, t) and o["length"] == t * hop
        for j in range(b):
            ident += 1
            assert (o["codes"][j] == ident).all() and (o["z"][j] == ident).all()


def test_decode_many_maps_back_to_list_order_and_selects():
    m = small()
    hop = m.hop_length
    seen = []

    def stub(zc, lens):
        seen.append((zc.clone(), lens.clone()))
        zc = K.zero_frames_past(zc, lens[0])
        return zc[:, :, :1].repeat_interleave(hop, dim=1).permute(0, 2, 1)   # (B, 1, T * hop)
    m._decode_launch = stub
    zs = [torch.full((1, m.latent_dim, 2), 1.0), torch.full((2, m.latent_dim, 4), 2.0),
          torch.full((1, m.latent_dim, 3), 3.0)]
    zs[1][1] = 4.0
    out = m.decode_many(zs, budget=2 * 4 * hop)
    assert [tuple(z.shape) for z, _ in seen] == [(2, 4, m.latent_dim), (2, 3, m.latent_dim)]
    assert seen[1][1].tolist() == K.decoder_lengths([3, 2], m.decoder_rates)
    assert [tuple(o["audio"].shape) for o in out] == [(1, 1, 2 * hop), (2, 1, 4 * hop), (1, 1, 3 * hop)]
    assert (out[0]["audio"] == 1).all() and (out[1]["audio"][0] == 2).all() and (out[1]["audio"][1] == 4).all()
    assert (out[2]["audio"] == 3).all()


def test_refusals():
    m = small()
    hop = m.hop_length
    with pytest.raises(ValueError, match="empty list"):
        m.encode_many([])
    with pytest.raises(ValueError, match="empty list"):
        m.decode_many([])
    with pytest.raises(ValueError, match="entry 1"):
        m.encode_many([torch.zeros(1, 1, hop), torch.zeros(1, 1, 0)])
    with pytest.raises(ValueError, match="entry 0"):
        m.decode_many([torch.zeros(1, m.latent_dim, 0)])
    with pytest.raises(ValueError, match="different sample rates"):
        m.encode_many([torch.zeros(1, 1, hop)] * 2, [44100, 48000])
    with pytest.raises(ValueError, match="multiple of"):
        m.encode_many([torch.zeros(1, 1, hop + 1)])
    with pytest.raises(ValueError, match="different latent counts"):
        m.decode_many([torch.zeros(1, m.latent_dim, 2), torch.zeros(1, m.latent_dim // 2, 2)])
