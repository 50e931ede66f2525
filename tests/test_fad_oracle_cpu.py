"""CPU: the float64 restatement of the Fréchet audio distance (oracle/fad_oracle.py) and the host half of
vampnet_b200.fad (the distance, the checkpoint checks that run before any device call)."""
import numpy as np
import pytest
import torch

from oracle import fad_oracle as fo
from vampnet_b200 import fad


@pytest.fixture(scope="module")
def sd():
    return fo.random_state_dict(5)


def test_oracle_network_equals_torchvggish_layer_list(sd):
    """The oracle's NHWC flatten is torchvggish's transpose(1, 3).transpose(1, 2).view: equal to float64 rounding."""
    ex = np.stack([fo.examples(fo.test_signal(15600, s)) [0] for s in (1, 2)])
    want = fo.torch_module(sd)(torch.from_numpy(ex).double()[:, None]).detach().numpy()
    got = fo.embed(ex, sd)
    assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max()


def test_module_state_dict_passes_the_checkpoint_checks(sd):
    """A torchvggish-layout state dict (with the checkpoint's pproc.* tensors) has every key and shape VGGish needs."""
    m = fo.torch_module(sd)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == fad.expected_shapes()


def test_bad_checkpoints_are_refused(sd):
    """Missing keys, wrong shapes and unexpected keys raise ValueError before any device work."""
    bad = dict(sd)
    del bad["features.8.bias"]
    with pytest.raises(ValueError, match="missing"):
        fad.VGGish(bad, device="cpu")
    bad = dict(sd)
    bad["embeddings.0.weight"] = torch.zeros(4096, 512 * 6 * 4 + 1)
    with pytest.raises(ValueError, match="shape"):
        fad.VGGish(bad, device="cpu")
    bad = dict(sd, **{"features.15.weight": torch.zeros(1)})
    with pytest.raises(ValueError, match="unexpected"):
        fad.VGGish(bad, device="cpu")


def test_unsupported_flags_are_refused(sd):
    with pytest.raises(ValueError, match="use_pca"):
        fad.FrechetAudioDistance(sd, use_pca=True)
    with pytest.raises(ValueError, match="use_activation"):
        fad.FrechetAudioDistance(sd, use_activation=True)


def test_htk_matrix():
    m = fo.htk_matrix()
    assert m.shape == (257, 64) and not m[0].any() and (m >= 0).all()
    edges = np.linspace(fo.hz_to_mel(125.0), fo.hz_to_mel(7500.0), 66)
    bins = fo.hz_to_mel(np.linspace(0, 8000, 257))
    for i in range(64):
        nz = np.nonzero(m[1:, i])[0] + 1
        # each band is nonzero strictly between its lower and upper edge, and peaks at the bin nearest its centre
        assert (bins[nz] > edges[i]).all() and (bins[nz] < edges[i + 2]).all()
        inside = np.nonzero((bins > edges[i]) & (bins < edges[i + 2]))[0]
        assert set(inside[inside > 0]) == set(nz)
    # mel = 1127 ln(1 + f / 700): 1000 Hz is 999.985 mel
    assert abs(fo.hz_to_mel(1000.0) - 1127.0 * np.log(1 + 1000 / 700)) < 1e-12


@pytest.mark.parametrize("n, want", [(15599, 0), (15600, 1), (160000, 10), (30959, 1), (30960, 2), (0, 0), (399, 0)])
def test_example_counts(n, want):
    assert fo.num_examples(n) == fad.num_examples(n) == want
    if n >= 400:
        assert fo.examples(np.zeros(n, np.float32)).shape == (want, 96, 64)


def _gauss(seed, m=400, d=128, scale=1.0):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((m, d)) * scale + rng.standard_normal(d)


def test_distance_of_a_set_with_itself_is_zero():
    mu, s = fo.stats(_gauss(1))
    assert abs(fad.frechet_distance(mu, s, mu, s)) < 1e-8 * np.trace(s)


def test_diagonal_gaussians_closed_form():
    rng = np.random.default_rng(2)
    a, b = rng.uniform(0.1, 2.0, 128), rng.uniform(0.1, 2.0, 128)
    m1, m2 = rng.standard_normal(128), rng.standard_normal(128)
    want = ((m1 - m2) ** 2).sum() + ((np.sqrt(a) - np.sqrt(b)) ** 2).sum()
    for f in (fad.frechet_distance, fo.frechet_distance):
        assert abs(f(m1, np.diag(a), m2, np.diag(b)) - want) <= 1e-10 * want


def test_distance_is_symmetric():
    m1, s1 = fo.stats(_gauss(3))
    m2, s2 = fo.stats(_gauss(4, scale=1.3))
    d12, d21 = fad.frechet_distance(m1, s1, m2, s2), fad.frechet_distance(m2, s2, m1, s1)
    assert abs(d12 - d21) <= 1e-9 * d12
    assert abs(d12 - fo.frechet_distance(m1, s1, m2, s2)) <= 1e-12 * d12


def test_complex_result_raises():
    """A product s1 s2 with a negative eigenvalue has a square root with an imaginary diagonal."""
    s1 = np.diag([1.0, 1.0])
    s2 = np.diag([-4.0, 1.0])
    with pytest.raises(ValueError, match="[Ii]maginary"):
        fad.frechet_distance(np.zeros(2), s1, np.zeros(2), s2)


def test_score_moments_and_fewer_than_two_embeddings():
    m1, m2 = fo.stats(_gauss(5)), fo.stats(_gauss(6))
    assert fad.FrechetAudioDistance.score_moments(m1, m2) == fad.frechet_distance(*m1, *m2)
    with pytest.raises(ValueError, match="two"):
        fad.moments(torch.zeros(1, 128))
