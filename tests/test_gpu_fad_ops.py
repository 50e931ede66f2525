"""GPU, op level: the kernels of the Fréchet audio distance against float64 (DESIGN.md §14): the VGGish log-mel
frontend (mel.cu's VGGISH_LOG mode) against oracle/fad_oracle.py, each layer kind of the embedding network through
vnb_dbg_vggish_layer against a float64 composition of the same split operands, and the moments against numpy."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from oracle import fad_oracle as fo
from vampnet_b200 import _lib, fad
from vampnet_b200.audio import AudioSignal

pytestmark = pytest.mark.gpu
DEV = "cuda"
# Layer tolerances, in the codec's model (tests/test_gpu_codec_ops.py): the tensor-core layers form exactly the products
# hi*hi + hi*lo + lo*hi of their split operands, and so does the float64 reference, so what remains is wgmma's fp32
# accumulation, at most K 2^-24 times the root-sum-square of the products (rss; it adds up rather than averaging out),
# 2^-22 of the magnitudes the epilogue adds, and the stored hi + lo representation (2^-17 |v|).  The first layer's fp32
# fmaf chain is held to K 2^-24 of the sum of |products|.  A 2x2 max-pool takes the largest bound of its four inputs.
# The measured largest error / bound per layer kind is in DESIGN.md §14.
TC_K_RSS = 2.0 ** -24
EPS_ADD = 2.0 ** -22
SPLIT_REL = 2.0 ** -17 + 2.0 ** -21


def _split(x):
    return fad._split(x.float().to(DEV))


def _frontend(x):
    xd = torch.as_tensor(x, dtype=torch.float32, device=DEV).reshape(1, -1).contiguous()
    n_ex = fad.num_examples(xd.shape[1])
    out = torch.empty((n_ex, 96, 64), dtype=torch.float32, device=DEV)
    _lib.check(_lib.lib().vnb_vggish_frontend(_lib.ptr(xd), 1, xd.shape[1], _lib.ptr(out), _lib.stream_ptr()))
    return out.cpu().numpy()


def _check_frontend(x):
    got, want = _frontend(x), fo.examples(x)
    assert got.shape == want.shape and got.shape[0] >= 1
    # both are float64 results rounded to fp32 once: they differ by at most a few fp32 ulps
    err = np.abs(got.astype(np.float64) - want) / np.maximum(1.0, np.abs(want))
    assert err.max() <= 1e-6, err.max()


@pytest.mark.parametrize("kind", ["tones", "silence", "dc", "one_example"])
def test_frontend_matches_oracle(kind):
    n = 15600 if kind == "one_example" else 3 * 16000 + 123
    x = {"tones": fo.test_signal(n, 3), "silence": np.zeros(n, np.float32), "dc": np.full(n, 0.25, np.float32),
         "one_example": fo.test_signal(n, 4)}[kind]
    _check_frontend(x)


@pytest.mark.parametrize("sr", [16000, 44100, 48000])
def test_frontend_after_resampling(sr):
    sig = AudioSignal(fo.test_signal(2 * sr, 5, sr=sr)[None, None], sr, device=DEV)
    x = sig.resample(16000).audio_data.reshape(-1).cpu().numpy()
    _check_frontend(x)


def test_frontend_rows_are_independent():
    x = np.stack([fo.test_signal(40000, s) for s in (6, 7, 8)])
    xd = torch.from_numpy(x).to(DEV)
    out = torch.empty((3 * 2, 96, 64), dtype=torch.float32, device=DEV)
    _lib.check(_lib.lib().vnb_vggish_frontend(_lib.ptr(xd), 3, 40000, _lib.ptr(out), _lib.stream_ptr()))
    for r in range(3):
        assert torch.equal(out[2 * r:2 * r + 2].cpu(), torch.from_numpy(_frontend(x[r])))


def _layer(x=None, w=None, a=None, wt=None, Bn=1, H=0, W=0, Cin=1, N=64, bias=None, relu=1, pool=0, out_shape=None,
           f32=False):
    L = _lib.lib()
    out_hi = out_lo = out_f = None
    if f32:
        out_f = torch.empty(out_shape, dtype=torch.float32, device=DEV)
    else:
        out_hi = torch.empty(out_shape, dtype=torch.bfloat16, device=DEV)
        out_lo = torch.empty(out_shape, dtype=torch.bfloat16, device=DEV)
    _lib.check(L.vnb_dbg_vggish_layer(_lib.ptr(x), _lib.ptr(w), _lib.ptr(a[0]) if a else None,
                                      _lib.ptr(a[1]) if a else None, Bn, H, W, Cin, _lib.ptr(wt[0]) if wt else None,
                                      _lib.ptr(wt[1]) if wt else None, N, _lib.ptr(bias), relu, pool, _lib.ptr(out_hi),
                                      _lib.ptr(out_lo), _lib.ptr(out_f), _lib.stream_ptr()))
    return out_f if f32 else out_hi.double() + out_lo.double()


def _check(got, want, tol):
    """Largest |got - want| / tol; asserts it is at most 1."""
    ratio = ((got.double() - want.double()).abs() / tol).max().item()
    assert ratio <= 1.0, ratio
    return ratio


def _tol(want, scale, K, bias):
    return TC_K_RSS * K * scale + EPS_ADD * (want.abs() + bias.abs()) + SPLIT_REL * want.abs()


def test_edge_layer():
    g = torch.Generator().manual_seed(1)
    Bn = 3
    x = torch.from_numpy(np.stack([fo.examples(fo.test_signal(15600, s))[0] for s in range(Bn)])).to(DEV)
    w = (torch.randn(64, 1, 3, 3, generator=g) * (2 / 9) ** 0.5).to(DEV)
    b = ((torch.rand(64, generator=g) - 0.5) * 0.2).to(DEV)
    got = _layer(x=x, w=w.reshape(64, 9).contiguous(), Bn=Bn, Cin=1, N=64, bias=b, out_shape=(Bn, 48, 32, 64))
    pre = Fn.relu(Fn.conv2d(x.double()[:, None], w.double(), b.double(), padding=1))
    abssum = Fn.conv2d(x.double().abs()[:, None], w.double().abs(), padding=1)
    tol = Fn.max_pool2d(_tol(pre, abssum, 9, b.double()[None, :, None, None]), 2)
    want = Fn.max_pool2d(pre, 2)
    print(f"edge layer: err / bound {_check(got, want.permute(0, 2, 3, 1), tol.permute(0, 2, 3, 1)):.3f}")


@pytest.mark.parametrize("H, W, Cin, N, pool", [(48, 32, 64, 128, 1), (24, 16, 128, 256, 0), (24, 16, 256, 256, 1),
                                                (12, 8, 256, 512, 0), (12, 8, 512, 512, 1), (48, 32, 64, 128, 0)])
def test_conv_layer(H, W, Cin, N, pool):
    g = torch.Generator().manual_seed(H * 1000 + Cin + pool)
    Bn = 3
    x = torch.rand(Bn, H, W, Cin, generator=g)  # post-ReLU activations are >= 0
    w = torch.randn(N, Cin, 3, 3, generator=g) * (2 / (9 * Cin)) ** 0.5
    b = (torch.rand(N, generator=g) - 0.5) * 0.2
    a = _split(x)
    wt = _split(w.permute(0, 2, 3, 1).reshape(N, 9 * Cin))
    shape = (Bn, H // 2, W // 2, N) if pool else (Bn, H, W, N)
    got = _layer(a=a, wt=wt, Bn=Bn, H=H, W=W, Cin=Cin, N=N, bias=b.to(DEV), pool=pool, out_shape=shape)
    xs = (a[0].double() + a[1].double()).permute(0, 3, 1, 2)
    ws = (wt[0].double() + wt[1].double()).reshape(N, 3, 3, Cin).permute(0, 3, 1, 2)
    bd = b.double().to(DEV)
    want = Fn.relu(Fn.conv2d(xs, ws, bd, padding=1))
    rss = Fn.conv2d(xs * xs, ws * ws, padding=1).sqrt()
    tol = _tol(want, rss, 9 * Cin, bd[None, :, None, None])
    if pool:
        want, tol = Fn.max_pool2d(want, 2), Fn.max_pool2d(tol, 2)
    ratio = _check(got, want.permute(0, 2, 3, 1), tol.permute(0, 2, 3, 1))
    print(f"conv {H}x{W}x{Cin}->{N} pool {pool}: err / bound {ratio:.3f}")


@pytest.mark.parametrize("M, K, N, relu", [(5, 12288, 4096, 1), (130, 4096, 4096, 1), (7, 4096, 128, 0),
                                           (1, 4096, 128, 0)])
def test_fc_layer(M, K, N, relu):
    g = torch.Generator().manual_seed(M + K + N)
    x = torch.rand(M, K, generator=g)
    w = torch.randn(N, K, generator=g) * (2 / K) ** 0.5
    b = (torch.rand(N, generator=g) - 0.5) * 0.2
    a, wt = _split(x), _split(w)
    got = _layer(a=a, wt=wt, Bn=M, Cin=K, N=N, bias=b.to(DEV), relu=relu, out_shape=(M, N), f32=not relu)
    xs, ws, bd = a[0].double() + a[1].double(), wt[0].double() + wt[1].double(), b.double().to(DEV)
    want = xs @ ws.T + bd
    if relu:
        want = want.clamp_min(0)
    rss = ((xs * xs) @ (ws * ws).T).sqrt()
    tol = _tol(want, rss, K, bd) if relu else TC_K_RSS * K * rss + EPS_ADD * (want.abs() + bd.abs())
    print(f"fc {M}x{K}->{N} relu {relu}: err / bound {_check(got, want, tol):.3f}")


def test_layer_refusals():
    L = _lib.lib()
    z = torch.zeros(1 << 16, device=DEV)
    p = _lib.ptr(z)
    # N not a multiple of 128, an image whose tile is not whole row pairs, a NULL output
    assert L.vnb_dbg_vggish_layer(None, None, p, p, 1, 0, 0, 64, p, p, 96, p, 1, 0, p, p, None, _lib.stream_ptr()) != 0
    assert L.vnb_dbg_vggish_layer(None, None, p, p, 1, 12, 12, 64, p, p, 128, p, 1, 1, p, p, None, _lib.stream_ptr()) != 0
    assert L.vnb_dbg_vggish_layer(None, None, p, p, 1, 0, 0, 64, p, p, 128, p, 0, 0, p, p, None, _lib.stream_ptr()) != 0


def test_moments_match_numpy_and_batching():
    g = torch.Generator().manual_seed(9)
    e = (torch.randn(1000, 128, generator=g) * 3 + 1).to(DEV)
    mu, sigma = fad.moments(e)
    en = e.double().cpu().numpy()
    np.testing.assert_allclose(mu.cpu().numpy(), en.mean(0), rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(sigma.cpu().numpy(), np.cov(en, rowvar=False), rtol=1e-10, atol=1e-11)
    assert torch.equal(sigma, sigma.T)
    mu2, sigma2 = fad.moments(torch.cat([e[:300].clone(), e[300:].clone()]))
    assert torch.equal(mu, mu2) and torch.equal(sigma, sigma2)


def test_frontend_and_moments_refusals():
    L = _lib.lib()
    z = torch.zeros(20000, device=DEV)
    assert L.vnb_vggish_frontend(_lib.ptr(z), 1, 15599, _lib.ptr(z), _lib.stream_ptr()) != 0
    assert b"15600" in L.vnb_last_error()
    assert L.vnb_vggish_frontend(_lib.ptr(z), 0, 15600, _lib.ptr(z), _lib.stream_ptr()) != 0
    assert L.vnb_fad_moments(_lib.ptr(z), 1, _lib.ptr(z), _lib.ptr(z), _lib.stream_ptr()) != 0
    assert L.vnb_fad_moments(None, 5, _lib.ptr(z), _lib.ptr(z), _lib.stream_ptr()) != 0
