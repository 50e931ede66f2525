"""CPU: the ABI-level float64 references of tests/codec_op_ref.py (channels-last, packed split-bf16 weights, the
offset / limit / batch-stride store) equal the codec oracle's layers (oracle/dac_oracle.py: F.conv1d,
F.conv_transpose1d, snake, the RVQ) on the same values, in float64.  The inputs are built by tools/codec_bits.py and
packed by the product's DAC._pack_conv_tc / _pack_convt_tc, so the packing and the kernels' index arithmetic are pinned
to the oracle here, and tests/test_gpu_codec_ops.py pins the kernels to these references."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import dac_oracle as do
from tests import codec_op_ref as R
from tools import codec_bits as CB

TOL = 1e-12


def unsplit(hi, lo):
    return hi.double() + lo.double()


def weight64(c):
    """The split weight in the oracle's layout, as float64: Conv1d (Cout, Cin, K) or ConvTranspose1d (Cin, Cout, 2s)."""
    hi, lo = CB.split(c["w"])
    return unsplit(hi, lo)


def abi_output(c, products=R.ALL_PRODUCTS):
    """The reference's stored fp32 stream and split value as (B, rows, cout) channels-last tensors."""
    y, rss = R.conv_tc_acc(c["a_hi"], c["a_lo"], c["w_hi"], c["w_lo"], c["s"], c["N"], c["taps"], c["dil"], c["pad"],
                           c["Tq"], products=products)
    resid = c["resid_init"] if c["resid"] is not None else None
    pos, f32, act, _, _ = R.conv_tc_store(y, rss, c["bias"], c["bias_mod"], c["alpha"], c["alpha_mod"], resid,
                                          c["out_batch_stride"], c["out_offset"], c["out_limit"], c["do_tanh"])
    B, rows, cout = c["B"], c["rows"], c["cout"]
    assert torch.equal(pos, torch.arange(rows * cout)), "the store must cover [0, out_limit) exactly once"
    return f32.view(B, rows, cout), act.view(B, rows, cout)


def oracle_conv(c):
    """The same layer through the oracle's functions, channels-first in, channels-last out."""
    x = unsplit(c["a_hi"], c["a_lo"]).permute(0, 2, 1)
    w, b = weight64(c), c["bias"].double()
    if c["kind"] == "convt":
        s = c["stride_s"]
        y = F.conv_transpose1d(x, w, b, stride=s, padding=math.ceil(s / 2))
    elif c["kind"] == "down":
        s = c["stride_s"]
        y = F.conv1d(x, w, b, stride=s, padding=math.ceil(s / 2))
    else:
        K = w.shape[-1]
        y = F.conv1d(x, w, b, dilation=c["dil"], padding=(K - 1) * c["dil"] // 2)
    if c["resid"] is not None:
        y = y + c["resid_init"][:, :c["rows"] * c["cout"]].double().view(c["B"], c["rows"], c["cout"]).permute(0, 2, 1)
    act = do.snake(y, c["alpha"].double()) if c["alpha"] is not None else y
    return y.permute(0, 2, 1), act.permute(0, 2, 1)


@pytest.mark.parametrize("kind,C,Tq,B,kw", [
    ("res7", 64, 37, 2, dict(dil=1)), ("res7", 96, 40, 1, dict(dil=3)), ("res7", 32, 50, 2, dict(dil=9)),
    ("res1", 128, 20, 2, {}), ("res1", 32, 9, 1, {}),
    ("down", 64, 13, 2, dict(s=2)), ("down", 32, 11, 1, dict(s=4)), ("down", 64, 5, 1, dict(s=8)),
    ("down", 32, 4, 2, dict(s=12)),
    ("convt", 192, 9, 2, dict(s=2)), ("convt", 128, 7, 1, dict(s=4)), ("convt", 64, 5, 1, dict(s=8)),
    ("convt", 64, 4, 2, dict(s=12)), ("convt", 64, 6, 1, dict(s=3)),
    ("conv", 128, 21, 1, dict(k=3, N=64, alpha=False, out_split=False, out_f32=True)),
    ("conv", 64, 15, 2, dict(k=7, N=96)),
])
def test_conv_tc_reference_equals_oracle_layers(kind, C, Tq, B, kw):
    c = CB.tc_layer(kind, C, Tq, B, seed=77, **kw)
    f32, act = abi_output(c)
    of32, oact = oracle_conv(c)
    assert f32.shape == of32.shape, (f32.shape, of32.shape)
    assert (f32 - of32).abs().max() < TOL
    assert (act - oact).abs().max() < TOL


def test_conv_tc_reference_forms_three_products():
    """The default reference leaves out exactly lo * lo, as the kernel does."""
    c = CB.tc_layer("res7", 64, 30, 1, seed=78)
    y3, _ = R.conv_tc_acc(c["a_hi"], c["a_lo"], c["w_hi"], c["w_lo"], 1, 64, 7, 1, 3, 30)
    y4, _ = R.conv_tc_acc(c["a_hi"], c["a_lo"], c["w_hi"], c["w_lo"], 1, 64, 7, 1, 3, 30, products=R.ALL_PRODUCTS)
    yl, _ = R.conv_tc_acc(c["a_hi"], c["a_lo"], c["w_hi"], c["w_lo"], 1, 64, 7, 1, 3, 30, products=("ll",))
    assert (y4 - y3 - yl).abs().max() < TOL
    assert yl.abs().max() > 0


def test_conv_tc_store_guard_rows_and_tanh():
    c = CB.tc_layer("res1", 64, 10, 2, seed=79, resid="copy", do_tanh=True)
    f32, _ = abi_output(c)
    of32, _ = oracle_conv(c)
    assert (f32 - torch.tanh(of32)).abs().max() < TOL
    assert c["out_batch_stride"] == (10 + CB.GUARD_ROWS) * 64


@pytest.mark.parametrize("T", [1, 5, 17])
def test_conv_in_reference_equals_oracle(T):
    c = CB.conv_in_case(32, T, 2, seed=80)
    y, _ = R.conv_in(c["x"], c["w"], c["bias"], 3)
    want = F.conv1d(c["x"].double()[:, None], c["w"].double(), c["bias"].double(), padding=3)
    assert (y - want.permute(0, 2, 1)).abs().max() < TOL


@pytest.mark.parametrize("T", [1, 33])
def test_conv_out_reference_equals_oracle(T):
    c = CB.conv_out_case(96, T, 2, seed=81)
    y, _ = R.conv_out(c["a_hi"], c["a_lo"], c["w"], c["bias"], 3)
    a = unsplit(c["a_hi"], c["a_lo"]).permute(0, 2, 1)
    want = torch.tanh(F.conv1d(a, c["w"].double(), c["bias"].double(), padding=3))[:, 0]
    assert (y - want).abs().max() < TOL


@pytest.mark.parametrize("name,args,kw", [
    ("res", ("res", 32, 32, 40, 2), dict(dil=3)), ("down", ("conv", 16, 32, 48, 1), dict(K=8, stride=4)),
    ("convt_s4", ("convt", 32, 16, 9, 2), dict(s=4)), ("convt_s3", ("convt", 32, 16, 9, 1), dict(s=3)),
    ("tanh", ("conv", 32, 1, 40, 1), dict(tanh=True)),
])
def test_conv1d_reference_equals_oracle(name, args, kw):
    c = CB.conv1d_case(*args, seed=82, **kw)
    want_init = c["resid"] if c["resid"] is not None else torch.zeros(c["B"], c["Cout"], c["Tout"])
    y = want_init.double()
    for w, stride, dil, pad, ostr, ooff, nq in CB.conv1d_launches(c):
        yy, wr, _, _ = R.conv1d(c["x"], w, c["bias"], c["alpha"], c["resid"], c["Tout"], stride, dil, pad, ostr, ooff,
                                nq, c["tanh"], y)
        y = torch.where(wr, yy, y)
    x = do.snake(c["x"].double(), c["alpha"].double())
    if c["kind"] == "convt":
        s = c["s"]
        want = F.conv_transpose1d(x, c["w"].double(), c["bias"].double(), stride=s, padding=math.ceil(s / 2))
    else:
        want = F.conv1d(x, c["w"].double(), c["bias"].double(), stride=c["stride"], dilation=c["dil"], padding=c["pad"])
        if c["resid"] is not None:
            want = want + c["resid"].double()
        if c["tanh"]:
            want = torch.tanh(want)
    assert y.shape == want.shape
    assert (y - want).abs().max() < TOL


def oracle_weights(wts, L, cfg):
    w = {}
    for i in range(L):
        p = f"quantizer.quantizers.{i}"
        w[p + ".in_proj.weight"] = wts["win"][i].double()[:, :, None]
        w[p + ".in_proj.bias"] = wts["bin"][i].double()
        w[p + ".out_proj.weight"] = wts["wout"][i].double()[:, :, None]
        w[p + ".out_proj.bias"] = wts["bout"][i].double()
        w[p + ".codebook.weight"] = wts["cb"][i].double()
    return w


def test_rvq_reference_equals_oracle():
    D, L, T, B = 64, 6, 9, 2
    cfg = do.CodecConfig(encoder_dim=4, n_codebooks=L)     # latent_dim 64
    wts = CB.rvq_weights(D, L, seed=83, V=128)
    w = oracle_weights(wts, L, cfg)
    cbn = F.normalize(wts["cb"].double(), dim=-1)
    args = (wts["win"], wts["bin"], wts["wout"], wts["bout"], wts["cb"], cbn)
    z = CB.rvq_inputs(0, wts, T, B, seed=84)["in_f"].double()
    got = R.rvq(0, z, None, *args, L)
    zq, codes, lat = do.rvq_encode(z, w, cfg)
    assert torch.equal(got["codes"], codes)
    assert (got["zq"] - zq).abs().max() < TOL and (got["latents"] - lat).abs().max() < TOL
    got_cl = R.rvq(0, z.permute(0, 2, 1), None, *args, L, channels_last=True)
    assert torch.equal(got_cl["codes"], codes) and (got_cl["zq"] - zq).abs().max() < TOL
    assert (got["scores"].max(-1)[1] == codes).all()
    got2 = R.rvq(2, None, codes, *args, L)
    assert (got2["zq"] - do.rvq_from_codes(codes, w, cfg)).abs().max() < TOL
    latents = CB.rvq_inputs(1, wts, T, B, seed=85)["in_f"].double()
    got1 = R.rvq(1, latents, None, *args, L)
    assert (got1["zq"] - do.rvq_from_latents(latents, w, cfg)[0]).abs().max() < TOL
