"""GPU: the ragged codec entry points (vnb_codec_conv_tc_ragged, vnb_codec_conv_in_ragged, vnb_codec_conv_out_ragged)
called directly, on every distinct layer of the full-size, the reduced-width (SMALL) and the odd-rate codec, and on
all four epilogue variants at MMA widths 32, 64 and 128.

One launch holds items whose output lengths are 1, 27, 127, 128, 129, 255 and the launch's own.  An item's valid input
rows are random, its next 128 rows (the halo the previous layer writes) are +0, and every row past that holds a NaN
sentinel; outputs start as the sentinel.  Required of every item:
  - valid rows equal, bit for bit, a launch of the item alone at its own length (the plain entry point);
  - halo rows [len, len + 128) are +0 (bit pattern 0) in every output;
  - rows past the halo keep the sentinel: the CTAs whose rows all lie there did not run, and the others stored nothing
    there.
"""
import pytest
import torch

from tools import codec_bits as CB
from tools.gemm_bits import SENTINEL_BF16, SENTINEL_F32, sentinel, untouched

pytestmark = pytest.mark.gpu

HALO = 128
ITEM_LENGTHS = (1, 27, 127, 128, 129, 255)
T_LAUNCH = 300


def L():
    from vampnet_b200 import _lib
    return _lib


def dev_lens(lens):
    return torch.tensor(lens, dtype=torch.int32, device="cuda")


def _layers():
    """(label, tc_layer arguments) of every distinct tensor-core layer of the three codecs, plus the epilogue variants
    the codec does not use at some widths."""
    out = {}

    def add(label, kind, C, **kw):
        out.setdefault((kind, C, tuple(sorted(kw.items()))), (label, kind, C, kw))

    for name, enc_dim, rates, dec_dim, dec_rates in (("full", 64, (2, 4, 8, 12), 1536, (8, 8, 4, 2)),
                                                      ("small", 32, (2, 4, 8, 12), 512, (8, 8, 4, 2)),
                                                      ("odd", 32, (3, 2), 256, (2, 3))):
        d = enc_dim
        for s in rates:
            for dil in (1, 3, 9):
                add(f"{name}_enc_res7_c{d}_d{dil}", "res7", d, dil=dil)
            add(f"{name}_enc_res1_c{d}", "res1", d)
            add(f"{name}_enc_down_c{d}_s{s}", "down", d, s=s)
            d *= 2
        latent = d
        add(f"{name}_enc_conv2_c{latent}", "conv", latent, N=latent, k=3, alpha=False, out_f32=True, out_split=False)
        add(f"{name}_dec_conv1_c{latent}", "conv", latent, N=dec_dim, k=7)
        c = dec_dim
        for s in dec_rates:
            add(f"{name}_dec_convt_c{c}_s{s}", "convt", c, s=s)
            for dil in (1, 3, 9):
                add(f"{name}_dec_res7_c{c // 2}_d{dil}", "res7", c // 2, dil=dil)
            add(f"{name}_dec_res1_c{c // 2}", "res1", c // 2)
            c //= 2
    # the run-time (generic) epilogue and the fp32-stream epilogue at the narrow widths
    add("generic_n32", "res7", 32, alpha=False)
    add("generic_n64", "res7", 64, alpha=False)
    add("generic_n128_tanh", "res7", 128, do_tanh=True)
    add("split_f32_n32", "res7", 32, out_f32=True)
    return sorted(out.values(), key=lambda v: v[0])


LAYERS = _layers()


def _geometry(c, t):
    """For an item of t rows at the layer's input rate (convt: input frames; else output rows): (Tin, Tq, rows)."""
    if c["kind"] == "convt":
        s = c["stride_s"]
        return t, t + 1, t * s - s % 2
    return t * c["s"], t, t


def _launch(c, a_hi, a_lo, Tin, Tq, rows, resid_rows, lens=None):
    """Runs the layer over a_hi / a_lo (B, Tin, Cin) into sentinel-filled outputs of `rows` rows; resid_rows: (B, rows,
    cout) initial fp32 stream of an in-place skip.  Returns the outputs as (B, rows, cout) tensors."""
    lib = L()
    B, cout = a_hi.shape[0], c["cout"]
    shape = (B, rows, cout)
    outs = {}
    if c["out_f32"]:
        outs["f32"] = resid_rows.clone() if c["resid"] == "inplace" else sentinel(shape, torch.float32)
    if c["out_split"]:
        outs["hi"], outs["lo"] = sentinel(shape, torch.bfloat16), sentinel(shape, torch.bfloat16)
    resid = outs["f32"] if c["resid"] == "inplace" else (resid_rows if c["resid"] == "copy" else None)
    w_hi, w_lo = c["w_hi"].cuda(), c["w_lo"].cuda()
    bias = None if c["bias"] is None else c["bias"].cuda()
    alpha = None if c["alpha"] is None else c["alpha"].cuda()
    off = c["out_offset"]
    args = (lib.ptr(a_hi), lib.ptr(a_lo), B, Tin, c["Cin"], c["s"], lib.ptr(w_hi), lib.ptr(w_lo), c["N"], c["taps"],
            c["dil"], c["pad"], Tq, lib.ptr(bias), c["bias_mod"], lib.ptr(alpha), c["alpha_mod"], lib.ptr(resid),
            lib.ptr(outs.get("f32")), lib.ptr(outs.get("hi")), lib.ptr(outs.get("lo")), rows * cout, off, rows * cout,
            1 if c["do_tanh"] else 0)
    if lens is None:
        lib.check(lib.lib().vnb_codec_conv_tc(*args, lib.stream_ptr()))
    else:
        lib.check(lib.lib().vnb_codec_conv_tc_ragged(*args, lib.ptr(lens), cout, lib.stream_ptr()))
    return outs


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _check_item(label, got, alone, n_valid, rows):
    """got / alone: dict of (rows, cout) / (n_valid, cout) tensors of one item."""
    for k, g in got.items():
        assert torch.equal(_bits(g[:n_valid]), _bits(alone[k])), f"{label}: {k} valid rows differ from the item alone"
        h = min(n_valid + HALO, rows)
        assert (_bits(g[n_valid:h]) == 0).all(), f"{label}: {k} halo rows are not +0"
        assert untouched(g[h:]).all(), f"{label}: {k} written past the halo"


@pytest.mark.parametrize("label,kind,C,kw", LAYERS, ids=[v[0] for v in LAYERS])
def test_conv_tc_ragged_matches_items_alone(label, kind, C, kw):
    c = CB.tc_layer(kind, C, T_LAUNCH, 1, seed=5, **kw)
    items = list(ITEM_LENGTHS) + [T_LAUNCH]           # convt: input frames; else output rows
    B = len(items)
    Tin, Tq, rows = _geometry(c, T_LAUNCH)
    g = torch.Generator().manual_seed(11)
    a = torch.randn(B, Tin, c["Cin"], generator=g)
    a_hi, a_lo = (t.cuda() for t in CB.split(a))
    skip = torch.randn(B, rows, c["cout"], generator=g).cuda()
    outs_len, skip_in = [], skip.clone()
    for b, t in enumerate(items):
        t_in, _, n = _geometry(c, t)
        outs_len.append(n)
        # the halo the previous layer leaves: +0 on [t_in, t_in + 128), a NaN sentinel past it
        a_hi[b, t_in:t_in + HALO] = 0
        a_lo[b, t_in:t_in + HALO] = 0
        a_hi[b, t_in + HALO:].view(torch.int16).fill_(SENTINEL_BF16)
        a_lo[b, t_in + HALO:].view(torch.int16).fill_(SENTINEL_BF16)
        skip_in[b, n:].view(torch.int32).fill_(SENTINEL_F32)
    got = _launch(c, a_hi, a_lo, Tin, Tq, rows, skip_in, lens=dev_lens(outs_len))
    for b, t in enumerate(items):
        t_in, tq, n = _geometry(c, t)
        alone = _launch(c, a_hi[b:b + 1, :t_in].contiguous(), a_lo[b:b + 1, :t_in].contiguous(), t_in, tq, n,
                        skip[b:b + 1, :n].contiguous())
        _check_item(f"{label} item {b} ({n} rows)", {k: v[b] for k, v in got.items()}, {k: v[0] for k, v in alone.items()},
                    n, rows)


@pytest.mark.parametrize("C", [32, 64])
def test_conv_in_ragged_matches_items_alone(C):
    lib = L()
    items = list(ITEM_LENGTHS) + [T_LAUNCH * 4]
    B, T = len(items), T_LAUNCH * 4
    c = CB.conv_in_case(C, T, B, seed=21)
    x = c["x"].clone()
    for b, n in enumerate(items):
        x[b, n:] = float("nan")                       # reads are bounded by the item's length, not by padding
    x = x.cuda()
    w, bias, al = (c[k].cuda() for k in ("w", "bias", "alpha"))

    def run(xx, BB, TT, lens=None):
        f, h, lo = sentinel((BB, TT, C), torch.float32), sentinel((BB, TT, C), torch.bfloat16), \
            sentinel((BB, TT, C), torch.bfloat16)
        args = (lib.ptr(xx), lib.ptr(w), lib.ptr(bias), lib.ptr(al), lib.ptr(f), lib.ptr(h), lib.ptr(lo), BB, TT, C, 7, 3)
        if lens is None:
            lib.check(lib.lib().vnb_codec_conv_in(*args, lib.stream_ptr()))
        else:
            lib.check(lib.lib().vnb_codec_conv_in_ragged(*args, lib.ptr(lens), lib.stream_ptr()))
        return dict(f32=f, hi=h, lo=lo)

    got = run(x, B, T, dev_lens(items))
    for b, n in enumerate(items):
        alone = run(x[b:b + 1, :n].contiguous(), 1, n)
        _check_item(f"conv_in C {C} item {b} ({n} samples)", {k: v[b] for k, v in got.items()},
                    {k: v[0] for k, v in alone.items()}, n, T)


@pytest.mark.parametrize("C", [32, 64, 96])
def test_conv_out_ragged_matches_items_alone(C):
    lib = L()
    items = list(ITEM_LENGTHS) + [T_LAUNCH * 4]
    B, T = len(items), T_LAUNCH * 4
    c = CB.conv_out_case(C, T, B, seed=22)
    ah, al = c["a_hi"].cuda(), c["a_lo"].cuda()
    for b, n in enumerate(items):
        ah[b, n:].view(torch.int16).fill_(SENTINEL_BF16)
        al[b, n:].view(torch.int16).fill_(SENTINEL_BF16)
    w, bias = c["w"].cuda(), c["bias"].cuda()

    def run(h, lo, BB, TT, lens=None):
        audio = sentinel((BB, TT), torch.float32)
        args = (lib.ptr(h), lib.ptr(lo), lib.ptr(w), lib.ptr(bias), lib.ptr(audio), BB, TT, C, 7, 3)
        if lens is None:
            lib.check(lib.lib().vnb_codec_conv_out(*args, lib.stream_ptr()))
        else:
            lib.check(lib.lib().vnb_codec_conv_out_ragged(*args, lib.ptr(lens), lib.stream_ptr()))
        return audio

    got = run(ah, al, B, T, dev_lens(items))
    for b, n in enumerate(items):
        alone = run(ah[b:b + 1, :n].contiguous(), al[b:b + 1, :n].contiguous(), 1, n)
        assert torch.equal(got[b, :n].view(torch.int32), alone[0].view(torch.int32)), f"conv_out C {C} item {b}"
        assert untouched(got[b, n:]).all(), f"conv_out C {C} item {b}: written past the item's samples"


def test_ragged_entry_points_refuse_a_missing_table():
    lib = L()
    x = torch.zeros(1, 768, device="cuda")
    with pytest.raises(RuntimeError, match="length table"):
        lib.check(lib.lib().vnb_codec_conv_in_ragged(lib.ptr(x), lib.ptr(x), lib.ptr(x), lib.ptr(x), lib.ptr(x),
                                                    lib.ptr(x), lib.ptr(x), 1, 4, 4, 7, 3, None, lib.stream_ptr()))
    with pytest.raises(RuntimeError, match="length table"):
        lib.check(lib.lib().vnb_codec_conv_out_ragged(lib.ptr(x), lib.ptr(x), lib.ptr(x), lib.ptr(x), lib.ptr(x), 1, 4,
                                                     4, 7, 3, None, lib.stream_ptr()))
