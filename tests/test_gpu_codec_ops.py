"""GPU: the codec kernels one at a time against float64 references of their C ABI (tests/codec_op_ref.py), at the layer
shapes of the real codec (encoder 64 .. 1024, decoder 1536 .. 96) and of the reduced-width one (32 ...), with ragged
frame counts and B > 1.

Every output buffer starts as a NaN sentinel, has guard regions before and after it and, for the tensor-core
convolutions, guard rows between batch items (out_batch_stride > out_limit); everything outside the valid range must
keep the sentinel.

Tolerances.  The tensor-core convolution forms exactly the products hi*hi + hi*lo + lo*hi of its split-bf16 operands,
and so does the reference, so what remains is fp32 accumulation, measured against the root-sum-square of the per-term
products (rss).  On an H100 80GB HBM3 (700 W) the largest error / rss per case grew with the reduction length
K = taps x Cin, from 1.1e-6 at K = 32 to 6.4e-5 at K = 12288, and stayed below 0.57 K 2^-24 (wgmma's fp32 accumulation
does not round to nearest, so its error adds up rather than averaging out).  The bound is therefore K 2^-24 rss, plus
2^-22 of the magnitudes the epilogue adds.  Leaving out one cross product costs about 2^-10 of the rss, above the bound
even at the largest K here (12288: 2^-10.4) and far above it at the others; a scale of sum |W||a| would hide it (it is
below 2^-16 of that at K ~ 1e4).
Snake's output adds the fp32 error carried through |snake'| <= 2, __sinf's error (< 1e-6 for |alpha v| < 1e4, divided
by alpha) and the hi + lo representation (2^-17 |v|).
"""
import math

import pytest
import torch

from tests import codec_op_ref as R
from tools import codec_bits as CB
from tools.gemm_bits import untouched

pytestmark = pytest.mark.gpu

TC_K_RSS = 2.0 ** -24          # f32 error <= TC_K_RSS * K * rss (measured at most 0.57x of it)
EPS_ADD = 2.0 ** -22            # rounding of bias / skip additions and of the stored value, relative
SIN_ERR = 1e-6 + 2.0 ** -20     # __sinf after the Cody-Waite reduction, plus the fp32 ops around it (abs, x 1/alpha)
SPLIT_REL = 2.0 ** -17 + 2.0 ** -21   # hi + lo representation of an fp32 value, plus fp32 rounding of alpha * v


def cuda64(t):
    return None if t is None else t.cuda()


def bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def snake_tol(v, alpha, err_v):
    return 2.0 * err_v + SIN_ERR / alpha.double() + SPLIT_REL * v.abs()


# ---------------------------------------------------------------------------------------------------- (a) conv_tc
def tc_reference(c):
    y, rss = R.conv_tc_acc(*(c[k].cuda() for k in ("a_hi", "a_lo", "w_hi", "w_lo")), c["s"], c["N"], c["taps"],
                           c["dil"], c["pad"], c["Tq"])
    resid = c["resid_init"].cuda() if c["resid"] is not None else None
    return R.conv_tc_store(y, rss, cuda64(c["bias"]), c["bias_mod"], cuda64(c["alpha"]), c["alpha_mod"], resid,
                           c["out_batch_stride"], c["out_offset"], c["out_limit"], c["do_tanh"])


def check_tc(c, outs, label):
    pos, f64, act64, rss, skip = tc_reference(c)
    B, stride = c["B"], c["out_batch_stride"]
    written = torch.zeros(stride, dtype=torch.bool, device="cuda")
    written[pos] = True
    nn = (pos - c["out_offset"]) % c["N"]
    bias = c["bias"].cuda().double()[nn % c["bias_mod"]].abs() if c["bias"] is not None else 0.0
    K = c["taps"] * c["Cin"]
    err_f32 = TC_K_RSS * K * rss + EPS_ADD * (f64.abs() + bias + skip)
    for k, full in outs.items():
        assert CB.guards_untouched(full), f"{label}: {k} written outside its buffer"
        v = CB.inner(full).cuda().view(B, stride)
        assert untouched(v[:, ~written]).all(), f"{label}: {k} written outside [0, out_limit) or in a guard row"
        assert not untouched(v[:, written]).any(), f"{label}: {k} not written inside [0, out_limit)"
    f32 = None
    if "f32" in outs:
        f32 = CB.inner(outs["f32"]).cuda().view(B, stride)[:, pos]
        err = (f32.double() - f64).abs()
        ratio = (err / rss.clamp_min(1e-30)).max().item()
        print(f"{label}: K {K}, f32 max err / rss {ratio:.3e} = {ratio / (K * 2.0 ** -24):.3f} K 2^-24, "
              f"max err {err.max().item():.3e}")
        bad = err > err_f32
        assert not bad.any(), f"{label}: f32 {int(bad.sum())} of {bad.numel()} outside tolerance, max err {err.max():.3e}"
    if "hi" in outs:
        hi = CB.inner(outs["hi"]).cuda().view(B, stride)[:, pos]
        lo = CB.inner(outs["lo"]).cuda().view(B, stride)[:, pos]
        if c["alpha"] is None:
            assert f32 is not None
            want_hi = f32.bfloat16()
            want_lo = (f32 - want_hi.float()).bfloat16()
            assert torch.equal(bits(hi), bits(want_hi)), f"{label}: hi != bf16_rn(out_f32)"
            assert torch.equal(bits(lo), bits(want_lo)), f"{label}: lo != bf16_rn(out_f32 - hi)"
        else:
            al = c["alpha"].cuda()[nn % c["alpha_mod"]]
            got = hi.double() + lo.double()
            err = (got - act64).abs()
            tol = snake_tol(act64, al, err_f32)
            print(f"{label}: split max err {err.max().item():.3e}  max err / tol {(err / tol).max().item():.3f}")
            bad = err > tol
            assert not bad.any(), f"{label}: split {int(bad.sum())} of {bad.numel()} outside tolerance"


TQ = (1, 127, 128, 129, 300)


def _cases():
    cs = []
    i = 0

    def add(name, kind, C, Tq, B, **kw):
        nonlocal i
        cs.append(pytest.param(kind, C, Tq, B, 2000 + i, kw, id=name))
        i += 1

    # encoder residual units (k = 7, dil 1 / 3 / 9) and their closing 1x1 with the skip updated in place
    for j, C in enumerate((64, 128, 256, 512)):
        for m, dil in enumerate((1, 3, 9)):
            Tq = TQ[(3 * j + m) % len(TQ)]
            add(f"enc_res7_c{C}_d{dil}_t{Tq}", "res7", C, Tq, 3 if m == 1 else 1, dil=dil)
        add(f"enc_res1_skip_c{C}", "res1", C, 300, 1 + 2 * (j % 2))
    # strided convolutions (A-box shift floor(e / s) < 0 on the first taps)
    for C, s, Tq in ((64, 2, 300), (128, 4, 129), (256, 8, 127), (512, 12, 1)):
        add(f"enc_down_c{C}_s{s}_t{Tq}", "down", C, Tq, 3 if s == 4 else 1, s=s)
    add("enc_conv2_k3_n1024", "conv", 1024, 129, 1, k=3, N=1024, alpha=False, out_split=False, out_f32=True)
    add("dec_conv1_1024_1536", "conv", 1024, 128, 1, k=7, N=1536)
    # transposed convolutions through the offset / limit store (N = 9216, 3072, 768, 192; 192 takes BN = 96), and an
    # odd stride
    for C, s, T in ((1536, 12, 24), (768, 8, 40), (384, 4, 127), (192, 2, 300), (192, 3, 129)):
        add(f"dec_convt_c{C}_s{s}_t{T}", "convt", C, T, 3 if s == 4 else 1, s=s)
    # decoder residual units (C = 96: BN = 96 on n128 MMAs, the second 64-channel block of Cin half empty)
    for j, C in enumerate((768, 384, 192, 96)):
        for m, dil in enumerate((1, 3, 9)):
            Tq = TQ[(3 * j + m + 1) % len(TQ)]
            add(f"dec_res7_c{C}_d{dil}_t{Tq}", "res7", C, Tq, 3 if m == 2 else 1, dil=dil)
        add(f"dec_res1_skip_c{C}", "res1", C, 129 if C == 768 else 300, 3 if C == 96 else 1)
    # reduced widths: n32 and n64, and a strided conv with Cin = 32 whose A box spans two phases of the (T/s, s*C) view
    add("red_res7_c32_d3", "res7", 32, 300, 3, dil=3)
    add("red_res1_skip_c32", "res1", 32, 129, 1)
    add("red_down_c32_s2", "down", 32, 300, 1, s=2)
    add("red_down_c32_s4", "down", 32, 129, 3, s=4)
    add("red_convt_c64_s2", "convt", 64, 300, 1, s=2)
    # CT_GENERIC explicitly
    add("generic_tanh_c64", "res7", 64, 129, 3, do_tanh=True, out_f32=True)
    add("generic_noalpha_f32_split_c128", "res7", 128, 300, 1, alpha=False, out_f32=True)
    add("generic_noalpha_f32_split_c32", "res1", 32, 128, 1, alpha=False, resid="copy")
    add("generic_resid_copy_c128", "res1", 128, 300, 3, resid="copy")
    add("generic_nobias_down_c64_s2", "down", 64, 300, 1, s=2, bias="none")
    return cs


@pytest.mark.parametrize("kind,C,Tq,B,seed,kw", _cases())
def test_conv_tc_against_float64(request, kind, C, Tq, B, seed, kw):
    c = CB.tc_layer(kind, C, Tq, B, seed, **kw)
    label = f"{request.node.callspec.id} [{CB.variant(c)}, n{CB.mma_width(c['N'])}, BN {CB.tile_bn(c['N'])}]"
    check_tc(c, CB.run_tc(c), label)


def row_case(c, b):
    r = dict(c, B=1)
    for k in ("a_hi", "a_lo", "resid_init"):
        if k in c:
            r[k] = c[k][b:b + 1].contiguous()
    return r


@pytest.mark.parametrize("kind,C,Tq,kw", [
    ("res1", 128, 300, {}), ("res7", 96, 129, dict(dil=9)), ("down", 64, 300, dict(s=2)),
    ("convt", 384, 127, dict(s=4)), ("res7", 32, 129, dict(dil=3)), ("res7", 64, 300, dict(do_tanh=True, out_f32=True)),
], ids=["res1_c128", "res7_c96", "down_c64_s2", "convt_c384_s4", "res7_c32", "generic_tanh_c64"])
def test_conv_tc_batch_rows_match_single_launches(kind, C, Tq, kw):
    c = CB.tc_layer(kind, C, Tq, 3, 3000 + C, **kw)
    full = CB.run_tc(c)
    for b in range(3):
        one = CB.run_tc(row_case(c, b))
        for k, t in full.items():
            rows = CB.inner(t).view(3, -1)
            assert torch.equal(bits(rows[b]), bits(CB.inner(one[k]))), f"row {b} of {k} differs from its own launch"


def test_conv_tc_skip_variant_matches_generic():
    """CT_SPLIT_SKIP (resid == out_f32, in place) against CT_GENERIC (resid read from a separate copy)."""
    a = CB.tc_layer("res1", 192, 300, 3, 4001)
    b = CB.tc_layer("res1", 192, 300, 3, 4001, resid="copy")
    assert (CB.variant(a), CB.variant(b)) == ("split_skip", "generic")
    oa, ob = CB.run_tc(a), CB.run_tc(b)
    for k in ("f32", "hi", "lo"):
        assert torch.equal(bits(oa[k]), bits(ob[k])), k


def test_conv_tc_f32_variant_matches_generic():
    """CT_SPLIT_F32 with a zero bias against CT_GENERIC with bias = NULL."""
    a = CB.tc_layer("down", 128, 129, 3, 4002, s=4, bias="zero")
    b = CB.tc_layer("down", 128, 129, 3, 4002, s=4, bias="none")
    assert (CB.variant(a), CB.variant(b)) == ("split_f32", "generic")
    oa, ob = CB.run_tc(a), CB.run_tc(b)
    for k in ("f32", "hi", "lo"):
        assert torch.equal(bits(oa[k]), bits(ob[k])), k


# ---------------------------------------------------------------------------------------------------- (b) snake
def test_snake_at_large_arguments():
    """The epilogue's Snake (Cody-Waite reduction + __sinf) at alpha in {0.05, 0.5, 1.5, 8} and |alpha v| up to 1e4,
    through an identity 1x1 convolution (the fp32 output is v exactly).  Beyond 1e4 the error is reported only.

    This pins Snake to within the resolution of its hi + lo output (2^-17 |v|); it cannot pin the range reduction.
    Dropping the second Cody-Waite constant moves r by k * 1.75e-7, about 2.8e-8 |alpha v| rad, so the output by at
    most 2.8e-8 |v|: under a quarter of an fp32 ulp, and the kernel's own fl32(alpha * v) is already off by up to
    2^-24 |alpha v|.  Only the bit record (tests/test_gpu_codec_bits.py) catches such a change."""
    C, T = 64, 512
    g = torch.Generator().manual_seed(5000)
    alphas = torch.tensor([0.05, 0.5, 1.5, 8.0]).repeat_interleave(16)
    mag = 10.0 ** (torch.rand(1, T, C, generator=g) * 8.0 - 3.0)          # |alpha v| in [1e-3, 1e5]
    sign = torch.where(torch.rand(1, T, C, generator=g) < 0.5, -1.0, 1.0)
    hi, lo = CB.split(sign * mag / alphas)
    v = hi.float() + lo.float()                                            # exactly representable as hi + lo
    c = CB.tc_layer("res1", C, T, 1, 5001, bias="none", resid=None, out_f32=True)
    c["resid"], c["alpha"], c["a_hi"], c["a_lo"] = None, alphas, hi, lo
    c["w_hi"], c["w_lo"] = CB.pack_conv(torch.eye(C)[:, :, None])
    assert CB.variant(c) == "generic"
    outs = CB.run_tc(c)
    n = T * C
    f32 = CB.inner(outs["f32"])[:n].view(T, C)
    assert torch.equal(f32, v[0]), "identity convolution must reproduce v"
    got = (CB.inner(outs["hi"])[:n].double() + CB.inner(outs["lo"])[:n].double()).view(T, C)
    want = R.snake(v[0].double(), alphas)
    err = (got - want).abs()
    tol = SIN_ERR / alphas.double() + SPLIT_REL * want.abs()
    t = (alphas.double() * v[0].double()).abs()
    inside = t <= 1e4
    for a in (0.05, 0.5, 1.5, 8.0):
        sel = alphas == a
        for lo_t, hi_t in ((0, 1e2), (1e2, 1e4), (1e4, 1e5)):
            m = sel[None, :] & (t > lo_t) & (t <= hi_t)
            if m.any():
                print(f"alpha {a}: |alpha v| in ({lo_t:g}, {hi_t:g}]: max err {err[m].max().item():.3e}, "
                      f"max err * alpha {(err[m] * a).max().item():.3e}, max err / tol {(err[m] / tol[m]).max().item():.3f}")
    bad = (err > tol) & inside
    assert not bad.any(), f"{int(bad.sum())} values outside tolerance for |alpha v| <= 1e4"


# ---------------------------------------------------------------------------------------------------- (c) conv_in
@pytest.mark.parametrize("T", [1, 5, 17, 2304 + 3])
@pytest.mark.parametrize("C", [32, 64])
def test_conv_in_against_float64(C, T):
    c = CB.conv_in_case(C, T, 2, 6000 + C + T)
    outs = CB.run_conv_in(c)
    for k, full in outs.items():
        assert CB.guards_untouched(full), k
        assert not untouched(CB.inner(full)).any(), f"{k} not fully written"
    y64, S = R.conv_in(c["x"].cuda(), c["w"].cuda(), c["bias"].cuda(), 3)
    f32 = CB.inner(outs["f32"]).cuda().view(2, T, C).double()
    tol = 7 * 2.0 ** -24 * S                     # seven FMA roundings, each below 2^-24 of the running |sum|
    err = (f32 - y64).abs()
    print(f"conv_in C={C} T={T}: max err {err.max().item():.3e}, max err / tol {(err / tol).max().item():.3f}")
    assert (err <= tol).all(), f"f32 outside 7 FMA roundings; edges: first {err[:, :3].max():.3e}, last {err[:, -3:].max():.3e}"
    al = c["alpha"].cuda()
    got = (CB.inner(outs["hi"]).cuda().double() + CB.inner(outs["lo"]).cuda().double()).view(2, T, C)
    act = R.snake(y64, al)
    tol_s = snake_tol(act, al, tol)
    assert ((got - act).abs() <= tol_s).all(), f"split max err {(got - act).abs().max():.3e}"


# ---------------------------------------------------------------------------------------------------- (d) conv_out
@pytest.mark.parametrize("T", [1, 31, 33, 255, 257, 4100])
@pytest.mark.parametrize("C", [32, 96, 128])
def test_conv_out_against_float64(C, T):
    c = CB.conv_out_case(C, T, 2, 7000 + C + T)
    full = CB.run_conv_out(c)["audio"]
    assert CB.guards_untouched(full), "samples past T (or before the buffer) were written"
    assert not untouched(CB.inner(full)).any(), "sample not written"
    got = CB.inner(full).cuda().view(2, T).double()
    want, S = R.conv_out(*(c[k].cuda() for k in ("a_hi", "a_lo", "w", "bias")), 3)
    tol = 8 * 2.0 ** -24 * S + 4 * 2.0 ** -24    # measured at most 0.8 2^-24 S (28 FMAs per lane, 5 adds, tanhf)
    err = (got - want).abs()
    print(f"conv_out C={C} T={T}: max err {err.max().item():.3e}, max err / tol {(err / tol).max().item():.3f}")
    assert (err <= tol).all()


# ---------------------------------------------------------------------------------------------------- (e) rvq
def rvq_ref(mode, wts, inp, L, cl, cb=None):
    cb = wts["cb"] if cb is None else cb
    return R.rvq(mode, cuda64(inp["in_f"]), cuda64(inp["in_codes"]), wts["win"].cuda(), wts["bin"].cuda(),
                 wts["wout"].cuda(), wts["bout"].cuda(), cb.cuda(), CB.normalized(cb).cuda(), L, channels_last=cl)


def unpack_rvq(outs, B, D, L, T, cl):
    r = {k: CB.inner(v).cuda() for k, v in outs.items()}
    zq = r["zq"].view(B, T, D).permute(0, 2, 1) if cl else r["zq"].view(B, D, T)
    r["zq_cf"] = zq
    if "codes" in r:
        r["codes"] = r["codes"].view(B, L, T)
        r["latents"] = r["latents"].view(B, 8 * L, T)
    return r


ZQ_REL = 2.0 ** -18     # zq against zq_scale = |z| + sum_l |out_proj_l| (float64), per element; measured <= 1.1e-6
LAT_REL = 2.0 ** -21    # latents against sum_d |win x res| + |bin|; measured <= 4.6e-8


@pytest.mark.parametrize("T", [1, 7, 8, 9, 575])
@pytest.mark.parametrize("D", [512, 1024])
@pytest.mark.parametrize("mode,cl", [(0, False), (0, True), (1, False), (2, False)], ids=["enc", "enc_cl", "latents", "codes"])
def test_rvq_against_float64(mode, cl, D, T):
    B = 2
    L = 14 if mode == 0 else 4
    wts = CB.rvq_weights(D, 14, 8000 + D)
    inp = CB.rvq_inputs(mode, {**wts, "L": L}, T, B, 8100 + T, channels_last=cl)
    outs = CB.run_rvq(mode, wts, inp, L, T, B, channels_last=cl, split_out=cl)
    for k, full in outs.items():
        assert CB.guards_untouched(full), f"{k}: written outside its buffer (frames >= T)"
        inn = CB.inner(full)
        assert not ((inn == CB.SENTINEL_CODE) if inn.dtype == torch.int64 else untouched(inn)).any(), f"{k} not written"
    got = unpack_rvq(outs, B, D, L, T, cl)
    ref = rvq_ref(mode, wts, inp, L, cl)
    zq_err = (got["zq_cf"].double() - ref["zq"]).abs() / ref["zq_scale"]
    if mode == 0:
        dv = R.code_divergence(got["codes"], got["latents"], ref)
        nmis = int((dv["first"] < L).sum())
        print(f"rvq enc D={D} T={T}: {nmis} of {B * T} frames diverge, delta {dv['delta']:.3e}, "
              f"max gap {dv['gap'].max().item():.3e}")
        assert (dv["gap"] < dv["delta"]).all(), "a code differs from float64 by more than a near-tie"
        lat_err = ((got["latents"].double() - ref["latents"]).abs().view(B, L, 8, T) / ref["lat_scale"])
        lat_err = lat_err.permute(0, 1, 3, 2)[dv["comparable"]].max().item()
        same = dv["first"] == L
        zq_max = zq_err.permute(0, 2, 1)[same].max().item() if same.any() else 0.0
        print(f"  latents max err / scale {lat_err:.3e}, zq max err / scale {zq_max:.3e}")
        assert lat_err <= LAT_REL and zq_max <= ZQ_REL
        assert nmis <= max(1, B * T // 50)
    elif mode == 1:
        sc = ref["scores"]
        top2 = sc.topk(2, dim=-1).values
        clear = ((top2[..., 0] - top2[..., 1]) >= 2.0 ** -18).all(1)       # (B, T): no near-tie on any level
        zq_max = zq_err.permute(0, 2, 1)[clear].max().item()
        print(f"rvq latents D={D} T={T}: {int((~clear).sum())} frames with a near-tie, zq max err / scale {zq_max:.3e}")
        assert zq_max <= ZQ_REL
    else:
        print(f"rvq codes D={D} T={T}: zq max err / scale {zq_err.max().item():.3e}")
        assert zq_err.max().item() <= ZQ_REL
    if cl:
        zq = got["zq"].view(B, T, D)
        hi, lo = got["zq_hi"].view(B, T, D), got["zq_lo"].view(B, T, D)
        assert torch.equal(bits(hi), bits(zq.bfloat16()))
        assert torch.equal(bits(lo), bits((zq - hi.float()).bfloat16()))


def test_rvq_exact_ties_pick_the_first_index():
    """Duplicated codebook rows give bit-identical scores; the lower index must win, as torch.max picks it, both
    between lanes (the shuffle reduction) and within one lane's strided walk over the codebook."""
    D, T, B, L = 1024, 575, 2, 1
    wts = CB.rvq_weights(D, 1, 8500)
    inp = CB.rvq_inputs(0, wts, T, B, 8501)
    ref0 = rvq_ref(0, wts, inp, L, False)
    picked = torch.unique(ref0["codes"][:, 0].flatten()).tolist()
    cb = wts["cb"].clone()
    pairs = []
    for i, c in enumerate(picked[:96]):
        p = (c + (32 if i % 3 == 0 else 1 + 7 * i)) % wts["V"]             # same lane every third pair
        if p in picked[:96] or any(p in q for q in pairs):
            continue
        cb[0, p] = cb[0, c]
        pairs.append((c, p))
    ref = rvq_ref(0, wts, inp, L, False, cb=cb)
    outs = CB.run_rvq(0, wts, inp, L, T, B, cb=cb)
    got = CB.inner(outs["codes"]).view(B, 1, T).cuda()
    low = {min(c, p) for c, p in pairs}
    tie = torch.tensor([int(x) in low for x in ref["codes"].flatten().tolist()], device="cuda").view(B, 1, T)
    sc = ref["scores"][:, 0]
    distinct = sc.clone()
    for c, p in pairs:
        distinct[..., max(c, p)] = -math.inf
    top2 = distinct.topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1] >= 2.0 ** -18)[:, None, :]
    chk = tie & clear
    print(f"exact ties: {len(pairs)} duplicated rows, {int(chk.sum())} frames checked")
    assert int(chk.sum()) >= 100
    assert torch.equal(got[chk], ref["codes"][chk]), "an exact tie did not go to the first index"


# ---------------------------------------------------------------------------------------------------- (f) conv1d
CONV1D = [
    ("res_k7_d3_snake_resid", ("res", 64, 64, 300, 2), dict(dil=3)),
    ("conv_k7_d9_snake", ("conv", 96, 64, 257, 2), dict(dil=9)),
    ("down_k8_s4", ("conv", 64, 128, 1200, 2), dict(K=8, stride=4)),
    ("down_k24_s12", ("conv", 32, 64, 1200, 1), dict(K=24, stride=12)),
    ("convt_s8", ("convt", 192, 96, 40, 2), dict(s=8)),
    ("convt_s3_odd", ("convt", 64, 32, 50, 2), dict(s=3)),
    ("out_k7_tanh", ("conv", 96, 1, 1000, 2), dict(tanh=True)),
]


@pytest.mark.parametrize("args,kw", [pytest.param(a, k, id=n) for n, a, k in CONV1D])
def test_conv1d_fp32_against_float64(args, kw):
    c = CB.conv1d_case(*args, seed=9000 + args[3], **kw)
    full = CB.run_conv1d(c)["y"]
    assert CB.guards_untouched(full)
    got = CB.inner(full).cuda().view(c["B"], c["Cout"], c["Tout"])
    y_init = (c["resid"] if c["resid"] is not None else torch.zeros(c["B"], c["Cout"], c["Tout"])).cuda()
    want = y_init.double()
    written = torch.zeros(c["Tout"], dtype=torch.bool, device="cuda")
    rss, scale = torch.zeros_like(want), torch.zeros_like(want)
    n = 0
    for w, stride, dil, pad, ostr, ooff, nq in CB.conv1d_launches(c):
        y, wr, r, s = R.conv1d(c["x"].cuda(), w.cuda(), c["bias"].cuda(), c["alpha"].cuda(),
                               cuda64(c["resid"]), c["Tout"], stride, dil, pad, ostr, ooff, nq, c["tanh"], want)
        want = torch.where(wr, y, want)
        rss, scale = torch.where(wr, r, rss), torch.where(wr, s, scale)
        written |= wr
        n = c["Cin"] * w.shape[-1]
    assert written.all(), "reference does not cover the output"
    assert not untouched(got).any(), "output not fully written"
    tol = 2.0 ** -22 * math.sqrt(n) * rss + 2.0 ** -21 * scale
    err = (got.double() - want).abs()
    print(f"conv1d {args}: max err {err.max().item():.3e}, max err / tol {(err / tol).max().item():.3f}")
    assert (err <= tol).all()
