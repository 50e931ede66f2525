"""GPU: the sampling step's kernels, one path at a time through vnb_dbg_sample (include/vampnet_b200.h), against the
float64 reference tests/sample_ref.py (pinned to the oracle's sampler by tests/test_sample_ref_cpu.py).

Every call starts from tokens and conf filled with a NaN sentinel.  Known positions must come back exactly (token =
zcur, conf = +inf); zcur after the call must equal the reference re-mask rule applied to the kernel's OWN conf and
tokens, exactly, conditioning codebooks included.

Tokens must equal the reference's wherever the reference calls the draw unambiguous (no crossing within AMBIGUOUS_REL
of its target, no uncertain nucleus token that changes the draw); greedy draws are never ambiguous.  At most
AMBIG_MAX of the masked positions of a call may be ambiguous.

Confidence bound.  The kernel computes log(expf(xs - m) / se) + fp32(temp_eff) * (-logf(-logf(u))) in fp32: se is a
sum of up to 1024 expf terms (relative error a few 1e-7, ~1e-6 worst case, i.e. an absolute error of that size in log
p), logf adds an ulp of |log p|, the Gumbel term an ulp or two of its own size (its inner log's relative error times 1,
and the product's rounding), and the final add half an ulp of |conf|.  The bound is therefore
    CONF_ABS + CONF_REL * (|log p| + |temp_eff * g|)   (+ the reference's logp_spread for a nucleus boundary token)
with CONF_ABS = 2e-5 and CONF_REL = 2^-21 (8 ulp-units of fp32).  sample_combine_kernel uses ex2.approx (2 ulp) and
fp32(inv_t * log2 e), which stays inside the same bound against a reference that starts from the same records.  Its
records, however, carry each strip's sum scaled by 2^delta, delta = max*c1 - fp32(max*c1) the rounding of the
epilogue's c0 (tests/gemm_sample_ref.py), |delta| <= 2^-24 |max * c1|; against float64 softmax of the logits the
confidence therefore also moves by up to ln 2 * 2 max |delta| <= 2^-23 max_v |x_v * inv_t| (COMBINE_REL), which is what
the logits of large row scales (|x| ~ 5e3) show.

Measured on an H100 80GB HBM3 (700 W): confidence error at most 1.0e-5 on the materialised draws (0.16 of the bound),
1.5e-4 where a nucleus boundary token is uncertain (0.85 of that bound, which includes logp_spread), 6.8e-4 on the
combine path with |x| ~ 5e3 (0.31 of its bound); 65 of 78 990 draws were ambiguous (0.08 %), at most 4 of 310 in one
call."""
import hashlib

import numpy as np
import pytest
import torch

from oracle import philox
from tests import gemm_sample_ref as GR
from tests import sample_ref as SR
from tests.sample_ref import Group
from tools import gemm_bits as GB
from tools import sample_bits as SB

pytestmark = pytest.mark.gpu

CONF_ABS = 2e-5
CONF_REL = 2.0 ** -21
COMBINE_REL = 2.0 ** -22    # twice the 2^-23 derived above
AMBIG_MAX, AMBIG_SLACK = 0.01, 2   # per call: 1 % of the masked draws, plus 2 for calls of a few hundred draws
SEED = (9001, 17)


def gen(*key):
    return torch.Generator().manual_seed(int(hashlib.sha256(repr(key).encode()).hexdigest()[:8], 16))


def n0_of(zcur, groups, ncc, V):
    """Each group's count of masked predicted entries (what gen_init_kernel computes at the first step)."""
    out, b = [], 0
    for g in groups:
        out.append(int((zcur[b:b + g.rows, :, ncc:] == V).sum()))
        b += g.rows
    return out


def group_refs(logits, groups, S, V):
    refs, b = [], 0
    for g in groups:
        refs.append(SR.sample_group(logits[b * S:(b + g.rows) * S].view(g.rows, S, V), g))
        b += g.rows
    return refs


def run(path, zcur0, groups, n0, ncc, V, logits=None, partials=None, zorig=None, tokens=None, conf=None):
    B, T, C = zcur0.shape
    S = T * (C - ncc)
    z = zcur0.clone()
    if tokens is None:
        tokens, conf = SB.sentinel((B, S), torch.int32), SB.sentinel((B, S), torch.float32)
    SB.dbg_sample(path, z, tokens, conf, n0, ncc, V, groups, logits=logits, partials=partials, zorig=zorig)
    return tokens, conf, z


def check_remask(z, zcur0, zorig, tokens, conf, groups, n0, ncc, V, what=""):
    want = SR.remask(conf, tokens, zcur0, zorig, ncc, V, groups, n0)
    bad = z != want
    assert not bool(bad.any()), (f"{what}: re-mask differs at {int(bad.sum())} entries, first "
                                 f"{bad.nonzero()[0].tolist()} (got {int(z[bad][0])}, want {int(want[bad][0])})")


def check_step(path, zcur0, groups, ncc, V, logits=None, partials=None, zorig=None, refs=None, what=""):
    """One call, everything checked; returns (tokens, conf, zcur, stats)."""
    B, T, C = zcur0.shape
    S = T * (C - ncc)
    n0 = n0_of(zcur0, groups, ncc, V)
    tokens, conf, z = run(path, zcur0, groups, n0, ncc, V, logits=logits, partials=partials, zorig=zorig)
    zp = zcur0[:, :, ncc:].reshape(B, S)
    known = zp != V
    assert torch.equal(tokens[known], zp[known]), what + ": known positions: token != zcur"
    assert bool((conf[known] == float("inf")).all()), what + ": known positions: conf != +inf"
    if refs is None:
        refs = group_refs(logits, groups, S, V)
    n_amb = n_cmp = 0
    max_err = max_ratio = 0.0
    b = 0
    for g, ref in zip(groups, refs):
        rows = slice(b, b + g.rows)
        m = ~known[rows]
        tk = tokens[rows].long()
        bad = m & ~ref["ambiguous"] & (tk != ref["token"])
        assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {int(m.sum())} tokens differ, first at row "
                                     f"{b + int(bad.nonzero()[0][0])} position {int(bad.nonzero()[0][1])}")
        n_amb += int((m & ref["ambiguous"]).sum())
        n_cmp += int(m.sum())
        same = m & (tk == ref["token"])
        err = (conf[rows].double() - ref["conf"]).abs()[same]
        tol = CONF_ABS + CONF_REL * (ref["logp"].abs() + ref["noise"].abs()) + ref["logp_spread"]
        tol = (tol + ref.get("tol_extra", 0.0))[same]
        if err.numel():
            assert bool((err <= tol).all()), (f"{what}: {int((err > tol).sum())} confidences outside the bound, "
                                              f"max error {err.max().item():.3e}")
            max_err = max(max_err, err.max().item())
            max_ratio = max(max_ratio, (err / tol).max().item())
        b += g.rows
    assert n_amb <= AMBIG_MAX * n_cmp + AMBIG_SLACK, f"{what}: {n_amb} of {n_cmp} draws ambiguous"
    check_remask(z, zcur0, zorig, tokens, conf, groups, n0, ncc, V, what)
    print(f"{what}: {n_amb} of {n_cmp} draws ambiguous; conf max |err| {max_err:.3e} ({max_ratio:.3f} of the bound)")
    return tokens, conf, z, dict(amb=n_amb, cmp=n_cmp, err=max_err)


# ------------------------------------------------------------------------------------ materialised draw (paths 0, 1)
DRAW = [(0.05, 0.0, 1), (1.0, 10.5, 1), (3.0, 4.0, 1), (-1.0, 10.5, 1), (0.7, 10.5, 0)]


@pytest.mark.parametrize("temperature,temp_eff,do_sample", DRAW,
                         ids=["T0.05_te0", "T1_te10.5", "T3_te4", "Tneg_te10.5", "greedy"])
@pytest.mark.parametrize("V", [128, 256, 512, 768, 1024])
@pytest.mark.parametrize("C,ncc", [(4, 0), (14, 4)], ids=["coarse", "c2f"])
@pytest.mark.parametrize("path", [0, 1], ids=["rows", "topp"])
def test_materialised_draw(path, C, ncc, V, temperature, temp_eff, do_sample):
    """B*S = 444 (coarse) or 1110 (c2f) positions: the last CTA of 8 warps is ragged.  Path 1 filters at top_p 0.9."""
    B, T = 3, 37
    S = T * (C - ncc)
    g = gen("draw", path, C, V, temperature, temp_eff, do_sample)
    zcur = SB.state(B, T, C, ncc, V, g)
    logits = SB.logits_for(B * S, V, g)
    grp = Group(rows=B, temperature=temperature, gamma=0.55, temp_eff=temp_eff, do_sample=do_sample, step=6,
                seed=SEED, top_p=0.9 if path == 1 else 0.0)
    check_step(path, zcur, [grp], ncc, V, logits=logits, what=f"path {path} V={V} C={C} T={temperature}")


# ------------------------------------------------------------------------------------ nucleus (path 1)
def nucleus_logits(kind, R, V, g):
    x = torch.randn(R, V, generator=g) * 2.5
    if kind == "top_alone":            # p(top) ~ 1 > top_p
        x[torch.arange(R), torch.randint(0, V, (R,), generator=g)] = 14.0
    elif kind in ("tie", "signed_zero"):
        # p(top) = e / (e + 2) = 0.576 <= top_p = 0.6 < p(top) + p(tie): the tied pair straddles the cut and must be
        # kept whole; indices in different lanes and 128-entry chunks, in both orders
        x.fill_(-30.0)
        for r in range(R):
            i, j, k = torch.randperm(V, generator=g)[:3].tolist()
            x[r, i] = 1.0
            lo, hi = (0.0, -0.0) if r % 2 else (-0.0, 0.0)
            x[r, j], x[r, k] = (lo, hi) if kind == "signed_zero" else (0.0, 0.0)
    elif kind == "tails":              # 40-token support, the rest at -30
        x.fill_(-30.0)
        for r in range(R):
            sup = torch.randperm(V, generator=g)[:40]
            x[r, sup] = torch.randn(40, generator=g) * 1.5
    return x


NUCLEUS = [("normal", 0.85), ("top_alone", 0.3), ("tie", 0.6), ("signed_zero", 0.6), ("tails", 0.999),
           ("normal", 0.999), ("normal", 0.3)]


@pytest.mark.parametrize("kind,top_p", NUCLEUS, ids=[f"{k}_{p}" for k, p in NUCLEUS])
@pytest.mark.parametrize("do_sample", [1, 0], ids=["sample", "greedy"])
def test_nucleus(kind, top_p, do_sample):
    """Path 1 at temperature 1.7 (a filter of the scaled logits would keep a different set) and temp_eff 0, so that
    exp(conf) is p(token) renormalised over the nucleus: the conf check pins the kept set, not just the token.  Every
    sampled token lies in the float64 nucleus (uncertain boundary tokens allowed)."""
    B, T, C, ncc, V = 4, 40, 4, 0, 1024
    S = T * (C - ncc)
    g = gen("nucleus", kind, top_p, do_sample)
    zcur = SB.state(B, T, C, ncc, V, g, p_masked=0.9)
    logits = nucleus_logits(kind, B * S, V, g).cuda()
    grp = Group(rows=B, temperature=1.7, gamma=0.4, temp_eff=0.0, do_sample=do_sample, step=3, seed=SEED, top_p=top_p)
    ref = group_refs(logits, [grp], S, V)[0]
    tokens, conf, _, _ = check_step(1, zcur, [grp], ncc, V, logits=logits, refs=[ref], what=f"nucleus {kind}")
    masked = (zcur[:, :, ncc:].reshape(B, S) == V)
    inside = (ref["keep"] | ref["uncertain"]).gather(2, tokens.long().clamp(0, V - 1)[..., None])[..., 0]
    assert bool(inside[masked].all()), f"{int((~inside & masked).sum())} tokens outside the nucleus"
    if kind == "top_alone":
        assert bool((conf[masked] == 0.0).all()), "a one-token nucleus must give log p = 0"
    if kind in ("tie", "signed_zero"):
        assert bool((ref["keep"].sum(-1)[masked] == 3).all())


def test_disabled_top_p_group_equals_path_0():
    """In a path-1 launch, the rows of a group whose top_p is disabled (0 and 1) equal path 0 bit for bit."""
    B, T, C, ncc, V = 6, 33, 14, 4, 1024
    S = T * (C - ncc)
    g = gen("disabled")
    zcur = SB.state(B, T, C, ncc, V, g)
    logits = SB.logits_for(B * S, V, g)
    mk = lambda tp: [Group(rows=2, temperature=0.8, gamma=0.5, temp_eff=3.0, seed=(5, 6), step=2, top_p=tp[0]),  # noqa: E731
                     Group(rows=2, temperature=1.2, gamma=0.5, temp_eff=3.0, seed=(7, 8), step=2, top_p=tp[1]),
                     Group(rows=2, temperature=0.9, gamma=0.7, temp_eff=0.0, seed=(9, 1), step=2, top_p=tp[2])]
    groups = mk((0.8, 0.0, 1.0))
    t1, c1, z1, _ = check_step(1, zcur, groups, ncc, V, logits=logits, what="path 1, groups 1 and 2 disabled")
    t0, c0, z0, _ = check_step(0, zcur, mk((0.0, 0.0, 0.0)), ncc, V, logits=logits, what="path 0")
    assert torch.equal(t1[2:], t0[2:]) and torch.equal(c1[2:].view(torch.int32), c0[2:].view(torch.int32))
    assert torch.equal(z1[2:], z0[2:])
    assert not torch.equal(t1[:2], t0[:2])   # the filtering group does filter


# ------------------------------------------------------------------------------------ combine (path 2)
def records_ref(rec, g, B, S, masked):
    """sample_combine_kernel's choice and confidence from float4 records rec (B*S, nt, 4), float64 apart from the
    kernel's fp32 constant c1 = fp32(inv_t * fp32(log2 e)); rows that are not `masked` are not evaluated."""
    R, nt, _ = rec.shape
    r = rec.clone()
    r[~masked.reshape(-1)] = 0.0                       # known positions' records may be anything (NaN): never read
    mx, s = r[..., 0], r[..., 1].double()
    bits = r[..., 3].contiguous().view(torch.int32).long()
    v0 = torch.arange(nt, device=rec.device) * GR.TILE
    cand, am = (bits & 0xFFFF) - v0, (bits >> 16) - v0
    inv_t = GR.inv_temperature(g.temperature)
    u1, _, uc = SR.uniforms(g.seed, g.step, B, S, rec.device)
    tok, amb = GR.combine(mx, s, cand, am, inv_t, u1.reshape(-1) if g.do_sample else None)
    c1 = float(np.float32(inv_t) * GR.LOG2E_F32)
    M = mx.max(-1, keepdim=True).values.double()
    total = (s * torch.exp2((mx.double() - M) * c1)).sum(-1)
    xc = r[..., 2].gather(1, (tok // GR.TILE)[:, None])[:, 0].double()
    logp = (xc - M[:, 0]) * c1 * np.log(2.0) - torch.log(total)
    noise = float(np.float32(g.temp_eff)) * SR.gumbel(uc.reshape(-1))
    rs = lambda t: t.reshape(B, S)  # noqa: E731
    return dict(token=rs(tok), ambiguous=rs(amb), logp=rs(logp), noise=rs(noise), conf=rs(logp + noise),
                logp_spread=torch.zeros(B, S, dtype=torch.float64, device=rec.device))


@pytest.mark.parametrize("C,ncc", [(4, 0), (14, 4)], ids=["coarse", "c2f"])
@pytest.mark.parametrize("temperature,do_sample,step", [(0.7, 1, 11), (1.0, 0, 0), (3.0, 1, 2)])
def test_combine_real_records(C, ncc, temperature, do_sample, step):
    """Records from the classifier GEMM's sampling epilogue (vnb_dbg_gemm_sample) on real operands: tokens equal
    gemm_sample_ref.combine of the float64 records of the same logits, confidences are within the bound against
    float64 softmax, and path 0 on the materialised logits gives the same tokens except on ambiguous rows.  Records of
    known positions are never written by the epilogue (they hold a NaN sentinel) and must not be read."""
    check_combine_real_records(C, ncc, temperature, do_sample, step, GB.V)


@pytest.mark.parametrize("C,ncc", [(4, 0), (14, 4), (1, 0)], ids=["coarse", "c2f", "cp1"])
@pytest.mark.parametrize("temperature,do_sample,step", [(0.7, 1, 11), (1.0, 0, 0), (3.0, 1, 2)])
def test_combine_real_records_v512(C, ncc, temperature, do_sample, step):
    """test_combine_real_records at a 512-entry vocabulary: four records per position."""
    check_combine_real_records(C, ncc, temperature, do_sample, step, 512)


def check_combine_real_records(C, ncc, temperature, do_sample, step, V):
    B, T, d = 3, 150, 1280
    Cp = C - ncc
    M, N, S, nt = B * T, Cp * V, T * Cp, V // 128
    A, W, gg = GB.operands(M, N, d, seed=31 + C + (V != GB.V) * V)
    bias = torch.randn(N, generator=gg)
    W = W.cpu()
    GB.tie_columns(W, bias, gg, V=V)
    W, bias = W.cuda(), bias.cuda()
    ss, inv_d, _ = GB.row_stats(M, d, d // 128, gg)
    zcur = GB.sample_inputs(M, C, ncc, gg, V=V)
    logits = GB.sentinel((M, N), torch.float32)
    GB.gemm_fused(GB.lib().EPI_BIAS_F32, A, W, logits, bias=bias, ss_in=ss, inv_d=inv_d)
    logits = logits.view(M * Cp, V)
    rec = GB.sentinel((M * Cp * nt, 4), torch.float32)
    GB.gemm_sample(A, W, bias, ss, inv_d, zcur, T, C, ncc, temperature, do_sample, step, SEED, rec, V=V)
    torch.cuda.synchronize()
    z3 = zcur.view(B, T, C)
    grp = Group(rows=B, temperature=temperature, gamma=0.45, temp_eff=10.5 * (1 - step / 12), do_sample=do_sample,
                step=step, seed=SEED)
    masked = z3[:, :, ncc:].reshape(B, S) == V
    # the token reference: float64 records of the same logits, then the tile pick
    u1 = u2 = None
    if do_sample:
        u1 = torch.from_numpy(philox.uniform_bs(SEED, step, B, S, stream=0, word=0)).reshape(-1).cuda()
        u2 = torch.from_numpy(philox.uniform_bs(SEED, step, B, S, stream=0, word=1)).reshape(-1).cuda()
    mx, am, s, cand, amb_s = GR.strip_records(logits.reshape(-1, 128), GR.inv_temperature(temperature),
                                              None if u2 is None else u2.repeat_interleave(nt))
    rs = lambda t: t.reshape(B * S, nt)  # noqa: E731
    tok, amb_t = GR.combine(rs(mx), rs(s), rs(cand), rs(am), GR.inv_temperature(temperature), u1)
    amb = amb_t | rs(amb_s).gather(1, (tok // 128)[:, None])[:, 0]
    ref = group_refs(logits, [grp], S, V)[0]
    ref["token"], ref["ambiguous"] = tok.view(B, S), amb.view(B, S)
    xs_max = (logits * torch.tensor(GR.inv_temperature(temperature), device="cuda")).abs().amax(-1).double()
    ref["tol_extra"] = COMBINE_REL * xs_max.view(B, S)
    t2, c2, _, st = check_step(2, z3, [grp], ncc, V, partials=rec, refs=[ref], what=f"combine C={C} T={temperature}")
    t0, _, _, _ = check_step(0, z3, [grp], ncc, V, logits=logits, what=f"rows C={C} T={temperature}")
    amb0 = group_refs(logits, [grp], S, V)[0]["ambiguous"]
    differ = (t2 != t0) & masked & ~amb.view(B, S) & ~amb0
    assert not bool(differ.any()), f"paths 0 and 2 differ at {int(differ.sum())} unambiguous positions"


@pytest.mark.parametrize("do_sample", [1, 0], ids=["sample", "greedy"])
def test_combine_synthetic_records(do_sample):
    """Hand-made logits turned into records: rows whose maximum is tied across two tiles (greedy takes the first
    tile), rows whose tile maxima are 0, 60, 120, ... below the top (ex2.approx.ftz flushes the far tiles' mass to
    0), and NaN records at every known position."""
    B, T, C, ncc, V = 2, 48, 4, 0, 1024
    S, nt = T * C, V // 128
    g = gen("synthetic", do_sample)
    zcur = SB.state(B, T, C, ncc, V, g)
    x = torch.randn(B * S, V, generator=g)
    x[0::2, 2 * 128 + 17] = x[0::2, 5 * 128 + 3] = 9.0                 # tied tile maxima in tiles 2 and 5
    x[1::2] -= (torch.arange(nt).repeat_interleave(128) * 60.0)[None]  # tile k sits 60 k below tile 0
    x = x.cuda()
    grp = Group(rows=B, temperature=1.0, gamma=0.6, temp_eff=2.0, do_sample=do_sample, step=4, seed=SEED)
    rec = SB.records_from_logits(x, 1.0, do_sample, SEED, 4, B, S).view(B * S, nt, 4)
    masked = zcur[:, :, ncc:].reshape(B, S) == V
    rec[~masked.reshape(-1)] = float("nan")
    ref = records_ref(rec, grp, B, S, masked)
    tokens, conf, _, _ = check_step(2, zcur, [grp], ncc, V, partials=rec.reshape(-1, 4), refs=[ref],
                                    what=f"synthetic records sample={do_sample}")
    assert bool(torch.isfinite(conf).logical_or(conf == float("inf")).all())
    if not do_sample:
        tied = masked.reshape(-1).clone()
        tied[1::2] = False
        assert bool((tokens.reshape(-1)[tied] == 2 * 128 + 17).all()), "greedy must take the first of tied tiles"


# ------------------------------------------------------------------------------------ re-mask (path 3)
# (name, B, T, C, ncc, conf kind, gamma, is_last, n0 ("cnt": the group's count, "big": S + 50, or a number))
REMASK = [
    ("S1", 2, 1, 1, 0, "randn", 0.5, 0, "cnt"),
    ("S7", 2, 7, 1, 0, "randn", 0.5, 0, "cnt"),
    ("S1024", 2, 256, 4, 0, "randn", 0.37, 0, "cnt"),
    ("S1025", 2, 1025, 1, 0, "randn", 0.61, 0, "cnt"),
    ("S30720", 2, 3072, 14, 4, "randn", 0.5, 0, "cnt"),
    ("all_equal", 2, 100, 4, 0, "equal", 0.5, 0, "cnt"),
    ("ties_at_cut", 3, 300, 4, 0, "ties", 0.5, 0, "cnt"),
    ("inf_mixed", 3, 300, 4, 0, "inf", 0.5, 0, "cnt"),
    ("gamma_n0_below_1", 2, 100, 4, 0, "randn", 0.005, 0, 100),      # floor(0.5) = 0, clamped up to 1
    ("n0_above_S_last", 2, 100, 4, 0, "randn", 1.0, 1, "big"),
    ("gamma0_last", 2, 100, 4, 0, "ties", 0.0, 1, "cnt"),
]


@pytest.mark.parametrize("zorig_kind", ["zorig", "null"])
@pytest.mark.parametrize("case", REMASK, ids=[c[0] for c in REMASK])
def test_remask(case, zorig_kind):
    """remask_kernel alone on given tokens and conf; zcur's conditioning entries are scrambled before the call (they
    must come back from zorig, or stay as they are when zorig is NULL)."""
    name, B, T, C, ncc, kind, gamma, is_last, n0k = case
    S = T * (C - ncc)
    V = 1024
    g = gen("remask", name, zorig_kind)
    zcur = SB.state(B, T, C, ncc, V, g)
    zorig = torch.randint(0, V, (B, T, C), generator=g, dtype=torch.int32).cuda()
    tokens = torch.randint(0, V, (B, S), generator=g, dtype=torch.int32).cuda()
    c = torch.randn(B, S, generator=g) * 3.0
    if kind == "equal":
        c.fill_(-1.25)
    elif kind == "ties":
        c = torch.round(c * 2.0) / 2.0
    elif kind == "inf":
        c = torch.round(c * 4.0) / 4.0
        c[torch.rand(B, S, generator=g) < 0.2] = float("inf")
        c[torch.rand(B, S, generator=g) < 0.2] = -float("inf")
    conf = c.cuda()
    groups = [Group(rows=B, gamma=gamma, is_last=is_last)]
    n0 = [S + 50] if n0k == "big" else [n0k] if isinstance(n0k, int) else n0_of(zcur, groups, ncc, V)
    tok_in, conf_in = tokens.clone(), conf.clone()
    zo = zorig if zorig_kind == "zorig" else None
    _, _, z = run(3, zcur, groups, n0, ncc, V, zorig=zo, tokens=tokens, conf=conf)
    torch.cuda.synchronize()
    assert torch.equal(tokens, tok_in) and torch.equal(conf, conf_in), "path 3 must not write tokens or conf"
    check_remask(z, zcur, zo, tokens, conf, groups, n0, ncc, V, name)
    if ncc and zo is None:
        assert torch.equal(z[:, :, :ncc], zcur[:, :, :ncc])


def test_remask_restores_conditioning_codebooks():
    """Every path: with ncc = 4, zcur's conditioning entries (set to other tokens than zorig's) come back from zorig."""
    B, T, C, ncc, V = 2, 20, 14, 4, 1024
    S = T * (C - ncc)
    g = gen("restore")
    zorig = torch.randint(0, V, (B, T, C), generator=g, dtype=torch.int32).cuda()
    zcur = SB.state(B, T, C, ncc, V, g)
    zcur[:, :, :ncc] = (zorig[:, :, :ncc] + 1) % V
    logits = SB.logits_for(B * S, V, g)
    grp = Group(rows=B, temperature=0.9, gamma=0.5, temp_eff=4.0, step=1, seed=SEED)
    rec = SB.records_from_logits(logits, 0.9, 1, SEED, 1, B, S)
    for path in (0, 1, 2):
        _, _, z, _ = check_step(path, zcur, [grp], ncc, V, logits=logits, partials=rec if path == 2 else None,
                                zorig=zorig, what=f"path {path} with zorig")
        assert torch.equal(z[:, :, :ncc], zorig[:, :, :ncc])


# ------------------------------------------------------------------------------------ groups
@pytest.mark.parametrize("path", [0, 2], ids=["rows", "combine"])
def test_groups_use_their_own_state(path):
    """One call with three groups of 2, 1 and 3 rows, each with its own seed, temperature, do_sample, N0, gamma and
    temp_eff: every row matches the reference run on its group alone (Philox row b - first), and equals, bit for bit,
    a call with that group alone."""
    B, T, C, ncc, V = 6, 25, 4, 0, 1024
    S = T * (C - ncc)
    g = gen("groups", path)
    zcur = SB.state(B, T, C, ncc, V, g)
    logits = SB.logits_for(B * S, V, g)
    groups = [Group(rows=2, temperature=0.8, gamma=0.5, temp_eff=6.0, do_sample=1, step=4, seed=(11, 1)),
              Group(rows=1, temperature=2.0, gamma=0.9, temp_eff=1.0, do_sample=0, step=4, seed=(12, 2)),
              Group(rows=3, temperature=-1.0, gamma=0.2, temp_eff=10.5, do_sample=1, step=4, seed=(13, 3))]
    recs, b = [], 0
    for gr in groups:
        recs.append(SB.records_from_logits(logits[b * S:(b + gr.rows) * S], gr.temperature, gr.do_sample, gr.seed,
                                           gr.step, gr.rows, S))
        b += gr.rows
    rec = torch.cat(recs) if path == 2 else None
    t, c, z, _ = check_step(path, zcur, groups, ncc, V, logits=logits, partials=rec, what=f"three groups path {path}")
    b = 0
    for gi, gr in enumerate(groups):
        rows = slice(b, b + gr.rows)
        t1, c1, z1 = run(path, zcur[rows], [gr], n0_of(zcur[rows], [gr], ncc, V), ncc, V,
                         logits=logits[b * S:(b + gr.rows) * S], partials=recs[gi] if path == 2 else None)
        assert torch.equal(t[rows], t1) and torch.equal(c[rows].view(torch.int32), c1.view(torch.int32)), gi
        assert torch.equal(z[rows], z1), gi
        b += gr.rows


def test_refusals():
    """Bad arguments are refused with a message, before any launch."""
    L = SB.lib()
    z = torch.zeros(2, 4, 4, dtype=torch.int32, device="cuda")
    tok = torch.zeros(2, 16, dtype=torch.int32, device="cuda")
    conf = torch.zeros(2, 16, device="cuda")
    logits = torch.zeros(32, 256, device="cuda")

    def call(path=0, groups=(Group(rows=2),), V=256, ncc=0, C=4, lg=logits, zc=z):
        arr = (L.SampleGroup * len(groups))()
        for a, g in zip(arr, groups):
            a.rows = g.rows
        n0 = torch.zeros(len(groups), dtype=torch.int32, device="cuda")
        rc = L.lib().vnb_dbg_sample(path, L.ptr(lg), None, L.ptr(zc), None, L.ptr(tok), L.ptr(conf), L.ptr(n0), 2, 4,
                                    C, ncc, V, V, arr, len(groups), L.stream_ptr())
        return rc, L.lib().vnb_last_error().decode()

    assert call()[0] == 0
    for kw, msg in [(dict(path=4), "path"), (dict(groups=(Group(rows=1),)), "sum"),
                    (dict(groups=(Group(rows=3), Group(rows=-1))), "rows"), (dict(ncc=4), "ncc"), (dict(V=200), "V"),
                    (dict(V=2048), "V"), (dict(lg=None), "logits"), (dict(path=2), "partials"), (dict(zc=None), "zcur")]:
        rc, err = call(**kw)
        assert rc != 0 and msg in err, (kw, err)
