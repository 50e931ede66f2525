"""CPU: the float64 reference of the sampling step (tests/sample_ref.py) reproduces the oracle's sampler
(OracleVampNet.sample_from_logits and mask_by_random_topk with rng="philox", oracle/vampnet_oracle.py) token for token
and mask for mask, with and without the nucleus filter.  tests/test_gpu_sampler_ops.py holds the kernels to this
reference, so the sampler is pinned to the oracle through it.  Positions whose draw or nucleus boundary lies within
AMBIGUOUS_REL of a crossing are excluded (the oracle works in fp32 and may round either way there), and so are rows
where a group of tied logits straddles the nucleus boundary, because the oracle's sort splits such a group
arbitrarily while the kernels keep it whole."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import vampnet_oracle as vo
from tests import sample_ref as SR
from tests.gemm_sample_ref import inv_temperature

MT = 1024


def _oracle():
    cfg = vo.OracleConfig(n_heads=4, n_layers=1, n_codebooks=4, n_conditioning_codebooks=0, embedding_dim=256)
    return vo.OracleVampNet(cfg, vo.make_state_dict(cfg, seed=0), "fp32")


def oracle_nucleus(x, top_p):
    """The oracle's sort-based filter (transformer.py:1001-1016 as restated in OracleVampNet.sample_from_logits):
    True where the logit survives."""
    v, si = x.sort(descending=True)
    rm = v.softmax(dim=-1).cumsum(dim=-1) > top_p
    rm = F.pad(rm, (1, 0), value=False)[..., :-1]
    return ~rm.scatter(-1, si, rm)


def logits_of(kind, B, S, V, g):
    x = torch.randn(B, S, V, generator=g) * 3.0
    if kind == "peaked":          # one tile holds almost all of the mass
        x[..., 256:384] += 12.0
    elif kind == "ties":          # exact ties of the maximum inside and across tiles, and many tied values
        x = torch.round(x)
        x[..., 5] = x[..., 77] = x[..., 600] = x.amax(-1) + 1.0
    elif kind == "heavy":         # heavy tails: a few logits far above the bulk
        x = torch.randn(B, S, V, generator=g) / torch.rand(B, S, V, generator=g).clamp_min(1e-3) ** 0.5
    return x.float()


@pytest.mark.parametrize("kind", ["normal", "peaked", "ties", "heavy"])
@pytest.mark.parametrize("temperature", [0.7, 1.0, 3.0])
@pytest.mark.parametrize("top_p", [None, 0.3, 0.85, 0.99])
@pytest.mark.parametrize("sample", [1, 0], ids=["sample", "greedy"])
def test_reference_equals_oracle_sampler(kind, temperature, top_p, sample):
    B, S, V, key, step = 6, 300, 1024, (321, 654), 5
    gamma, n0, temp_eff = 0.4, 250, 3.5
    logits = logits_of(kind, B, S, V, torch.Generator().manual_seed(11))
    orc = _oracle()
    want, p32 = orc.sample_from_logits(logits.clone(), bool(sample), temperature, top_p, rng="philox",
                                       philox_key=key, step=step)
    g = SR.Group(rows=B, temperature=temperature, gamma=gamma, temp_eff=temp_eff, do_sample=sample, step=step,
                 seed=key, top_p=0.0 if top_p is None else top_p)
    ref = SR.sample_group(logits, g)
    amb = ref["ambiguous"]
    n_amb = int(amb.sum())
    print(f"{kind} T={temperature} top_p={top_p} sample={sample}: {n_amb} of {amb.numel()} positions ambiguous")
    if not sample and top_p is None:
        assert n_amb == 0
    assert n_amb <= amb.numel() // 100
    x = logits.reshape(-1, V)
    if top_p is not None:
        # the nucleus, token by token away from its uncertain boundary, on rows where no tie group straddles the cut
        # (the oracle's sort splits such a group arbitrarily; the kernels keep it whole)
        keep, unc = ref["keep"].reshape(-1, V), ref["uncertain"].reshape(-1, V)
        cut = x.masked_fill(~keep, float("inf")).min(-1, keepdim=True).values
        tie_at_cut = ((x == cut).sum(-1) > 1).reshape(B, S)
        if kind != "ties":
            assert not tie_at_cut.any()
        rows = ~tie_at_cut.reshape(-1)
        same = (keep == oracle_nucleus(x, top_p)) | unc
        assert bool(same[rows].all()), f"{int((~same[rows]).sum())} nucleus entries differ"
        amb = amb | tie_at_cut
    bad = (ref["token"] != want) & ~amb
    assert not bad.any(), f"{int(bad.sum())} tokens differ, first at {bad.nonzero()[0].tolist()}"

    # the confidence and the re-mask: every position still masked, so cnt = S
    ok = ~amb
    # the oracle's fp32 filter may keep or drop an uncertain boundary token: that moves log p by up to logp_spread
    tol = 1e-4 + ref["logp_spread"][ok]
    assert bool(((ref["logp"][ok] - torch.log(p32.double())[ok]).abs() <= tol).all())
    n = SR.num_to_mask(gamma, n0, S, S, False)
    mask_want, conf_want = orc.mask_by_random_topk(torch.full((B, 1), n, dtype=torch.long), p32,
                                                   torch.full((B,), temp_eff), rng="philox", philox_key=key, step=step)
    assert bool(((ref["conf"][ok] - conf_want.double()[ok]).abs() <= tol + 1e-4).all())
    # the re-mask rule on the oracle's own probabilities (so that an ambiguous draw does not change the input)
    zcur = torch.full((B, S, 1), MT, dtype=torch.int32)
    z = SR.remask(torch.log(p32.double()) + ref["noise"], want.int(), zcur, None, 0, MT, [g], [n0])
    assert torch.equal(z[..., 0] == MT, mask_want)
    assert torch.equal(z[..., 0][~mask_want], want.int()[~mask_want])


def test_nucleus_edges():
    """Hand-made rows: a top token whose probability exceeds top_p is kept alone; a uniform row is kept whole (every
    pre-mass is 0); -inf logits are never kept; a +0 / -0 pair is one tie, kept or dropped together."""
    V = 256
    x = torch.full((5, V), -5.0)
    x[0, 17] = 10.0                                   # p(top) ~ 1 > 0.3
    x[1] = 0.0                                        # uniform
    x[2, :100] = -float("inf")
    x[2, 100:] = torch.linspace(-1, 1, V - 100)
    x[3, :3] = torch.tensor([1.0, 0.0, -0.0])         # with top_p = 0.5 the zeros straddle the boundary ...
    x[4, :3] = torch.tensor([-0.0, 0.0, -0.0])
    keep, amb = SR.nucleus(x, 0.3)
    assert not amb.any()
    assert keep[0].nonzero().flatten().tolist() == [17]
    assert keep[1].all()
    assert not keep[2, :100].any() and keep[2, 100:].any()
    p = torch.softmax(x[3].double(), 0)
    assert p[0] <= 0.5 < p[0] + p[1]                  # ... and float comparison keeps both zeros with the top
    keep3, unc3 = SR.nucleus(x[3:4], 0.5)
    assert not unc3.any() and keep3[0].nonzero().flatten().tolist() == [0, 1, 2]
    assert keep[4].nonzero().flatten().tolist() == [0, 1, 2]
    keep_all, _ = SR.nucleus(x, 1.0)
    assert keep_all.all()
    keep_off, _ = SR.nucleus(x, 0.0)
    assert keep_off.all()


def test_draw_and_confidence_on_hand_made_rows():
    """Greedy takes the lowest index of a tied maximum; a one-token nucleus draws that token with log p = 0."""
    V = 256
    x = torch.full((2, V), -3.0)
    x[0, 40] = x[0, 200] = 2.0
    x[1, 7] = 50.0
    keep = torch.ones_like(x, dtype=torch.bool)
    tok, amb = SR.draw(x, keep, np.float32(1.0), None, None)
    assert tok.tolist() == [40, 7] and not amb.any()
    keep1, _ = SR.nucleus(x[1:], 0.5)
    u = torch.tensor([0.999], dtype=torch.float32)
    tok1, _ = SR.draw(x[1:], keep1, inv_temperature(0.3), u, u)
    assert tok1.tolist() == [7]
    assert SR.log_prob(x[1:], keep1, inv_temperature(0.3), tok1).item() == 0.0


@pytest.mark.parametrize("gamma,n0,cnt,S,is_last", [(0.4, 250, 300, 300, 0), (0.001, 250, 300, 300, 0),
                                                    (1.0, 17, 10, 64, 0), (1.0, 90, 90, 64, 1), (0.0, 90, 0, 64, 1),
                                                    (0.9999, 30720, 30720, 30720, 0)])
def test_num_to_mask_matches_the_oracle_schedule(gamma, n0, cnt, S, is_last):
    """num_to_mask is the oracle's floor(gamma * N0) with its clamps (OracleVampNet.generate), plus the [0, S - 1] clamp
    that keeps the cut inside the row."""
    n = torch.floor(torch.tensor(gamma, dtype=torch.float32) * torch.tensor(n0)).long()
    if not is_last:
        n = torch.maximum(torch.tensor(1), torch.minimum(torch.tensor(cnt) - 1, n))
    assert SR.num_to_mask(gamma, n0, cnt, S, bool(is_last)) == min(max(int(n), 0), S - 1)
