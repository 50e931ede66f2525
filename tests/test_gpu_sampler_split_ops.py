"""GPU: the pieces of a fused launch that mixes nucleus (top-p) and plain groups, at op level.

vnb_dbg_gemm_sample_split (the classifier GEMM with the split sampling epilogue) must give, bit for bit,
  - at the still-masked positions of nucleus groups' rows: the logits of vnb_dbg_gemm_fused(VNB_EPI_BIAS_F32);
  - at the still-masked positions of plain groups' rows: the records of vnb_dbg_gemm_sample run on that group alone;
and write nothing else (every output starts as a NaN sentinel).  vnb_dbg_sample_split (split combine, split nucleus
draw, re-mask) must give path 1's tokens, confidences and re-masked row on nucleus rows and path 2's on plain rows.
Groups of one row at T = 40 put rows of both kinds in every 128-row tile."""
import dataclasses

import pytest
import torch

from tests.sample_ref import Group, top_p_on
from tools import gemm_bits as GB
from tools import sample_bits as SB

pytestmark = pytest.mark.gpu

T = 40
GROUPS = [Group(rows=1, temperature=0.7, do_sample=1, step=3, seed=(11, 2), top_p=0.9),
          Group(rows=1, temperature=1.0, do_sample=1, step=3, seed=(12, 2), top_p=0.0),
          Group(rows=2, temperature=1.3, do_sample=0, step=5, seed=(13, 2), top_p=0.8),
          Group(rows=1, temperature=0.9, do_sample=1, step=0, seed=(14, 2), top_p=1.0),
          Group(rows=1, temperature=1.0, do_sample=1, step=7, seed=(15, 2), top_p=0.5),
          Group(rows=2, temperature=0.6, do_sample=0, step=1, seed=(16, 2), top_p=0.0),
          Group(rows=1, temperature=1.0, do_sample=1, step=2, seed=(17, 2), top_p=0.95)]
B = sum(g.rows for g in GROUPS)


def sample_groups(groups):
    L = GB.lib()
    arr = (L.SampleGroup * len(groups))()
    for a, g in zip(arr, groups):
        a.rows, a.temperature, a.gamma, a.temp_eff = g.rows, g.temperature, g.gamma, g.temp_eff
        a.do_sample, a.is_last, a.step = g.do_sample, g.is_last, g.step
        a.seed_lo, a.seed_hi, a.top_p = g.seed[0], g.seed[1], g.top_p
    return arr


def row_ranges(groups):
    b = 0
    for g in groups:
        yield g, b, b + g.rows
        b += g.rows


@pytest.mark.parametrize("C,ncc", [(4, 0), (14, 4)], ids=["coarse", "c2f"])
def test_split_epilogue_equals_bias_f32_and_sample_records(C, ncc):
    check_split_epilogue(C, ncc, GB.V)


@pytest.mark.parametrize("V,C,ncc", [(256, 1, 0), (256, 3, 1), (768, 9, 2)], ids=["v256_cp1", "v256_cp2", "v768_cp7"])
def test_split_epilogue_vocab_sizes(V, C, ncc):
    """The split epilogue at 2 and 6 strips per codebook, with one, two and seven predicted codebooks."""
    check_split_epilogue(C, ncc, V)


def check_split_epilogue(C, ncc, V):
    L = GB.lib()
    d = 512
    Cp = C - ncc
    M, N, nt = B * T, Cp * V, V // 128
    A, W, gg = GB.operands(M, N, d, seed=50 + C + (V != GB.V) * V)
    bias = torch.randn(N, generator=gg)
    W = W.cpu()
    GB.tie_columns(W, bias, gg, V=V)
    W, bias = W.cuda(), bias.cuda()
    ss, inv_d, _ = GB.row_stats(M, d, d // 128, gg)
    zcur = GB.sample_inputs(M, C, ncc, gg, V=V)
    # the materialised logits and, per plain group, the records of the group launched alone
    want_logits = GB.sentinel((M, N), torch.float32)
    GB.gemm_fused(L.EPI_BIAS_F32, A, W, want_logits, bias=bias, ss_in=ss, inv_d=inv_d)
    want_rec = GB.sentinel((M * Cp * nt, 4), torch.float32)
    for g, b0, b1 in row_ranges(GROUPS):
        if not top_p_on(g.top_p):
            rows = slice(b0 * T, b1 * T)
            GB.gemm_sample(A[rows], W, bias, ss[:, rows].contiguous(), inv_d, zcur[rows].contiguous(), T, C, ncc,
                           g.temperature, g.do_sample, g.step, g.seed, want_rec[b0 * T * Cp * nt:b1 * T * Cp * nt],
                           V=V)
    logits = GB.sentinel((M, N), torch.float32)
    rec = GB.sentinel((M * Cp * nt, 4), torch.float32)
    L.check(L.lib().vnb_dbg_gemm_sample_split(L.ptr(A), L.ptr(W), L.ptr(bias), M, N, d, L.ptr(ss), ss.shape[0], inv_d,
                                              GB.EPS, L.ptr(zcur), T, C, ncc, V, V, sample_groups(GROUPS), len(GROUPS),
                                              L.ptr(rec), L.ptr(logits), L.stream_ptr()))
    torch.cuda.synchronize()
    nucleus_row = torch.zeros(M, dtype=torch.bool, device="cuda")
    for g, b0, b1 in row_ranges(GROUPS):
        nucleus_row[b0 * T:b1 * T] = top_p_on(g.top_p)
    masked = zcur[:, ncc:] == V                                    # (M, Cp)
    stored = (masked & nucleus_row[:, None]).repeat_interleave(V, 1)  # (M, N): logits the epilogue must store
    lb, wb = logits.view(torch.int32), want_logits.view(torch.int32)
    assert bool(stored.any()) and bool((masked & ~nucleus_row[:, None]).any())
    assert torch.equal(lb[stored], wb[stored]), f"{int((lb != wb)[stored].sum())} stored logits differ from BIAS_F32"
    assert bool(GB.untouched(logits)[~stored].all()), f"{int((~GB.untouched(logits))[~stored].sum())} stray logits"
    # records: bit-equal to the plain groups' own launches everywhere (both hold the sentinel where nothing is written,
    # the nucleus rows included)
    rb, wrb = rec.view(torch.int32), want_rec.view(torch.int32)
    drawn = (masked & ~nucleus_row[:, None]).repeat_interleave(nt, 1).reshape(-1)
    assert bool(GB.untouched(rec)[~drawn].all()), "records written outside the plain rows' masked positions"
    assert torch.equal(rb, wrb), f"{int((rb != wrb).any(-1).sum())} records differ from the plain groups' launches"


@pytest.mark.parametrize("C,ncc", [(4, 0), (14, 4)], ids=["coarse", "c2f"])
def test_split_sampler_equals_path_1_and_path_2(C, ncc):
    L = GB.lib()
    V = 1024
    S = T * (C - ncc)
    g = torch.Generator().manual_seed(1000 + C)
    zcur = SB.state(B, T, C, ncc, V, g)
    zorig = zcur.clone()
    zorig[:, :, :ncc] = torch.randint(0, V, (B, T, ncc), generator=g, dtype=torch.int32).cuda()
    groups = [dataclasses.replace(x, gamma=0.3 + 0.1 * i, temp_eff=(0.0, 4.5, 10.5)[i % 3])
              for i, x in enumerate(GROUPS)]
    logits = SB.logits_for(B * S, V, g)
    # each group's records as its own launch's classifier epilogue would leave them (Philox row = b - first)
    parts = []
    for q, b0, b1 in row_ranges(groups):
        parts.append(SB.records_from_logits(logits[b0 * S:b1 * S], q.temperature, q.do_sample, q.seed, q.step,
                                            q.rows, S))
    partials = torch.cat(parts).contiguous()
    n0 = []
    for q, b0, b1 in row_ranges(groups):
        n0.append(int((zcur[b0:b1, :, ncc:] == V).sum()))

    def run(path):
        z = zcur.clone()
        tok, conf = SB.sentinel((B, S), torch.int32), SB.sentinel((B, S), torch.float32)
        if path == "split":
            n0d = torch.tensor(n0, dtype=torch.int32, device="cuda")
            L.check(L.lib().vnb_dbg_sample_split(L.ptr(logits), L.ptr(partials), L.ptr(z), L.ptr(zorig), L.ptr(tok),
                                                 L.ptr(conf), L.ptr(n0d), B, T, C, ncc, V, V, sample_groups(groups),
                                                 len(groups), L.stream_ptr()))
        else:
            SB.dbg_sample(path, z, tok, conf, n0, ncc, V, groups, logits=logits, partials=partials, zorig=zorig)
        torch.cuda.synchronize()
        return tok, conf.view(torch.int32), z

    ts, cs, zs = run("split")
    t1, c1, z1 = run(1)
    t2, c2, z2 = run(2)
    for q, b0, b1 in row_ranges(groups):
        t, c, z = (t1, c1, z1) if top_p_on(q.top_p) else (t2, c2, z2)
        what = f"rows {b0}..{b1 - 1} (top_p {q.top_p})"
        assert torch.equal(ts[b0:b1], t[b0:b1]), what + ": tokens differ"
        assert torch.equal(cs[b0:b1], c[b0:b1]), what + ": confidences differ"
        assert torch.equal(zs[b0:b1], z[b0:b1]), what + ": re-masked rows differ"
    # the two draws do differ on the plain rows, so the equality above pins which kernel served them
    plain = torch.tensor([not top_p_on(q.top_p) for q, b0, b1 in row_ranges(groups) for _ in range(q.rows)],
                         device="cuda")
    assert not torch.equal(c1[plain], c2[plain])


def test_split_op_refusals():
    L = GB.lib()
    z = torch.full((2, 4, 4), 1024, dtype=torch.int32, device="cuda")
    tok = torch.empty(2, 16, dtype=torch.int32, device="cuda")
    conf = torch.empty(2, 16, device="cuda")
    n0 = torch.zeros(1, dtype=torch.int32, device="cuda")
    lg = torch.zeros(32, 1024, device="cuda")
    rec = torch.zeros(32 * 8, 4, device="cuda")
    grp = sample_groups([Group(rows=2, top_p=0.9)])

    def call(logits=lg, partials=rec, groups=grp, n=1):
        rc = L.lib().vnb_dbg_sample_split(L.ptr(logits), L.ptr(partials), L.ptr(z), None, L.ptr(tok), L.ptr(conf),
                                          L.ptr(n0), 2, 4, 4, 0, 1024, 1024, groups, n, L.stream_ptr())
        L.check(rc)
    call()
    with pytest.raises(RuntimeError, match="needs logits"):
        call(logits=None)
    with pytest.raises(RuntimeError, match="needs partials"):
        call(partials=None)
    with pytest.raises(RuntimeError, match="sum to"):
        call(groups=sample_groups([Group(rows=1)]))
    # path 4 is not a vnb_dbg_sample path
    with pytest.raises(RuntimeError, match="outside 0..3"):
        L.check(L.lib().vnb_dbg_sample(4, L.ptr(lg), L.ptr(rec), L.ptr(z), None, L.ptr(tok), L.ptr(conf), L.ptr(n0),
                                       2, 4, 4, 0, 1024, 1024, grp, 1, L.stream_ptr()))
