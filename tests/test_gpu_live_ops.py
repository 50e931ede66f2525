"""GPU: the live bound of launches of calls with different step counts, one kernel at a time (vnb_dbg_set_live; see
include/vampnet_b200.h).  At an iteration where only batch rows b < R are live:

  * a GEMM tile whose first row is at or past R * T (CTA pair: the cluster's first row) writes nothing, and so does an
    attention CTA of a row b >= R; the LoRA down-projection writes no u row at or past R * T;
  * the sampler (materialised draw, combine, re-mask) leaves tokens, confidences and zcur of rows b >= R untouched;
  * everything the bounded launch does write for live rows is bit-equal to the same launch without a bound.

Outputs start as a NaN sentinel (tools/gemm_bits.py, tools/sample_bits.py), so a stray store shows up.  T = 100 puts
the bound inside 128-row tiles (straddling tiles run whole; their dead rows are unspecified and not compared)."""
import contextlib

import pytest
import torch

from tests.test_gpu_adapter_ops import make_adapters, row_map, run_adapted
from tests.test_gpu_attention_ragged import ragged_inputs, sentinel_out
from tools import gemm_bits as GB
from tools import sample_bits as SB
from tests.sample_ref import Group

pytestmark = pytest.mark.gpu

B, T, D = 5, 100, 256
M = B * T


@pytest.fixture(scope="module")
def L():
    return GB.lib()


@pytest.fixture(params=[0, 1], ids=["single_cta", "cta_pair"])
def pair(request, L):
    prev = GB.set_pair(request.param)
    yield request.param
    GB.set_pair(prev)


@contextlib.contextmanager
def live_bound(L, R):
    """The unit-level entry points run with batch rows [0, R) live while inside."""
    r = torch.tensor([R], dtype=torch.int32, device="cuda")
    L.check(L.lib().vnb_dbg_set_live(L.ptr(r)))
    try:
        yield
    finally:
        torch.cuda.synchronize()
        L.check(L.lib().vnb_dbg_set_live(None))


def dead_from(R, pair_on):
    """First GEMM row of the tiles that must do nothing: tiles (pair: clusters of two) start at multiples of 128 (256)."""
    tm = 256 if pair_on else 128
    return min(M, -(-(R * T) // tm) * tm)


def assert_bound(got, want, live_rows, dead_rows, what):
    """Rows [0, live_rows) equal `want` bit for bit; rows [dead_rows, ...) still hold the sentinel."""
    assert torch.equal(got[:live_rows].view(torch.int16 if got.dtype == torch.bfloat16 else torch.int32),
                       want[:live_rows].view(torch.int16 if want.dtype == torch.bfloat16 else torch.int32)), \
        f"{what}: live rows differ from the unbounded launch"
    assert bool(GB.untouched(got[dead_rows:]).all()), f"{what}: a tile past the live rows wrote"


@pytest.mark.parametrize("R", [1, 3])
@pytest.mark.parametrize("epi", ["BF16", "QKV", "RESID", "GEGLU", "BIAS_F32"])
def test_gemm_tiles_past_the_bound_write_nothing(L, pair, epi, R):
    """Every epilogue, single-CTA and CTA-pair; GEGLU without a pair is the persistent FFN-up kernel."""
    e = getattr(L, "EPI_" + epi)
    N = {"QKV": 3 * D, "GEGLU": 4 * D}.get(epi, D)
    A, W, g = GB.operands(M, N, D, seed=40 + R)
    ss_in, inv_d, _ = GB.row_stats(M, D, D // 128, g) if epi in ("QKV", "GEGLU") else (None, 0.0, None)
    bias = (torch.randn(N, generator=g) * 0.1).cuda() if epi == "BIAS_F32" else None
    Tpad = (T + 7) // 8 * 8
    x0 = torch.randn(M, N, generator=g).cuda() if epi == "RESID" else None

    def run(bounded):
        width = {"QKV": 2 * D, "GEGLU": N // 2}.get(epi, N)
        dtype = torch.float32 if epi in ("RESID", "BIAS_F32") else torch.bfloat16
        out = x0.clone() if epi == "RESID" else GB.sentinel((M, width), dtype)
        vT = GB.sentinel((B, D, Tpad), torch.bfloat16) if epi == "QKV" else None
        obf = GB.sentinel((M, N), torch.bfloat16) if epi == "RESID" else None
        ss = GB.sentinel((N // 128, M), torch.float32) if epi == "RESID" else None
        ctx = live_bound(L, R) if bounded else contextlib.nullcontext()
        with ctx:
            GB.gemm_fused(e, A, W, out, out2=vT, bias=bias, T=T, Tpad=Tpad, ss_in=ss_in, inv_d=inv_d, out_bf16=obf,
                          ss_out=ss)
        torch.cuda.synchronize()
        return out, vT, obf, ss

    want, got = run(False), run(True)
    live, dead = R * T, dead_from(R, pair)
    if epi == "RESID":  # in place: dead tiles leave the residual rows as they were
        assert torch.equal(got[0][:live], want[0][:live]), "RESID: live rows differ"
        assert torch.equal(got[0][dead:], x0[dead:]), "RESID: a tile past the live rows wrote"
        assert_bound(got[2], want[2], live, dead, "RESID bf16 copy")
        assert_bound(got[3].t(), want[3].t(), live, dead, "RESID sums of squares")
    else:
        assert_bound(got[0], want[0], live, dead, epi)
    if epi == "QKV":  # v^T of a batch row wholly inside dead tiles is never written
        assert torch.equal(got[1][:R].view(torch.int16), want[1][:R].view(torch.int16)), "QKV: live v^T differs"
        first_dead_b = -(-dead // T)
        assert bool(GB.untouched(got[1][first_dead_b:]).all()), "QKV: v^T of a dead row written"


@pytest.mark.parametrize("R", [1, 4])
@pytest.mark.parametrize("epi", ["QKV", "GEGLU", "RESID"])
def test_adapted_gemm_and_lora_down_respect_the_bound(L, pair, epi, R):
    g = torch.Generator().manual_seed(7 + R)
    ads = make_adapters(D, g)
    rmap = row_map(B, T, "rows", g)
    e = getattr(L, "EPI_" + epi)
    N = {"QKV": 3 * D, "GEGLU": 4 * D}.get(epi, D)
    A, W, _ = GB.operands(M, N, D, seed=90 + R)
    Tpad = (T + 7) // 8 * 8
    Ru = 16 if epi == "QKV" else 8
    x0 = torch.randn(M, N, generator=g).cuda() if epi == "RESID" else None

    def run(bounded):
        width = {"QKV": 2 * D, "GEGLU": N // 2}.get(epi, N)
        out = x0.clone() if epi == "RESID" else GB.sentinel((M, width), torch.bfloat16)
        vT = GB.sentinel((B, D, Tpad), torch.bfloat16) if epi == "QKV" else None
        u = GB.sentinel((M, Ru), torch.float32)
        ctx = live_bound(L, R) if bounded else contextlib.nullcontext()
        with ctx:
            run_adapted(L, e, A, W, out, out2=vT, T=T, Tpad=Tpad, ads=ads, rmap=rmap, u=u)
        torch.cuda.synchronize()
        return out, u

    (want, u_want), (got, u_got) = run(False), run(True)
    live, dead = R * T, dead_from(R, pair)
    if epi == "RESID":
        assert torch.equal(got[:live], want[:live]) and torch.equal(got[dead:], x0[dead:]), "adapted RESID"
    else:
        assert_bound(got, want, live, dead, "adapted " + epi)
    # the down-projection's bound is exact: no u row at or past R * T
    assert torch.equal(u_got[:live].view(torch.int32), u_want[:live].view(torch.int32)), "u of live rows differs"
    assert bool(GB.untouched(u_got[live:]).all()), "lora_down wrote a row past the bound"


@pytest.mark.parametrize("R", [1, 3])
def test_classifier_records_respect_the_bound(L, pair, R):
    """The sampling epilogue of the generate loop's classifier: no record for rows of dead tiles."""
    C, ncc = 4, 0
    N = (C - ncc) * GB.V
    A, W, g = GB.operands(M, N, D, seed=60 + R)
    bias = (torch.randn(N, generator=g) * 0.1).cuda()
    ss_in, inv_d, _ = GB.row_stats(M, D, D // 128, g)
    zcur = GB.sample_inputs(M, C, ncc, g)
    nt = GB.V // 128

    def run(bounded):
        partials = GB.sentinel((M, C - ncc, nt, 4), torch.float32)
        ctx = live_bound(L, R) if bounded else contextlib.nullcontext()
        with ctx:
            GB.gemm_sample(A, W, bias, ss_in, inv_d, zcur, T, C, ncc, 1.0, 1, 3, (5, 6), partials)
        torch.cuda.synchronize()
        return partials

    want, got = run(False), run(True)
    assert_bound(got, want, R * T, dead_from(R, pair), "classifier records")


@pytest.mark.parametrize("R", [1, 2, 4])
def test_attention_ctas_of_idle_rows_write_nothing(L, R):
    H = 4
    qk, vT, rel, sat, Tpad = ragged_inputs((T,) * B, T, H, seed=12)

    def run(bounded):
        out = sentinel_out(B, T, H * 64)
        ctx = live_bound(L, R) if bounded else contextlib.nullcontext()
        with ctx:
            L.check(L.lib().vnb_op_attention(L.ptr(qk), L.ptr(vT), L.ptr(out), L.ptr(rel), sat, B, T, Tpad, H,
                                             L.stream_ptr()))
        torch.cuda.synchronize()
        return out

    want, got = run(False), run(True)
    assert torch.equal(got[:R].view(torch.int16), want[:R].view(torch.int16)), "live rows differ"
    assert bool(GB.untouched(got[R:]).all()), "an idle row's attention CTA wrote"


@pytest.mark.parametrize("path", [0, 1, 2, 3], ids=["rows", "topp", "combine", "remask"])
def test_sampler_leaves_idle_rows_untouched(L, path):
    """Two groups of two rows each, then a third group of one; rows 3 and 4 are idle (R = 3)."""
    Bs, Ts, C, ncc, V, R = 5, 37, 4, 0, 1024, 3
    g = torch.Generator().manual_seed(100 + path)
    S = Ts * (C - ncc)
    zcur0 = SB.state(Bs, Ts, C, ncc, V, g)
    top_p = 0.85 if path == 1 else 0.0
    groups = [Group(rows=2, temperature=0.8, gamma=0.5, temp_eff=4.0, do_sample=1, is_last=0, step=3, seed=(1, 2),
                    top_p=top_p),
              Group(rows=2, temperature=1.2, gamma=0.3, temp_eff=0.0, do_sample=0, is_last=0, step=0, seed=(3, 4),
                    top_p=top_p),
              Group(rows=1, temperature=1.0, gamma=0.9, temp_eff=10.5, do_sample=1, is_last=1, step=7, seed=(5, 6),
                    top_p=top_p)]
    n0 = [int((zcur0[b0:b0 + gr.rows] == V).sum()) for b0, gr in zip((0, 2, 4), groups)]
    logits = SB.logits_for(Bs * S, V, g).cuda() if path in (0, 1) else None
    partials = (SB.records_from_logits(SB.logits_for(Bs * S, V, g).cuda(), 1.0, 1, (1, 2), 3, Bs, S)
                if path == 2 else None)
    tokens0 = conf0 = None
    if path == 3:  # the re-mask alone reads the step's tokens and confidences
        tokens0 = torch.randint(0, V, (Bs, S), generator=g, dtype=torch.int32).cuda()
        conf0 = torch.randn(Bs, S, generator=g).cuda()

    def run(bounded):
        z = zcur0.clone()
        tokens = tokens0.clone() if path == 3 else SB.sentinel((Bs, S), torch.int32)
        conf = conf0.clone() if path == 3 else SB.sentinel((Bs, S), torch.float32)
        ctx = live_bound(L, R) if bounded else contextlib.nullcontext()
        with ctx:
            SB.dbg_sample(path, z, tokens, conf, n0, ncc, V, groups, logits=logits, partials=partials)
        torch.cuda.synchronize()
        return tokens, conf, z

    want, got = run(False), run(True)
    for w, x, name in zip(want, got, ("tokens", "conf", "zcur")):
        assert torch.equal(x[:R].view(torch.int32), w[:R].view(torch.int32)), f"{name} of live rows differ"
    assert torch.equal(got[2][R:], zcur0[R:]), "zcur of an idle row changed"
    if path != 3:
        assert bool((got[0][R:].view(torch.int32) == SB.SENTINEL).all()), "tokens of an idle row written"
        assert bool((got[1][R:].view(torch.int32) == SB.SENTINEL).all()), "confidences of an idle row written"
    else:
        assert torch.equal(got[0][R:], tokens0[R:]) and torch.equal(got[1][R:], conf0[R:])
