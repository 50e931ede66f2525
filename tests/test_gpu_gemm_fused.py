"""GPU: the GEMM family's fused epilogues, one kernel at a time, at the forward's shapes, against float64 references of
the same bf16 operands (vnb_dbg_gemm_fused, vnb_dbg_gemm_sample; include/vampnet_b200.h).  Every test runs with both
tile variants ("gemm_pair" 0 and 1).  Output buffers start as a NaN sentinel bit pattern and guard regions around them
must keep it, so a missed or a stray store fails.

Row scale (fused RMSNorm of the A operand): rs = rsqrt(sum_p ss_in[p] / d + eps), with rows whose rs spans 1e-2 .. 1e3
and rows where eps alone sets it (tools/gemm_bits.py row_stats).  The references use rs64, float64 from the same fp32
partials; the kernel's fp32 rs is within a few 1e-7 of it, far inside every bound below.

Bounds (acc = A . W^T, exact in float64): the existing op tests bound the tensor-core fp32 accumulator by 2e-4 and a
bf16 output by 2^-7 |want| + 2e-3 (tests/test_gpu_gemm.py); here every absolute term is multiplied by the row scale
it passes through."""
import numpy as np
import pytest
import torch

from oracle import philox
from tests import gemm_sample_ref as SR
from tools import gemm_bits as GB

pytestmark = pytest.mark.gpu

ACC_ABS = 2e-4          # fp32 accumulator vs float64, |acc| ~ 1 (tests/test_gpu_gemm.py)
BF16_REL, BF16_ABS = 2.0 ** -7, 2e-3
CHUNK = 4096            # rows per float64 reference block


@pytest.fixture(scope="module")
def L():
    return GB.lib()


@pytest.fixture(params=[0, 1], ids=["single_cta", "cta_pair"])
def pair(request, L):
    prev = GB.set_pair(request.param)
    yield request.param
    GB.set_pair(prev)


def acc64(A, W, rows=None):
    """float64 A[rows] . W^T on the GPU."""
    a = A if rows is None else A[rows]
    return a.double() @ W.double().t()


def gelu_tanh(x):
    return 0.5 * x * (1.0 + torch.tanh(np.sqrt(2.0 / np.pi) * (x + 0.044715 * x ** 3)))


def assert_within(got, want, tol, what):
    err = (got.double() - want).abs()
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = int(bad.reshape(-1).nonzero()[0])
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.numel()} outside the bound; first flat index {i}: got "
                    f"{got.reshape(-1)[i].item():.6e} want {want.reshape(-1)[i].item():.6e} tol {tol.reshape(-1)[i].item():.3e}")


def assert_untouched(t, what):
    ok = GB.untouched(t)
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} entries written outside the output"


# (d, ss_parts, B, T): the coarse-tiny model (ragged M = 300, batch boundaries every 75 rows) and the real d = 1280
# at 3 x 575 (ragged, boundaries inside tiles) and 4 x 768
SHAPES = [(256, 2, 4, 75), (1280, 10, 3, 575), (1280, 10, 4, 768)]
SHAPE_IDS = ["d256_M300", "d1280_M1725", "d1280_M3072"]


@pytest.mark.parametrize("d,parts,B,T", SHAPES, ids=SHAPE_IDS)
def test_bf16_row_scaled(L, pair, d, parts, B, T):
    """BF16 with a row scale: bf16(rs * acc) within 2^-7 |want| + 2e-3 rs."""
    M, N = B * T, d
    A, W, g = GB.operands(M, N, d, seed=11 + M + d)
    ss, inv_d, rs = GB.row_stats(M, d, parts, g)
    out = GB.sentinel((M + 8, N), torch.bfloat16)
    GB.gemm_fused(L.EPI_BF16, A, W, out, ss_in=ss, inv_d=inv_d)
    torch.cuda.synchronize()
    want = rs[:, None] * acc64(A, W)
    assert_within(out[:M], want, BF16_REL * want.abs() + BF16_ABS * rs[:, None], "bf16")
    assert_untouched(out[M:], "rows >= M")


@pytest.mark.parametrize("d,parts,B,T", SHAPES, ids=SHAPE_IDS)
def test_qkv_row_scaled(L, pair, d, parts, B, T):
    """QKV (N = 3d, K = d) with a row scale: qk = bf16(rs * acc[:, :2d]) and the transposed v store
    vT[b, :, t] = bf16(rs * acc[b*T + t, 2d:]), each within 2^-7 |want| + 2e-3 rs; vT's padding columns t >= T and
    qk's rows >= M stay untouched."""
    M, N = B * T, 3 * d
    Tpad = (T + 7) // 8 * 8
    A, W, g = GB.operands(M, N, d, seed=12 + M + d)
    ss, inv_d, rs = GB.row_stats(M, d, parts, g)
    qk = GB.sentinel((M + 8, 2 * d), torch.bfloat16)
    vT = GB.sentinel((B + 1, d, Tpad), torch.bfloat16)
    GB.gemm_fused(L.EPI_QKV, A, W, qk, vT, T=T, Tpad=Tpad, ss_in=ss, inv_d=inv_d)
    torch.cuda.synchronize()
    want = rs[:, None] * acc64(A, W)
    tol = BF16_REL * want.abs() + BF16_ABS * rs[:, None]
    assert_within(qk[:M], want[:, :2 * d], tol[:, :2 * d], "qk")
    assert_untouched(qk[M:], "qk rows >= M")
    v_want = want[:, 2 * d:].reshape(B, T, d).permute(0, 2, 1)
    v_tol = tol[:, 2 * d:].reshape(B, T, d).permute(0, 2, 1)
    assert_within(vT[:B, :, :T], v_want, v_tol, "vT")
    assert_untouched(vT[:B, :, T:], "vT padding")
    assert_untouched(vT[B:], "vT past the last batch item")


@pytest.mark.parametrize("d,parts,B,T", SHAPES, ids=SHAPE_IDS)
def test_geglu_row_scaled(L, pair, d, parts, B, T):
    """GEGLU (N = 4d, K = d; W rows per 256-row tile = [128 value | 128 gate]) with a row scale on value AND gate:
    out = bf16((v rs) * gelu_tanh(g rs)).  Bound: 2^-7 |want| + rs 2e-4 (|gelu(g rs)| + 1.13 |v rs|) (the accumulator
    bound through the product; |gelu'| <= 1.13) + 2e-6 |v rs| |g rs| (the fp32 tanh form of the kernel near gelu's
    tail) + 1e-6."""
    M, N = B * T, 4 * d
    A, W, g = GB.operands(M, N, d, seed=13 + M + d)
    ss, inv_d, rs = GB.row_stats(M, d, parts, g)
    out = GB.sentinel((M + 8, N // 2), torch.bfloat16)
    GB.gemm_fused(L.EPI_GEGLU, A, W, out, ss_in=ss, inv_d=inv_d)
    torch.cuda.synchronize()
    a = acc64(A, W).reshape(M, N // 256, 2, 128)
    v = a[:, :, 0].reshape(M, N // 2) * rs[:, None]
    gt = a[:, :, 1].reshape(M, N // 2) * rs[:, None]
    gl = gelu_tanh(gt)
    want = v * gl
    tol = BF16_REL * want.abs() + rs[:, None] * ACC_ABS * (gl.abs() + 1.13 * v.abs()) + 2e-6 * (v * gt).abs() + 1e-6
    assert_within(out[:M], want, tol, "geglu")
    assert_untouched(out[M:], "rows >= M")


@pytest.mark.parametrize("d,parts,B,T,N", [s + (n,) for s in SHAPES for n in (4096, 10240) if s[0] == 1280 or n == 4096],
                         ids=[i + f"_N{n}" for s, i in zip(SHAPES, SHAPE_IDS) for n in (4096, 10240)
                              if s[0] == 1280 or n == 4096])
def test_classifier_bias_f32_row_scaled(L, pair, d, parts, B, T, N):
    """BIAS_F32 with a row scale (the classifier, N = Cp * 1024): out = fp32(rs * acc) + bias, within
    rs (2e-4 + 4e-6 |acc|) + 1e-6 |bias| (accumulator bound through rs; fp32 rounding of rs and of the product)."""
    M = B * T
    A, W, g = GB.operands(M, N, d, seed=14 + M + N)
    ss, inv_d, rs = GB.row_stats(M, d, parts, g)
    bias = torch.randn(N, generator=g).cuda()
    out = GB.sentinel((M + 8, N), torch.float32)
    GB.gemm_fused(L.EPI_BIAS_F32, A, W, out, bias=bias, ss_in=ss, inv_d=inv_d)
    torch.cuda.synchronize()
    for r0 in range(0, M, CHUNK):
        rows = slice(r0, min(M, r0 + CHUNK))
        a = acc64(A, W, rows)
        want = rs[rows, None] * a + bias.double()
        tol = rs[rows, None] * (ACC_ABS + 4e-6 * a.abs()) + 1e-6 * bias.double().abs()
        assert_within(out[rows], want, tol, "classifier")
    assert_untouched(out[M:], "rows >= M")


def check_partials(ss_out, x, per_tile, what):
    """ss_out (parts, M) against float64 sums of squares of the kernel's own fp32 output x (M, N), per part and chunk
    set: per_tile 2 (RESID): part 2j = 32-column chunks {0, 2, 4, 6} of 256-column tile j, part 2j+1 = {1, 3, 5, 7};
    per_tile 1 (BIAS_F32): part j = all of tile j.  Relative bound: one fp32 rounding per term of the longest
    sequential chain (16 resp. 32 terms per lane, then 3 shuffle adds), 2e-6 resp. 3e-6."""
    M, N = x.shape
    sq = (x.double() ** 2).reshape(M, N // 256, 4, 2, 32)   # (row, tile, chunk pair, even/odd, column)
    if per_tile == 2:
        want = sq.sum(dim=(2, 4)).reshape(M, N // 128).t()   # part 2j + h
        rel = 2e-6
    else:
        want = sq.sum(dim=(2, 3, 4)).t()
        rel = 3e-6
    got = ss_out[: want.shape[0]]
    assert_within(got, want, rel * want, what)


@pytest.mark.parametrize("K", [1280, 2560])
@pytest.mark.parametrize("M", [1, 300, 1725, 24576])
def test_resid_producer(L, pair, M, K):
    """RESID with the bf16 copy and the sum-of-squares partials (attention-out K = 1280, FFN-down K = 2560; N = 1280):
    out = x0 + acc within 2e-4 of float64; out_bf16 == bf16(out) bit for bit; N/128 = 10 partials, each checked
    against float64 on its own chunk set; nothing written past row M-1 or past the last part."""
    N, G = 1280, 8
    A, W, g = GB.operands(M, N, K, seed=15 + M + K)
    x0 = torch.randn(M, N, generator=g).cuda()
    out = GB.sentinel((M + G, N), torch.float32)
    out[:M] = x0
    y = GB.sentinel((M + G, N), torch.bfloat16)
    parts = N // 128
    ss = GB.sentinel(((parts + 1) * M + G,), torch.float32)
    GB.gemm_fused(L.EPI_RESID, A, W, out, out_bf16=y, ss_out=ss)
    torch.cuda.synchronize()
    for r0 in range(0, M, CHUNK):
        rows = slice(r0, min(M, r0 + CHUNK))
        assert_within(out[rows], x0[rows].double() + acc64(A, W, rows), torch.full((1,), ACC_ABS, device="cuda"),
                      "resid out")
    assert torch.equal(y[:M].view(torch.int16), out[:M].bfloat16().view(torch.int16)), "out_bf16 != bf16(out)"
    check_partials(ss[: parts * M].view(parts, M), out[:M], 2, "resid ss_out")
    assert_untouched(out[M:], "out rows >= M")
    assert_untouched(y[M:], "out_bf16 rows >= M")
    assert_untouched(ss[parts * M:], "ss_out past the last part")


@pytest.mark.parametrize("K", [192, 384])
@pytest.mark.parametrize("M", [300, 1725])
def test_embedding_producer(L, pair, M, K):
    """BIAS_F32 with the bf16 copy and partials (the embedding projection, K = 3 Kp, N = 1280): out = acc + bias
    within 2e-4; out_bf16 == bf16(out); ONE partial per 256-column tile; parts >= N/256 of the workspace's N/128 stay
    untouched (launch_embed_gather zeroes them in the forward)."""
    N, G = 1280, 8
    A, W, g = GB.operands(M, N, K, seed=16 + M + K)
    bias = torch.randn(N, generator=g).cuda()
    out = GB.sentinel((M + G, N), torch.float32)
    y = GB.sentinel((M + G, N), torch.bfloat16)
    ss = GB.sentinel((N // 128, M), torch.float32)
    GB.gemm_fused(L.EPI_BIAS_F32, A, W, out, bias=bias, out_bf16=y, ss_out=ss)
    torch.cuda.synchronize()
    assert_within(out[:M], acc64(A, W) + bias.double(), torch.full((1,), ACC_ABS, device="cuda"), "embed out")
    assert torch.equal(y[:M].view(torch.int16), out[:M].bfloat16().view(torch.int16)), "out_bf16 != bf16(out)"
    check_partials(ss, out[:M], 1, "embed ss_out")
    assert_untouched(ss[N // 256:], "parts >= N/256")
    assert_untouched(out[M:], "out rows >= M")
    assert_untouched(y[M:], "out_bf16 rows >= M")


@pytest.mark.parametrize("B,T", [(3, 575), (4, 768)])
def test_producer_to_consumer_chain(L, pair, B, T):
    """RESID writes x, y = bf16(x) and N/128 partials; QKV consumes y with ss_parts = N/128, as in the forward.  The
    result equals float64 rmsnorm(x) . W^T, x the fp32 residual the producer wrote and y the operand the design
    prescribes, within the bf16 bounds (scaled by the row's rms scale)."""
    d = 1280
    M = B * T
    Tpad = (T + 7) // 8 * 8
    A, Wo, g = GB.operands(M, d, d, seed=17 + M)
    x = (torch.randn(M, d, generator=g) * (10.0 ** (torch.rand(M, 1, generator=g) * 4 - 2))).cuda()
    y = GB.sentinel((M, d), torch.bfloat16)
    ss = GB.sentinel((d // 128, M), torch.float32)
    GB.gemm_fused(L.EPI_RESID, A, Wo, x, out_bf16=y, ss_out=ss)
    Wqkv = (torch.randn(3 * d, d, generator=g) / d ** 0.5).bfloat16().cuda()
    qk = GB.sentinel((M, 2 * d), torch.bfloat16)
    vT = GB.sentinel((B, d, Tpad), torch.bfloat16)
    GB.gemm_fused(L.EPI_QKV, y, Wqkv, qk, vT, T=T, Tpad=Tpad, ss_in=ss, inv_d=float(np.float32(1.0 / d)))
    torch.cuda.synchronize()
    assert torch.equal(y.view(torch.int16), x.bfloat16().view(torch.int16))
    x64 = x.double()
    rs = 1.0 / torch.sqrt((x64 ** 2).mean(-1) + GB.EPS)
    want = rs[:, None] * acc64(y, Wqkv)
    tol = BF16_REL * want.abs() + BF16_ABS * rs[:, None]
    assert_within(qk, want[:, :2 * d], tol[:, :2 * d], "qk")
    assert_within(vT[:, :, :T], want[:, 2 * d:].reshape(B, T, d).permute(0, 2, 1),
                  tol[:, 2 * d:].reshape(B, T, d).permute(0, 2, 1), "vT")


# ------------------------------------------------------------------------------------------ sampling epilogue
SAMPLE_GRID = [(t, s, st) for t in (0.05, 0.7, 1.0, 3.0) for s in (0, 1) for st in (0, 11)]
SEED = (2024, 77)


def check_sample_records(L, A, W, bias, ss, inv_d, zcur, T, C, ncc, grid, V=GB.V):
    """Runs the sampling epilogue for every (temperature, do_sample, step) of `grid` and checks every record against
    tests/gemm_sample_ref.py, with the logits L from BIAS_F32 on the same operands and row scale (the epilogue
    computes each logit with the same two roundings):  max exact; arg-max exact (lowest index on ties); sum within
    1e-5 relative of float64 (ex2.approx and a 128-term fp32 sum); candidate exact unless its crossing lies within
    1e-5 * sum of the target; the record's logit == L[candidate]; greedy: candidate == arg-max; known positions and
    everything past the last row keep the sentinel.  V is the vocabulary size (and the mask token)."""
    M, K = A.shape
    Cp, nt = C - ncc, V // 128
    N = Cp * V
    Bn = M // T
    G = 64
    logits = GB.sentinel((M, N), torch.float32)
    GB.gemm_fused(L.EPI_BIAS_F32, A, W, logits, bias=bias, ss_in=ss, inv_d=inv_d)
    masked = (zcur[:, ncc:] == V)                                      # (M, Cp)
    rows_m, cps_m = masked.nonzero(as_tuple=True)
    ambiguous = compared = 0
    for temperature, do_sample, step in grid:
        rec = GB.sentinel((M * Cp * nt + G, 4), torch.float32)
        GB.gemm_sample(A, W, bias, ss, inv_d, zcur, T, C, ncc, temperature, do_sample, step, SEED, rec, V=V)
        torch.cuda.synchronize()
        what = f"V={V} T={temperature} sample={do_sample} step={step}"
        assert_untouched(rec[M * Cp * nt:], what + ": records past the last row")
        recs = rec[: M * Cp * nt].view(M, Cp, nt, 4)
        assert bool(GB.untouched(recs[~masked]).all()), what + ": a known position's record was written"
        u2_all = None
        if do_sample:
            u2_all = torch.from_numpy(philox.uniform_bs(SEED, step, Bn, T * Cp, stream=0, word=1)).cuda()
        inv_t = SR.inv_temperature(temperature)
        for i0 in range(0, rows_m.numel(), 65536):
            r, cp = rows_m[i0:i0 + 65536], cps_m[i0:i0 + 65536]
            x = logits[r[:, None], cp[:, None] * V + torch.arange(V, device="cuda")].reshape(-1, 128)
            u2 = None
            if do_sample:
                u2 = u2_all[r // T, (r % T) * Cp + cp].repeat_interleave(nt)
            mx, am, s, cand, amb = SR.strip_records(x, inv_t, u2)
            got = recs[r, cp].reshape(-1, 4)
            bits = got[:, 3].contiguous().view(torch.int32)
            g_cand, g_am = bits & 0xFFFF, bits >> 16
            v0 = (torch.arange(nt, device="cuda") * 128).repeat(r.numel())
            assert torch.equal(got[:, 0], mx), what + ": strip max"
            assert torch.equal(g_am, v0 + am), what + ": arg-max"
            assert_within(got[:, 1], s, 1e-5 * s, what + ": sum of exp")
            ok = ~amb
            bad = (g_cand != v0 + cand) & ok
            assert not bool(bad.any()), f"{what}: {int(bad.sum())} candidates differ of {int(ok.sum())}"
            if not do_sample:
                assert torch.equal(g_cand, g_am), what + ": greedy candidate != arg-max"
            xc = x.gather(1, (g_cand - v0).clamp(0, 127).long()[:, None])[:, 0]
            assert torch.equal(got[:, 2], xc), what + ": record logit != L[candidate]"
            ambiguous += int(amb.sum())
            compared += amb.numel()
    assert ambiguous <= compared // 1000 + 1, f"{ambiguous} of {compared} draws too close to call"


def sample_case(M, T, C, ncc, d=1280, seed=0, V=GB.V):
    N = (C - ncc) * V
    A, W, g = GB.operands(M, N, d, seed=seed)
    bias = torch.randn(N, generator=g)
    W = W.cpu()
    GB.tie_columns(W, bias, g, V=V)
    ss, inv_d, _ = GB.row_stats(M, d, d // 128, g)
    return A, W.cuda(), bias.cuda(), ss, inv_d, GB.sample_inputs(M, C, ncc, g, V=V)


@pytest.mark.parametrize("C,ncc", [(4, 0), (14, 4)], ids=["coarse", "c2f"])
@pytest.mark.parametrize("B,T", [(3, 150), (4, 768)])
def test_sample_records(L, pair, B, T, C, ncc):
    A, W, bias, ss, inv_d, zcur = sample_case(B * T, T, C, ncc, seed=18 + B * T + C)
    check_sample_records(L, A, W, bias, ss, inv_d, zcur, T, C, ncc, SAMPLE_GRID)


def test_sample_records_benchmark_size(L, pair):
    """The c2f classifier at the benchmark's 32 x 768 rows."""
    B, T, C, ncc = 32, 768, 14, 4
    A, W, bias, ss, inv_d, zcur = sample_case(B * T, T, C, ncc, seed=19)
    check_sample_records(L, A, W, bias, ss, inv_d, zcur, T, C, ncc, [(0.7, 1, 11)])


VOCAB_GRID = [(0.05, 1, 11), (0.7, 1, 0), (1.0, 0, 0), (3.0, 1, 11)]


@pytest.mark.parametrize("C,ncc", [(1, 0), (4, 1), (9, 2)], ids=["cp1", "cp3", "cp7"])
@pytest.mark.parametrize("V", [256, 512, 768])
def test_sample_records_vocab_sizes(L, pair, V, C, ncc):
    """Every vocabulary size the library accepts below 1024 (2, 4 and 6 strips per codebook; the record index and the
    mask token both depend on it) with one, three and seven predicted codebooks, at d = 512 and ragged M = 3 x 150:
    each record must equal the float64 reference and nothing outside the masked positions' records may be written."""
    B, T = 3, 150
    A, W, bias, ss, inv_d, zcur = sample_case(B * T, T, C, ncc, d=512, seed=20 + V + C, V=V)
    check_sample_records(L, A, W, bias, ss, inv_d, zcur, T, C, ncc, VOCAB_GRID, V=V)


# ------------------------------------------------------------------------------------------ determinism
@pytest.mark.parametrize("case", GB.CASES, ids=[GB.case_name(*c) for c in GB.CASES])
def test_fused_variants_deterministic(L, case):
    """Every fused variant, the sampling epilogue included, is bit-identical across two runs and across the two tile
    variants."""
    prev = GB.set_pair(0)
    try:
        first = GB.run_case(*case)
        again = GB.run_case(*case)
        GB.set_pair(1)
        paired = GB.run_case(*case)
    finally:
        GB.set_pair(prev)
    assert GB.digest(first) == GB.digest(again), "two runs differ"
    assert GB.digest(first) == GB.digest(paired), "the tile variants differ"
