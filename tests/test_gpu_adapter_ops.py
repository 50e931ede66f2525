"""GPU: the per-request LoRA kernels one launch at a time (vnb_dbg_gemm_adapted; include/vampnet_b200.h), at the forward's
shapes, against float64: the down-projection u = A . A'^T, and the adapted QKV (with vT), RESID (with the bf16 copy
and the sum-of-squares partials) and GEGLU epilogues, acc' = acc + u . B'^T before the row scale and everything else.
Row maps mix several adapters and base rows inside one 128-row tile (T < 128, and batch boundaries inside tiles).
Base rows must equal the plain kernel (vnb_dbg_gemm_fused) bit for bit, and so must the k columns of QKV.  Outputs
start as a NaN sentinel with guard regions (tools/gemm_bits.py), and u rows of the base stay untouched."""
import pytest
import torch

from tests.test_gpu_gemm_fused import (ACC_ABS, BF16_ABS, BF16_REL, acc64, assert_untouched, assert_within,
                                       check_partials, gelu_tanh)
from tools import gemm_bits as GB

pytestmark = pytest.mark.gpu

LAYERS, LAYER = 2, 1   # the adapters hold two layers; the launch reads layer 1 (layer offsets are exercised)
N_ADAPTERS = 3


@pytest.fixture(scope="module")
def L():
    return GB.lib()


@pytest.fixture(params=[0, 1], ids=["single_cta", "cta_pair"])
def pair(request, L):
    prev = GB.set_pair(request.param)
    yield request.param
    GB.set_pair(prev)


def make_adapters(d, g):
    """N_ADAPTERS random adapters in the vnb_adapter_weights layout (fp32, device); u ~ 1 and the update ~ 0.1."""
    shapes = dict(a_qkv=(d, 16), b_qkv=(2 * d, 8), a_wo=(d, 8), b_wo=(d, 8), a_w1=(d, 8), b_w1=(4 * d, 8),
                  a_w2=(2 * d, 8), b_w2=(d, 8))
    ads = []
    for _ in range(N_ADAPTERS):
        ads.append({k: (torch.randn(LAYERS, *s, generator=g) * (s[0] ** -0.5 if k[0] == "a" else 0.05)).cuda()
                    for k, s in shapes.items()})
    return ads


def row_map(B, T, kind, g):
    """Adapter of every row: 'groups' = one adapter (or -1) per batch row, cycling base, 0, 1, 2; 'rows' = random per
    row (several adapters and base rows inside every tile)."""
    if kind == "groups":
        per_b = torch.tensor([(b % (N_ADAPTERS + 1)) - 1 for b in range(B)], dtype=torch.int32)
        return per_b.repeat_interleave(T).cuda()
    return (torch.randint(0, N_ADAPTERS + 1, (B * T,), generator=g, dtype=torch.int32) - 1).cuda()


def run_adapted(L, epi, A, W, out, out2=None, T=1, Tpad=8, ss_in=None, inv_d=0.0, out_bf16=None, ss_out=None,
                ads=None, rmap=None, u=None):
    lib = L.lib()
    M, K = A.shape
    N = W.shape[0]
    arr = (L.AdapterWeights * len(ads))(*[L.AdapterWeights(**{k: v.data_ptr() for k, v in a.items()}) for a in ads])
    parts = 0 if ss_in is None else ss_in.shape[0]
    L.check(lib.vnb_dbg_gemm_adapted(epi, L.ptr(A), L.ptr(W), M, N, K, L.ptr(out), L.ptr(out2), T, Tpad, L.ptr(ss_in),
                                     parts, inv_d, GB.EPS, L.ptr(out_bf16), L.ptr(ss_out), arr, len(ads), LAYER,
                                     L.ptr(rmap), L.ptr(u), L.stream_ptr()))


def check_u(u, A, ads, rmap, slot, R):
    """u of adapted rows against float64 (bound: K 2^-24 sum_k |a_k w_k|, the fp32 fma chain); base rows untouched."""
    M, K = A.shape
    ad = rmap >= 0
    for i, a in enumerate(ads):
        rows = (rmap == i).nonzero().flatten()
        if rows.numel() == 0:
            continue
        Ap = a["a_" + slot][LAYER].double()                       # (K, R)
        x = A[rows].double()
        want = x @ Ap
        tol = K * 2.0 ** -24 * (x.abs() @ Ap.abs()) + 1e-30
        assert_within(u[rows, :R], want, tol, f"u ({slot}, adapter {i})")
    assert bool(GB.untouched(u[:M][~ad]).all()), "u written for a base row"
    assert_untouched(u[M:], "u rows >= M")


def delta64(u, ads, rmap, b_key, N, brow=None):
    """(M, N) float64 u . B'^T of every adapted row (0 for base rows), from the kernel's own u; brow(n) maps output
    column n to (B' row, u offset), None = no update."""
    M = u.shape[0] - 8
    out = torch.zeros(M, N, dtype=torch.float64, device="cuda")
    for i, a in enumerate(ads):
        rows = (rmap == i).nonzero().flatten()
        if rows.numel() == 0:
            continue
        Bp = a[b_key][LAYER].double()
        uu = u[rows].double()
        if brow is None:
            out[rows] = uu[:, :8] @ Bp.t()
        else:
            for (c0, c1), (b0, uoff) in brow:
                out[rows, c0:c1] = uu[:, uoff:uoff + 8] @ Bp[b0:b0 + (c1 - c0)].t()
    return out


# (d, ss_parts, B, T): tiny models (d = 256, ragged M = 300), d = 1280 at 3 x 575 (boundaries inside tiles) and at
# T = 37 < 128 (several batch rows per tile)
SHAPES = [(256, 2, 4, 75), (1280, 10, 3, 575), (1280, 10, 12, 37)]
SHAPE_IDS = ["d256_M300", "d1280_M1725", "d1280_T37"]
KINDS = ["groups", "rows"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d,parts,B,T", SHAPES, ids=SHAPE_IDS)
def test_adapted_qkv(L, pair, d, parts, B, T, kind):
    """QKV: q and v columns get the update (u[:, :8] . B'_q, u[:, 8:] . B'_v) before the row scale; k columns none."""
    M, N = B * T, 3 * d
    Tpad = (T + 7) // 8 * 8
    A, W, g = GB.operands(M, N, d, seed=41 + M + d)
    ss, inv_d, rs = GB.row_stats(M, d, parts, g)
    ads, rmap = make_adapters(d, g), row_map(B, T, kind, g)
    u = GB.sentinel((M + 8, 16), torch.float32)
    qk, vT = GB.sentinel((M + 8, 2 * d), torch.bfloat16), GB.sentinel((B + 1, d, Tpad), torch.bfloat16)
    run_adapted(L, L.EPI_QKV, A, W, qk, vT, T=T, Tpad=Tpad, ss_in=ss, inv_d=inv_d, ads=ads, rmap=rmap, u=u)
    qk0, vT0 = GB.sentinel((M + 8, 2 * d), torch.bfloat16), GB.sentinel((B + 1, d, Tpad), torch.bfloat16)
    GB.gemm_fused(L.EPI_QKV, A, W, qk0, vT0, T=T, Tpad=Tpad, ss_in=ss, inv_d=inv_d)
    torch.cuda.synchronize()
    check_u(u, A, ads, rmap, "qkv", 16)
    dl = delta64(u, ads, rmap, "b_qkv", N, brow=[((0, d), (0, 0)), ((2 * d, 3 * d), (d, 8))])   # k columns: none
    want = rs[:, None] * (acc64(A, W) + dl)
    tol = BF16_REL * want.abs() + BF16_ABS * rs[:, None]
    assert_within(qk[:M], want[:, :2 * d], tol[:, :2 * d], "qk")
    assert_untouched(qk[M:], "qk rows >= M")
    v_want = want[:, 2 * d:].reshape(B, T, d).permute(0, 2, 1)
    v_tol = tol[:, 2 * d:].reshape(B, T, d).permute(0, 2, 1)
    assert_within(vT[:B, :, :T], v_want, v_tol, "vT")
    assert_untouched(vT[:B, :, T:], "vT padding")
    assert_untouched(vT[B:], "vT past the last batch item")
    base = rmap < 0
    assert torch.equal(qk[:M][base].view(torch.int16), qk0[:M][base].view(torch.int16)), "base rows of qk differ"
    assert torch.equal(qk[:M, d:2 * d].view(torch.int16), qk0[:M, d:2 * d].view(torch.int16)), "k columns updated"
    vb = base.reshape(B, T)
    assert torch.equal(vT[:B, :, :T].permute(0, 2, 1)[vb].view(torch.int16),
                       vT0[:B, :, :T].permute(0, 2, 1)[vb].view(torch.int16)), "base rows of vT differ"


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d,parts,B,T", SHAPES, ids=SHAPE_IDS)
def test_adapted_geglu(L, pair, d, parts, B, T, kind):
    """GEGLU (packed w1 rows, B'_w1 permuted alike): value and gate both updated, then row-scaled, then gelu."""
    M, N = B * T, 4 * d
    A, W, g = GB.operands(M, N, d, seed=43 + M + d)
    ss, inv_d, rs = GB.row_stats(M, d, parts, g)
    ads, rmap = make_adapters(d, g), row_map(B, T, kind, g)
    u = GB.sentinel((M + 8, 8), torch.float32)
    out = GB.sentinel((M + 8, N // 2), torch.bfloat16)
    run_adapted(L, L.EPI_GEGLU, A, W, out, ss_in=ss, inv_d=inv_d, ads=ads, rmap=rmap, u=u)
    out0 = GB.sentinel((M + 8, N // 2), torch.bfloat16)
    GB.gemm_fused(L.EPI_GEGLU, A, W, out0, ss_in=ss, inv_d=inv_d)
    torch.cuda.synchronize()
    check_u(u, A, ads, rmap, "w1", 8)
    a = (acc64(A, W) + delta64(u, ads, rmap, "b_w1", N)).reshape(M, N // 256, 2, 128)
    v = a[:, :, 0].reshape(M, N // 2) * rs[:, None]
    gt = a[:, :, 1].reshape(M, N // 2) * rs[:, None]
    gl = gelu_tanh(gt)
    want = v * gl
    tol = BF16_REL * want.abs() + rs[:, None] * ACC_ABS * (gl.abs() + 1.13 * v.abs()) + 2e-6 * (v * gt).abs() + 1e-6
    assert_within(out[:M], want, tol, "geglu")
    assert_untouched(out[M:], "rows >= M")
    base = rmap < 0
    assert torch.equal(out[:M][base].view(torch.int16), out0[:M][base].view(torch.int16)), "base rows differ"


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("K_of_d", [1, 2], ids=["attn_out", "ffn_down"])
@pytest.mark.parametrize("d,B,T", [(256, 4, 75), (1280, 3, 575), (1280, 12, 37)], ids=SHAPE_IDS)
def test_adapted_resid(L, pair, d, B, T, K_of_d, kind):
    """RESID (fc: K = d, w_2: K = 2d) with the bf16 copy and the partials: out = x0 + acc + u . B'^T within 2e-4 plus
    the update's fp32 rounding; out_bf16 == bf16(out) and the partials of the kernel's own out, as for the plain
    kernel; base rows bit-identical to it (out, bf16 copy and partials)."""
    M, N, K = B * T, d, K_of_d * d
    slot = "wo" if K_of_d == 1 else "w2"
    A, W, g = GB.operands(M, N, K, seed=45 + M + K)
    ads, rmap = make_adapters(d, g), row_map(B, T, kind, g)
    x0 = torch.randn(M, N, generator=g).cuda()
    parts = N // 128

    def fresh():
        out = GB.sentinel((M + 8, N), torch.float32)
        out[:M] = x0
        return out, GB.sentinel((M + 8, N), torch.bfloat16), GB.sentinel(((parts + 1) * M + 8,), torch.float32)
    out, y, ss = fresh()
    u = GB.sentinel((M + 8, 8), torch.float32)
    run_adapted(L, L.EPI_RESID, A, W, out, out_bf16=y, ss_out=ss, ads=ads, rmap=rmap, u=u)
    out0, y0, ss0 = fresh()
    GB.gemm_fused(L.EPI_RESID, A, W, out0, out_bf16=y0, ss_out=ss0)
    torch.cuda.synchronize()
    check_u(u, A, ads, rmap, slot, 8)
    dl = delta64(u, ads, rmap, "b_" + slot, N)
    want = x0.double() + acc64(A, W) + dl
    assert_within(out[:M], want, ACC_ABS + 2e-6 * dl.abs(), "resid out")
    assert torch.equal(y[:M].view(torch.int16), out[:M].bfloat16().view(torch.int16)), "out_bf16 != bf16(out)"
    check_partials(ss[: parts * M].view(parts, M), out[:M], 2, "resid ss_out")
    assert_untouched(out[M:], "out rows >= M")
    assert_untouched(y[M:], "out_bf16 rows >= M")
    assert_untouched(ss[parts * M:], "ss_out past the last part")
    base = rmap < 0
    assert torch.equal(out[:M][base], out0[:M][base]) and torch.equal(y[:M][base].view(torch.int16),
                                                                        y0[:M][base].view(torch.int16))
    sp, sp0 = ss[: parts * M].view(parts, M), ss0[: parts * M].view(parts, M)
    assert torch.equal(sp[:, base], sp0[:, base]), "base rows' partials differ"


def test_row_arithmetic_does_not_depend_on_tile_neighbours(L):
    """An adapted row gives the same bits whoever shares its tile: the same rows under two different row maps that agree
    on them (QKV and RESID at d = 1280, T = 37)."""
    d, B, T = 1280, 12, 37
    M = B * T
    g = torch.Generator().manual_seed(7)
    A, W, _ = GB.operands(M, 3 * d, d, seed=90)
    ss, inv_d, _ = GB.row_stats(M, d, 10, g)
    ads = make_adapters(d, g)
    m1 = row_map(B, T, "rows", g)
    m2 = m1.clone()
    flip = torch.arange(M, device="cuda") % 3 == 0          # every third row changes adapter (or base / adapted)
    m2[flip] = (m1[flip] + 2) % (N_ADAPTERS + 1) - 1
    keep = ~flip
    outs = []
    for rm in (m1, m2):
        qk, vT = GB.sentinel((M, 2 * d), torch.bfloat16), GB.sentinel((B, d, 40), torch.bfloat16)
        u = GB.sentinel((M + 8, 16), torch.float32)
        run_adapted(L, L.EPI_QKV, A, W, qk, vT, T=T, Tpad=40, ss_in=ss, inv_d=inv_d, ads=ads, rmap=rm, u=u)
        outs.append(qk)
    torch.cuda.synchronize()
    assert torch.equal(outs[0][keep].view(torch.int16), outs[1][keep].view(torch.int16))


def test_refusals(L):
    lib = L.lib()
    A = torch.zeros(8, 256, dtype=torch.bfloat16, device="cuda")
    W = torch.zeros(256, 256, dtype=torch.bfloat16, device="cuda")
    arr = (L.AdapterWeights * 1)()
    rc = lib.vnb_dbg_gemm_adapted(L.EPI_BF16, L.ptr(A), L.ptr(W), 8, 256, 256, L.ptr(A), None, 1, 8, None, 0, 0.0,
                                  1e-6, None, None, arr, 1, 0, L.ptr(A), L.ptr(A), L.stream_ptr())
    assert rc != 0 and b"no adapted variant" in lib.vnb_last_error()
