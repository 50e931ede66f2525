"""GPU: the two kernels that let calls of different lengths share one generate launch, one launch at a time.

Attention with a key length per batch row (vnb_dbg_attention_ragged): batch row b of a launch at T is a call of
frames[b] <= T frames padded to T.  Its padded q / k rows hold NaN and its padded v^T columns hold zeros, as a ragged
generate launch leaves them.  Each row's first frames[b] output rows must equal, bit for bit, a standalone
vnb_op_attention launch of that row at T = frames[b]; the rows past frames[b] must keep their sentinel.

The QKV epilogue with a frames table (vnb_dbg_gemm_qkv_frames): v^T columns t >= frames[b] are exactly 0, and every
other output is bit-equal to the same GEMM without the table, plain (single CTA and CTA pair) and adapted."""
import pytest
import torch

from tests.test_gpu_adapter_ops import LAYER, make_adapters, row_map
from tools import gemm_bits as GB

pytestmark = pytest.mark.gpu

BOUNDARIES = (1, 63, 64, 65, 127, 128, 129, 200)   # one query tile / key block and either side of their edges


@pytest.fixture(scope="module")
def L():
    from vampnet_b200 import _lib
    _lib.lib()
    return _lib


def ragged_inputs(lengths, T, H, seed, sat=128):
    """qk (B, T, 2d) with NaN past every row's length, vT (B, d, Tpad) zero there, rel (2 sat + 1, H)."""
    B, d = len(lengths), H * 64
    g = torch.Generator().manual_seed(seed)
    qk = torch.randn(B, T, 2 * d, generator=g).bfloat16()
    v = torch.randn(B, T, d, generator=g).bfloat16()
    rel = torch.randn(2 * sat + 1, H, generator=g) * 0.5
    rel[:36] = rel[36]
    rel[-36:] = rel[-37]
    Tpad = (T + 7) // 8 * 8
    vT = torch.zeros(B, d, Tpad, dtype=torch.bfloat16)
    for b, n in enumerate(lengths):
        qk[b, n:] = float("nan")
        vT[b, :, :n] = v[b, :n].t()
    return qk.cuda(), vT.cuda(), rel.cuda(), sat, Tpad


def sentinel_out(B, T, d):
    return GB.sentinel((B, T, d), torch.bfloat16)


def standalone(L, qk, vT, rel, sat, b, n, H):
    """Row b alone at T = n: its own q / k rows and v^T columns, zero-padded to its own Tpad."""
    d = H * 64
    Tp = (n + 7) // 8 * 8
    q1 = qk[b:b + 1, :n].contiguous()
    v1 = torch.zeros(1, d, Tp, device="cuda", dtype=torch.bfloat16)
    v1[:, :, :n] = vT[b:b + 1, :, :n]
    out = sentinel_out(1, n, d)
    L.check(L.lib().vnb_op_attention(L.ptr(q1), L.ptr(v1), L.ptr(out), L.ptr(rel), sat, 1, n, Tp, H, L.stream_ptr()))
    return out


def run_ragged(L, qk, vT, rel, sat, lengths, T, Tpad, H):
    B = len(lengths)
    frames = torch.tensor(lengths, dtype=torch.int32, device="cuda")
    out = sentinel_out(B, T, H * 64)
    L.check(L.lib().vnb_dbg_attention_ragged(L.ptr(qk), L.ptr(vT), L.ptr(out), L.ptr(rel), sat, B, T, Tpad, H,
                                             L.ptr(frames), L.stream_ptr()))
    return out


@pytest.mark.parametrize("T,H,lengths", [
    (768, 4, BOUNDARIES + (768,)),
    (768, 20, BOUNDARIES + (768,)),
    (3072, 4, BOUNDARIES + (1000, 3071, 3072)),
], ids=["T768_d256", "T768_d1280", "T3072_d256"])
def test_ragged_rows_equal_their_standalone_launch(L, T, H, lengths):
    qk, vT, rel, sat, Tpad = ragged_inputs(lengths, T, H, seed=T + H)
    got = run_ragged(L, qk, vT, rel, sat, lengths, T, Tpad, H)
    torch.cuda.synchronize()
    for b, n in enumerate(lengths):
        want = standalone(L, qk, vT, rel, sat, b, n, H)
        torch.cuda.synchronize()
        assert torch.equal(got[b, :n].view(torch.int16), want[0].view(torch.int16)), f"row {b} (length {n}) differs"
        assert bool(GB.untouched(got[b, n:]).all()), f"row {b} (length {n}) wrote past its length"


def test_full_length_table_equals_the_plain_launch(L):
    """A table that gives every row T is the launch without one (same inputs, no padding)."""
    T, H, B = 575, 20, 3
    qk, vT, rel, sat, Tpad = ragged_inputs([T] * B, T, H, seed=3)
    got = run_ragged(L, qk, vT, rel, sat, [T] * B, T, Tpad, H)
    want = sentinel_out(B, T, H * 64)
    L.check(L.lib().vnb_op_attention(L.ptr(qk), L.ptr(vT), L.ptr(want), L.ptr(rel), sat, B, T, Tpad, H, L.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


# ------------------------------------------------------------------------------------------------ QKV epilogue
def qkv_frames(L, A, W, qk, vT, T, Tpad, ss, inv_d, frames, ads=None, rmap=None, u=None):
    M, K = A.shape
    N = W.shape[0]
    arr = None
    if ads is not None:
        arr = (L.AdapterWeights * len(ads))(*[L.AdapterWeights(**{k: v.data_ptr() for k, v in a.items()}) for a in ads])
    L.check(L.lib().vnb_dbg_gemm_qkv_frames(L.ptr(A), L.ptr(W), M, N, K, L.ptr(qk), L.ptr(vT), T, Tpad, L.ptr(ss),
                                            ss.shape[0], inv_d, GB.EPS, L.ptr(frames), arr, 0 if ads is None else len(ads),
                                            LAYER, L.ptr(rmap), L.ptr(u), L.stream_ptr()))


@pytest.fixture(params=[0, 1], ids=["single_cta", "cta_pair"])
def pair(request, L):
    prev = GB.set_pair(request.param)
    yield request.param
    GB.set_pair(prev)


@pytest.mark.parametrize("adapted", [False, True], ids=["plain", "adapted"])
@pytest.mark.parametrize("d,parts,T,lengths", [(256, 2, 200, (1, 63, 64, 65, 127, 128, 129, 200)),
                                               (1280, 10, 575, (575, 502, 271, 133))], ids=["d256_T200", "d1280_T575"])
def test_qkv_zeroes_padded_vT_columns_only(L, pair, d, parts, T, lengths, adapted):
    B = len(lengths)
    M, N = B * T, 3 * d
    Tpad = (T + 7) // 8 * 8
    A, W, g = GB.operands(M, N, d, seed=7 + M + d)
    A = A.view(B, T, d)
    for b, n in enumerate(lengths):   # padded rows of the A operand hold NaN, as after a ragged layer
        A[b, n:] = float("nan")
    A = A.view(M, d)
    ss, inv_d, _ = GB.row_stats(M, d, parts, g)
    frames = torch.tensor(lengths, dtype=torch.int32, device="cuda")
    kw = {}
    if adapted:
        kw = dict(ads=make_adapters(d, g), rmap=row_map(B, T, "groups", g))
    outs = []
    for with_frames in (True, False):
        qk, vT = GB.sentinel((M + 8, 2 * d), torch.bfloat16), GB.sentinel((B + 1, d, Tpad), torch.bfloat16)
        u = GB.sentinel((M + 8, 16), torch.float32) if adapted else None
        if with_frames:
            qkv_frames(L, A, W, qk, vT, T, Tpad, ss, inv_d, frames, u=u, **kw)
        elif adapted:
            from tests.test_gpu_adapter_ops import run_adapted
            run_adapted(L, L.EPI_QKV, A, W, qk, vT, T=T, Tpad=Tpad, ss_in=ss, inv_d=inv_d, u=u, **kw)
        else:
            GB.gemm_fused(L.EPI_QKV, A, W, qk, vT, T=T, Tpad=Tpad, ss_in=ss, inv_d=inv_d)
        outs.append((qk, vT, u))
    torch.cuda.synchronize()
    (qk1, vT1, u1), (qk0, vT0, u0) = outs
    assert torch.equal(qk1.view(torch.int16), qk0.view(torch.int16)), "qk differs"
    if adapted:
        assert torch.equal(u1.view(torch.int32), u0.view(torch.int32)), "u differs"
    for b, n in enumerate(lengths):
        assert torch.equal(vT1[b, :, :n].view(torch.int16), vT0[b, :, :n].view(torch.int16)), f"vT row {b} differs"
        assert bool((vT1[b, :, n:T].view(torch.int16) == 0).all()), f"vT row {b}: padded columns are not +0"
    assert torch.equal(vT1[:, :, T:].view(torch.int16), vT0[:, :, T:].view(torch.int16)), "vT past T touched"
    assert torch.equal(vT1[B:].view(torch.int16), vT0[B:].view(torch.int16)), "vT past the last batch row touched"
