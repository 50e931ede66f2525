"""GPU: the fused attention kernel (vnb_op_attention through the C ABI) against the float64 reference of the same bf16
operands (tests/attention_ref.py) — reference vampnet/modules/transformer.py:234-254: softmax(q.k^T/8 + bias[h, k-q]).v,
heads merged.

Tolerance: the elementwise bound attention_ref.bound derives from the kernel's rounding points (the bf16 output and
softmax numerators, the fp32 score, exponential and sum errors); the mean error must also stay below 5e-4 (2e-3 below
64 keys, where a row has too few keys to average the rounding of the numerators).
"""
import pytest
import torch

from tests import attention_ref as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from vampnet_b200 import _lib
    _lib.lib()
    return _lib


def attention_inputs(B, T, H, seed, sat=128):
    d = H * 64
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, T, d, generator=g).bfloat16().cuda() for _ in range(3))
    rel = (torch.randn(2 * sat + 1, H, generator=g) * 0.5).cuda()
    rel[:36] = rel[36]       # like the T5 buckets: constant beyond a distance (sat 91 of 128 here)
    rel[-36:] = rel[-37]
    Tpad = (T + 7) // 8 * 8
    qk = torch.cat([q, k], dim=-1).contiguous()
    vT = torch.zeros(B, d, Tpad, device="cuda", dtype=torch.bfloat16)
    vT[:, :, :T] = v.permute(0, 2, 1)
    return q, k, v, rel, sat, qk, vT, Tpad


def within_bound(name, got, qk, vT, rel, sat):
    """Asserts the kernel's output is within attention_ref.bound of the float64 reference; returns |error|."""
    o, A, D, n = R.attention_ref(qk, vT, rel, sat)
    tol = R.bound(o, A, D, n, vT)
    err = (got.double() - o).abs()
    print(f"{name}: max err/tol {(err / tol).max().item():.3f}  max err {err.max().item():.3e}  "
          f"mean {err.mean().item():.3e}")
    assert not torch.isnan(got.float()).any()
    assert bool((err <= tol).all()), (err / tol).max().item()
    return err


def run_attention(L, qk, vT, rel, sat, B, T, Tpad, H):
    out = torch.full((B, T, H * 64), float("nan"), device="cuda", dtype=torch.bfloat16)
    L.check(L.lib().vnb_op_attention(L.ptr(qk), L.ptr(vT), L.ptr(out), L.ptr(rel), sat, B, T, Tpad, H, L.stream_ptr()))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("B,T,H", [(1, 64, 1), (1, 65, 1), (1, 128, 1), (1, 129, 2), (2, 100, 4), (1, 3, 2), (1, 256, 2),
                                   (1, 257, 1), (2, 768, 4), (1, 1000, 2), (1, 3072, 1), (3, 575, 20)])
def test_attention_vs_fp32_torch(L, B, T, H):
    """Ragged T (partial last key block / query tile, T < one block), one to 48 key blocks, the table-lookup and the
    constant-bias regimes (T > 2*sat), the reference's 10 s chunk length (575) at full width (20 heads)."""
    q, k, v, rel, sat, qk, vT, Tpad = attention_inputs(B, T, H, seed=T + 1)
    got = run_attention(L, qk, vT, rel, sat, B, T, Tpad, H)
    err = within_bound(f"attention B={B} T={T} H={H}", got, qk, vT, rel, sat)
    assert err.mean() < (2e-3 if T < 64 else 5e-4)


def test_attention_saturated_table_matches_unsaturated_lookup(L):
    """A table given with sat = 128 and one given cut at the distance where it stops changing are the same bias."""
    B, T, H = 1, 300, 2
    q, k, v, rel, sat, qk, vT, Tpad = attention_inputs(B, T, H, seed=7)
    a = run_attention(L, qk, vT, rel, sat, B, T, Tpad, H)
    cut = 128 - 36 + 1   # entries beyond +-92 repeat the edge value
    rel_small = rel[sat - cut: sat + cut + 1].contiguous()
    b = run_attention(L, qk, vT, rel_small, cut, B, T, Tpad, H)
    assert torch.equal(a, b)


@pytest.mark.parametrize("first,later", [(1.0, 40.0), (40.0, 1.0), (40.0, 160.0)])
def test_attention_reference_moves_when_logits_grow(L, first, later):
    """The online softmax moves its row maximum to max(m, block maximum) at every key block and rescales O and l by
    exp2(m_old - m_new).  Keys scaled so that (a) the maximum grows at the later blocks, far beyond block 0's (O and l
    rescaled by factors that flush to 0), (b) block 0 dominates and the later blocks' weights flush to 0 against it,
    (c) both."""
    B, T, H = 1, 640, 2
    q, k, v, rel, sat, qk, vT, Tpad = attention_inputs(B, T, H, seed=5)
    qk = qk.clone()
    qk[:, :64, H * 64:] *= first     # keys of block 0
    qk[:, 400:, H * 64:] *= later    # keys of the later blocks
    got = run_attention(L, qk, vT, rel, sat, B, T, Tpad, H)
    within_bound(f"keys x{first} / x{later}", got, qk, vT, rel, sat)


def test_attention_rows_are_independent_of_batch_and_head_neighbours(L):
    """(b, h, query tile) are independent CTAs: a batch-of-3 / 4-head call equals the calls on its slices bit for bit."""
    B, T, H = 3, 200, 4
    q, k, v, rel, sat, qk, vT, Tpad = attention_inputs(B, T, H, seed=11)
    full = run_attention(L, qk, vT, rel, sat, B, T, Tpad, H)
    one = run_attention(L, qk[1:2].contiguous(), vT[1:2].contiguous(), rel, sat, 1, T, Tpad, H)
    assert torch.equal(full[1:2], one)


def test_attention_timing_bench_shapes(L):
    """Printed for the record (pytest -s): the benchmark's shapes, CUDA-event timed."""
    for (B, T, H) in ((32, 768, 20), (8, 3072, 20)):
        q, k, v, rel, sat, qk, vT, Tpad = attention_inputs(B, T, H, seed=1)
        out = torch.empty(B, T, H * 64, device="cuda", dtype=torch.bfloat16)
        call = lambda: L.lib().vnb_op_attention(L.ptr(qk), L.ptr(vT), L.ptr(out), L.ptr(rel), sat, B, T, Tpad, H,  # noqa: E731
                                                L.stream_ptr())
        for _ in range(3):
            call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            call()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 20
        print(f"attention B={B} T={T} H={H}: {ms * 1e3:.1f} us  {4.0 * B * H * T * T * 64 / ms / 1e9:.0f} TFLOP/s")
