"""GPU: the persistent QKV GEMM (single-CTA mode without adapters: gemm_persistent_kernel, one CTA per SM walking the
tiles, each tile's stores overlapping the next tile's MMAs) against the CTA-pair kernel, which keeps the one-tile
epilogue.  Same operands and the same k order per output element, so q / k and the whole v^T buffer (padding columns
t >= T and any batch row the launch does not reach included, all sentinel-filled) must agree bit for bit:

  * more tiles than SMs, so every CTA loops over several tiles and both staging layouts (q / k row-major, v transposed):
    the benchmark's M = 24 576 at T = 768, and B = 32 at T = 575, where tiles span two batch rows at unaligned t;
  * an odd T with a frames table shorter than T on some rows (v^T columns past a row's length are 0);
  * a live bound that leaves idle rows: the tiles past it write nothing."""
import pytest
import torch

from tests.test_gpu_attention_ragged import qkv_frames
from tests.test_gpu_live_ops import live_bound
from tools import gemm_bits as GB

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    return GB.lib()


def run_both(fn):
    """fn() under the persistent kernel (gemm_pair 0) and under the CTA-pair kernel (gemm_pair 1)."""
    prev = GB.set_pair(0)
    try:
        got = fn()
        GB.set_pair(1)
        want = fn()
    finally:
        GB.set_pair(prev)
    torch.cuda.synchronize()
    return got, want


def bits(t):
    return t.view(torch.int16)


def buffers(B, T, d, extra_rows=0):
    Tpad = (T + 7) // 8 * 8
    return GB.sentinel((B * T + extra_rows, 2 * d), torch.bfloat16), GB.sentinel((B + 1, d, Tpad), torch.bfloat16), Tpad


@pytest.mark.parametrize("B,T,d", [(32, 768, 1280), (32, 575, 1280), (3, 75, 256)],
                         ids=["M24576_T768", "B32_T575", "B3_T75"])
def test_persistent_qkv_equals_the_one_tile_epilogue(L, B, T, d):
    M, N = B * T, 3 * d
    A, W, g = GB.operands(M, N, d, seed=B + T + d)
    ss, inv_d, _ = GB.row_stats(M, d, d // 128, g)

    def fn():
        qk, vT, Tpad = buffers(B, T, d, extra_rows=8)
        GB.gemm_fused(L.EPI_QKV, A, W, qk, vT, T=T, Tpad=Tpad, ss_in=ss, inv_d=inv_d)
        return qk, vT

    (qk1, vT1), (qk0, vT0) = run_both(fn)
    assert torch.equal(bits(qk1), bits(qk0)), "q / k differ"
    assert torch.equal(bits(vT1), bits(vT0)), "v^T differs"
    assert bool(GB.untouched(qk1[M:]).all()) and bool(GB.untouched(vT1[:, :, T:]).all()) and \
        bool(GB.untouched(vT1[B:]).all()), "a store past the rows or frames of the launch"


@pytest.mark.parametrize("T,lengths", [(201, (201, 13, 150, 1, 77, 200)), (575, (575, 502, 271, 133))],
                         ids=["T201", "T575"])
def test_persistent_qkv_zeroes_frames_past_each_length(L, T, lengths):
    B, d = len(lengths), 256
    M, N = B * T, 3 * d
    A, W, g = GB.operands(M, N, d, seed=T + 11)
    ss, inv_d, _ = GB.row_stats(M, d, d // 128, g)
    A = A.view(B, T, d)
    for b, n in enumerate(lengths):   # padded rows of the A operand hold NaN, as after a ragged layer
        A[b, n:] = float("nan")
    A = A.view(M, d)
    frames = torch.tensor(lengths, dtype=torch.int32, device="cuda")

    def fn():
        qk, vT, Tpad = buffers(B, T, d)
        qkv_frames(L, A, W, qk, vT, T, Tpad, ss, inv_d, frames)
        return qk, vT

    (qk1, vT1), (qk0, vT0) = run_both(fn)
    assert torch.equal(bits(qk1), bits(qk0)), "q / k differ"
    assert torch.equal(bits(vT1), bits(vT0)), "v^T differs"
    for b, n in enumerate(lengths):
        assert bool((bits(vT1[b, :, n:T]) == 0).all()), f"v^T row {b}: frames past {n} are not +0"


@pytest.mark.parametrize("R", [1, 5])
def test_persistent_qkv_tiles_past_the_live_bound_write_nothing(L, R):
    B, T, d = 12, 99, 256
    M, N = B * T, 3 * d
    A, W, g = GB.operands(M, N, d, seed=70 + R)
    ss, inv_d, _ = GB.row_stats(M, d, d // 128, g)

    def fn():
        qk, vT, Tpad = buffers(B, T, d)
        with live_bound(L, R):
            GB.gemm_fused(L.EPI_QKV, A, W, qk, vT, T=T, Tpad=Tpad, ss_in=ss, inv_d=inv_d)
        return qk, vT

    (qk1, vT1), (qk0, vT0) = run_both(fn)
    live = R * T
    dead = -(-live // 128) * 128   # first row of the persistent kernel's tiles past the bound
    assert torch.equal(bits(qk1[:live]), bits(qk0[:live])), "q / k of live rows differ"
    assert torch.equal(bits(vT1[:R]), bits(vT0[:R])), "v^T of live rows differs"
    assert bool(GB.untouched(qk1[dead:]).all()), "q / k: a tile past the live rows wrote"
    assert bool(GB.untouched(vT1[-(-dead // T):]).all()), "v^T: a batch row past the live tiles was written"
