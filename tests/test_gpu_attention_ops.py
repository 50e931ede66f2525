"""GPU: the fused attention kernel at op level against the float64 reference of tests/attention_ref.py.

Every output starts as the NaN sentinel (tools/gemm_bits.sentinel) with a guard region past the last row, which must
keep it; rows past a ragged row's length must keep it too, and no other output may be NaN.

a. Bias probes (q = 0: every score is the bias alone, one table entry per head holds +100): rows whose peak lands on
   one key must equal that key's v bit for bit, rows that average (r* = +-sat, or no key at the peak) must be within
   the bound for weights that are exactly 1 or 0.  sat sweeps the one-value branch's edges, T the ragged block.
b. Needle probes (one score 60 nats above every other): out[b, i] = v[b, pi(i)] bit for bit, so every K and v^T
   offset of every (b, h, block, ring stage) is checked exactly, plain and with a length per batch row.
c. Random inputs within the derived bound: every case of tools/attention_bits.py (whose recorded hashes must also
   match), the same shapes with a generic table, and the ragged length sets of test_gpu_attention_ragged.py.
d. The mask excludes padding: 1e4 in the v^T columns past each row's length leaves the output bit-identical.
e. Refusals: sat outside 1..128 and Tpad < T, with the library working afterwards."""
import os

import numpy as np
import pytest
import torch

from tests import attention_ref as R
from tests.test_gpu_attention_ragged import BOUNDARIES, ragged_inputs
from tools import attention_bits as AB
from tools import gemm_bits as GB

pytestmark = pytest.mark.gpu

GUARD_ROWS = 4


@pytest.fixture(scope="module")
def L():
    from vampnet_b200 import _lib
    _lib.lib()
    return _lib


def launch(L, qk, vT, rel, sat, frames=None):
    """The kernel's output (B, T, d) on a sentinel buffer; checks the guard rows, the rows past each length and NaN."""
    B, T, d2 = qk.shape
    d, H = d2 // 2, d2 // 128
    qk, vT, rel = qk.cuda(), vT.cuda(), rel.cuda()
    buf = GB.sentinel(((B * T + GUARD_ROWS) * d,), torch.bfloat16)
    out = buf[:B * T * d].view(B, T, d)
    if frames is None:
        L.check(L.lib().vnb_op_attention(L.ptr(qk), L.ptr(vT), L.ptr(out), L.ptr(rel), sat, B, T, vT.shape[2], H,
                                         L.stream_ptr()))
    else:
        f = torch.tensor(list(frames), dtype=torch.int32, device="cuda")
        L.check(L.lib().vnb_dbg_attention_ragged(L.ptr(qk), L.ptr(vT), L.ptr(out), L.ptr(rel), sat, B, T,
                                                 vT.shape[2], H, L.ptr(f), L.stream_ptr()))
    torch.cuda.synchronize()
    assert bool(GB.untouched(buf[B * T * d:]).all()), "store past the last row"
    lens = [T] * B if frames is None else list(frames)
    for b, n in enumerate(lens):
        assert bool(GB.untouched(out[b, n:]).all()), f"row {b} wrote past its length {n}"
        assert not bool(torch.isnan(out[b, :n].float()).any()), f"NaN in row {b}"
    return out


def within_bound(name, got, o, tol, lens):
    got = got.double()
    err = (got - o).abs()
    valid = torch.arange(got.shape[1], device=got.device)[None, :] < torch.tensor(lens, device=got.device)[:, None]
    ratio = (err / tol)[valid]
    bad = (err > tol) & valid[..., None]
    print(f"{name}: max err/tol {ratio.max().item():.3f}  mean err {err[valid].mean().item():.2e}  "
          f"max err {err[valid].max().item():.2e}")
    if bool(bad.any()):
        b, q, c = bad.nonzero()[0].tolist()
        pytest.fail(f"{name}: {int(bad.sum())} elements outside the bound; first [b={b}, q={q}, col={c}]: got "
                    f"{got[b, q, c].item():.8e} want {o[b, q, c].item():.17e} tol {tol[b, q, c].item():.3e}")


# ------------------------------------------------------------------------------------------- a. bias probes
@pytest.mark.parametrize("sat,T", [(s, T) for s in R.BIAS_SATS for T in R.BIAS_TS])
def test_bias_probe(L, sat, T):
    qk, vT, rel, rs = R.bias_probe(2, T, sat, seed=1000 * sat + T)
    got = launch(L, qk, vT, rel, sat).cpu().double()
    exp, exact, A = R.bias_probe_expect(vT, T, sat, rs)
    wrong = exact & (got != exp)
    if bool(wrong.any()):
        b, q, c = wrong.nonzero()[0].tolist()
        pytest.fail(f"{int(wrong.sum())} single-key rows differ; first [b={b}, q={q}, col={c}, r*={rs[c // 64]}]: "
                    f"got {got[b, q, c].item()} want {exp[b, q, c].item()}")
    tol = R.bound(exp, A, None, torch.tensor([T, T]), vT, exps=False)
    within_bound(f"bias sat={sat} T={T} (means)", got, exp, torch.where(exact, torch.ones_like(tol), tol), [T, T])


# ------------------------------------------------------------------------------------------ b. needle probes
def needle_check(L, lens, T, H):
    qk, vT, rel, pi = R.needle_probe(lens, T, H, seed=T + H)
    assert R.needle_gap(qk.cuda(), rel, pi) >= 60.0
    frames = None if all(n == T for n in lens) else lens
    got = launch(L, qk, vT, rel, 128, frames=frames).cpu()
    exp = R.needle_expect(vT, pi)
    for b, n in enumerate(lens):
        wrong = got[b, :n].double() != exp[b, :n]
        if bool(wrong.any()):
            i, c = wrong.nonzero()[0].tolist()
            pytest.fail(f"row {b} (length {n}): {int(wrong.sum())} outputs differ; first query {i} col {c}: want key "
                        f"{int(pi[b, i])}, got {got[b, i, c].item()} want {exp[b, i, c].item()}")


@pytest.mark.parametrize("B,T,H", R.NEEDLE_SHAPES)
def test_needle_probe(L, B, T, H):
    needle_check(L, [T] * B, T, H)


def test_needle_probe_ragged(L):
    needle_check(L, list(R.NEEDLE_RAGGED), R.NEEDLE_RAGGED_T, 2)


# ----------------------------------------------------------------------------------------- c. random inputs
@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "attention_bits.npz"))


def random_check(L, name, qk, vT, rel, sat, frames=None):
    got = launch(L, qk, vT, rel, sat, frames=frames)
    f = None if frames is None else torch.tensor(list(frames))
    o, A, D, n = R.attention_ref(qk.cuda(), vT.cuda(), rel.cuda(), sat, frames=f)
    within_bound(name, got, o, R.bound(o, A, D, n, vT.cuda()), n.tolist())
    return got


@pytest.mark.parametrize("B,T,H,sat", AB.CASES, ids=[AB.case_name(*c) for c in AB.CASES])
def test_recorded_cases_within_bound(L, golden, B, T, H, sat):
    qk, vT, rel, _ = AB.make_inputs(B, T, H, sat, 1000 * sat + T + B + H)
    got = random_check(L, AB.case_name(B, T, H, sat), qk, vT, rel, sat)
    assert AB.digest(got.cpu()) == str(golden["sha256_" + AB.case_name(B, T, H, sat)])


@pytest.mark.parametrize("B,T,H,sat", AB.CASES, ids=[AB.case_name(*c) for c in AB.CASES])
def test_generic_table_within_bound(L, B, T, H, sat):
    """Every table entry distinct (std 1), so no index error can hide behind a repeated value."""
    qk, vT, _, _ = AB.make_inputs(B, T, H, sat, 7 + sat + T + B + H)
    rel = torch.randn(2 * sat + 1, H, generator=torch.Generator().manual_seed(sat + H))
    random_check(L, f"generic {AB.case_name(B, T, H, sat)}", qk, vT, rel, sat)


@pytest.mark.parametrize("T,H,lengths", [
    (768, 4, BOUNDARIES + (768,)),
    (768, 20, BOUNDARIES + (768,)),
    (3072, 4, BOUNDARIES + (1000, 3071, 3072)),
], ids=["T768_d256", "T768_d1280", "T3072_d256"])
def test_ragged_within_bound(L, T, H, lengths):
    qk, vT, rel, sat, _ = ragged_inputs(lengths, T, H, seed=T + H)
    random_check(L, f"ragged T={T} H={H}", qk, vT, rel, sat, frames=lengths)


# ----------------------------------------------------------------------------------------------- d. padding
@pytest.mark.parametrize("T,lens", [(3, None), (65, None), (575, None), (3071, None),
                                    (R.NEEDLE_RAGGED_T, R.NEEDLE_RAGGED)], ids=["T3", "T65", "T575", "T3071", "ragged"])
def test_padding_is_masked(L, T, lens):
    qk, vT, rel = R.padding_probe(lens, T)
    big = launch(L, qk, vT, rel, 128, frames=lens)
    zero = launch(L, qk, R.pad_with(vT, lens, T, 0.0), rel, 128, frames=lens)
    assert torch.equal(big.view(torch.int16), zero.view(torch.int16))


# ---------------------------------------------------------------------------------------------- e. refusals
def test_refusals_leave_the_library_working(L):
    B, T, H = 1, 100, 2
    g = torch.Generator().manual_seed(5)
    qk = torch.randn(B, T, 256, generator=g).bfloat16().cuda()
    vT = R.vT_of(torch.randn(B, T, 128, generator=g).bfloat16(), 104).cuda()
    rel = (torch.randn(2 * 128 + 1, H, generator=g) * 0.5).cuda()
    want = launch(L, qk, vT, rel, 128)
    out = GB.sentinel((B, T, 128), torch.bfloat16)
    frames = torch.tensor([T], dtype=torch.int32, device="cuda")
    short = vT[:, :, :96].contiguous()
    calls = {
        "sat 0": lambda: L.lib().vnb_op_attention(L.ptr(qk), L.ptr(vT), L.ptr(out), L.ptr(rel), 0, B, T, 104, H,
                                                  L.stream_ptr()),
        "sat 129": lambda: L.lib().vnb_op_attention(L.ptr(qk), L.ptr(vT), L.ptr(out), L.ptr(rel), 129, B, T, 104, H,
                                                    L.stream_ptr()),
        "ragged sat 129": lambda: L.lib().vnb_dbg_attention_ragged(L.ptr(qk), L.ptr(vT), L.ptr(out), L.ptr(rel), 129,
                                                                   B, T, 104, H, L.ptr(frames), L.stream_ptr()),
        "Tpad < T": lambda: L.lib().vnb_op_attention(L.ptr(qk), L.ptr(short), L.ptr(out), L.ptr(rel), 128, B, T, 96,
                                                     H, L.stream_ptr()),
        "ragged Tpad < T": lambda: L.lib().vnb_dbg_attention_ragged(L.ptr(qk), L.ptr(short), L.ptr(out), L.ptr(rel),
                                                                    128, B, T, 96, H, L.ptr(frames), L.stream_ptr()),
    }
    for name, call in calls.items():
        assert call() != 0, f"{name} accepted"
        print(f"{name}: {L.lib().vnb_last_error().decode()}")
        torch.cuda.synchronize()
        assert bool(GB.untouched(out).all()), f"{name} wrote output"
    again = launch(L, qk, vT, rel, 128)
    assert torch.equal(again.view(torch.int16), want.view(torch.int16))
