"""CPU: ties the float64 attention reference (tests/attention_ref.py) to the oracle and to its probes, and shows that
the probes of tests/test_gpu_attention_ops.py see the kernel bugs listed in attention_ref.MUTANTS.

- With the real models' table (rel_bias_table, as VampNet.pack_weights builds it), the reference equals a float64
  attention with the oracle's full (H, T, T) position bias.
- On every probe input the reference equals the probe's closed-form expectation.
- Every mutated reference leaves the GPU test's bound on at least one element of the probe inputs: it differs from
  the expectation by more than the probe's tolerance plus the bound on the mutated kernel's own rounding."""
from types import SimpleNamespace

import pytest
import torch

from oracle import vampnet_oracle as vo
from tests import attention_ref as R
from vampnet_b200.modules.transformer import rel_bias_table


def plain_attention(q, k, v, bias):
    """float64 softmax(q k^T / 8 + bias) v over (H, T, 64) operands and an (H, T, T) bias."""
    p = torch.softmax(q @ k.transpose(1, 2) / 8 + bias, -1)
    return p @ v


@pytest.mark.parametrize("T", [3, 64, 65, 200, 575, 1000, 3072])
def test_reference_equals_oracle_position_bias(T):
    H = 2
    g = torch.Generator().manual_seed(T)
    w = torch.randn(32, H, generator=g) * 0.5
    rel, sat = rel_bias_table(w)
    assert sat == 91 and rel.shape == (2 * sat + 1, H)
    q, k, v = (torch.randn(1, T, 64 * H, generator=g).bfloat16() for _ in range(3))
    qk = torch.cat([q, k], -1)
    o, A, D, lens = R.attention_ref(qk, R.vT_of(v, (T + 7) // 8 * 8), rel, sat)
    bias = vo.OracleVampNet.position_bias(SimpleNamespace(rel_bias=w.double()), T)
    heads = lambda x: x[0].double().view(T, H, 64).transpose(0, 1)  # noqa: E731
    want = plain_attention(heads(q), heads(k), heads(v), bias).transpose(0, 1).reshape(T, 64 * H)
    assert float((o[0] - want).abs().max()) <= 1e-12
    assert bool((A[0] >= o[0].abs() - 1e-12).all())


def bias_cases():
    return [(sat, T) for sat in R.BIAS_SATS for T in R.BIAS_TS]


@pytest.mark.parametrize("sat,T", bias_cases())
def test_bias_probe_reference_equals_closed_form(sat, T):
    qk, vT, rel, rs = R.bias_probe(2, T, sat, seed=1000 * sat + T)
    o, A, D, lens = R.attention_ref(qk, vT, rel, sat)
    exp, exact, A_exp = R.bias_probe_expect(vT, T, sat, rs)
    assert torch.equal(o[exact], exp[exact])
    assert float((o - exp).abs().max()) <= 1e-12
    assert float((A - A_exp).abs().max()) <= 1e-12


def needle_cases():
    return [(B, T, H, None) for B, T, H in R.NEEDLE_SHAPES] + [(len(R.NEEDLE_RAGGED), R.NEEDLE_RAGGED_T, 2,
                                                                 R.NEEDLE_RAGGED)]


@pytest.mark.parametrize("B,T,H,lens", needle_cases(), ids=lambda x: str(x) if x is None or isinstance(x, int)
                         else "ragged")
def test_needle_probe_reference_equals_closed_form(B, T, H, lens):
    lens = [T] * B if lens is None else list(lens)
    qk, vT, rel, pi = R.needle_probe(lens, T, H, seed=T + H)
    assert R.needle_gap(qk, rel, pi) >= 60.0
    o, A, D, _ = R.attention_ref(qk, vT, rel, 128, frames=torch.tensor(lens))
    exp = R.needle_expect(vT, pi)
    for b, n in enumerate(lens):
        assert torch.equal(o[b, :n], exp[b, :n])
    for b, n in enumerate(lens):
        p = pi[b, :n]
        for a, c in R.needle_pairs(n):
            assert p[a] == c and p[c] == a
        assert torch.equal(p.sort().values, torch.arange(n))


# ------------------------------------------------------------------------------------------------- power checks
def probe_inputs():
    """(name, qk, vT, rel, sat, lens, expected, exact, tolerance) of the GPU test's exact probes: every bias probe, the
    needle probes up to T = 1000 and the ragged one, then the padding probe (1e4 in the excluded v^T columns, against
    the same reference on the zero-padded operands: expected None)."""
    for sat, T in bias_cases():
        qk, vT, rel, rs = R.bias_probe(2, T, sat, seed=1000 * sat + T)
        exp, exact, A = R.bias_probe_expect(vT, T, sat, rs)
        lens = torch.tensor([T, T])
        tol = torch.where(exact, torch.zeros_like(exp), R.bound(exp, A, None, lens, vT, exps=False))
        yield f"bias sat={sat} T={T}", qk, vT, rel, sat, None, exp, exact, tol
    for B, T, H, lens in needle_cases():
        if T > 1000:
            continue
        lens = [T] * B if lens is None else list(lens)
        qk, vT, rel, pi = R.needle_probe(lens, T, H, seed=T + H)
        exp = R.needle_expect(vT, pi)
        yield f"needle T={T} H={H}", qk, vT, rel, 128, lens, exp, torch.ones_like(exp, dtype=torch.bool), \
            torch.zeros_like(exp)
    for lens, T in ((None, 65), (R.NEEDLE_RAGGED, R.NEEDLE_RAGGED_T)):
        qk, vT, rel = R.padding_probe(lens, T)
        yield f"padding T={T}", qk, vT, rel, 128, lens, None, None, None


@pytest.mark.parametrize("mutant", R.MUTANTS)
def test_probes_see_mutant(mutant):
    for name, qk, vT, rel, sat, lens, exp, exact, tol in probe_inputs():
        frames = None if lens is None else torch.tensor(lens)
        o, A, D, n = R.attention_ref(qk, vT, rel, sat, frames=frames, mutant=mutant)
        mb = R.bound(o.nan_to_num(), A.nan_to_num(), D.nan_to_num(), n, vT)
        if exp is None:   # the padding probe: against the same (mutated) kernel on zero-padded operands
            exp, A0, D0, _ = R.attention_ref(qk, R.pad_with(vT, lens, qk.shape[1], 0.0), rel, sat, frames=frames,
                                             mutant=mutant)
            tol = R.bound(exp.nan_to_num(), A0.nan_to_num(), D0.nan_to_num(), n, vT)
        if lens is not None:
            valid = torch.arange(qk.shape[1])[None, :] < torch.tensor(lens)[:, None]
        else:
            valid = torch.ones(qk.shape[:2], dtype=torch.bool)
        seen = (torch.isnan(o) | ((o - exp).abs() > tol + mb)) & valid[..., None]
        if bool(seen.any()):
            print(f"{mutant}: first seen by {name} ({int(seen.sum())} elements)")
            return
    pytest.fail(f"no probe sees {mutant}")
