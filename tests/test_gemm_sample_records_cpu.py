"""CPU: the reference of the classifier GEMM's sampling records (tests/gemm_sample_ref.py), followed by the tile pick
of sample_combine_kernel with uniform 1, reproduces the oracle's two-level Philox draw
(OracleVampNet.sample_from_logits, rng="philox") token for token.  tests/test_gpu_gemm_fused.py holds the kernel's
records to this reference, so the fused sampler is pinned to the oracle through it.  Rows whose draw lies within
1e-5 of a crossing (relative to the mass) are excluded: the two definitions round differently there."""
import numpy as np
import pytest
import torch

from oracle import philox
from oracle import vampnet_oracle as vo
from tests import gemm_sample_ref as R


def _oracle():
    cfg = vo.OracleConfig(n_heads=4, n_layers=1, n_codebooks=4, n_conditioning_codebooks=0, embedding_dim=256)
    return vo.OracleVampNet(cfg, vo.make_state_dict(cfg, seed=0), "fp32")


def records_then_combine(logits, temperature, sample, key, step):
    """logits (B, S, V) fp32 -> token (B, S) and the ambiguity mask, by way of the per-strip records."""
    B, S, V = logits.shape
    nt = V // R.TILE
    inv_t = R.inv_temperature(temperature)
    u1 = u2 = None
    if sample:
        u1 = torch.from_numpy(philox.uniform_bs(key, step, B, S, stream=0, word=0)).reshape(-1)
        u2 = torch.from_numpy(philox.uniform_bs(key, step, B, S, stream=0, word=1)).reshape(-1)
    mx, am, s, cand, amb = R.strip_records(logits.reshape(-1, R.TILE), inv_t,
                                           None if u2 is None else u2.repeat_interleave(nt))
    rs = lambda t: t.reshape(B * S, nt)  # noqa: E731
    tok, amb_t = R.combine(rs(mx), rs(s), rs(cand), rs(am), inv_t, u1)
    amb_in = rs(amb).gather(1, (tok // R.TILE)[:, None])[:, 0]  # the picked tile's in-strip draw
    return tok.reshape(B, S), (amb_in | amb_t).reshape(B, S)


def _logits(kind, B, S, V, g):
    x = torch.randn(B, S, V, generator=g) * 3.0
    if kind == "peaked":          # one tile holds almost all of the mass
        x[..., 256:384] += 12.0
    elif kind == "ties":          # exact ties of the maximum inside and across tiles
        x = torch.round(x)
        x[..., 5] = x[..., 77] = x[..., 600] = x.amax(-1) + 1.0
    return x.float()


@pytest.mark.parametrize("kind", ["normal", "peaked", "ties"])
@pytest.mark.parametrize("temperature", [0.05, 0.7, 1.0, 3.0])
@pytest.mark.parametrize("sample", [True, False], ids=["sample", "greedy"])
def test_records_then_tile_pick_equal_the_oracle_draw(kind, temperature, sample):
    B, S, V, key, step = 2, 600, 1024, (123, 45), 11
    logits = _logits(kind, B, S, V, torch.Generator().manual_seed(7))
    want, _ = _oracle().sample_from_logits(logits.clone(), sample, temperature, rng="philox", philox_key=key, step=step)
    got, amb = records_then_combine(logits, temperature, sample, key, step)
    if not sample:
        assert not amb.any()
    assert int(amb.sum()) <= amb.numel() // 100, f"{int(amb.sum())} ambiguous rows"
    ok = ~amb
    bad = (got != want) & ok
    assert not bad.any(), f"{int(bad.sum())} of {int(ok.sum())} tokens differ, first at {bad.nonzero()[0].tolist()}"


def test_strip_records_fields():
    """The record fields on hand-made strips: exact max, first arg-max on ties, the sum of exp, and the candidate is
    the first entry whose running sum passes u2 * sum."""
    x = torch.full((3, R.TILE), -1000.0)
    x[0, 10] = x[0, 20] = 2.0            # tie: arg-max 10, half the mass each
    x[1, :] = 0.0                        # uniform strip
    x[2, 127] = 5.0
    u2 = torch.tensor([0.75, 0.503, 0.3], dtype=torch.float32)
    mx, am, s, cand, amb = R.strip_records(x, np.float32(1.0), u2)
    assert mx.tolist() == [2.0, 0.0, 5.0] and am.tolist() == [10, 0, 127]
    assert np.allclose(s.numpy(), [2.0, 128.0, 1.0], rtol=1e-6)
    assert cand.tolist() == [20, 64, 127] and not amb.any()
    _, _, _, cand_g, _ = R.strip_records(x, np.float32(1.0), None)
    assert cand_g.tolist() == [10, 0, 127]
