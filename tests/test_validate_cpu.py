"""CPU: the validation-metric oracle (oracle/validate_oracle.py) against the reference's own val_loop values
(tests/golden/validate_*.npz, oracle/gen_validate_golden.py) and torch's CrossEntropyLoss, and the host-side argument
checks of VampNet.validate."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from oracle import validate_oracle as vor

TINY_COARSE = dict(n_heads=4, n_layers=2, n_codebooks=4, n_conditioning_codebooks=0, embedding_dim=256)


def goldens(golden_dir):
    paths = sorted(glob.glob(os.path.join(golden_dir, "validate_*.npz")))
    assert len(paths) == 4, paths
    return paths


def test_oracle_reproduces_reference_values(golden_dir):
    """From each golden's own (reference fp32) logits: the loss within 1e-6 relative of the reference's fp32 value,
    every accuracy exactly, NaN where the reference has NaN; no tie decides any of them."""
    seen_nan = seen_value = 0
    for path in goldens(golden_dir):
        g = np.load(path)
        ncc = json.loads(str(g["cfg"]))["n_conditioning_codebooks"]
        target, flat_mask = vor.targets(g["z"], g["mask"], ncc)
        vals, amb, _ = vor.metrics(g["logits"], target, flat_mask, g["r"], float(g["label_smoothing"]))
        ref = dict(zip(vor.KEYS, g["values"]))
        assert abs(vals["loss"] - ref["loss"]) <= 1e-6 * abs(ref["loss"]), (path, vals["loss"], ref["loss"])
        for k in vor.KEYS[1:]:
            assert amb[k] == 0, (path, k)
            if np.isnan(ref[k]):
                assert np.isnan(vals[k]), (path, k)
                seen_nan += 1
            else:
                assert np.float32(vals[k]) == ref[k], (path, k, vals[k], ref[k])
                seen_value += 1
    assert seen_nan and seen_value


def test_oracle_loss_is_torch_cross_entropy():
    """The closed form against nn.CrossEntropyLoss(label_smoothing, ignore_index=-100) in float64, the empty case NaN."""
    g = torch.Generator().manual_seed(0)
    B, S, V = 3, 20, 64
    x = torch.randn(B, S, V, generator=g, dtype=torch.float64) * 3
    t = torch.randint(0, V, (B, S), generator=g)
    m = torch.rand(B, S, generator=g) < 0.6
    for eps in (0.0, 0.1, 0.5, 1.0):
        want = torch.nn.CrossEntropyLoss(label_smoothing=eps, ignore_index=-100)(x.permute(0, 2, 1), t.masked_fill(~m, -100))
        got, _, _ = vor.metrics(x.numpy(), t.numpy(), m.numpy(), np.zeros(B), eps)
        assert abs(got["loss"] - float(want)) <= 1e-12 * abs(float(want)), eps
    got, _, _ = vor.metrics(x.numpy(), t.numpy(), np.zeros((B, S), bool), np.zeros(B), 0.1)
    assert np.isnan(got["loss"])


def test_oracle_ranks_ties_and_margins():
    x = np.array([[3.0, 1.0, 3.0, 2.0] + [0.0] * 28,    # target 0 ties column 2 at the top: top-1 ambiguous
                  [1.0, 5.0, 4.0, 3.0] + [0.0] * 28])   # target 0: below three, above the 28 zeros
    st = vor.row_stats(x, np.array([0, 0]))
    assert list(st["gt"]) == [0, 3] and list(st["eq"]) == [1, 0]
    assert st["margin"][1][0] == 0.0 and st["margin"][1][1] == 4.0 and st["margin"][25][1] == 1.0
    vals, amb, _ = vor.metrics(x[None], np.array([[0, 0]]), np.array([[1, 1]]), np.array([0.2]))
    assert amb["accuracy-0-0.5/top1/masked"] == 1 and vals["accuracy-0-0.5/top1/masked"] == 0.0
    assert amb["accuracy-0-0.5/top25/masked"] == 0 and vals["accuracy-0-0.5/top25/masked"] == 1.0


def test_keys_match_the_reference_order():
    from vampnet_b200.metrics import KEYS
    assert KEYS == vor.KEYS and len(KEYS) == 9
    assert KEYS[1] == "accuracy-0-0.5/top1/unmasked" and KEYS[-1] == "accuracy-0.5-1.0/top25/masked"


def test_validate_argument_checks():
    """Refused on the host before any device work, so a CPU model shows them."""
    from vampnet.modules.transformer import VampNet as DropIn
    from vampnet_b200.modules.transformer import VampNet
    assert DropIn is VampNet
    from vampnet.interface import Interface
    assert callable(Interface.validate)
    model = VampNet(**TINY_COARSE)
    z = torch.randint(0, 1024, (2, 4, 6))
    rng = torch.quasirandom.SobolEngine(1, scramble=True, seed=0)
    with pytest.raises(ValueError, match="exactly one of r and rng"):
        model.validate(None, z)
    with pytest.raises(ValueError, match="exactly one of r and rng"):
        model.validate(None, z, r=0.5, rng=rng)
    with pytest.raises(ValueError, match="r must be"):
        model.validate(None, z, r=torch.tensor([0.1, 0.2, 0.3]))
    with pytest.raises(ValueError, match="r must be"):
        model.validate(None, z, r=torch.tensor([[0.1, 0.2]]))
    for ls in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError, match="label_smoothing"):
            model.validate(None, z, r=0.5, label_smoothing=ls)
    with pytest.raises(ValueError, match="z must be"):
        model.validate(None, z[:, :3], r=0.5)
    with pytest.raises(ValueError, match="mask .* must be"):
        model.validate(None, z, r=0.5, mask=torch.ones(2, 4, 5, dtype=torch.long))
    bad = torch.ones_like(z)
    bad[0, 0, 0] = 2
    with pytest.raises(ValueError, match="binary"):
        model.validate(None, z, r=0.5, mask=bad)
    with pytest.raises(ValueError, match="binary"):
        model.validate(None, z, r=0.5, mask=-torch.ones_like(z))
