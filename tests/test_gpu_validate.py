"""GPU: VampNet.validate and Interface.validate end to end (the reference training script's val_loop from codes on).

* On the reference's goldens (tests/golden/validate_*.npz, its own fp32 CPU run): validate with the golden's mask and r
  equals the float64 oracle applied to the kernels' own logits (forward_codes of the same masked codes): loss within
  1e-6 relative, accuracies bit for bit (the tie rule is the oracle's too).
* Against the reference's values.  The bf16-operand forward is within 0.09 max (1.2e-2 mean) of the fp32 reference on
  logits of std ~1 (DESIGN.md §2; asserted again here).  A logit error of at most d moves lse by at most d, x[target] by
  at most d and the row mean by at most d, so each row's nll and smooth move by at most 2 d, and so does their average:
  the loss is within 2 x 0.09 = 0.18 of the reference's.  A top-k decision cannot change where the target's distance
  to the k-th largest other logit (its margin) exceeds 2 d, so the decisions must equal the reference's on every such
  row, and such rows must exist.
* The adapter path: validate(adapter=) on the base model against the oracle on forward_codes(adapter=).
* Interface.validate on a seeded 10 s signal equals encode followed by VampNet.validate bit for bit under the same torch
  seed (the mask is a torch.bernoulli draw on the device), with torch's sync debug mode erroring from the forward on.
* Full-size coarse (d = 1280, 20 layers, random weights) at the reference's validation size B = 8, T = 575."""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import validate_oracle as vor
from tests.test_gpu_adapters import base_with_adapters
from tests.test_gpu_interface import iface  # noqa: F401  (fixture)
from tests.test_gpu_parity import build
from tests.test_gpu_parity_shapes import FULL_COARSE

pytestmark = pytest.mark.gpu

LOGIT_MAX, LOGIT_MEAN = 0.09, 1.2e-2  # bf16-operand forward vs fp32 reference, DESIGN.md §2


def masked_codes(model, z, mask):
    from vampnet_b200 import mask as pmask
    return pmask.apply_mask(z, mask, model.mask_token, check=False)[0]


def oracle_on(logits, z, mask, r, ncc, eps=0.1):
    target, flat_mask = vor.targets(z.cpu().numpy(), mask.cpu().numpy(), ncc)
    return vor.metrics(logits.cpu().numpy(), target, flat_mask, np.asarray(r, dtype=np.float64), eps)


def assert_matches(got: dict, vals: dict):
    from vampnet_b200.metrics import KEYS
    assert tuple(got) == KEYS
    for k, v in got.items():
        assert v.dtype == torch.float32 and v.ndim == 0 and v.is_cuda, k
    out = np.array([float(got[k]) for k in KEYS], dtype=np.float32)
    want = np.array([vals[k] for k in KEYS])
    assert (np.isnan(out[0]) and np.isnan(want[0])) or abs(out[0] - want[0]) <= 1e-6 * abs(want[0]), (out[0], want[0])
    assert np.array_equal(out[1:], want[1:].astype(np.float32), equal_nan=True), (out, want)
    return out


def decisions(stats, k):
    return stats["gt"] + stats["eq"] < k


@pytest.mark.parametrize("name", ["validate_tiny_coarse", "validate_tiny_coarse_empty", "validate_tiny_c2f",
                                  "validate_tiny_coarse_lora"])
def test_validate_vs_oracle_and_reference(golden_dir, name):
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    cfgd = json.loads(str(g["cfg"]))
    if int(g["lora"]):
        _, _, model, _, codec = base_with_adapters(cfgd, seed=int(g["weight_seed"]), cb_seed=int(g["codebook_seed"]))
        adapter = "ft0"
    else:
        _, _, model, _, codec = build(cfgd, seed=int(g["weight_seed"]), cb_seed=int(g["codebook_seed"]))
        adapter = None
    ncc = cfgd["n_conditioning_codebooks"]
    z, mask = torch.from_numpy(g["z"]).cuda(), torch.from_numpy(g["mask"]).cuda()
    r = torch.from_numpy(g["r"])
    got = model.validate(codec, z, r=r, mask=mask, adapter=adapter)
    logits = model.forward_codes(masked_codes(model, z, mask), codec, adapter=adapter)
    vals, amb, st = oracle_on(logits, z, mask, r, ncc)
    out = assert_matches(got, vals)
    # against the reference's fp32 run
    ref_logits = torch.from_numpy(g["logits"])
    e = (logits.cpu() - ref_logits).abs()
    print(f"[{name}] logits vs reference: max {e.max():.3e} mean {e.mean():.3e}; loss {out[0]:.6f} vs "
          f"{g['values'][0]:.6f}")
    assert e.max() < LOGIT_MAX and e.mean() < LOGIT_MEAN
    assert abs(out[0] - g["values"][0]) <= 2 * LOGIT_MAX
    assert np.array_equal(np.isnan(out), np.isnan(g["values"]))
    target, _ = vor.targets(g["z"], g["mask"], ncc)
    ref_st = vor.row_stats(g["logits"].reshape(-1, g["logits"].shape[-1]), target.reshape(-1))
    safe_total = 0
    for k in vor.TOPK:
        safe = ref_st["margin"][k] > 2 * LOGIT_MAX
        safe_total += int(safe.sum())
        assert np.array_equal(decisions(st, k)[safe], decisions(ref_st, k)[safe]), k
    assert safe_total > 0


def test_validate_is_deterministic_and_draws_like_the_reference():
    """Without a mask: the mask is pmask.random(z, r) with the conditioning books unmasked, drawn from torch's RNG, so
    the same seed gives the same bits; an rng draws r as rng.draw(B)[:, 0]."""
    from vampnet_b200 import mask as pmask
    from tests.test_gpu_parity import TINY_C2F
    cfg, _, model, _, codec = build(TINY_C2F)
    g = torch.Generator().manual_seed(5)
    z = torch.randint(0, 1024, (3, 14, 20), generator=g).cuda()
    runs = []
    for _ in range(2):
        torch.manual_seed(1)
        runs.append(model.validate(codec, z, rng=torch.quasirandom.SobolEngine(1, scramble=True, seed=0)))
    for k in runs[0]:
        assert runs[0][k].cpu().numpy().tobytes() == runs[1][k].cpu().numpy().tobytes(), k
    r = torch.quasirandom.SobolEngine(1, scramble=True, seed=0).draw(3)[:, 0]
    torch.manual_seed(1)
    mask = pmask.codebook_unmask(pmask.random(z, r.cuda()), 4)
    vals, _, _ = oracle_on(model.forward_codes(masked_codes(model, z, mask), codec), z, mask, r, 4)
    assert_matches(runs[0], vals)


def test_interface_validate_equals_encode_then_validate_without_sync(iface):  # noqa: F811
    from vampnet_b200.audio import AudioSignal
    torch.manual_seed(0)
    sr = 44100
    t = torch.arange(sr * 10) / sr
    sig = AudioSignal((0.3 * torch.sin(2 * math.pi * 220 * t) + 0.05 * torch.randn_like(t))[None, None], sr)
    for which in ("coarse", "c2f"):
        vn = getattr(iface, which)
        codes = iface.encode(sig)
        torch.manual_seed(3)
        want = vn.validate(iface.codec, codes, rng=torch.quasirandom.SobolEngine(1, scramble=True, seed=0))
        torch.cuda.synchronize()
        calls = []
        orig = vn.forward_codes

        def armed(*a, **k):
            torch.cuda.set_sync_debug_mode("error")
            calls.append(1)
            return orig(*a, **k)
        vn.forward_codes = armed
        torch.manual_seed(3)
        try:
            got = iface.validate(sig, model=which, rng=torch.quasirandom.SobolEngine(1, scramble=True, seed=0))
        finally:
            torch.cuda.set_sync_debug_mode("default")
            del vn.forward_codes
        assert calls == [1]
        assert tuple(got) == tuple(want)
        for k in want:
            assert got[k].is_cuda and got[k].dtype == torch.float32 and got[k].ndim == 0
            assert got[k].cpu().numpy().tobytes() == want[k].cpu().numpy().tobytes(), (which, k)
        assert not math.isnan(float(got["loss"]))
    with pytest.raises(ValueError, match="coarse' or 'c2f"):
        iface.validate(sig, model="fine", r=0.5)


def test_full_coarse_at_the_reference_validation_size():
    from vampnet_b200 import mask as pmask
    _, _, model, _, codec = build(FULL_COARSE)
    g = torch.Generator().manual_seed(8)
    z = torch.randint(0, 1024, (8, 4, 575), generator=g).cuda()
    r = torch.quasirandom.SobolEngine(1, scramble=True, seed=0).draw(8)[:, 0]
    torch.manual_seed(2)
    mask = pmask.codebook_unmask(pmask.random(z, r.cuda()), 0)
    got = model.validate(codec, z, r=r, mask=mask)
    vals, _, _ = oracle_on(model.forward_codes(masked_codes(model, z, mask), codec), z, mask, r, 0)
    out = assert_matches(got, vals)
    assert np.isfinite(out[0])
