"""CPU: the oracle restatement against the ORIGINAL project's own outputs, stored by oracle/gen_reference_golden.py
(tests/golden/reference_vampnet.npz): the same seeded weights, codes and masks go through the oracle here, and the
embedding, logits, per-layer activations (seeded samples of their entries) and generated tokens must match what the
original code produced."""
import numpy as np
import pytest
import torch

from oracle import vampnet_oracle as vo
from oracle.gen_reference_golden import CFGS, GEN_KWS, GEN_STEPS, sample_idx, vampnet_case


@pytest.fixture(scope="module")
def golden(golden_dir):
    import os
    return np.load(os.path.join(golden_dir, "reference_vampnet.npz"))


def sampled(t, seed):
    return t.flatten()[torch.from_numpy(sample_idx(t.numel(), seed))]


@pytest.mark.parametrize("tag", ["coarse", "c2f"])
@pytest.mark.parametrize("lora", [False, True])
def test_forward_and_generate_live(golden, tag, lora):
    key = f"{tag}_lora{int(lora)}"
    cfgd, cfg, sd, cb, z, zm, mask = vampnet_case(tag, lora)
    orc = vo.OracleVampNet(cfg, sd, "fp32")
    lat = orc.from_codes(zm, cb)
    assert torch.equal(sampled(lat, 1), torch.from_numpy(golden[f"{key}_latents"]))
    lo = orc.forward(lat)
    assert (sampled(lo, 2) - torch.from_numpy(golden[f"{key}_logits"])).abs().max() < 3e-5
    lo2, acts = orc.forward(lat, return_activations=True)  # residual stream after every layer (transformer.py:443-461)
    assert tuple(acts.shape) == tuple(golden[f"{key}_acts_shape"]) == (cfg.n_layers, 3, 31, cfg.embedding_dim)
    scale = max(1.0, float(golden[f"{key}_acts_absmax"]))
    assert (sampled(acts, 3) - torch.from_numpy(golden[f"{key}_acts"])).abs().max() < 3e-5 * scale
    assert torch.equal(lo2, lo)
    for ki, kw in enumerate(GEN_KWS):
        for steps in GEN_STEPS:
            zo = orc.generate(cb, z.clone(), mask.clone(), _sampling_steps=steps, seed=9, rng="torch", **kw)
            assert torch.equal(zo, torch.from_numpy(golden[f"{key}_gen{ki}_s{steps}"]).long()), (kw, steps)


def test_typical_filter_is_a_noop_in_the_reference(golden):
    """SURVEY.md §0.4: the reference discards typical_filter's result (transformer.py:989-993): its draws with and
    without the filter are identical, which is why the oracle and the kernels leave it out."""
    on = sorted(k for k in golden.files if k.startswith("typical_on_"))
    assert on and len(on) == len([k for k in golden.files if k.startswith("typical_off_")])
    for k in on:
        assert np.array_equal(golden[k], golden[k.replace("_on_", "_off_")])


def test_mask_2d_and_default_mask(golden):
    cfgd = CFGS["c2f"]
    cfg = vo.OracleConfig(**cfgd)
    sd = vo.make_state_dict(cfg, seed=4)
    cb = vo.make_codebooks(cfg.n_codebooks, seed=2)
    orc = vo.OracleVampNet(cfg, sd, "fp32")
    z = torch.randint(0, 1024, (2, 14, 12), generator=torch.Generator().manual_seed(1))
    m2 = torch.ones(2, 12, dtype=torch.long)
    m2[:, ::3] = 0
    for name, mask in (("mask_default", None), ("mask_2d", m2)):
        zo = orc.generate(cb, z.clone(), None if mask is None else mask.clone(), _sampling_steps=3, seed=1)
        assert torch.equal(zo, torch.from_numpy(golden[name]).long()), name
