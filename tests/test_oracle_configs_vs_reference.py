"""CPU: the oracle against the ORIGINAL project's own outputs off the shipped geometry (tests/golden/
reference_vampnet_configs.npz, written by oracle/gen_reference_golden.py): a 256-entry vocabulary with one predicted
codebook, and a 768-entry vocabulary with seven predicted codebooks under two conditioning ones.  The mask token is
the vocabulary size, so these pin every place the oracle uses it (masking, the embedding's MASK row, the re-mask) at a
value other than 1024, which is what makes the GPU tests of tests/test_gpu_model_configs.py meaningful there.  The
agreement required is that of tests/test_oracle_vs_reference.py."""
import os

import numpy as np
import pytest
import torch

from oracle import vampnet_oracle as vo
from oracle.gen_reference_golden import CONFIG_CFGS, GEN_KWS, GEN_STEPS, sample_idx, vampnet_case


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "reference_vampnet_configs.npz"))


def sampled(t, seed):
    return t.flatten()[torch.from_numpy(sample_idx(t.numel(), seed))]


@pytest.mark.parametrize("tag", sorted(CONFIG_CFGS))
def test_forward_and_generate_live(golden, tag):
    key = f"{tag}_lora0"
    cfgd, cfg, sd, cb, z, zm, mask = vampnet_case(tag, False, CONFIG_CFGS)
    assert cfg.vocab_size != 1024 and (zm == cfg.mask_token).any()
    orc = vo.OracleVampNet(cfg, sd, "fp32")
    lat = orc.from_codes(zm, cb)
    assert torch.equal(sampled(lat, 1), torch.from_numpy(golden[f"{key}_latents"]))
    lo = orc.forward(lat)
    assert lo.shape == (3, cfg.vocab_size, 31 * cfg.n_predict_codebooks)
    assert (sampled(lo, 2) - torch.from_numpy(golden[f"{key}_logits"])).abs().max() < 3e-5
    lo2, acts = orc.forward(lat, return_activations=True)
    assert tuple(acts.shape) == tuple(golden[f"{key}_acts_shape"]) == (cfg.n_layers, 3, 31, cfg.embedding_dim)
    scale = max(1.0, float(golden[f"{key}_acts_absmax"]))
    assert (sampled(acts, 3) - torch.from_numpy(golden[f"{key}_acts"])).abs().max() < 3e-5 * scale
    assert torch.equal(lo2, lo)
    for ki, kw in enumerate(GEN_KWS):
        for steps in GEN_STEPS:
            zo = orc.generate(cb, z.clone(), mask.clone(), _sampling_steps=steps, seed=9, rng="torch", **kw)
            want = torch.from_numpy(golden[f"{key}_gen{ki}_s{steps}"]).long()
            assert torch.equal(zo, want), (kw, steps)
            assert zo.max() < cfg.vocab_size
