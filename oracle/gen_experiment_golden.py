"""Run the ORIGINAL project's vampnet/mask.py once and store the masks the experiment script's conditions build.

    VAMPNET_REFERENCE_ROOT=<checkout of the original vampnet> python -m oracle.gen_experiment_golden

Writes tests/golden/reference_experiment_masks.npz: for each case, the mask of scripts/exp/experiment.py's CoarseCond
(full_mask, codebook_unmask, periodic_mask of the result) or of num_sampling_steps (periodic_mask(z, 16)) under
torch.manual_seed(seed), and the four torch.rand draws that follow it (the CPU generator's position afterwards).
tests/test_experiment_cpu.py recomputes them with vampnet_b200.experiment and compares.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_shims  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
# (kind, num_conditioning_codebooks, factor, frames, seed): the registry's four CoarseCond settings and the sampling
# steps' period at an excerpt's 575 frames and at a length that is no multiple of any factor
CASES = [("coarse_cond", n, x, T, 10 + k) for k, (n, x) in enumerate(((1, 1), (4, 4), (4, 16), (4, 32)))
         for T in (575, 37)] + [("periodic", None, 16, T, 30) for T in (575, 37)]


def codes(T: int) -> torch.Tensor:
    return torch.randint(0, 1024, (1, 14, T), generator=torch.Generator().manual_seed(T))


def gen(rm) -> dict:
    out = {}
    for c, (kind, n, x, T, seed) in enumerate(CASES):
        z = codes(T)
        torch.manual_seed(seed)
        if kind == "coarse_cond":
            mask = rm.periodic_mask(rm.codebook_unmask(rm.full_mask(z), n), x)
        else:
            mask = rm.periodic_mask(z, x)
        out[f"mask{c}"] = mask.numpy().astype(np.int8)
        out[f"next{c}"] = torch.rand(4).numpy()
    return out


def main():
    if not ref_shims.available():
        raise SystemExit(f"the original project is not at {ref_shims.REFERENCE_ROOT} (set VAMPNET_REFERENCE_ROOT)")
    _, rm, _ = ref_shims.load_reference()
    try:
        path = os.path.join(GOLDEN, "reference_experiment_masks.npz")
        np.savez_compressed(path, **gen(rm))
    finally:
        ref_shims.uninstall()
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
