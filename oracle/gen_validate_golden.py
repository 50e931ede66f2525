"""TEST INFRASTRUCTURE — write tests/golden/validate_*.npz by running the reference's own validation step: its
training script's val_loop (scripts/exp/train.py:327-371) from codes on, on the tiny models of oracle/gen_golden.py
(same weight and codebook seeds, fp32, CPU).

    VAMPNET_REFERENCE_ROOT=<checkout> python -m oracle.gen_validate_golden

The model, mask and codebook_flatten come from the checkout through oracle/ref_shims.py.  train.py itself imports
argbind, audiotools, lac and tensorboard, so it is not imported: its `accuracy` and `_metrics` definitions and its
IGNORE_INDEX are parsed out of the file and executed with torch and einops in scope.  Each file holds the cfg and
seeds, z, r, the reference's mask, its fp32 logits transposed to the kernels' (B, S, V) row order, and the 9 values in
the reference's key order (`values`, float32, NaN where the reference's is NaN).
"""
from __future__ import annotations

import ast
import json
import os
import sys
from typing import Optional

import numpy as np
import torch
import torch.nn as nn
from einops import rearrange

from . import ref_shims
from . import vampnet_oracle as vo
from .gen_golden import OUT, TINY_C2F, TINY_COARSE, build_ref
from .validate_oracle import KEYS


def load_train_metrics():
    """`accuracy`, `_metrics` and IGNORE_INDEX of the checkout's scripts/exp/train.py, executed on their own."""
    path = os.path.join(ref_shims.REFERENCE_ROOT, "scripts", "exp", "train.py")
    tree = ast.parse(open(path).read(), path)
    keep = [n for n in tree.body
            if (isinstance(n, ast.FunctionDef) and n.name in ("accuracy", "_metrics"))
            or (isinstance(n, ast.Assign) and any(getattr(t, "id", None) == "IGNORE_INDEX" for t in n.targets))]
    assert len(keep) == 3, [getattr(n, "name", "IGNORE_INDEX") for n in keep]
    ns = dict(torch=torch, rearrange=rearrange, Optional=Optional)
    exec(compile(ast.Module(body=keep, type_ignores=[]), path, "exec"), ns)
    return ns["_metrics"], ns["IGNORE_INDEX"]


# name, cfg, LoRA fine-tune, B, T, r, mask seed: every r range is populated somewhere, r = 1.0 (in neither range) is
# present, and validate_tiny_coarse_empty has no item in [0.5, 1.0)
CASES = (
    ("validate_tiny_coarse", TINY_COARSE, False, 4, 8, (0.25, 0.45, 0.7, 1.0), 1),
    ("validate_tiny_coarse_empty", TINY_COARSE, False, 3, 4, (0.2, 1.0, 0.35), 2),
    ("validate_tiny_c2f", TINY_C2F, False, 3, 4, (0.4, 0.55, 0.9), 3),
    ("validate_tiny_coarse_lora", TINY_COARSE, True, 2, 8, (0.3, 0.8), 4),
)


def main():
    tr, mk, ut = ref_shims.load_reference()
    _metrics, ignore_index = load_train_metrics()
    criterion = nn.CrossEntropyLoss(label_smoothing=0.1, ignore_index=ignore_index)
    for name, cfgd, lora, B, T, rs, mask_seed in CASES:
        cfg, sd, vn = build_ref(tr, cfgd, seed=0, lora=lora)
        codec = ref_shims.StubCodec(vo.make_codebooks(cfg.n_codebooks, seed=1))
        g = torch.Generator().manual_seed(40 + mask_seed)
        z = torch.randint(0, 1024, (B, cfg.n_codebooks, T), generator=g)
        r = torch.tensor(rs, dtype=torch.float32)
        torch.manual_seed(mask_seed)
        # val_loop, train.py:339-371, from the codes on
        mask = mk.random(z, r)
        mask = mk.codebook_unmask(mask, vn.n_conditioning_codebooks)
        z_mask, mask = mk.apply_mask(z, mask, vn.mask_token)
        with torch.no_grad():
            z_hat = vn(vn.embedding.from_codes(z_mask, codec))
        target = ut.codebook_flatten(z[:, vn.n_conditioning_codebooks:, :])
        flat_mask = ut.codebook_flatten(mask[:, vn.n_conditioning_codebooks:, :])
        output = {}
        t_masked = target.masked_fill(~flat_mask.bool(), ignore_index)
        output["loss"] = criterion(z_hat, t_masked)
        _metrics(r=r, z_hat=z_hat, target=target, flat_mask=flat_mask, output=output)
        assert tuple(output) == KEYS, tuple(output)
        values = np.array([float(output[k]) for k in KEYS], dtype=np.float32)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, cfg=json.dumps(cfgd), weight_seed=0, lora=int(lora), codebook_seed=1, z=z.numpy(),
                            r=r.numpy(), mask=mask.numpy(), logits=z_hat.permute(0, 2, 1).contiguous().numpy(),
                            values=values, label_smoothing=0.1)
        print(f"wrote {path} ({os.path.getsize(path) / 1024:.1f} KiB): " +
              ", ".join(f"{k.replace('accuracy-', '')} {v:.4g}" for k, v in zip(KEYS, values)))


if __name__ == "__main__":
    sys.exit(main())
