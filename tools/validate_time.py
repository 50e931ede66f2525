"""CUDA-event time of the validation metrics (DESIGN.md §12) at the reference's validation size, B = 8 ten-second clips
(T = 575), for full-size coarse (4 codebooks) and c2f (14 codebooks, 4 conditioning) models with random weights:

    python tools/validate_time.py [--iters 20] [--out FILE]

Times the metric kernels alone (vampnet_b200.metrics.xent_metrics on the forward's logits) and the whole
VampNet.validate (mask draw, forward, metrics).  Each is warmed, then timed over --iters back-to-back calls between two
CUDA events, three times; the median is reported.  The metric kernels' achieved bandwidth is the logits' B * S * V * 4
bytes (read once; the codes, mask and records add under 1 %) over their time, against the H100 SXM data sheet's
3.35 TB/s.  The card's name, power limit and SM clocks are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.onset_time import time_us  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
MODELS = {
    "coarse": dict(n_heads=20, n_layers=20, n_codebooks=4, n_conditioning_codebooks=0, embedding_dim=1280),
    "c2f": dict(n_heads=20, n_layers=16, n_codebooks=14, n_conditioning_codebooks=4, embedding_dim=1280),
}


def main():
    from tests.test_gpu_parity import build
    from vampnet_b200 import mask as pmask
    from vampnet_b200.metrics import xent_metrics
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    card = os.popen("nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv,noheader").read().strip()
    B, T = 8, 575
    res = dict(card=card, B=B, T=T, iters=a.iters, models={})
    for name, cfgd in MODELS.items():
        _, _, model, _, codec = build(cfgd)
        ncc = cfgd["n_conditioning_codebooks"]
        g = torch.Generator().manual_seed(0)
        z = torch.randint(0, 1024, (B, cfgd["n_codebooks"], T), generator=g).cuda()
        r = torch.quasirandom.SobolEngine(1, scramble=True, seed=0).draw(B)[:, 0].cuda()
        mask = pmask.codebook_unmask(pmask.random(z, r), ncc)
        logits = model.forward_codes(pmask.apply_mask(z, mask, model.mask_token, check=False)[0], codec)
        S, V = logits.shape[1], logits.shape[2]
        nbytes = B * S * V * 4
        t_metrics, all_m = time_us(lambda: xent_metrics(logits, z, mask, r, ncc), a.iters)
        t_validate, all_v = time_us(lambda: model.validate(codec, z, r=r), max(1, a.iters // 4))
        t_forward, _ = time_us(lambda: model.forward_codes(z, codec), max(1, a.iters // 4))
        bw = nbytes / (t_metrics * 1e-6)
        res["models"][name] = dict(S=S, V=V, logits_bytes=nbytes, metrics_us=t_metrics, metrics_runs_us=all_m,
                                   validate_us=t_validate, validate_runs_us=all_v, forward_us=t_forward,
                                   metrics_bytes_per_s=bw, share_of_3_35_TBps=bw / HBM_BYTES_PER_S)
        print(f"[{name}] B={B} T={T} S={S}: metric kernels {t_metrics:.1f} us ({nbytes / 1e6:.1f} MB of logits, "
              f"{bw / 1e12:.2f} TB/s = {100 * bw / HBM_BYTES_PER_S:.0f} % of 3.35 TB/s); forward {t_forward:.0f} us; "
              f"whole validate {t_validate:.0f} us")
        del model, logits
        torch.cuda.empty_cache()
    print(f"card: {card}")
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
