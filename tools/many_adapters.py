"""Mixed fine-tune traffic: one Interface.vamp_many() with per-request adapters against the per-model loop.

    python tools/many_adapters.py [--requests 16] [--repeats 3] [--out result.json]

The request mix is tools/many_requests.py's (5-30 s, batch_size=2, 36 coarse steps, the pinned 2-step fine stage) on the
same seeded full-size coarse (20 layers) and c2f (16 layers) models at d = 1280, spread round-robin over the base model
and four fine-tunes of it with seeded random rank-8 LoRA on w_qs, w_vs, fc, w_1 and w_2.  Two paths serve it:

  * loop: for each model (base, ft0 .. ft3) a hot swap of both models to it (load_state_dict of the fine-tune's state
    dict, held in memory: the swap re-folds LoRA and rewrites the packed weights in place; reading a checkpoint from disk,
    which the app also does, is not included), then one vamp_many of that model's requests;
  * adapters: the four fine-tunes registered once as adapters (VampNet.add_adapter on both models, from the same
    in-memory state dicts), then one vamp_many of all requests with adapter=name.

Each path has its own pair of models.  Both are warmed once, then alternated `--repeats` times with the global RNGs
reseeded before every run; every timed run ends in a device synchronise.  The two paths do not give the same tokens
(a folded fine-tune rounds W + BA to bf16; an adapter adds the update to the accumulator), so only times are compared.
The card's name, power limit and maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.many_requests import build_iface, card, make_requests, reseed, timed  # noqa: E402

N_FINETUNES = 4


def lora_tensors(model, seed):
    """Seeded random LoRA of one fine-tune of `model` (make_state_dict's scales)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, p in model.named_parameters():
        if name.endswith("lora_A"):
            out[name] = torch.randn(p.shape, generator=g) / math.sqrt(p.shape[1])
        elif name.endswith("lora_B"):
            out[name] = torch.randn(p.shape, generator=g) * 0.05
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    loop_iface, ad_iface = build_iface(), build_iface()
    names = [None] + [f"ft{i}" for i in range(N_FINETUNES)]
    base = {tag: {k: v.detach().cpu().clone() for k, v in m.state_dict().items() if ".lora_" not in k}
            for tag, m in (("coarse", loop_iface.coarse), ("c2f", loop_iface.c2f))}
    loras = {tag: {n: lora_tensors(m, 1 + 10 * i + (tag == "c2f")) for i, n in enumerate(names[1:])}
             for tag, m in (("coarse", loop_iface.coarse), ("c2f", loop_iface.c2f))}
    zero = {tag: {k: torch.zeros_like(v) for k, v in loras[tag]["ft0"].items() if k.endswith("lora_B")}
            for tag in loras}
    for n in names[1:]:  # what Interface.add_finetuned(n) does with loras/<n>/{coarse,c2f}.pth, from memory
        ad_iface.coarse.add_adapter(n, {**base["coarse"], **loras["coarse"][n]})
        ad_iface.c2f.add_adapter(n, {**base["c2f"], **loras["c2f"][n]})

    reqs = make_requests(loop_iface, a.requests, a.seed)
    for i, r in enumerate(reqs):
        r["adapter"] = names[i % len(names)]
    frames = [r["codes"].shape[-1] for r in reqs]

    def run_loop():
        out = []
        for n in names:
            for tag, m in (("coarse", loop_iface.coarse), ("c2f", loop_iface.c2f)):
                m.load_state_dict({**base[tag], **(zero[tag] if n is None else loras[tag][n])}, strict=False)
            mine = [{k: v for k, v in r.items() if k != "adapter"} for r in reqs if r["adapter"] == n]
            out += loop_iface.vamp_many(mine)
        return out

    runs = {"loop": run_loop, "adapters": lambda: ad_iface.vamp_many(reqs)}
    for fn in runs.values():  # warm-up: workspaces, graph captures
        reseed(1)
        fn()
    times = {k: [] for k in runs}
    for rep in range(a.repeats):
        for name in (("loop", "adapters") if rep % 2 == 0 else ("adapters", "loop")):
            reseed(1000 + rep)
            _, dt = timed(runs[name])
            times[name].append(dt)
    tokens = 2 * sum(frames)
    res = {
        "card": card(),
        "requests": a.requests, "frames": frames, "models": [n or "base" for n in names],
        "request_model": [r["adapter"] or "base" for r in reqs], "batch_size": 2, "coarse_steps": 36, "c2f_steps": 2,
        "seconds": {k: [round(t, 4) for t in v] for k, v in times.items()},
        "median_s": {k: round(float(np.median(v)), 4) for k, v in times.items()},
        "tokens_per_s": {k: round(tokens / float(np.median(v)), 1) for k, v in times.items()},
        "speedup_median": round(float(np.median(times["loop"]) / np.median(times["adapters"])), 3),
    }
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
