"""Nucleus (top-p) and plain-sampling requests in shared launches: Interface.vamp_many with and without
mixed_top_p=True on an app-shaped request mix.

    python tools/many_top_p.py [--requests 16] [--repeats 3] [--out result.json]

The app's "top p" slider is 0 (off) for most requests, so a real mix has both kinds.  Without mixed_top_p, vamp_many
buckets on top-p on/off: every coarse feedback pass of such a mix is two launches, and the top-p launch materialises
the fp32 logits of every position of every row.  With mixed_top_p=True the mix shares one launch: the classifier's split
epilogue draws the plain rows in place and stores logits only for the still-masked positions of the nucleus rows.

The requests are those of tools/many_requests.py --mixed-steps (the full-size coarse and c2f models at d = 1280 from
seeded weights, 5-30 s of seeded codes, batch_size=2, seeded coarse step counts from {12, 24, 36, 48, 64}); a seeded half
of them also take top_p from {0.8, 0.9, 0.95}, the rest None.  The arms,

  * iface.vamp_many(requests, mixed_lengths=True, mixed_steps=True) and
  * iface.vamp_many(requests, mixed_lengths=True, mixed_steps=True, mixed_top_p=True),

are each warmed once, then run `--repeats` times in alternating order with the global RNGs reseeded before every run;
every timed run ends in a device synchronise.  The two arms' outputs are compared bit for bit in every repeat (a
mismatch fails the run).  Also recorded: the generate launches per arm, the device time per kernel family of one
profiled run of each arm (vnb_profile_begin / end; graphs are bypassed while profiling), and the card's name, power
limit and maximum SM clock, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.many_requests import build_iface, card, family_times, make_requests, reseed, timed  # noqa: E402

TOP_P_CHOICES = (0.8, 0.9, 0.95)
ENTRIES = ("vnb_generate", "vnb_generate_many", "vnb_generate_many_adapted", "vnb_generate_ragged",
           "vnb_generate_steps", "vnb_generate_mixed_top_p")


def with_top_p(reqs, seed):
    """A seeded half of the requests get a top_p from TOP_P_CHOICES, the others None."""
    g = torch.Generator().manual_seed(seed)
    on = torch.randperm(len(reqs), generator=g)[:len(reqs) // 2].tolist()
    out = []
    for i, r in enumerate(reqs):
        r = dict(r)
        r["top_p"] = TOP_P_CHOICES[int(torch.randint(0, len(TOP_P_CHOICES), (1,), generator=g))] if i in on else None
        out.append(r)
    return out


class LaunchCount:
    """Counts the generate launches made through vampnet_b200._lib while installed, per entry point."""

    def __init__(self):
        from vampnet_b200 import _lib as L
        self.L, self.real, self.counts = L, L.lib, {}

    def __enter__(self):
        lib, counts = self.real(), self.counts

        class Spy:
            def __getattr__(self, name):
                fn = getattr(lib, name)
                if name not in ENTRIES:
                    return fn

                def counted(*a):
                    counts[name] = counts.get(name, 0) + 1
                    return fn(*a)
                return counted
        self.L.lib = lambda: Spy()
        return self

    def __exit__(self, *exc):
        self.L.lib = self.real


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    info = card()
    iface = build_iface()
    reqs = with_top_p(make_requests(iface, a.requests, a.seed, mixed_steps=True), a.seed + 1)
    runs = {"split_by_top_p": lambda: iface.vamp_many(reqs, mixed_lengths=True, mixed_steps=True),
            "mixed_top_p": lambda: iface.vamp_many(reqs, mixed_lengths=True, mixed_steps=True, mixed_top_p=True)}
    names = list(runs)
    for fn in runs.values():  # warm-up: workspaces, graph captures
        reseed(1)
        fn()
    times = {k: [] for k in runs}
    launches = {}
    identical = True
    for rep in range(a.repeats):
        outs = {}
        for name in names[rep % 2:] + names[:rep % 2]:
            reseed(1000 + rep)
            with LaunchCount() as c:
                outs[name], dt = timed(runs[name])
            launches[name] = c.counts
            times[name].append(dt)
        identical &= all(torch.equal(x, y) for x, y in zip(outs[names[0]], outs[names[1]]))
    med = {k: float(np.median(v)) for k, v in times.items()}
    res = {
        "card": info,
        "requests": a.requests, "frames": [r["codes"].shape[-1] for r in reqs], "batch_size": 2,
        "coarse_steps": [r["_sampling_steps"] for r in reqs], "top_p": [r["top_p"] for r in reqs], "c2f_steps": 2,
        "seconds": {k: [round(t, 4) for t in v] for k, v in times.items()},
        "median_s": {k: round(v, 4) for k, v in med.items()},
        "mixed_top_p_speedup": round(med["split_by_top_p"] / med["mixed_top_p"], 3),
        "generate_launches": launches,
        "bit_identical": bool(identical),
        "family_ms": {}, "family_launches": {},
    }
    for name in names:
        reseed(1)
        res["family_ms"][name], res["family_launches"][name] = family_times(iface, runs[name])
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    if not identical:
        sys.exit("vamp_many(mixed_top_p=True) differs from vamp_many without it")


if __name__ == "__main__":
    main()
