"""Throughput of an app-shaped request mix: sequential Interface.vamp() calls against one Interface.vamp_many(), with and
without mixed-length launches.

    python tools/many_requests.py [--requests 16] [--repeats 3] [--out result.json]

The app serves one vamp(batch_size=2) per request; a 10 s coarse chunk at B = 2 is M = 1150 GEMM rows, far below the
batches the kernels are tuned at.  vamp_many runs every request's chunks stage by stage through generate_many, so
chunks of equal length share a launch; with mixed_lengths=True chunks of any length do, padded to the launch's longest.  This script builds the full-size coarse (20 layers) and c2f (16 layers)
models at d = 1280 from seeded random weights, makes `--requests` requests of 5-30 s of seeded codes with a periodic
prompt mask, batch_size=2, 36 coarse sampling steps (the UI default) and the pinned 2-step fine stage, and times

  * the sequential loop [iface.vamp(**r) for r in requests],
  * iface.vamp_many(requests), and
  * iface.vamp_many(requests, mixed_lengths=True),

each warmed once, then run `--repeats` times in rotating order with the global RNGs reseeded before every run.  Every
timed run ends in a device synchronise.  The outputs of the three arms are compared bit for bit in every repeat; a
mismatch fails the run.  Per arm and timed run it also records the generate graphs captured
(vnb_graph_capture_count), the generate launches, and the fraction of GEMM rows (batch rows x launch T) that are
padding.  The card's name, power limit and maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

COARSE = dict(n_heads=20, n_layers=20, n_codebooks=4, n_conditioning_codebooks=0, embedding_dim=1280)
C2F = dict(n_heads=20, n_layers=16, n_codebooks=14, n_conditioning_codebooks=4, embedding_dim=1280)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def build_iface():
    import types
    from oracle import vampnet_oracle as vo
    from vampnet_b200.interface import Interface
    from vampnet_b200.modules.transformer import VampNet
    cb = vo.make_codebooks(14, seed=1).cuda()
    codec = types.SimpleNamespace(
        quantizer=types.SimpleNamespace(quantizers=[types.SimpleNamespace(codebook=types.SimpleNamespace(weight=cb[i]))
                                                    for i in range(14)]),
        sample_rate=44100, hop_length=768, to=lambda device: codec)
    models = []
    for seed, cfg in ((0, COARSE), (1, C2F)):
        m = VampNet(**cfg)
        m.load_state_dict(vo.make_state_dict(vo.OracleConfig(**cfg), seed=seed), strict=False)
        models.append(m)
    return Interface.from_models(codec, models[0], models[1], device="cuda")


def make_requests(iface, n, seed):
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for _ in range(n):
        secs = 5 + 25 * torch.rand(1, generator=g).item()
        T = iface.s2t(secs)
        z = torch.randint(0, 1024, (1, 14, T), generator=g)
        mask = torch.ones_like(z)
        mask[:, :, ::7] = 0          # periodic prompt
        mask[:, 3:, :] = 1           # codebooks >= 3 always regenerated
        reqs.append(dict(codes=z.cuda(), mask=mask.cuda(), batch_size=2, _sampling_steps=36, return_mask=False))
    return reqs


def reseed(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


class LaunchTally:
    """Counts the generate launches made through vampnet_b200._lib while installed, with their GEMM rows (B x T) and
    how many of those rows are padding (vnb_generate_ragged: rows of a call past its own frames)."""
    NAMES = ("vnb_generate", "vnb_generate_many", "vnb_generate_many_adapted", "vnb_generate_ragged")

    def __init__(self):
        from vampnet_b200 import _lib as L
        self.L, self.real = L, L.lib
        self.launches = self.rows = self.pad_rows = 0

    def __enter__(self):
        lib, tally = self.real(), self

        class Spy:
            def __getattr__(self, name):
                fn = getattr(lib, name)
                if name not in LaunchTally.NAMES:
                    return fn

                def counted(*a):
                    B, T = a[3], a[4]
                    tally.launches += 1
                    tally.rows += B * T
                    if name == "vnb_generate_ragged" and a[9] is not None:
                        tally.pad_rows += sum(a[7][g].rows * (T - a[9][g]) for g in range(a[8]))
                    return fn(*a)
                return counted
        self.L.lib = lambda: Spy()
        return self

    def __exit__(self, *exc):
        self.L.lib = self.real


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    iface = build_iface()
    reqs = make_requests(iface, a.requests, a.seed)
    frames = [r["codes"].shape[-1] for r in reqs]
    from vampnet_b200 import _lib as L
    runs = {"sequential": lambda: [iface.vamp(**r) for r in reqs], "vamp_many": lambda: iface.vamp_many(reqs),
            "vamp_many_mixed": lambda: iface.vamp_many(reqs, mixed_lengths=True)}
    names = list(runs)
    warm_captures = {}
    for name, fn in runs.items():  # warm-up: workspaces, graph captures
        reseed(1)
        c0 = L.lib().vnb_graph_capture_count()
        fn()
        warm_captures[name] = int(L.lib().vnb_graph_capture_count() - c0)
    times = {k: [] for k in runs}
    captures = {k: [] for k in runs}
    tallies = {}
    identical = True
    for rep in range(a.repeats):
        outs = {}
        for name in names[rep % len(names):] + names[:rep % len(names)]:
            reseed(1000 + rep)
            c0 = L.lib().vnb_graph_capture_count()
            with LaunchTally() as t:
                outs[name], dt = timed(runs[name])
            captures[name].append(int(L.lib().vnb_graph_capture_count() - c0))
            tallies[name] = t
            times[name].append(dt)
        for name in names[1:]:
            identical &= all(torch.equal(x, y) for x, y in zip(outs["sequential"], outs[name]))
    tokens = 2 * sum(frames)  # batch_size 2 per request
    res = {
        "card": card(),
        "requests": a.requests, "frames": frames, "batch_size": 2, "coarse_steps": 36, "c2f_steps": 2,
        "seconds": {k: [round(t, 4) for t in v] for k, v in times.items()},
        "median_s": {k: round(float(np.median(v)), 4) for k, v in times.items()},
        "tokens_per_s": {k: round(tokens / float(np.median(v)), 1) for k, v in times.items()},
        "speedup_median": round(float(np.median(times["sequential"]) / np.median(times["vamp_many"])), 3),
        "speedup_median_mixed": round(float(np.median(times["sequential"]) / np.median(times["vamp_many_mixed"])), 3),
        "mixed_vs_vamp_many": round(float(np.median(times["vamp_many"]) / np.median(times["vamp_many_mixed"])), 3),
        "graph_captures_warmup": warm_captures,
        "graph_captures_timed": captures,
        "generate_launches": {k: t.launches for k, t in tallies.items()},
        "gemm_rows": {k: t.rows for k, t in tallies.items()},
        "padding_row_fraction": {k: round(t.pad_rows / max(t.rows, 1), 4) for k, t in tallies.items()},
        "bit_identical": bool(identical),
    }
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    if not identical:
        sys.exit("vamp_many differs from the sequential vamp calls")


if __name__ == "__main__":
    main()
