"""Throughput of an app-shaped request mix: sequential Interface.vamp() calls against one Interface.vamp_many(), with and
without mixed-length launches.

    python tools/many_requests.py [--requests 16] [--repeats 3] [--mixed-steps] [--out result.json]

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

--mixed-steps: every request draws its coarse sampling steps (seeded) from {12, 24, 36, 48, 64}, and the arms are the
sequential loop, iface.vamp_many(requests, mixed_lengths=True) and iface.vamp_many(requests, mixed_lengths=True,
mixed_steps=True).  The run also records the device time per kernel family of one profiled run of each vamp_many arm
(vnb_profile_begin / end; graphs are bypassed while profiling), and times one coarse launch of two B = 2, T = 575 calls
of 48 and 12 steps (generate_many(mixed_steps=True)) against the two calls launched one by one.
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


STEP_CHOICES = (12, 24, 36, 48, 64)


def make_requests(iface, n, seed, mixed_steps=False):
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for _ in range(n):
        secs = 5 + 25 * torch.rand(1, generator=g).item()
        T = iface.s2t(secs)
        z = torch.randint(0, 1024, (1, 14, T), generator=g)
        mask = torch.ones_like(z)
        mask[:, :, ::7] = 0          # periodic prompt
        mask[:, 3:, :] = 1           # codebooks >= 3 always regenerated
        steps = 36
        if mixed_steps:
            steps = STEP_CHOICES[int(torch.randint(0, len(STEP_CHOICES), (1,), generator=g))]
        reqs.append(dict(codes=z.cuda(), mask=mask.cuda(), batch_size=2, _sampling_steps=steps, return_mask=False))
    return reqs


def reseed(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


class LaunchTally:
    """Counts the generate launches made through vampnet_b200._lib while installed, with their GEMM rows (B x T) and
    how many of those rows are padding (vnb_generate_ragged: rows of a call past its own frames)."""
    NAMES = ("vnb_generate", "vnb_generate_many", "vnb_generate_many_adapted", "vnb_generate_ragged",
             "vnb_generate_steps")

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
                    if name in ("vnb_generate_ragged", "vnb_generate_steps") and a[9] is not None:
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


def family_times(iface, fn):
    """Device ms and launches per kernel family, summed over both models, of one profiled run of fn."""
    import ctypes as C
    from vampnet_b200 import _lib as L
    n = len(L.FAMILIES) + 1
    handles = [iface.coarse._handle, iface.c2f._handle]
    for h in handles:
        L.check(L.lib().vnb_profile_begin(h))
    fn()
    torch.cuda.synchronize()
    names = list(L.FAMILIES) + ["lora_down"]
    ms, cnt = dict.fromkeys(names, 0.0), dict.fromkeys(names, 0)
    for h in handles:
        t, k = (C.c_float * n)(), (C.c_int32 * n)()
        L.check(L.lib().vnb_profile_end(h, t, k, n))
        for i, name in enumerate(names):
            ms[name] += t[i]
            cnt[name] += k[i]
    return {k: round(v, 2) for k, v in ms.items() if cnt[k]}, {k: v for k, v in cnt.items() if v}


def pair_launch(iface, repeats=5):
    """One coarse launch of a 48-step and a 12-step call (B = 2, T = 575 each) against the two launched alone."""
    g = torch.Generator().manual_seed(5)
    model, codec = iface.coarse, iface.codec

    def call(steps, seed):
        z = torch.randint(0, 1024, (2, 4, 575), generator=g).cuda()
        mask = (torch.rand(2, 4, 575, generator=g) < 0.7).long().cuda()
        return dict(start_tokens=z, mask=mask, _sampling_steps=steps, seed=seed, return_signal=False)
    c48, c12 = call(48, 1), call(12, 2)
    arms = {"mixed_48_12": lambda: model.generate_many(codec, [c48, c12], mixed_steps=True),
            "alone_48": lambda: [model.generate(codec, **c48)], "alone_12": lambda: [model.generate(codec, **c12)]}
    times, outs = {}, {}
    for name, fn in arms.items():
        fn()
        ts = []
        for _ in range(repeats):
            o, dt = timed(fn)
            ts.append(dt)
        outs[name], times[name] = o, ts
    med = {k: round(float(np.median(v)) * 1e3, 2) for k, v in times.items()}
    return {"ms": {k: [round(t * 1e3, 2) for t in v] for k, v in times.items()}, "median_ms": med,
            "separate_sum_ms": round(med["alone_48"] + med["alone_12"], 2),
            "extra_over_alone_48_ms": round(med["mixed_48_12"] - med["alone_48"], 2),
            "bit_identical": bool(torch.equal(outs["mixed_48_12"][0], outs["alone_48"][0]) and
                                  torch.equal(outs["mixed_48_12"][1], outs["alone_12"][0]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--mixed-steps", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    iface = build_iface()
    reqs = make_requests(iface, a.requests, a.seed, a.mixed_steps)
    frames = [r["codes"].shape[-1] for r in reqs]
    from vampnet_b200 import _lib as L
    if a.mixed_steps:
        runs = {"sequential": lambda: [iface.vamp(**r) for r in reqs],
                "vamp_many_mixed": lambda: iface.vamp_many(reqs, mixed_lengths=True),
                "vamp_many_mixed_steps": lambda: iface.vamp_many(reqs, mixed_lengths=True, mixed_steps=True)}
    else:
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
    med = {k: float(np.median(v)) for k, v in times.items()}
    res = {
        "card": card(),
        "requests": a.requests, "frames": frames, "batch_size": 2,
        "coarse_steps": [r["_sampling_steps"] for r in reqs] if a.mixed_steps else 36, "c2f_steps": 2,
        "seconds": {k: [round(t, 4) for t in v] for k, v in times.items()},
        "median_s": {k: round(v, 4) for k, v in med.items()},
        "tokens_per_s": {k: round(tokens / v, 1) for k, v in med.items()},
        "graph_captures_warmup": warm_captures,
        "graph_captures_timed": captures,
        "generate_launches": {k: t.launches for k, t in tallies.items()},
        "gemm_rows": {k: t.rows for k, t in tallies.items()},
        "padding_row_fraction": {k: round(t.pad_rows / max(t.rows, 1), 4) for k, t in tallies.items()},
        "bit_identical": bool(identical),
    }
    if a.mixed_steps:
        res["speedup_median"] = {k: round(med["sequential"] / v, 3) for k, v in med.items() if k != "sequential"}
        res["mixed_steps_vs_mixed"] = round(med["vamp_many_mixed"] / med["vamp_many_mixed_steps"], 3)
        res["family_ms"], res["family_launches"] = {}, {}
        for name in ("vamp_many_mixed", "vamp_many_mixed_steps"):
            reseed(1)
            res["family_ms"][name], res["family_launches"][name] = family_times(iface, runs[name])
        res["pair_launch_48_12"] = pair_launch(iface)
        identical &= res["pair_launch_48_12"]["bit_identical"]
        res["bit_identical"] = bool(identical)
    else:
        res["speedup_median"] = round(med["sequential"] / med["vamp_many"], 3)
        res["speedup_median_mixed"] = round(med["sequential"] / med["vamp_many_mixed"], 3)
        res["mixed_vs_vamp_many"] = round(med["vamp_many"] / med["vamp_many_mixed"], 3)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    if not identical:
        sys.exit("vamp_many differs from the sequential vamp calls")


if __name__ == "__main__":
    main()
