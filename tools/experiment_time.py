"""Throughput of the experiment script's gen-compression conditions: the sequential condition functions against
vampnet_b200.experiment.run_experiment, on blocks of 10 s excerpts.

    python tools/experiment_time.py [--blocks 8 32] [--repeats 2] [--out result.json]

Builds the shipped shapes from seeded random weights: the coarse (20 layers) and c2f (16 layers) models at d = 1280 and
the codec (encoder 64, decoder 1536, hop 768, 14 codebooks).  The excerpts are 10 s of seeded noise under a click every
half second at 44.1 kHz (the coarse chunk, as the script's dataset cuts them).  For each block size the two arms are
warmed once, then run `--repeats` times in alternating order with the global RNGs reseeded before every run, each timed
run ending in a device synchronise.  Their audio is compared bit for bit in every repeat; a mismatch fails the run.  Per
arm it records excerpts/s, the generate launches made through vampnet_b200._lib and the codec's encoder and decoder
launches.  The card's name, power limit and maximum SM clock are read in the same run.
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
GENERATE = ("vnb_generate_many", "vnb_generate_many_adapted", "vnb_generate_ragged", "vnb_generate_steps",
            "vnb_generate_mixed_top_p")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def build_iface():
    from oracle import dac_oracle as do
    from oracle import vampnet_oracle as vo
    from vampnet_b200.codec import DAC
    from vampnet_b200.interface import Interface
    from vampnet_b200.modules.transformer import VampNet
    cfg = do.CodecConfig()
    codec = DAC(encoder_dim=cfg.encoder_dim, encoder_rates=cfg.encoder_rates, decoder_dim=cfg.decoder_dim)
    codec.load_flat(do.make_codec_weights(cfg, seed=0))
    models = []
    for seed, c in ((0, COARSE), (1, C2F)):
        m = VampNet(**c)
        m.load_state_dict(vo.make_state_dict(vo.OracleConfig(**c), seed=seed), strict=False)
        models.append(m)
    return Interface.from_models(codec, models[0], models[1], device="cuda")


def excerpts(n, seed=0):
    from vampnet_b200.audio import AudioSignal
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        x = 0.05 * torch.randn(441000, generator=g)
        x[::22050] += 0.9
        out.append(AudioSignal(x[None, None].cuda(), 44100))
    return out


def reseed(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


class Tally:
    """Counts generate launches through vampnet_b200._lib and the codec's encoder / decoder launches while installed."""

    def __init__(self, iface):
        from vampnet_b200 import _lib as L
        self.L, self.real, self.codec = L, L.lib, iface.codec
        self.generate = self.encode = self.decode = 0

    def __enter__(self):
        lib, tally = self.real(), self

        class Spy:
            def __getattr__(self, name):
                fn = getattr(lib, name)
                if name not in GENERATE:
                    return fn

                def counted(*a):
                    tally.generate += 1
                    return fn(*a)
                return counted
        self.L.lib = lambda: Spy()
        c = self.codec
        enc, dec, enc1, dec1 = c._encode_launch, c._decode_launch, c.encode, c.decode

        def count(fn, attr):
            def counted(*a, **k):
                setattr(tally, attr, getattr(tally, attr) + 1)
                return fn(*a, **k)
            return counted
        c._encode_launch, c.encode = count(enc, "encode"), count(enc1, "encode")
        c._decode_launch, c.decode = count(dec, "decode"), count(dec1, "decode")
        return self

    def __exit__(self, *exc):
        self.L.lib = self.real
        for name in ("_encode_launch", "_decode_launch", "encode", "decode"):
            del self.codec.__dict__[name]


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--exp_type", default="gen-compression")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from vampnet_b200 import experiment as ex
    iface = build_iface()
    conds = ex.conditions(a.exp_type)
    res = {"card": card(), "exp_type": a.exp_type, "conditions": list(conds), "excerpt_s": 10.0, "blocks": {}}
    identical = True
    for n in a.blocks:
        sigs = excerpts(n)

        def sequential():
            out = {name: [] for name in conds}
            for s in sigs:
                for name, cond in conds.items():
                    out[name].append(cond(s, iface))
            return out
        runs = {"sequential": sequential, "batched": lambda: ex.run_experiment(iface, sigs, a.exp_type, block_size=n)}
        for fn in runs.values():  # warm-up: workspaces, graph captures, tables
            reseed(1)
            fn()
        times, tallies = {k: [] for k in runs}, {}
        for rep in range(a.repeats):
            outs = {}
            for name in (list(runs) if rep % 2 == 0 else list(runs)[::-1]):
                reseed(100 + rep)
                with Tally(iface) as t:
                    outs[name], dt = timed(runs[name])
                times[name].append(dt)
                tallies[name] = t
            identical &= all(torch.equal(x.audio_data, y.audio_data)
                             for c in conds for x, y in zip(outs["sequential"][c], outs["batched"][c]))
            del outs
        med = {k: float(np.median(v)) for k, v in times.items()}
        res["blocks"][n] = {
            "seconds": {k: [round(t, 3) for t in v] for k, v in times.items()},
            "median_s": {k: round(v, 3) for k, v in med.items()},
            "excerpts_per_s": {k: round(n / v, 3) for k, v in med.items()},
            "speedup": round(med["sequential"] / med["batched"], 3),
            "generate_launches": {k: t.generate for k, t in tallies.items()},
            "encoder_launches": {k: t.encode for k, t in tallies.items()},
            "decoder_launches": {k: t.decode for k, t in tallies.items()},
        }
        print(json.dumps({n: res["blocks"][n]}), flush=True)
    res["bit_identical"] = bool(identical)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    if not identical:
        sys.exit("run_experiment differs from the sequential condition functions")


if __name__ == "__main__":
    main()
