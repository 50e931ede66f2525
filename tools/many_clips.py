"""Codec time of an app-shaped request mix: clips coded one request at a time against DAC.encode_many / decode_many,
alone and inside the whole request path.

    python tools/many_clips.py [--requests 16] [--repeats 3] [--steps 36] [--out result.json]

An app request (reference app.py:175-264) starts and ends as audio: encode one clip, build a mask, vamp(batch_size=2),
decode the two result rows.  This script makes `--requests` seeded clips of 5-30 s at 44.1 kHz (the mix of
tools/many_requests.py), builds the full-size codec (encoder 64 .. 1024, decoder 1536 .. 96) and, for the second pair
of arms, the full-size coarse (20 layers) and c2f (16 layers) models at d = 1280, all from seeded random weights, and
times

  codec:       [iface.encode(s) for s in signals] + [iface.decode(z) for z in codes x 2 rows]
               against iface.encode_many(signals) + iface.decode_many(codes x 2 rows);
  end to end:  per request encode -> build_mask -> vamp(batch_size=2, `--steps` coarse steps) -> decode
               against encode_many -> build_mask per request -> vamp_many(mixed_lengths=True, mixed_steps=True)
               -> decode_many.

Masks are built with torch's RNG reseeded per request and every request carries its own generate seed, so both paths
draw the same masks and keys.  Each arm is warmed once, then the two arms of a pair alternate `--repeats` times; every
timed run ends in a device synchronise, and the outputs of the two arms are compared bit for bit in every repeat (a
mismatch fails the run).  Per arm it records the kernel launches of one run (vnb_launch_count) and, for the many-clip
arms, the padding samples of the launches (rows x launch length minus the rows' own lengths).  The card's name, power
limit and SM clocks are read in the same run, before and after the timed runs.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.many_requests import C2F, COARSE  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def build_iface(with_models: bool):
    from oracle import vampnet_oracle as vo
    from tools.codec_bits import full_codec
    from vampnet_b200.interface import Interface
    from vampnet_b200.modules.transformer import VampNet
    codec = full_codec(seed=0)[2]
    models = []
    for seed, cfg in ((0, COARSE), (1, C2F)):
        m = VampNet(**(cfg if with_models else dict(cfg, n_layers=1, n_heads=4, embedding_dim=256)))
        if with_models:
            m.load_state_dict(vo.make_state_dict(vo.OracleConfig(**cfg), seed=seed), strict=False)
        models.append(m)
    return Interface.from_models(codec, models[0], models[1], device="cuda")


def make_signals(n, seed):
    from vampnet_b200.audio import AudioSignal
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        secs = 5 + 25 * torch.rand(1, generator=g).item()
        out.append(AudioSignal((torch.randn(1, 1, int(44100 * secs), generator=g) * 0.3).cuda(), 44100))
    return out


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def launches(fn):
    from vampnet_b200 import _lib
    n0 = _lib.lib().vnb_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return int(_lib.lib().vnb_launch_count() - n0), out


def padding(lengths, budget):
    from vampnet_b200.codec import plan_launches
    plan = plan_launches(lengths, budget)
    return sum(len(p) * lengths[p[0]] - sum(lengths[k] for k in p) for p in plan), len(plan)


def flat(x):
    """Every tensor of a nested result, as int32 bit patterns (AudioSignals by their samples)."""
    if isinstance(x, (list, tuple)):
        return [t for y in x for t in flat(y)]
    if hasattr(x, "audio_data"):
        x = x.audio_data
    return [x.contiguous().view(torch.int32) if x.dtype == torch.float32 else x]


def same(a, b):
    fa, fb = flat(a), flat(b)
    return len(fa) == len(fb) and all(x.shape == y.shape and torch.equal(x, y) for x, y in zip(fa, fb))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=36)
    ap.add_argument("--codec-only", action="store_true", help="skip the end-to-end pair (no transformer models)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from vampnet_b200.codec import CODEC_MANY_MAX_SAMPLES
    res = {"card_before": card(), "requests": args.requests, "repeats": args.repeats, "steps": args.steps}
    iface = build_iface(with_models=not args.codec_only)
    signals = make_signals(args.requests, seed=0)
    hop = iface.codec.hop_length
    samples = [-(-s.signal_length // hop) * hop for s in signals]
    res["clip_seconds"] = [round(s.signal_length / 44100, 2) for s in signals]

    # ---- codec pair
    codes = [iface.encode(s) for s in signals]
    pairs = [c.expand(2, -1, -1).contiguous() for c in codes]     # what decode sees after vamp(batch_size=2)
    arms = {
        "codec_loop": lambda: ([iface.encode(s) for s in signals], [iface.decode(z) for z in pairs]),
        "codec_many": lambda: (iface.encode_many(signals), iface.decode_many(pairs)),
    }
    enc_pad, enc_launches = padding(samples, CODEC_MANY_MAX_SAMPLES)
    dec_pad, dec_launches = padding([n for n in samples for _ in range(2)], CODEC_MANY_MAX_SAMPLES)
    res["codec_many_plan"] = {"encode_launches": enc_launches, "encode_padding_samples": enc_pad,
                              "encode_samples": sum(samples), "decode_launches": dec_launches,
                              "decode_padding_samples": dec_pad, "decode_samples": 2 * sum(samples)}

    # ---- end-to-end pair
    def mask_for(i, z):
        torch.manual_seed(1000 + i)
        return iface.build_mask(z, periodic_prompt=7, upper_codebook_mask=3)

    def e2e_loop():
        out = []
        for i, s in enumerate(signals):
            z = iface.encode(s)
            zv = iface.vamp(z, mask_for(i, z), batch_size=2, _sampling_steps=args.steps, seed=i + 1)
            out.append(iface.decode(zv))
        return out

    def e2e_many():
        zs = iface.encode_many(signals)
        reqs = [dict(codes=z, mask=mask_for(i, z), batch_size=2, _sampling_steps=args.steps, seed=i + 1)
                for i, z in enumerate(zs)]
        return iface.decode_many(iface.vamp_many(reqs, mixed_lengths=True, mixed_steps=True))

    if not args.codec_only:
        arms["e2e_loop"], arms["e2e_many"] = e2e_loop, e2e_many
    names = list(arms)
    res["launches"], res["seconds"], ref = {}, {k: [] for k in names}, {}
    for k in names:                                                 # warm, count launches, keep the reference
        res["launches"][k], ref[k] = launches(arms[k])
    for a, b in (("codec_loop", "codec_many"), ("e2e_loop", "e2e_many")):
        if a in ref:
            assert same(ref[a], ref[b]), f"{a} and {b} differ"
    for r in range(args.repeats):
        for pair in (("codec_loop", "codec_many"), ("e2e_loop", "e2e_many")):
            for k in (pair if r % 2 == 0 else pair[::-1]):
                if k not in arms:
                    continue
                t, out = timed(arms[k])
                assert same(out, ref[k.replace("_many", "_loop")]), f"{k} differs from the loop in repeat {r}"
                res["seconds"][k].append(round(t, 4))
    res["median_seconds"] = {k: statistics.median(v) for k, v in res["seconds"].items()}
    res["card_after"] = card()
    res["bit_identical"] = True
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
