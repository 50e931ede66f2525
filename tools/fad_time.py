"""CUDA-event time of the Fréchet audio distance's device work (DESIGN.md §14): the VGGish embed per example and the
log-mel frontend, beside the fp32 torch composition of the same network with the same weights (conv2d / max_pool2d /
linear, what torchvggish runs), with achieved FLOP/s from the network's 1.73 GFLOP per example.

    python tools/fad_time.py [--batch 1 64 512] [--iters 10] [--out fad_time.json]

Seeded random weights (oracle/fad_oracle.random_state_dict); the card's name and power limit are printed with the
numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as Fn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import fad_oracle as fo  # noqa: E402
from vampnet_b200 import fad  # noqa: E402


def flops_per_example():
    f, H, W = 0, 96, 64
    for i, (ci, co) in fo.CONVS.items():
        f += 2 * H * W * co * 9 * ci
        if i in (0, 3, 8, 13):
            H, W = H // 2, W // 2
    return f + sum(2 * k * n for k, n in fo.FCS.values())


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(3):
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / iters)
    return float(np.median(times))


def torch_fp32(sd):
    w = {k: v.cuda().float() for k, v in sd.items()}

    def run(x):
        x = x[:, None]
        for i in (0, 3, 6, 8, 11, 13):
            x = Fn.relu(Fn.conv2d(x, w[f"features.{i}.weight"], w[f"features.{i}.bias"], padding=1))
            if i in (0, 3, 8, 13):
                x = Fn.max_pool2d(x, 2)
        x = x.permute(0, 2, 3, 1).reshape(x.shape[0], -1)
        x = Fn.relu(Fn.linear(x, w["embeddings.0.weight"], w["embeddings.0.bias"]))
        x = Fn.relu(Fn.linear(x, w["embeddings.2.weight"], w["embeddings.2.bias"]))
        return Fn.linear(x, w["embeddings.4.weight"], w["embeddings.4.bias"])
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 64, 512])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "fad_time measures on the GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd = fo.random_state_dict(1)
    model = fad.VGGish(sd, device="cuda")
    ref = torch_fp32(sd)
    gf = flops_per_example()
    res = {"card": card, "gflop_per_example": gf / 1e9, "embed": []}
    for n in a.batch:
        x = torch.from_numpy(np.concatenate([fo.examples(fo.test_signal(16000 * 10, s)) for s in range((n + 9) // 10)])[:n]).cuda()
        t = timed(lambda: model.embed(x), a.iters)
        tr = timed(lambda: ref(x), a.iters)
        diff = (model.embed(x) - ref(x)).abs().max().item()
        row = dict(batch=n, ms=t, us_per_example=1e3 * t / n, tflops=gf * n / (t * 1e-3) / 1e12, torch_fp32_ms=tr,
                   torch_fp32_us_per_example=1e3 * tr / n, speedup=tr / t, max_abs_diff_vs_torch=diff)
        res["embed"].append(row)
        print(json.dumps(row))
    x = torch.from_numpy(np.stack([fo.test_signal(16000 * 10, s) for s in range(64)])).cuda()
    t = timed(lambda: model.examples(x), a.iters)
    res["frontend"] = dict(rows=64, seconds_each=10, ms=t, us_per_10s_clip=1e3 * t / 64)
    print(card)
    print(json.dumps(res["frontend"]))
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
