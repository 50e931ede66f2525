"""Bit-level record of the fused attention kernel (vnb_op_attention) on seeded inputs:

    python tools/attention_bits.py --write tests/golden/attention_bits.npz

Every case builds q, k, v and the bias table on the CPU from a fixed seed (as tests/test_gpu_attention.py does), runs
the library's attention on cuda:0 and stores the SHA-256 of the bf16 output plus a fixed seeded sample of its values
(for diagnosing a mismatch).  tests/test_gpu_attention_bits.py requires a build to reproduce every hash, so a change
to the kernel's schedule that alters any float operation or its order is caught bit for bit.

The cases cover the three bias regimes of a (2*sat+1)-entry table: sat = 1, sat = 91 (the table the real models use,
built from relative_position_bucket) and sat = 128 (the table of tests/test_gpu_attention.py); lengths below one key
block, exactly one, one plus a ragged one, the reference's 10 s chunk (575) and the benchmark's 768 and 3072; more
than one batch item and head; and the benchmark's full shapes (32, 768, 20) and (8, 3072, 20).
"""
from __future__ import annotations

import argparse
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

N_SAMPLE = 256  # sampled output values stored per case

# (B, T, H, sat)
CASES = [(B, T, H, sat) for sat in (1, 91, 128)
         for (B, T, H) in ((2, 3, 2), (1, 64, 2), (2, 65, 3), (3, 575, 4), (2, 768, 4), (2, 1000, 2), (1, 3072, 2))]
CASES += [(32, 768, 20, sat) for sat in (91, 128)] + [(8, 3072, 20, sat) for sat in (91, 128)]


def case_name(B, T, H, sat):
    return f"B{B}_T{T}_H{H}_sat{sat}"


def make_inputs(B, T, H, sat, seed):
    """q, k, v (B, T, H*64) bf16 and the (2*sat+1, H) fp32 bias table on the CPU, then the kernel's operand layouts
    on cuda:0: qk = [q | k] (B, T, 2d) and v^T (B, d, Tpad) zero-padded to Tpad = T rounded up to 8."""
    d = H * 64
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, T, d, generator=g).bfloat16() for _ in range(3))
    if sat == 128:      # tests/test_gpu_attention.py's table: constant beyond distance 92 on both sides
        rel = torch.randn(2 * sat + 1, H, generator=g) * 0.5
        rel[:36] = rel[36]
        rel[-36:] = rel[-37]
    elif sat == 91:     # the real models' table: one weight per T5 bucket (32 buckets, max_distance 128)
        from vampnet_b200.modules.transformer import relative_position_bucket
        w = torch.randn(32, H, generator=g) * 0.5
        rel = w[relative_position_bucket(torch.arange(-sat, sat + 1))]
    else:
        rel = torch.randn(2 * sat + 1, H, generator=g) * 0.5
    Tpad = (T + 7) // 8 * 8
    qk = torch.cat([q, k], dim=-1).contiguous().cuda()
    vT = torch.zeros(B, d, Tpad, dtype=torch.bfloat16)
    vT[:, :, :T] = v.permute(0, 2, 1)
    return qk, vT.cuda(), rel.contiguous().cuda(), Tpad


def run_case(B, T, H, sat):
    """The kernel's output for one case as a CPU bf16 tensor."""
    from vampnet_b200 import _lib as L
    seed = 1000 * sat + T + B + H
    qk, vT, rel, Tpad = make_inputs(B, T, H, sat, seed)
    out = torch.full((B, T, H * 64), float("nan"), device="cuda", dtype=torch.bfloat16)
    L.check(L.lib().vnb_op_attention(L.ptr(qk), L.ptr(vT), L.ptr(out), L.ptr(rel), sat, B, T, Tpad, H, L.stream_ptr()))
    torch.cuda.synchronize()
    return out.cpu()


def digest(out):
    return hashlib.sha256(out.contiguous().view(torch.int16).numpy().tobytes()).hexdigest()


def sample_index(n, name):
    g = np.random.default_rng(int(hashlib.sha256(name.encode()).hexdigest()[:8], 16))
    return np.sort(g.choice(n, size=min(N_SAMPLE, n), replace=False))


def record():
    rec = {}
    for case in CASES:
        name = case_name(*case)
        out = run_case(*case)
        flat = out.float().reshape(-1).numpy()
        rec["sha256_" + name] = np.array(digest(out))
        rec["sample_" + name] = flat[sample_index(flat.size, name)]
        print(f"{name}: {rec['sha256_' + name]}", flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--write", metavar="NPZ", required=True, help="where to store the hashes and samples")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    rec = record()
    dev = torch.cuda.get_device_properties(0)
    rec["device"] = np.array(dev.name)
    os.makedirs(os.path.dirname(os.path.abspath(args.write)), exist_ok=True)
    np.savez_compressed(args.write, **rec)
    print(f"wrote {len(CASES)} cases to {args.write}")


if __name__ == "__main__":
    main()
