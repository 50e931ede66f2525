"""CUDA-event time of each layer GEMM of the default benchmark workload (config [2]: B = 32, T = 768, d = 1280), run
through vnb_dbg_gemm_fused with the epilogues and fused-RMSNorm operands the forward gives them:

    python tools/gemm_time.py [--iters 50] [--out FILE]

QKV (row-scaled A, q/k plus transposed V), FFN-up (row-scaled A, GEGLU), attention-out and FFN-down (residual add, bf16
copy and sum-of-squares partials).  Each GEMM is warmed, then timed over --iters back-to-back launches between two
CUDA events, three times; the median is reported as us per launch and TFLOP/s (2 M N K flop).  The card's name, power
limit and SM clocks are read in the same run, right after the timing.
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

from tools import gemm_bits as GB  # noqa: E402

B, T, D = 32, 768, 1280
M = B * T


def shapes():
    """name -> (epilogue, N, K) of the four layer GEMMs"""
    from vampnet_b200 import _lib as L
    return {"qkv": (L.EPI_QKV, 3 * D, D), "attn_out": (L.EPI_RESID, D, D), "ffn_up": (L.EPI_GEGLU, 4 * D, D),
            "ffn_down": (L.EPI_RESID, D, 2 * D)}


def launcher(epi, N, K, seed):
    """A closure that launches one GEMM of this shape on fixed operands."""
    from vampnet_b200 import _lib as L
    A, W, g = GB.operands(M, N, K, seed)
    if epi == L.EPI_RESID:
        x = torch.randn(M, N, generator=g).cuda()
        y = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        ss_out = torch.empty(N // 128, M, device="cuda")
        return lambda: GB.gemm_fused(epi, A, W, x, out_bf16=y, ss_out=ss_out)
    ss, inv_d, _ = GB.row_stats(M, K, K // 128, g)
    if epi == L.EPI_QKV:
        Tpad = (T + 7) // 8 * 8
        qk = torch.empty(M, 2 * D, dtype=torch.bfloat16, device="cuda")
        vT = torch.empty(B, D, Tpad, dtype=torch.bfloat16, device="cuda")
        return lambda: GB.gemm_fused(epi, A, W, qk, vT, T=T, Tpad=Tpad, ss_in=ss, inv_d=inv_d)
    h = torch.empty(M, N // 2, dtype=torch.bfloat16, device="cuda")
    return lambda: GB.gemm_fused(epi, A, W, h, ss_in=ss, inv_d=inv_d)


def time_us(fn, iters, reps=3):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        out.append(1e3 * e0.elapsed_time(e1) / iters)
    return sorted(out)[len(out) // 2], out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    res = {"shape": dict(B=B, T=T, d=D, M=M), "gemms": {}}
    for i, (name, (epi, N, K)) in enumerate(shapes().items()):
        us, runs = time_us(launcher(epi, N, K, 1000 + i), a.iters)
        res["gemms"][name] = {"N": N, "K": K, "us": round(us, 2), "runs_us": [round(r, 2) for r in runs],
                              "tflops": round(2.0 * M * N * K / us * 1e-6, 1)}
    q = os.popen("nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv,noheader").read().strip()
    res["card"] = torch.cuda.get_device_name(0)
    res["nvidia_smi"] = q
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
