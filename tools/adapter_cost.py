"""What per-request adapters cost at a benchmarked generate shape: the coarse generate of BASELINE.json configs[2]
(full-size coarse model, 20 layers, d = 1280, T = 768, B = 32, 12 sampling steps), as 16 generate_many calls of B = 2,
with no adapter and with every call adapted (four seeded random rank-8 fine-tunes, round-robin).

    python tools/adapter_cost.py [--repeats 5] [--out result.json]

* ms per sampling step: one graph-replayed generate_many per run, warmed, the two variants alternated `--repeats`
  times; host clock around work that ends in a device synchronise.
* the per-family device time of one run of each variant with vnb_profile_begin/end (CUDA events around every launch,
  graph replay bypassed; a separate run from the timed ones): the LoRA down-projections' share, and the LoRA'd GEMM
  families (QKV, attention out, FFN up, FFN down) adapted against plain.
The card's name, power limit and clocks are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.many_requests import COARSE, card  # noqa: E402

B_CALL, N_CALLS, T, STEPS = 2, 16, 768, 12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from oracle import vampnet_oracle as vo
    from tests.test_gpu_parity import StubCodec
    from vampnet_b200 import _lib as L
    from vampnet_b200.modules.transformer import VampNet
    sd = vo.make_state_dict(vo.OracleConfig(**COARSE), seed=0)
    model = VampNet(**COARSE)
    model.load_state_dict(sd, strict=False)
    model = model.to("cuda")
    for i in range(4):
        g = torch.Generator().manual_seed(1 + i)
        lora = {}
        for name, p in model.named_parameters():
            if name.endswith("lora_A"):
                lora[name] = torch.randn(p.shape, generator=g) / math.sqrt(p.shape[1])
            elif name.endswith("lora_B"):
                lora[name] = torch.randn(p.shape, generator=g) * 0.05
        model.add_adapter(f"ft{i}", {**sd, **lora})
    codec = StubCodec(vo.make_codebooks(4, seed=1).cuda())
    g = torch.Generator().manual_seed(0)
    z = torch.randint(0, 1024, (B_CALL * N_CALLS, 4, T), generator=g).cuda()

    def calls(adapted):
        return [dict(start_tokens=z[B_CALL * i:B_CALL * (i + 1)], _sampling_steps=STEPS, seed=i, return_signal=False,
                     **(dict(adapter=f"ft{i % 4}") if adapted else {})) for i in range(N_CALLS)]
    variants = {"base": calls(False), "adapted": calls(True)}

    def run(name):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.generate_many(codec, variants[name])
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    for name in variants:
        run(name)
    times = {k: [] for k in variants}
    for rep in range(a.repeats):
        for name in (("base", "adapted") if rep % 2 == 0 else ("adapted", "base")):
            times[name].append(run(name))
    lib = L.lib()
    fams = list(L.FAMILIES) + ["lora_down"]
    prof = {}
    for name in variants:
        L.check(lib.vnb_profile_begin(model._handle))
        model.generate_many(codec, variants[name])
        ms, n = (C.c_float * len(fams))(), (C.c_int32 * len(fams))()
        L.check(lib.vnb_profile_end(model._handle, ms, n, len(fams)))
        prof[name] = {f: round(ms[i], 3) for i, f in enumerate(fams)}
    lora_gemms = ("gemm_qkv", "gemm_attn_out", "gemm_ffn_up", "gemm_ffn_down")
    tot = {k: sum(v.values()) for k, v in prof.items()}
    gb, ga = (sum(prof[k][f] for f in lora_gemms) for k in ("base", "adapted"))
    q = os.popen("nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv,noheader").read().strip()
    res = {
        "card": card(), "clocks_after": q,
        "shape": dict(B=B_CALL * N_CALLS, calls=N_CALLS, T=T, steps=STEPS, d=1280, layers=20),
        "seconds": {k: [round(t, 4) for t in v] for k, v in times.items()},
        "ms_per_step_median": {k: round(1e3 * float(np.median(v)) / STEPS, 3) for k, v in times.items()},
        "adapted_over_base": round(float(np.median(times["adapted"]) / np.median(times["base"])), 4),
        "profile_ms": prof,
        "lora_down_share_of_adapted": round(prof["adapted"]["lora_down"] / tot["adapted"], 4),
        "lora_gemm_families_ms": {"base": round(gb, 3), "adapted": round(ga, 3)},
        "adapted_epilogue_extra_share_of_adapted": round((ga - gb) / tot["adapted"], 4),
    }
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
