"""Bit-level record of the sampling step (vnb_dbg_sample: sample_rows_kernel with and without the nucleus filter,
sample_combine_kernel and remask_kernel) on seeded inputs:

    python tools/sample_bits.py --write tests/golden/sample_bits.npz

Every case builds its inputs on the CPU from a fixed seed, runs one vnb_dbg_sample call on cuda:0 and stores the
SHA-256 of tokens, conf and zcur after the call (bit patterns, in that order) plus a fixed seeded sample of the conf
values (for diagnosing a mismatch).  tests/test_gpu_sample_bits.py requires a build to reproduce every hash, so a
rewrite of the sampler that alters any float operation, its order or a decision is caught bit for bit.

The cases cover every path, both codebook layouts (C, ncc) = (4, 0) and (14, 4), vocabulary sizes 256 and 1024, a
nucleus case, a re-mask with ties, infinities and a row longer than the CTA, and a three-group launch.

The input builders and the library wrapper here are shared with tests/test_gpu_sampler_ops.py.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests import gemm_sample_ref as GR  # noqa: E402
from tests.sample_ref import Group  # noqa: E402

N_SAMPLE = 256
SENTINEL = 0x7FBADBAD   # a NaN bit pattern (and an int32 no token equals): a missed store shows up


def lib():
    from vampnet_b200 import _lib as L
    L.lib()
    return L


def sentinel(shape, dtype):
    return torch.full(shape, SENTINEL, dtype=torch.int32, device="cuda").view(dtype)


# ---------------------------------------------------------------------------------------------------- inputs
def state(B, T, C, ncc, V, g, p_masked=0.7):
    """zcur (B, T, C) int32 on cuda:0 with mask token V: conditioning codebooks hold tokens, each predicted entry is
    masked with probability p_masked, and the last position of every row is known (a row is never fully masked)."""
    z = torch.randint(0, V, (B, T, C), generator=g, dtype=torch.int32)
    m = torch.rand(B, T, C, generator=g) < p_masked
    m[:, :, :ncc] = False
    m[:, -1, -1] = False
    z[m] = V
    return z.cuda()


def logits_for(R, V, g, scale=2.5):
    """(R, V) fp32 on cuda:0: N(0, scale^2); every 5th row rounded (many exact ties), and every 7th row with its
    maximum tied at indices 5, 77 and V - 1 - 128 (different lanes and, for V >= 256, different 128-entry chunks)."""
    x = torch.randn(R, V, generator=g) * scale
    x[::5] = torch.round(x[::5])
    t = x[::7]
    top = t.amax(-1) + 1.0
    for i in (5, 77, V - 1 - 128 if V >= 256 else 100):
        t[:, i] = top
    x[::7] = t
    return x.cuda()


def records_from_logits(x, temperature, do_sample, seed, step, B, S):
    """The classifier epilogue's float4 records of logits x (B*S, V) fp32 (tests/gemm_sample_ref.py strip_records,
    float64 sums stored as fp32), in the layout sample_combine_kernel reads: ((b*S + s) * V/128 + k, 4)."""
    from oracle import philox
    R, V = x.shape
    nt = V // GR.TILE
    u2 = None
    if do_sample:
        u2 = torch.from_numpy(philox.uniform_bs(seed, step, B, S, stream=0, word=1)).reshape(-1).cuda()
        u2 = u2.repeat_interleave(nt)
    mx, am, s, cand, _ = GR.strip_records(x.reshape(-1, GR.TILE), GR.inv_temperature(temperature), u2)
    v0 = (torch.arange(nt, device=x.device) * GR.TILE).repeat(R)
    xc = x.reshape(-1, GR.TILE).gather(1, cand[:, None])[:, 0]
    bits = ((v0 + cand) | ((v0 + am) << 16)).int()
    return torch.stack([mx, s.float(), xc, bits.view(torch.float32)], -1).contiguous()


# ---------------------------------------------------------------------------------------------------- library call
def dbg_sample(path, zcur, tokens, conf, n0, ncc, V, groups, logits=None, partials=None, zorig=None, mask_token=None):
    """One vnb_dbg_sample call; zcur (B, T, C) int32 is updated in place, n0 a list of per-group counts."""
    L = lib()
    B, T, C = zcur.shape
    arr = (L.SampleGroup * len(groups))()
    for a, g in zip(arr, groups):
        a.rows, a.temperature, a.gamma, a.temp_eff = g.rows, g.temperature, g.gamma, g.temp_eff
        a.do_sample, a.is_last, a.step = g.do_sample, g.is_last, g.step
        a.seed_lo, a.seed_hi, a.top_p = g.seed[0], g.seed[1], g.top_p
    n0d = torch.tensor(list(n0), dtype=torch.int32, device="cuda")
    L.check(L.lib().vnb_dbg_sample(path, L.ptr(logits), L.ptr(partials), L.ptr(zcur), L.ptr(zorig), L.ptr(tokens),
                                   L.ptr(conf), L.ptr(n0d), B, T, C, ncc, V, V if mask_token is None else mask_token,
                                   arr, len(groups), L.stream_ptr()))


# ---------------------------------------------------------------------------------------------------- cases
# (name, path, B, T, C, ncc, V, groups); groups: tuples (rows, temperature, gamma, temp_eff, do_sample, is_last, step,
# top_p)
CASES = [
    ("rows_coarse_V1024", 0, 3, 37, 4, 0, 1024, [(3, 0.7, 0.6, 4.5, 1, 0, 3, 0.0)]),
    ("rows_c2f_V1024_greedy", 0, 2, 29, 14, 4, 1024, [(2, 1.0, 0.3, 0.0, 0, 0, 7, 0.0)]),
    ("rows_coarse_V256", 0, 2, 50, 4, 0, 256, [(2, 3.0, 0.8, 10.5, 1, 1, 11, 0.0)]),
    ("topp_c2f_V1024", 1, 2, 23, 14, 4, 1024, [(2, 1.3, 0.5, 2.0, 1, 0, 2, 0.85)]),
    ("combine_coarse_V1024", 2, 3, 37, 4, 0, 1024, [(3, 0.7, 0.6, 4.5, 1, 0, 3, 0.0)]),
    ("combine_c2f_V1024_greedy", 2, 2, 29, 14, 4, 1024, [(2, 1.0, 0.3, 0.0, 0, 0, 7, 0.0)]),
    ("remask_c2f_S1030", 3, 2, 103, 14, 4, 1024, [(1, 1.0, 0.45, 0.0, 1, 0, 5, 0.0), (1, 1.0, 1.0, 0.0, 1, 1, 5, 0.0)]),
    ("groups_coarse_V768", 0, 6, 31, 4, 0, 768, [(2, 0.8, 0.5, 6.0, 1, 0, 4, 0.0), (1, 2.0, 0.9, 1.0, 0, 0, 9, 0.0),
                                                 (3, -1.0, 0.2, 10.5, 1, 0, 1, 0.0)]),
]


def run_case(name, path, B, T, C, ncc, V, gspec):
    """tokens, conf and zcur after one call, as CPU tensors (sentinel-filled outputs)."""
    g = torch.Generator().manual_seed(int(hashlib.sha256(name.encode()).hexdigest()[:8], 16))
    S = T * (C - ncc)
    groups = [Group(rows=r, temperature=t, gamma=ga, temp_eff=te, do_sample=ds, is_last=il, step=st,
                    seed=(1000 + 17 * i, 77 + i), top_p=tp) for i, (r, t, ga, te, ds, il, st, tp) in enumerate(gspec)]
    zcur = state(B, T, C, ncc, V, g)
    zorig = torch.randint(0, V, (B, T, C), generator=g, dtype=torch.int32).cuda()
    n0 = [int(S * 0.8) + 3 * i for i in range(len(groups))]
    tokens, conf = sentinel((B, S), torch.int32), sentinel((B, S), torch.float32)
    logits = partials = None
    if path == 3:
        tokens = torch.randint(0, V, (B, S), generator=g, dtype=torch.int32).cuda()
        c = torch.round(torch.randn(B, S, generator=g) * 4.0) / 4.0       # many ties
        c[:, ::11] = float("inf")
        c[:, 3::13] = -float("inf")
        conf = c.cuda()
    else:
        logits = logits_for(B * S, V, g)
        if path == 2:
            g0 = groups[0]
            partials = records_from_logits(logits, g0.temperature, g0.do_sample, g0.seed, g0.step, B, S)
    dbg_sample(path, zcur, tokens, conf, n0, ncc, V, groups, logits=logits, partials=partials, zorig=zorig)
    torch.cuda.synchronize()
    return [tokens.cpu(), conf.cpu(), zcur.cpu()]


def digest(outs):
    h = hashlib.sha256()
    for o in outs:
        h.update(o.contiguous().view(torch.uint8).numpy().tobytes())
    return h.hexdigest()


def sample_values(outs, name):
    flat = outs[1].reshape(-1).numpy()
    g = np.random.default_rng(int(hashlib.sha256(name.encode()).hexdigest()[:8], 16))
    return flat[np.sort(g.choice(flat.size, size=min(N_SAMPLE, flat.size), replace=False))]


def record():
    rec = {}
    for case in CASES:
        name = case[0]
        outs = run_case(*case)
        rec["sha256_" + name] = np.array(digest(outs))
        rec["sample_" + name] = sample_values(outs, name)
        print(f"{name}: {rec['sha256_' + name]}", flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--write", metavar="NPZ", required=True, help="where to store the hashes and samples")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    rec = record()
    rec["device"] = np.array(torch.cuda.get_device_properties(0).name)
    os.makedirs(os.path.dirname(os.path.abspath(args.write)), exist_ok=True)
    np.savez_compressed(args.write, **rec)
    print(f"wrote {len(CASES)} cases to {args.write}")


if __name__ == "__main__":
    main()
