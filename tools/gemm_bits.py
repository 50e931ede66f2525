"""Bit-level record of the GEMM family's fused epilogues (vnb_dbg_gemm_fused, vnb_dbg_gemm_sample) on seeded inputs:

    python tools/gemm_bits.py --write tests/golden/gemm_bits.npz
    python tools/gemm_bits.py --add-to tests/golden/gemm_bits.npz --write <new record>   # new cases only

Every case builds its operands on the CPU from a fixed seed, runs the library on cuda:0 and stores the SHA-256 of
all of its outputs (bit patterns, in a fixed order) plus a fixed seeded sample of its first output's values (for
diagnosing a mismatch).  tests/test_gpu_gemm_bits.py requires a build to reproduce every hash with both tile variants,
so a rewrite of the epilogues that alters any float operation or its order is caught bit for bit.

The cases cover every fused variant the forward launches, at d_model 256 (ss_parts 2) and 1280 (ss_parts 10), with
ragged M: the row-scaled consumers (BF16, QKV with vT and batch boundaries inside a tile, GEGLU, the classifier's
BIAS_F32), the producers (RESID with its bf16 copy and two sum-of-squares partials per tile, the embedding projection's
BIAS_F32 with one partial per tile) and the sampling epilogue for both codebook layouts (C, ncc) = (4, 0) and (14, 4)
at vocab_size 1024, and at vocab sizes 256 (one predicted codebook), 512 (three) and 768 (seven).

The input builders and library wrappers here are shared with tests/test_gpu_gemm_fused.py.
"""
from __future__ import annotations

import argparse
import hashlib
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

N_SAMPLE = 256
EPS = 1e-6
V = 1024                    # the vocabulary size of the sampling cases unless a case names another
SENTINEL_F32 = 0x7FBADBAD   # NaN bit patterns that no kernel produces: a missed or stray store shows up
SENTINEL_BF16 = 0x7FA5


def lib():
    from vampnet_b200 import _lib as L
    L.lib()
    return L


# ---------------------------------------------------------------------------------------------------- inputs
def operands(M, N, K, seed):
    """A (M, K) and W (N, K) bf16 on cuda:0 (W scaled so that A . W^T is about unit size) and the CPU generator."""
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).bfloat16()
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).bfloat16()
    return A.cuda(), W.cuda(), g


def row_stats(M, d, parts, g):
    """ss_in (parts, M) fp32 on cuda:0 whose row scales rs = rsqrt(sum_p ss_in[p] / d + eps) span about 1e-2 .. 1e3:
    the mean square of a row is 10^U(-9, 4), and every 7th row has none at all (eps alone: rs = 1e3); the total is
    split over the parts with random positive weights.  Returns ss_in, inv_d (fp32) and rs64 (M,) float64 on cuda:0,
    the row scale computed in float64 from the fp32 partials."""
    ms = 10.0 ** (torch.rand(M, generator=g, dtype=torch.float64) * 13.0 - 9.0)
    ms[::7] = 0.0
    w = torch.rand(parts, M, generator=g, dtype=torch.float64) + 0.05
    ss = (ms * d * w / w.sum(0)).float()
    inv_d = float(np.float32(1.0 / d))
    rs64 = 1.0 / torch.sqrt(ss.double().sum(0) * inv_d + EPS)
    return ss.contiguous().cuda(), inv_d, rs64.cuda()


def sentinel(shape, dtype):
    if dtype == torch.bfloat16:
        return torch.full(shape, SENTINEL_BF16, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    return torch.full(shape, SENTINEL_F32, dtype=torch.int32, device="cuda").view(dtype)


def untouched(t):
    """True where t still holds the sentinel bit pattern."""
    if t.dtype == torch.bfloat16:
        return t.view(torch.int16) == SENTINEL_BF16
    return t.view(torch.int32) == SENTINEL_F32


def sample_inputs(M, C, ncc, g, V=V):
    """zcur (M, C) int32 on cuda:0: conditioning codebooks hold tokens; each predicted position is masked (= V, the mask
    token) with probability 0.7, and rows 32 .. 95 are known in every codebook (whole epilogue warps with nothing to
    sample)."""
    z = torch.randint(0, V, (M, C), generator=g, dtype=torch.int32)
    masked = torch.rand(M, C, generator=g) < 0.7
    masked[:, :ncc] = False
    masked[32:96] = False
    z[masked] = V
    return z.cuda()


def tie_columns(W, bias, g, per=4, V=V):
    """Make exact ties: in `per` strips of every V-column codebook block (all of them if it has fewer), a scaled copy of
    one W row and its bias entry also goes to a later column of the same 128-column strip, so those logits are equal
    bit for bit and are the strip's maximum for many rows."""
    N = W.shape[0]
    for blk in range(N // V):
        for k in torch.randperm(V // 128, generator=g)[:per].tolist():
            base = blk * V + k * 128
            i, j = sorted(torch.randperm(128, generator=g)[:2].tolist())
            W[base + i] = (W[base + i].float() * 4.0).bfloat16()
            W[base + j] = W[base + i]
            bias[base + j] = bias[base + i]


# ---------------------------------------------------------------------------------------------------- library calls
def gemm_fused(epi, A, W, out, out2=None, bias=None, T=1, Tpad=8, ss_in=None, inv_d=0.0, out_bf16=None, ss_out=None):
    L = lib()
    M, K = A.shape
    N = W.shape[0]
    parts = 0 if ss_in is None else ss_in.shape[0]
    L.check(L.lib().vnb_dbg_gemm_fused(epi, L.ptr(A), L.ptr(W), M, N, K, L.ptr(out), L.ptr(out2), L.ptr(bias), T, Tpad,
                                       L.ptr(ss_in), parts, inv_d, EPS, L.ptr(out_bf16), L.ptr(ss_out),
                                       L.stream_ptr()))


def gemm_sample(A, W, bias, ss_in, inv_d, zcur, T, C, ncc, temperature, do_sample, step, seed, partials, V=V):
    L = lib()
    M, K = A.shape
    N = W.shape[0]
    parts = 0 if ss_in is None else ss_in.shape[0]
    L.check(L.lib().vnb_dbg_gemm_sample(L.ptr(A), L.ptr(W), L.ptr(bias), M, N, K, L.ptr(ss_in), parts, inv_d, EPS,
                                        L.ptr(zcur), T, C, ncc, V, V, temperature, do_sample, step, seed[0], seed[1],
                                        L.ptr(partials), L.stream_ptr()))


def set_pair(value):
    """Sets the "gemm_pair" option and returns its previous value."""
    L = lib()
    prev = L.C.c_int32()
    L.check(L.lib().vnb_get_option(b"gemm_pair", L.C.byref(prev)))
    L.check(L.lib().vnb_set_option(b"gemm_pair", value))
    return prev.value


# ---------------------------------------------------------------------------------------------------- cases
# (kind, d, M, extra): d sets K (and ss_parts = d / 128 for the consumers); M is ragged (not a multiple of 128)
CASES = [
    ("bf16", 256, 300, None), ("bf16", 1280, 1725, None),
    ("qkv", 256, 300, 75), ("qkv", 1280, 1725, 575),          # extra = T
    ("geglu", 256, 300, None), ("geglu", 1280, 1725, None),
    ("cls", 256, 300, 4096), ("cls", 1280, 1725, 10240),       # extra = N
    ("resid", 256, 300, 512), ("resid", 1280, 1725, 2560),     # extra = K
    ("embed", 256, 300, 192), ("embed", 1280, 1725, 384),      # extra = K = 3 Kp
    ("sample", 256, 450, (4, 0)), ("sample", 1280, 1725, (14, 4)),   # extra = (C, ncc)
    ("sample", 256, 450, (1, 0, 256)), ("sample", 512, 450, (4, 1, 512)),  # extra = (C, ncc, V)
    ("sample", 1280, 1725, (9, 2, 768)),
]


def case_name(kind, d, M, extra):
    ex = "" if extra is None else "_" + ("x".join(map(str, extra)) if isinstance(extra, tuple) else str(extra))
    return f"{kind}_d{d}_M{M}{ex}"


def run_case(kind, d, M, extra):
    """All outputs of one case as CPU tensors, in a fixed order (sentinel-filled buffers, so untouched entries are
    part of the record too)."""
    from vampnet_b200 import _lib as L
    seed = len(kind) * 100003 + d * 7 + M
    parts = d // 128
    if kind in ("bf16", "qkv", "geglu", "cls"):
        N = {"bf16": d, "qkv": 3 * d, "geglu": 4 * d, "cls": extra}[kind]
        A, W, g = operands(M, N, d, seed)
        ss, inv_d, _ = row_stats(M, d, parts, g)
        if kind == "qkv":
            T = extra
            B, Tpad = M // T, (T + 7) // 8 * 8
            qk, vT = sentinel((M, 2 * d), torch.bfloat16), sentinel((B, d, Tpad), torch.bfloat16)
            gemm_fused(L.EPI_QKV, A, W, qk, vT, T=T, Tpad=Tpad, ss_in=ss, inv_d=inv_d)
            outs = [qk, vT]
        elif kind == "cls":
            bias = torch.randn(N, generator=g).cuda()
            out = sentinel((M, N), torch.float32)
            gemm_fused(L.EPI_BIAS_F32, A, W, out, bias=bias, ss_in=ss, inv_d=inv_d)
            outs = [out]
        else:
            out = sentinel((M, N if kind == "bf16" else N // 2), torch.bfloat16)
            gemm_fused(L.EPI_BF16 if kind == "bf16" else L.EPI_GEGLU, A, W, out, ss_in=ss, inv_d=inv_d)
            outs = [out]
    elif kind in ("resid", "embed"):
        A, W, g = operands(M, d, extra, seed)
        y, ss_out = sentinel((M, d), torch.bfloat16), sentinel((d // 128, M), torch.float32)
        if kind == "resid":
            out = torch.randn(M, d, generator=g).cuda()
            gemm_fused(L.EPI_RESID, A, W, out, out_bf16=y, ss_out=ss_out)
        else:
            bias = torch.randn(d, generator=g).cuda()
            out = sentinel((M, d), torch.float32)
            gemm_fused(L.EPI_BIAS_F32, A, W, out, bias=bias, out_bf16=y, ss_out=ss_out)
        outs = [out, y, ss_out]
    else:
        C, ncc, Vc = extra if len(extra) == 3 else (*extra, V)
        T = 150 if M == 450 else 575
        N = (C - ncc) * Vc
        A, W, g = operands(M, N, d, seed)
        bias = torch.randn(N, generator=g)
        W = W.cpu()
        tie_columns(W, bias, g, V=Vc)
        W, bias = W.cuda(), bias.cuda()
        ss, inv_d, _ = row_stats(M, d, parts, g)
        zcur = sample_inputs(M, C, ncc, g, V=Vc)
        outs = []
        for temperature, do_sample, step in ((0.7, 1, 11), (1.0, 0, 0)):
            rec = sentinel((M * (C - ncc) * (Vc // 128), 4), torch.float32)
            gemm_sample(A, W, bias, ss, inv_d, zcur, T, C, ncc, temperature, do_sample, step, (1234, 5678), rec, V=Vc)
            outs.append(rec)
    torch.cuda.synchronize()
    return [o.cpu() for o in outs]


def digest(outs):
    h = hashlib.sha256()
    for o in outs:
        h.update(o.contiguous().view(torch.uint8).numpy().tobytes())
    return h.hexdigest()


def sample_index(n, name):
    g = np.random.default_rng(int(hashlib.sha256(name.encode()).hexdigest()[:8], 16))
    return np.sort(g.choice(n, size=min(N_SAMPLE, n), replace=False))


def sample_values(outs, name):
    flat = outs[0].float().reshape(-1).numpy()
    return flat[sample_index(flat.size, name)]


def record(cases=CASES):
    rec = {}
    prev = set_pair(0)
    try:
        for case in cases:
            name = case_name(*case)
            outs = run_case(*case)
            rec["sha256_" + name] = np.array(digest(outs))
            rec["sample_" + name] = sample_values(outs, name)
            print(f"{name}: {rec['sha256_' + name]}", flush=True)
    finally:
        set_pair(prev)
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--write", metavar="NPZ", required=True, help="where to store the hashes and samples")
    ap.add_argument("--add-to", metavar="NPZ", help="keep this record's entries as they are and record only the cases "
                    "it lacks")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    dev = torch.cuda.get_device_properties(0)
    old = dict(np.load(args.add_to)) if args.add_to else {}
    cases = [c for c in CASES if "sha256_" + case_name(*c) not in old]
    rec = record(cases)
    if old:
        rec["device_added"] = np.array(dev.name)
    else:
        rec["device"] = np.array(dev.name)
    os.makedirs(os.path.dirname(os.path.abspath(args.write)), exist_ok=True)
    np.savez_compressed(args.write, **old, **rec)
    print(f"wrote {len(cases)} new cases ({len(CASES)} in all) to {args.write}")


if __name__ == "__main__":
    main()
