"""Bit-level record of the codec kernels (vnb_codec_conv_tc, vnb_codec_conv_in, vnb_codec_conv_out, vnb_codec_rvq,
vnb_codec_conv1d) on seeded inputs:

    python tools/codec_bits.py --write tests/golden/codec_bits.npz

Every case builds its inputs on the CPU from a fixed seed, runs the library on cuda:0 and stores the SHA-256 of all of
its outputs (bit patterns, in a fixed order, guard regions included) plus a fixed seeded sample of its first output's
values (for diagnosing a mismatch).  tests/test_gpu_codec_bits.py requires a build to reproduce every hash, so a rewrite
of a codec kernel that alters any float operation or its order is caught bit for bit.

The cases cover each epilogue variant of conv_wgmma_kernel (CT_GENERIC, CT_SPLIT, CT_SPLIT_SKIP, CT_SPLIT_F32) at each
MMA width (32, 64, 128) on the codec's layer shapes, the transposed convolutions' offset / limit store, the two edge
layers, the RVQ in its three modes, the fp32 CUDA-core convolution, and a short full-size encode + decode.

Weights are packed with the product's own DAC._split / _pack_conv_tc / _pack_convt_tc, so the packing is under test
too.  The input builders and library wrappers here are shared with tests/test_gpu_codec_ops.py; the float64
references are in tests/codec_op_ref.py.
"""
from __future__ import annotations

import argparse
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.gemm_bits import SENTINEL_F32, digest, lib, sample_index, sentinel, untouched  # noqa: E402

GUARD = 256          # sentinel elements before and after every output buffer
GUARD_ROWS = 3       # sentinel rows between the batch items of a tensor-core convolution's output
SENTINEL_CODE = -1


# ---------------------------------------------------------------------------------------------------- buffers
def guarded(n, dtype):
    """(full, view): a sentinel-filled buffer of n elements with GUARD sentinel elements on each side."""
    if dtype == torch.int64:
        full = torch.full((n + 2 * GUARD,), SENTINEL_CODE, dtype=torch.int64, device="cuda")
    else:
        full = sentinel((n + 2 * GUARD,), dtype)
    return full, full[GUARD:GUARD + n]


def inner(full):
    return full[GUARD:full.numel() - GUARD]


def guards_untouched(full):
    if full.dtype == torch.int64:
        ok = full == SENTINEL_CODE
    else:
        ok = untouched(full)
    return bool(ok[:GUARD].all()) and bool(ok[full.numel() - GUARD:].all())


# ---------------------------------------------------------------------------------------------------- packing
def _dac():
    from vampnet_b200.codec import DAC
    return DAC


def split(x):
    """fp32 -> (hi, lo) bf16 as the product splits activations (DAC._split)."""
    return _dac()._split(x.float())


def pack_conv(w):
    """Conv1d weight (Cout, Cin, K) -> the product's packed split-bf16 (Cout, K * cblocks * 64) pair."""
    D = _dac()
    return D._pack_conv_tc(D, w.float())   # uses only the static _split


def pack_convt(w, s):
    """ConvTranspose1d weight (Cin, Cout, 2s) -> the product's packed (s * Cout, 2 * cblocks * 64) pair."""
    D = _dac()
    return D._pack_convt_tc(D, w.float(), s)


def tile_bn(N):
    """The column tile vnb_codec_conv_tc picks for N columns."""
    bn = 128 if N >= 128 else N
    if N > 128 and N % 128 != 0:
        bn = 96 if N % 96 == 0 else 64
    return bn


def mma_width(N):
    bn = tile_bn(N)
    return 32 if bn <= 32 else 64 if bn <= 64 else 128


def variant(c):
    """The epilogue variant launch_conv selects for case c."""
    fast = c["bias"] is not None and c["alpha"] is not None and c["out_split"] and not c["do_tanh"]
    if fast and c["resid"] == "inplace":
        return "split_skip"
    if fast and c["resid"] is None and c["out_f32"]:
        return "split_f32"
    if fast and c["resid"] is None and not c["out_f32"]:
        return "split"
    return "generic"


# ---------------------------------------------------------------------------------------------------- tc layers
def tc_layer(kind, C, Tq, B, seed, dil=1, s=1, N=None, k=7, bias="rand", alpha=True, resid=None, out_f32=None,
             out_split=True, do_tanh=False):
    """One tensor-core convolution of the codec, as CPU tensors plus its ABI geometry.

    kind  res7:   residual unit's k = 7 conv, C -> C, dilation dil (CT_SPLIT as the product runs it)
          res1:   residual unit's closing 1x1 conv, fp32 skip updated in place (CT_SPLIT_SKIP)
          down:   encoder block's strided conv, k = 2s, pad ceil(s/2), C -> 2C, input viewed as (T/s, s*C)
          convt:  decoder block's ConvTranspose1d(k = 2s, stride s, pad ceil(s/2)), C -> C/2, as one GEMM of
                  N = s * C/2 phase-major columns over the taps (x[q], x[q-1]), stored through the offset / limit view
          conv:   a plain kernel-k conv C -> N, pad k // 2: encoder.conv2 (k 3) and decoder.conv1 (k 7)
    Tq is the number of output rows (for convt: input frames T; the GEMM has T + 1 rows).  The keyword arguments
    override the layer's defaults to reach the other epilogues: bias "rand" / "zero" / "none", alpha (next layer's
    Snake), resid None / "inplace" / "copy", out_f32, out_split, do_tanh.  All random draws happen in a fixed order
    whatever the overrides, so two cases that differ only in them see the same inputs."""
    g = torch.Generator().manual_seed(seed)
    taps, pad, s_view = 7, 3 * dil, 1
    if kind == "res7":
        Cin, Nn, K = C, C, 7
    elif kind == "res1":
        Cin, Nn, K, taps, pad = C, C, 1, 1, 0
    elif kind == "down":
        Cin, Nn, K, taps, pad, s_view = C, 2 * C, 2 * s, 2 * s, math.ceil(s / 2), s
    elif kind == "convt":
        Cin, Nn, K, taps, pad = C, (C // 2) * s, 2 * s, 2, 0
    elif kind == "conv":
        Cin, Nn, K, taps, pad = C, N, k, k, k // 2
    else:
        raise ValueError(kind)
    if kind == "convt":
        Tin, rows_q, cout = Tq, Tq + 1, C // 2
    else:
        Tin, rows_q, cout = Tq * s_view, Tq, Nn
    a = torch.randn(B, Tin, Cin, generator=g)
    if kind == "convt":
        w = torch.randn(Cin, cout, K, generator=g) / math.sqrt(2 * Cin)
        w_hi, w_lo = pack_convt(w, s)
    else:
        w = torch.randn(Nn, Cin, K, generator=g) / math.sqrt(Cin * K)
        w_hi, w_lo = pack_conv(w)
    b = torch.randn(cout, generator=g) * 0.1
    al = 0.5 + torch.rand(cout, generator=g)
    skip_vals = torch.randn(B, Tq * Nn, generator=g)
    if kind == "convt":
        rows, off = Tq * s - s % 2, -math.ceil(s / 2) * cout
    else:
        rows, off = Tq, 0
    limit = rows * cout
    stride = (rows + GUARD_ROWS) * cout
    if resid is None and kind == "res1":
        resid = "inplace"
    if out_f32 is None:
        out_f32 = kind in ("down", "convt") or resid is not None
    a_hi, a_lo = split(a)
    c = dict(kind=kind, C=C, B=B, Tin=Tin, Cin=Cin, s=s_view, N=Nn, taps=taps, dil=-1 if kind == "convt" else dil,
             pad=pad, Tq=rows_q, cout=cout, a=a, a_hi=a_hi, a_lo=a_lo, w=w, w_hi=w_hi, w_lo=w_lo,
             bias=None if bias == "none" else (torch.zeros_like(b) if bias == "zero" else b), bias_mod=cout,
             alpha=al if alpha else None, alpha_mod=cout, resid=resid, out_f32=out_f32, out_split=out_split,
             do_tanh=do_tanh, rows=rows, out_offset=off, out_limit=limit, out_batch_stride=stride, stride_s=s)
    if resid is not None:
        r = torch.full((B, stride), SENTINEL_F32, dtype=torch.int32).view(torch.float32)
        r[:, :Tq * Nn] = skip_vals          # normal convs only: rows [0, Tq) are the valid range
        c["resid_init"] = r
    return c


def run_tc(c):
    """Runs vnb_codec_conv_tc on case c; returns the guarded output buffers on the CPU: dict with f32 / hi / lo."""
    L = lib()
    B, stride = c["B"], c["out_batch_stride"]
    n = B * stride
    dev = lambda t: None if t is None else t.cuda()  # noqa: E731
    outs, ptrs = {}, {}
    if c["out_f32"]:
        outs["f32"], v = guarded(n, torch.float32)
        if c["resid"] == "inplace":
            v.copy_(c["resid_init"].reshape(-1))
        ptrs["f32"] = v
    resid = None
    if c["resid"] == "inplace":
        resid = ptrs["f32"]
    elif c["resid"] == "copy":
        resid = c["resid_init"].reshape(-1).cuda()
    if c["out_split"]:
        outs["hi"], ptrs["hi"] = guarded(n, torch.bfloat16)
        outs["lo"], ptrs["lo"] = guarded(n, torch.bfloat16)
    a_hi, a_lo, w_hi, w_lo = (c[k].cuda() for k in ("a_hi", "a_lo", "w_hi", "w_lo"))
    bias, alpha = dev(c["bias"]), dev(c["alpha"])
    L.check(L.lib().vnb_codec_conv_tc(
        L.ptr(a_hi), L.ptr(a_lo), B, c["Tin"], c["Cin"], c["s"], L.ptr(w_hi), L.ptr(w_lo), c["N"], c["taps"], c["dil"],
        c["pad"], c["Tq"], L.ptr(bias), c["bias_mod"], L.ptr(alpha), c["alpha_mod"], L.ptr(resid),
        L.ptr(ptrs.get("f32")), L.ptr(ptrs.get("hi")), L.ptr(ptrs.get("lo")), stride, c["out_offset"], c["out_limit"],
        1 if c["do_tanh"] else 0, L.stream_ptr()))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in outs.items()}


# ---------------------------------------------------------------------------------------------------- edge layers
def conv_in_case(C, T, B, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, generator=g) * 0.3
    w = torch.randn(C, 1, 7, generator=g) / math.sqrt(7)
    b = torch.randn(C, generator=g) * 0.1
    al = 0.5 + torch.rand(C, generator=g)
    return dict(C=C, T=T, B=B, x=x, w=w, bias=b, alpha=al, pad=3)


def run_conv_in(c):
    L = lib()
    n = c["B"] * c["T"] * c["C"]
    (f, fv), (h, hv), (lo, lv) = guarded(n, torch.float32), guarded(n, torch.bfloat16), guarded(n, torch.bfloat16)
    x, w, b, al = (c[k].cuda() for k in ("x", "w", "bias", "alpha"))
    L.check(L.lib().vnb_codec_conv_in(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(al), L.ptr(fv), L.ptr(hv), L.ptr(lv),
                                      c["B"], c["T"], c["C"], 7, c["pad"], L.stream_ptr()))
    torch.cuda.synchronize()
    return dict(f32=f.cpu(), hi=h.cpu(), lo=lo.cpu())


def conv_out_case(C, T, B, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(B, T, C, generator=g)
    w = torch.randn(1, C, 7, generator=g) * (0.4 / math.sqrt(7 * C))
    b = torch.randn(1, generator=g) * 0.02
    hi, lo = split(a)
    return dict(C=C, T=T, B=B, a_hi=hi, a_lo=lo, w=w, bias=b, pad=3)


def run_conv_out(c):
    L = lib()
    full, v = guarded(c["B"] * c["T"], torch.float32)
    ah, al, w, b = (c[k].cuda() for k in ("a_hi", "a_lo", "w", "bias"))
    L.check(L.lib().vnb_codec_conv_out(L.ptr(ah), L.ptr(al), L.ptr(w), L.ptr(b), L.ptr(v), c["B"], c["T"], c["C"], 7,
                                       c["pad"], L.stream_ptr()))
    torch.cuda.synchronize()
    return dict(audio=full.cpu())


# ---------------------------------------------------------------------------------------------------- fp32 conv
def conv1d_case(kind, Cin, Cout, T, B, seed, K=7, stride=1, dil=1, s=2, tanh=False):
    """kind conv: a Conv1d with Snake on its input, pad ceil(stride / 2) when strided (k = 2 * stride, as the encoder's
    blocks) and (K - 1) * dil / 2 otherwise; res: the same with a residual added in place; convt: ConvTranspose1d(2s,
    stride s, pad ceil(s/2)) as s phase launches through out_stride / out_off."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, T, generator=g)
    al = 0.5 + torch.rand(Cin, generator=g)
    b = torch.randn(Cout, generator=g) * 0.1
    if kind == "convt":
        w = torch.randn(Cin, Cout, 2 * s, generator=g) / math.sqrt(2 * Cin)
        pad = math.ceil(s / 2)
        Tout = T * s - s % 2
        return dict(kind=kind, x=x, w=w, bias=b, alpha=al, resid=None, s=s, pad=pad, Tout=Tout, B=B, Cin=Cin,
                    Cout=Cout, T=T, tanh=False)
    w = torch.randn(Cout, Cin, K, generator=g) / math.sqrt(Cin * K)
    pad = math.ceil(stride / 2) if stride > 1 else (K - 1) * dil // 2
    Tout = (T + 2 * pad - dil * (K - 1) - 1) // stride + 1
    resid = torch.randn(B, Cout, Tout, generator=g) if kind == "res" else None
    return dict(kind=kind, x=x, w=w, bias=b, alpha=al, resid=resid, K=K, stride=stride, dil=dil, pad=pad, Tout=Tout,
                B=B, Cin=Cin, Cout=Cout, T=T, tanh=tanh)


def conv1d_launches(c):
    """The (weight, stride, dil, pad, out_stride, out_off, nq) of each vnb_codec_conv1d launch of case c, with the
    weights in the layout the launch takes (codec.py's per-phase ConvTranspose1d packing for convt)."""
    if c["kind"] == "convt":
        s, pad = c["s"], c["pad"]
        return [(c["w"][:, :, r::s].permute(1, 0, 2).contiguous(), 1, -1, 0, s, r - pad, c["T"] + 1) for r in range(s)]
    return [(c["w"], c["stride"], c["dil"], c["pad"], 1, 0, c["Tout"])]


def run_conv1d(c):
    L = lib()
    B, Cout, Tout = c["B"], c["Cout"], c["Tout"]
    full, y = guarded(B * Cout * Tout, torch.float32)
    x, b, al = c["x"].cuda(), c["bias"].cuda(), c["alpha"].cuda()
    resid = None
    if c["resid"] is not None:
        y.copy_(c["resid"].reshape(-1))
        resid = y
    for w, stride, dil, pad, ostr, ooff, nq in conv1d_launches(c):
        w = w.cuda()
        L.check(L.lib().vnb_codec_conv1d(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(al), L.ptr(resid), L.ptr(y), B, c["Cin"],
                                         c["T"], Cout, Tout, w.shape[-1], stride, dil, pad, ostr, ooff, nq,
                                         1 if c["tanh"] else 0, L.stream_ptr()))
    torch.cuda.synchronize()
    return dict(y=full.cpu())


# ---------------------------------------------------------------------------------------------------- rvq
def rvq_weights(D, L, seed, V=1024):
    """Seeded quantiser weights as the codec packs them: win (L, 8, D), bin (L, 8), wout (L, D, 8), bout (L, D),
    cb (L, V, 8) and cbn = F.normalize(cb) (computed as the product does, in fp32)."""
    g = torch.Generator().manual_seed(seed)
    win = torch.randn(L, 8, D, generator=g) / math.sqrt(D)
    bin_ = torch.randn(L, 8, generator=g) * 0.02
    wout = torch.randn(L, D, 8, generator=g) / math.sqrt(8 * L)
    bout = torch.randn(L, D, generator=g) * 0.02
    cb = torch.randn(L, V, 8, generator=g)
    return dict(win=win, bin=bin_, wout=wout, bout=bout, cb=cb, D=D, L=L, V=V)


def normalized(cb):
    return torch.nn.functional.normalize(cb, dim=-1).contiguous()


def rvq_inputs(mode, wts, T, B, seed, channels_last=False):
    """Seeded input of each mode: z (B, D, T) or (B, T, D); latents near codebook vectors; codes."""
    g = torch.Generator().manual_seed(seed)
    D, L, V = wts["D"], wts["L"], wts["V"]
    if mode == 0:
        z = torch.randn(B, T, D, generator=g) if channels_last else torch.randn(B, D, T, generator=g)
        return dict(in_f=z, in_codes=None)
    codes = torch.randint(0, V, (B, L, T), generator=g)
    if mode == 2:
        return dict(in_f=None, in_codes=codes)
    lat = torch.stack([wts["cb"][l][codes[:, l]] for l in range(L)], 1)        # (B, L, T, 8)
    lat = lat + 0.3 * torch.randn(lat.shape, generator=g)
    return dict(in_f=lat.permute(0, 1, 3, 2).reshape(B, 8 * L, T).contiguous(), in_codes=None)


def run_rvq(mode, wts, inp, L, T, B, channels_last=False, split_out=False, cb=None):
    """Runs vnb_codec_rvq; returns guarded codes / latents (mode 0), zq and, with split_out, zq_hi / zq_lo."""
    Lb = lib()
    D, V = wts["D"], wts["V"]
    cb = wts["cb"] if cb is None else cb
    win, bin_, wout, bout = (wts[k].contiguous().cuda() for k in ("win", "bin", "wout", "bout"))
    cbg, cbn = cb.contiguous().cuda(), normalized(cb).cuda()
    in_f = None if inp["in_f"] is None else inp["in_f"].cuda()
    in_codes = None if inp["in_codes"] is None else inp["in_codes"].cuda()
    outs, ptrs = {}, {}
    if mode == 0:
        outs["codes"], ptrs["codes"] = guarded(B * L * T, torch.int64)
        outs["latents"], ptrs["latents"] = guarded(B * 8 * L * T, torch.float32)
    outs["zq"], ptrs["zq"] = guarded(B * D * T, torch.float32)
    if split_out:
        outs["zq_hi"], ptrs["zq_hi"] = guarded(B * D * T, torch.bfloat16)
        outs["zq_lo"], ptrs["zq_lo"] = guarded(B * D * T, torch.bfloat16)
    Lb.check(Lb.lib().vnb_codec_rvq(mode, Lb.ptr(in_f), Lb.ptr(in_codes), Lb.ptr(win), Lb.ptr(bin_), Lb.ptr(wout),
                                    Lb.ptr(bout), Lb.ptr(cbg), Lb.ptr(cbn), Lb.ptr(ptrs.get("codes")),
                                    Lb.ptr(ptrs["zq"]), Lb.ptr(ptrs.get("latents")), B, D, T, L, V,
                                    1 if channels_last else 0, Lb.ptr(ptrs.get("zq_hi")), Lb.ptr(ptrs.get("zq_lo")),
                                    Lb.stream_ptr()))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in outs.items()}


# ---------------------------------------------------------------------------------------------------- full codec
def full_codec(seed=0):
    """The full-size codec (encoder 64 .. 1024, decoder 1536 .. 96, 14 x 1024 x 8 RVQ) on seeded oracle weights."""
    from oracle import dac_oracle as do
    from vampnet_b200.codec import DAC
    cfg = do.CodecConfig()
    w = do.make_codec_weights(cfg, seed=seed)
    m = DAC(encoder_dim=cfg.encoder_dim, encoder_rates=cfg.encoder_rates, decoder_dim=cfg.decoder_dim,
            n_codebooks=cfg.n_codebooks, codebook_size=cfg.codebook_size, codebook_dim=cfg.codebook_dim,
            sample_rate=cfg.sample_rate)
    m.load_flat(w)
    return cfg, w, m.to("cuda")


# ---------------------------------------------------------------------------------------------------- cases
# One tensor-core case per (epilogue variant, MMA width), on the codec's layer shapes (width 32 only exists in the
# reduced-width codec), plus the transposed convolutions' store at both column tiles.
TC_CASES = [
    # (name, kind, C, Tq, B, keyword arguments)
    ("split_n128_res7_c128_d3", "res7", 128, 300, 2, dict(dil=3)),
    ("split_n64_res7_c64_d9", "res7", 64, 300, 2, dict(dil=9)),
    ("split_n32_res7_c32_d1", "res7", 32, 300, 2, dict(dil=1)),
    ("skip_n128_res1_c768", "res1", 768, 129, 2, {}),
    ("skip_n128_res1_c96", "res1", 96, 300, 2, {}),
    ("skip_n64_res1_c64", "res1", 64, 300, 2, {}),
    ("skip_n32_res1_c32", "res1", 32, 300, 2, {}),
    ("f32_n128_down_c256_s8", "down", 256, 129, 2, dict(s=8)),
    ("f32_n128_convt_c1536_s12", "convt", 1536, 24, 2, dict(s=12)),
    ("f32_n128_convt_c192_s2", "convt", 192, 300, 2, dict(s=2)),
    ("f32_n64_down_c32_s2", "down", 32, 300, 2, dict(s=2)),
    ("f32_n32_res7_c32", "res7", 32, 300, 2, dict(out_f32=True)),
    ("generic_n128_conv2", "conv", 1024, 129, 2, dict(k=3, N=1024, alpha=False, out_split=False, out_f32=True)),
    ("generic_n64_tanh_c64", "res7", 64, 300, 2, dict(do_tanh=True, out_f32=True)),
    ("generic_n32_resid_c32", "res1", 32, 300, 2, dict(resid="copy")),
]


def tc_bits_case(i):
    name, kind, C, Tq, B, kw = TC_CASES[i]
    return tc_layer(kind, C, Tq, B, seed=1000 + i, **kw)


def _flat(o, keys):
    return [o[k] for k in keys if k in o]


def run_named(name):
    """All outputs of the record case `name`, as CPU tensors in a fixed order."""
    for i, (n, *_rest) in enumerate(TC_CASES):
        if n == name:
            return _flat(run_tc(tc_bits_case(i)), ("f32", "hi", "lo"))
    if name == "conv_in_c64_t2307":
        return _flat(run_conv_in(conv_in_case(64, 2307, 2, 11)), ("f32", "hi", "lo"))
    if name == "conv_out_c96_t4100":
        return _flat(run_conv_out(conv_out_case(96, 4100, 2, 12)), ("audio",))
    if name == "conv1d_res_c64":
        return _flat(run_conv1d(conv1d_case("res", 64, 64, 300, 2, 13, dil=3)), ("y",))
    if name == "conv1d_down_c64_s4":
        return _flat(run_conv1d(conv1d_case("conv", 64, 128, 1200, 2, 14, K=8, stride=4)), ("y",))
    if name == "conv1d_convt_c192_s8":
        return _flat(run_conv1d(conv1d_case("convt", 192, 96, 40, 2, 15, s=8)), ("y",))
    if name.startswith("rvq_mode"):
        mode, cl = int(name[8]), name.endswith("_cl")
        L = 14 if mode == 0 else 4
        wts = rvq_weights(1024, 14, 16)
        inp = rvq_inputs(mode, {**wts, "L": L}, 575, 2, 17 + mode, channels_last=cl)
        return _flat(run_rvq(mode, wts, inp, L, 575, 2, channels_last=cl, split_out=cl),
                     ("zq", "codes", "latents", "zq_hi", "zq_lo"))
    if name == "full_codec_encode_decode":
        _, _, m = full_codec(seed=0)
        x = torch.randn(2, 1, 768 * 5, generator=torch.Generator().manual_seed(18)) * 0.3
        enc = m.encode(x.cuda())
        audio = m.decode(enc["z"])["audio"]
        torch.cuda.synchronize()
        return [audio.cpu(), enc["codes"].cpu(), enc["z"].cpu(), enc["latents"].cpu()]
    raise KeyError(name)


CASES = [c[0] for c in TC_CASES] + ["conv_in_c64_t2307", "conv_out_c96_t4100", "conv1d_res_c64",
                                    "conv1d_down_c64_s4", "conv1d_convt_c192_s8", "rvq_mode0", "rvq_mode0_cl",
                                    "rvq_mode1", "rvq_mode2", "full_codec_encode_decode"]


def sample_values(outs, name):
    flat = outs[0].double().reshape(-1).numpy()
    return flat[sample_index(flat.size, name)]


def record():
    rec = {}
    for name in CASES:
        outs = run_named(name)
        rec["sha256_" + name] = np.array(digest(outs))
        rec["sample_" + name] = sample_values(outs, name)
        print(f"{name}: {rec['sha256_' + name]}", flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--write", metavar="NPZ", help="where to store the hashes and samples (default: only print them)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    rec = record()
    dev = torch.cuda.get_device_properties(0)
    rec["device"] = np.array(dev.name)
    if args.write:
        os.makedirs(os.path.dirname(os.path.abspath(args.write)), exist_ok=True)
        np.savez_compressed(args.write, **rec)
        print(f"wrote {len(CASES)} cases to {args.write}")


if __name__ == "__main__":
    main()
