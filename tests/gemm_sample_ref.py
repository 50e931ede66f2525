"""Reference of the classifier GEMM's sampling records (VNB_EPI_SAMPLE; include/vampnet_b200.h, vnb_dbg_gemm_sample) and
of the tile pick that sample_combine_kernel makes from them.  Plain torch in float64, on whatever device the logits are
on: tests/test_gemm_sample_records_cpu.py pins it to the oracle's sampler on the CPU, tests/test_gpu_gemm_fused.py
holds the kernel to it on the GPU.

The record of a 128-entry strip x (fp32 logits) is {max x, sum, x[cand], cand | argmax << 16} with
    sum  = sum_v 2^(x_v * c1 + c0),  c1 = fp32(inv_temp * fp32(log2 e)),  c0 = -fp32(max x * c1)
(= sum_v exp((x_v - max x) * inv_temp) up to the fp32 rounding of c1 and c0, which scales every term of the strip by
the same factor and which sample_combine_kernel undoes with the same c1).  The two constants are taken as the kernel
forms them; every other operation here is float64.  cand = the first v whose running sum exceeds u2 * sum (u2: word 1
of the Philox counter (t*Cp + cp, b, step, 0)), the arg-max (lowest index on ties) on greedy steps.
"""
from __future__ import annotations

import numpy as np
import torch

TILE = 128
LOG2E_F32 = np.float32(1.4426950408889634)
AMBIGUOUS_REL = 1e-5  # a crossing this close to its target (relative to the sum) may go either way in fp32


def first_true(mask: torch.Tensor) -> torch.Tensor:
    """Index of the first True along the last axis, mask.shape[-1] where there is none."""
    n = mask.shape[-1]
    idx = torch.arange(n, device=mask.device).expand_as(mask)
    return torch.where(mask, idx, n).min(-1).values


def inv_temperature(temperature: float) -> np.float32:
    """The kernels' 1/temperature: fp32(1/T) computed in double, 1 when T <= 0."""
    return np.float32(1.0 / temperature) if temperature > 0 else np.float32(1.0)


def strip_records(x: torch.Tensor, inv_temp: np.float32, u2: torch.Tensor | None):
    """x (R, 128) fp32 strips, u2 (R,) fp32 uniforms (None: greedy).  Returns (max fp32, argmax int64, sum fp64,
    cand int64, ambiguous bool), each (R,); `ambiguous` marks strips whose candidate is within AMBIGUOUS_REL * sum of
    flipping (never on greedy steps)."""
    assert x.dtype == torch.float32 and x.shape[-1] == TILE
    mx = x.max(-1).values
    am = first_true(x == mx[:, None])
    c1 = np.float32(inv_temp) * LOG2E_F32    # fp32 product, as the kernel forms it
    c0 = -(mx * torch.tensor(c1, device=x.device))   # fp32 product
    e = torch.exp2(x.double() * float(c1) + c0.double()[:, None])
    cum = e.cumsum(-1)
    s = cum[:, -1]
    if u2 is None:
        return mx, am, s, am.clone(), torch.zeros_like(am, dtype=torch.bool)
    target = u2.double() * s
    hit = cum > target[:, None]
    cand = torch.where(hit.any(-1), first_true(hit), am)
    ambiguous = ((cum - target[:, None]).abs() <= AMBIGUOUS_REL * s[:, None]).any(-1)
    return mx, am, s, cand, ambiguous


def combine(mx: torch.Tensor, s: torch.Tensor, cand: torch.Tensor, am: torch.Tensor, inv_temp: np.float32,
            u1: torch.Tensor | None):
    """sample_combine_kernel's choice from the records of one row's V/128 tiles: mx, s, cand, am (R, nt) as from
    strip_records, u1 (R,) word 0 of the same counter (None: greedy).  Returns (token, ambiguous), (R,) each: the tile
    whose running mass first exceeds u1 * total gives its candidate; greedy takes the arg-max of the tile with the
    largest maximum (the first such tile)."""
    R, nt = mx.shape
    M = mx.max(-1, keepdim=True).values
    kmax = first_true(mx == M)
    if u1 is None:
        return kmax * TILE + am.gather(1, kmax[:, None])[:, 0], torch.zeros(R, dtype=torch.bool, device=mx.device)
    c1 = float(np.float32(inv_temp) * LOG2E_F32)
    mass = s * torch.exp2((mx.double() - M.double()) * c1)
    cum = mass.cumsum(-1)
    total = cum[:, -1]
    target = u1.double() * total
    hit = cum > target[:, None]
    k = torch.where(hit.any(-1), first_true(hit), kmax)
    ambiguous = ((cum - target[:, None]).abs() <= AMBIGUOUS_REL * total[:, None]).any(-1)
    return k * TILE + cand.gather(1, k[:, None])[:, 0], ambiguous
