"""Validation metrics of the reference's training script (scripts/exp/train.py:155-213, 327-371) from a forward's
logits: the label-smoothed cross-entropy over the masked tokens and top-1 / top-25 accuracy split by mask ratio and by
masked / unmasked position, computed by the kernels of csrc/validate.cu (DESIGN.md §12).  VampNet.validate is the
user-facing entry; xent_metrics is the launch it makes."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib

# the reference's output keys, in its order (train.py:366, 182-213); also the order of the kernel's 9 outputs
KEYS = ("loss",) + tuple(f"accuracy-{s}-{e}/top{k}/{sel}" for s, e in ((0, 0.5), (0.5, 1.0)) for k in (1, 25)
                         for sel in ("unmasked", "masked"))


def xent_metrics(logits: torch.Tensor, z: torch.Tensor, mask: torch.Tensor, r: torch.Tensor, n_conditioning_codebooks: int,
                 label_smoothing: float = 0.1, return_ambiguous: bool = False):
    """logits (B, S, V) fp32, z and mask (B, C, T) int64, r (B,): all on one CUDA device; S = T * (C - ncc).
    Returns the 9 metrics in KEYS order as an fp32 (9,) tensor on that device without synchronising, and with
    return_ambiguous also the int32 (9,) counts of rows whose top-k decision is a tie at the k-th place."""
    B, C_, T = z.shape
    ncc = int(n_conditioning_codebooks)
    V = logits.shape[-1]
    dev = logits.device
    if logits.dtype != torch.float32 or tuple(logits.shape) != (B, T * (C_ - ncc), V):
        raise ValueError(f"xent_metrics: logits must be fp32 (B, T * (C - ncc), V) = ({B}, {T * (C_ - ncc)}, V), got "
                         f"{logits.dtype} {tuple(logits.shape)}")
    if tuple(mask.shape) != (B, C_, T):
        raise ValueError(f"xent_metrics: mask {tuple(mask.shape)} must have z's shape {(B, C_, T)}")
    logits = logits.contiguous()
    z = z.to(dev, torch.int64).contiguous()
    mask = mask.to(dev, torch.int64).contiguous()
    r = r.to(dev, torch.float64).contiguous()
    L = _lib.lib()
    need = C.c_uint64()
    _lib.check(L.vnb_xent_metrics_workspace_bytes(B, T * (C_ - ncc), C.byref(need)))
    ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
    out = torch.empty(len(KEYS), dtype=torch.float32, device=dev)
    amb = torch.empty(len(KEYS), dtype=torch.int32, device=dev) if return_ambiguous else None
    with torch.cuda.device(dev):
        _lib.check(L.vnb_xent_metrics(_lib.ptr(logits), _lib.ptr(z), _lib.ptr(mask), _lib.ptr(r), B, C_, T, ncc, V,
                                      float(label_smoothing), _lib.ptr(ws), need.value, _lib.ptr(out),
                                      _lib.ptr(amb) if amb is not None else None, _lib.stream_ptr(dev)))
    return (out, amb) if return_ambiguous else out
