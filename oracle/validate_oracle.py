"""TEST INFRASTRUCTURE — the validation metrics of the reference's training script (scripts/exp/train.py val_loop,
_metrics, accuracy; :155-213, 327-371) restated in float64 numpy from given logits (DESIGN.md §12).

    target    = codebook_flatten(z[:, ncc:])       (B, S), s = t * Cp + c, the logits' row order
    flat_mask = codebook_flatten(mask[:, ncc:])
    loss      = ((1 - eps) sum nll + eps sum smooth) / n over the n masked rows, nll = lse - x[t], smooth = lse - mean x
                (nn.CrossEntropyLoss(label_smoothing=eps, ignore_index=-100)); NaN for n = 0
    accuracy  = correct / rows over the rows of the items whose r lies in [0, 0.5) or [0.5, 1.0), masked or unmasked;
                NaN for no rows.  gt = #{c : x[c] > x[t]}, eq = #{c != t : x[c] == x[t]}: correct iff gt + eq < k,
                a tie (gt < k <= gt + eq) counts as not correct and as ambiguous (torch.topk breaks it its own way)

row_stats also gives each row's top-k decision margin |x[t] - o[k-1]|, o the other logits in descending order: the
decision cannot change under logit errors below half of it.
"""
from __future__ import annotations

import numpy as np

KEYS = ("loss",) + tuple(f"accuracy-{s}-{e}/top{k}/{sel}" for s, e in ((0, 0.5), (0.5, 1.0)) for k in (1, 25)
                         for sel in ("unmasked", "masked"))
RANGES = ((0.0, 0.5), (0.5, 1.0))
TOPK = (1, 25)


def codebook_flatten(x: np.ndarray) -> np.ndarray:
    """(B, C, T) -> (B, T * C), s = t * C + c (the reference's rearrange "b c t -> b (t c)", util.py)."""
    B, C, T = x.shape
    return np.ascontiguousarray(np.transpose(x, (0, 2, 1))).reshape(B, T * C)


def targets(z: np.ndarray, mask: np.ndarray, ncc: int):
    """(target, flat_mask), both (B, S) int64."""
    return codebook_flatten(np.asarray(z)[:, ncc:]).astype(np.int64), codebook_flatten(np.asarray(mask)[:, ncc:]).astype(np.int64)


def row_stats(logits: np.ndarray, target: np.ndarray) -> dict:
    """logits (N, V), target (N,) -> float64 lse, nll, smooth; int64 gt, eq; margin[k] for k in TOPK."""
    x = np.asarray(logits, dtype=np.float64)
    t = np.asarray(target, dtype=np.int64)
    N, V = x.shape
    m = x.max(axis=1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(x - m).sum(axis=1))
    xt = x[np.arange(N), t]
    gt = (x > xt[:, None]).sum(axis=1)
    eq = (x == xt[:, None]).sum(axis=1) - 1
    others = x.copy()
    others[np.arange(N), t] = -np.inf
    o = -np.sort(-others, axis=1)  # descending; the target's own column last
    margin = {k: np.abs(xt - o[:, k - 1]) if k <= V - 1 else np.full(N, np.inf) for k in TOPK}
    return dict(lse=lse, nll=lse - xt, smooth=lse - x.mean(axis=1), gt=gt, eq=eq, margin=margin)


def metrics(logits: np.ndarray, target: np.ndarray, flat_mask: np.ndarray, r: np.ndarray, label_smoothing: float = 0.1):
    """logits (B, S, V), target / flat_mask (B, S), r (B,) -> (values, ambiguous, stats): values and ambiguous are
    dicts over KEYS (float64 metrics; tie counts, 0 for the loss), stats the row_stats of all B * S rows."""
    B, S, V = logits.shape
    st = row_stats(np.asarray(logits).reshape(B * S, V), np.asarray(target).reshape(-1))
    sel_m = np.asarray(flat_mask).reshape(-1) != 0
    n = int(sel_m.sum())
    eps = float(label_smoothing)
    values = {"loss": ((1 - eps) * st["nll"][sel_m].sum() + eps * st["smooth"][sel_m].sum()) / n if n else np.nan}
    ambiguous = {"loss": 0}
    item = np.repeat(np.arange(B), S)
    r = np.asarray(r, dtype=np.float64)
    keys = iter(KEYS[1:])
    for lo, hi in RANGES:
        in_range = ((r >= lo) & (r < hi))[item]
        for k in TOPK:
            correct = st["gt"] + st["eq"] < k
            tie = (st["gt"] < k) & ~correct
            for sel in (~sel_m, sel_m):
                rows = in_range & sel
                key = next(keys)
                cnt = int(rows.sum())
                values[key] = np.float32(correct[rows].sum()) / np.float32(cnt) if cnt else np.nan
                ambiguous[key] = int(tie[rows].sum())
    return values, ambiguous, st
