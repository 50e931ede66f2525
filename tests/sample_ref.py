"""Float64 reference of one sampling step of the generate loop as vampnet_b200/csrc/sampler.cu makes it
(include/vampnet_b200.h, vnb_dbg_sample): the nucleus filter, the two-level inverse-CDF draw, the confidence and the
re-mask.  Plain torch on whatever device the inputs are on, in the style of tests/gemm_sample_ref.py, whose
`first_true`, `inv_temperature` and `AMBIGUOUS_REL` it shares.  tests/test_sample_ref_cpu.py pins it to the oracle's
sampler (OracleVampNet.sample_from_logits and mask_by_random_topk, rng="philox") on the CPU;
tests/test_gpu_sampler_ops.py holds the kernels to it on the GPU.

The kernels' inputs are fp32; the few fp32 roundings the kernels make before any arithmetic that matters are taken as
the kernels make them (fp32(1/T), the fp32 product x * inv_t, fp32(gamma * N0)); every other operation is float64.
Uniforms are oracle/philox.py's: counter (s, b - first, step, 0) words 0 and 1 for the draw, (s, b - first, step, 1)
word 0 for the confidence's Gumbel noise, where b - first is the row's index within its own group (generate call).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from oracle import philox
from tests.gemm_sample_ref import AMBIGUOUS_REL, first_true, inv_temperature

TILE = 128


@dataclass
class Group:
    """One generate() call's rows of a launch and its sampling scalars at one step (vnb_sample_group)."""
    rows: int
    temperature: float = 1.0
    gamma: float = 1.0
    temp_eff: float = 0.0
    do_sample: int = 1
    is_last: int = 0
    step: int = 0
    seed: tuple = (0, 0)
    top_p: float = 0.0


def top_p_on(top_p: float) -> bool:
    return 0.0 < top_p < 1.0


def nucleus(x: torch.Tensor, top_p: float):
    """x (R, V) fp32 RAW logits.  Returns (keep, uncertain), (R, V) bool each: v is kept iff the softmax mass of the
    tokens strictly above it, sum_{u: x_u > x_v} p_u, is <= top_p (float64), so tied logits are kept or dropped
    together (+0 and -0 are tied).  `uncertain` marks the tokens whose pre-mass lies within AMBIGUOUS_REL of top_p
    (fp32 sums may put them on either side; a row with one is an ambiguous row of the filter).  Disabled (everything
    kept, nothing uncertain) when top_p <= 0 or >= 1."""
    R, V = x.shape
    if not top_p_on(top_p):
        return torch.ones_like(x, dtype=torch.bool), torch.zeros_like(x, dtype=torch.bool)
    x64 = x.double()
    p = torch.softmax(x64, -1)
    xa, order = x64.sort(-1)                                    # ascending
    pd = p.gather(-1, order).flip(-1)                           # masses in descending order of x
    cum = torch.cat([torch.zeros(R, 1, dtype=torch.float64, device=x.device), pd.cumsum(-1)], -1)
    above = V - torch.searchsorted(xa.contiguous(), x64.contiguous(), right=True)   # entries strictly greater
    pre = cum.gather(-1, above)
    return pre <= top_p, (pre - top_p).abs() <= AMBIGUOUS_REL


def scaled(x: torch.Tensor, keep: torch.Tensor, inv_t: np.float32) -> torch.Tensor:
    """fp32(x * inv_t) with the filtered entries at -inf, as float64."""
    xs = x.masked_fill(~keep, -float("inf")) * torch.tensor(np.float32(inv_t), device=x.device)
    return xs.double()


def draw(x: torch.Tensor, keep: torch.Tensor, inv_t: np.float32, u1: torch.Tensor | None, u2: torch.Tensor | None):
    """The token of each row: x (R, V) fp32 raw logits, keep (R, V) the nucleus, u1 / u2 (R,) fp32 uniforms (None:
    greedy).  Sampling: with e = exp(xs - max xs) over the kept entries, the 128-entry tile whose running mass first
    exceeds u1 * sum(e) (tiles in vocabulary order), then the first entry of that tile whose running sum exceeds
    u2 * mass(tile).  Greedy: the arg-max of the raw logits, lowest index on ties.  Returns (token int64, ambiguous
    bool), (R,) each; a row is ambiguous where either crossing is within AMBIGUOUS_REL (relative to its sum) of its
    target, never on greedy steps."""
    R, V = x.shape
    if u1 is None:
        xf = x.masked_fill(~keep, -float("inf"))
        return first_true(xf == xf.max(-1, keepdim=True).values), torch.zeros(R, dtype=torch.bool, device=x.device)
    xs = scaled(x, keep, inv_t)
    e = torch.exp(xs - xs.max(-1, keepdim=True).values).view(R, V // TILE, TILE)
    cum_t = e.sum(-1).cumsum(-1)
    total = cum_t[:, -1]
    target = u1.double() * total
    k = first_true(cum_t > target[:, None])
    amb = ((cum_t - target[:, None]).abs() <= AMBIGUOUS_REL * total[:, None]).any(-1)
    cin = e.gather(1, k[:, None, None].expand(R, 1, TILE))[:, 0].cumsum(-1)
    tt = cin[:, -1]
    target_in = u2.double() * tt
    j = first_true(cin > target_in[:, None])
    amb |= ((cin - target_in[:, None]).abs() <= AMBIGUOUS_REL * tt[:, None]).any(-1)
    return k * TILE + j, amb


def log_prob(x: torch.Tensor, keep: torch.Tensor, inv_t: np.float32, token: torch.Tensor) -> torch.Tensor:
    """log softmax(filtered xs)[token] in float64, (R,)."""
    return torch.log_softmax(scaled(x, keep, inv_t), -1).gather(1, token[:, None].long())[:, 0]


def gumbel(u: torch.Tensor) -> torch.Tensor:
    """-log(-log u) in float64 of the fp32 uniforms u."""
    return -torch.log(-torch.log(u.double()))


def uniforms(seed, step: int, rows: int, S: int, device):
    """(u1, u2, u_conf), each (rows, S) fp32 on `device`, for rows 0 .. rows-1 of one group."""
    u = [philox.uniform_bs(seed, step, rows, S, stream=st, word=w) for st, w in ((0, 0), (0, 1), (1, 0))]
    return [torch.from_numpy(a).to(device) for a in u]


def sample_group(logits: torch.Tensor, g: Group):
    """One group's draw on its own: logits (rows, S, V) fp32 raw.  Returns a dict of (rows, S) tensors: token (int64),
    conf (float64: log p64(token) + fp32(temp_eff) * gumbel(u_conf)), logp, noise (fp32(temp_eff) * gumbel),
    ambiguous, logp_spread, and keep / uncertain (rows, S, V) from `nucleus`.  Known positions are the caller's
    business.  Where the nucleus has uncertain tokens, the draw is also made from the nucleus without them and with
    them: the position is ambiguous unless all three draws give the same unambiguous token, and logp_spread is how far
    log p(token) moves between the three sets (0 without uncertain tokens)."""
    rows, S, V = logits.shape
    x = logits.reshape(-1, V)
    keep, unc = nucleus(x, g.top_p)
    inv_t = inv_temperature(g.temperature)
    u1, u2, uc = uniforms(g.seed, g.step, rows, S, x.device)
    uu = (u1.reshape(-1), u2.reshape(-1)) if g.do_sample else (None, None)
    token, amb = draw(x, keep, inv_t, *uu)
    logp = log_prob(x, keep, inv_t, token)
    spread = torch.zeros_like(logp)
    if bool(unc.any()):
        for k in (keep & ~unc, keep | unc):
            t_k, a_k = draw(x, k, inv_t, *uu)
            amb |= a_k | (t_k != token)
            spread = torch.maximum(spread, (log_prob(x, k, inv_t, token) - logp).abs())
    noise = float(np.float32(g.temp_eff)) * gumbel(uc.reshape(-1))
    rs = lambda t: t.reshape(rows, S, *t.shape[1:])  # noqa: E731
    return dict(token=rs(token), conf=rs(logp + noise), logp=rs(logp), noise=rs(noise), ambiguous=rs(amb),
                logp_spread=rs(spread), keep=rs(keep), uncertain=rs(unc))


def num_to_mask(gamma: float, n0: int, cnt: int, S: int, is_last: bool) -> int:
    """remask_kernel's count: floor(fp32(gamma * N0)); unless last, clamped to [1, cnt - 1]; then to [0, S - 1]."""
    n = int(np.floor(np.float32(gamma) * np.float32(n0)))
    if not is_last:
        n = max(min(n, cnt - 1), 1)
    return max(min(n, S - 1), 0)


def remask(conf: torch.Tensor, tokens: torch.Tensor, zcur: torch.Tensor, zorig: torch.Tensor | None, ncc: int,
           mask_token: int, groups, n0) -> torch.Tensor:
    """zcur after the re-mask: conf, tokens (B, S) (conf compared as floats, so the kernel's own fp32 conf gives an
    exact answer), zcur / zorig (B, T, C) before the call, groups a list of Group, n0 the per-group initial mask
    counts.  For every row: cnt = masked positions of its predicted codebooks, n = num_to_mask(...), cut =
    sort(conf)[n], predicted entries = where(conf < cut, MASK, token); conditioning entries from zorig (unchanged when
    zorig is None)."""
    B, T, C = zcur.shape
    Cp = C - ncc
    S = T * Cp
    out = zcur.clone()
    b = 0
    for gi, g in enumerate(groups):
        for _ in range(g.rows):
            cnt = int((zcur[b, :, ncc:] == mask_token).sum())
            n = num_to_mask(g.gamma, int(n0[gi]), cnt, S, bool(g.is_last))
            cut = conf[b].sort().values[n]
            pred = torch.where(conf[b] < cut, torch.full_like(tokens[b], mask_token), tokens[b])
            out[b, :, ncc:] = pred.view(T, Cp).to(out.dtype)
            if zorig is not None and ncc > 0:
                out[b, :, :ncc] = zorig[b, :, :ncc]
            b += 1
    return out
