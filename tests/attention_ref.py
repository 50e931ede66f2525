"""Float64 reference of the fused attention kernel's C ABI (vnb_op_attention / vnb_dbg_attention_ragged), the bound on
the kernel's error derived from its rounding points, and the probes whose correct outputs are known exactly.

Operands as the kernel takes them: qk (B, T, 2d) bf16 = [q | k], vT (B, d, Tpad) bf16, rel (2 sat + 1, H) fp32, sat,
frames (B,) key length per batch row or None (every row T); d = 64 H.  For batch row b with n = frames[b] keys, head h
and query q < n, over the keys k < n:

    x_k = q.k / 8 + rel[clamp(k - q, -sat, sat) + sat, h],   p = softmax(x),   o = sum_k p_k v_k,   A = sum_k p_k |v_k|

The bound.  The kernel (attention_wgmma.cu) works in the log2 domain and rounds at these points; u = 2^-24 (fp32),
u_b = 2^-8 (bf16, round to nearest: half an ulp of an 8-bit significand):

  1. S = q.k on the tensor cores: 64 exact bf16 products in four k16 steps.  A step adds its products to the
     accumulator with an error of at most E_STEP = 48 * 2^-23 of the sum of magnitudes it adds (any grouping of the
     products with alignment truncation and a truncating normalisation: a group of g terms errs by at most
     (g + 2) 2^-23 of the magnitudes, 16 / g groups per step), so |S - s| <= 4 E_STEP sum_i |q_i k_i|.
  2. t = fma(S, c, rel * log2 e) with c = fl(0.125 fl(log2 e)): c, the table entry and the fma round once each.
  3. m = the running maximum of the computed t (exact); t - m and the rescale exponent m_old - m_new round once each;
     over a row the rescale exponents telescope to at most 2 max|t|.
  Together, in natural units, every key's exponent is off by at most
     Delta = (4 E_STEP + 3 * 2^-23 + 2^-22) max_k D_k,   D_k = sum_i |q_i k_i| / 8 + |rel_k|   (per row),
  plus the relative error of ex2.approx (2 ulp = 2^-22) of its own exponential and of each rescale factor alpha it
  passes through: at most nblk + 1 of them, nblk = ceil(n / 64).  These errors are common to the numerator and to l,
  so the normalised weights move by a factor in [e^-2D, e^2D] with D = Delta + (nblk + 1) * -log(1 - 2^-22), and
  the exact softmax output moves by at most (e^2D - 1) A.
  4. P is rounded to bf16 before P.V (numerator only): u_b per weight.
  5. O accumulates P.V on the tensor cores, four k16 steps per key block, and is rescaled by alpha once per block:
     eps_O = nblk (4 E_STEP + u) of the sum of magnitudes.  l is summed on the CUDA cores in fp32 (16 keys per
     thread per block in pairs, one rescale per block, two shuffle adds): every term carries a factor within
     gamma(17 nblk + 2), gamma(k) = k u / (1 - k u).
  6. 1 / l and O * (1 / l) round (an approximate reciprocal included): gamma(3).
  7. ex2.approx.ftz flushes weights below 2^-126 (relative to a row maximum of weight 1, and l >= 1/2), and the tensor
     core may flush products below 2^-126: at most n 2^-125 (1 + max|v|) in all.
  8. The bf16 output: u_b |o_k|, and a bf16 subnormal half ulp 2^-134.

With e2 = e^2D - 1 and gamma_l = gamma(17 nblk + 2):

    |o_k - o| <= e2 A                                                         (3: weights)
               + [gamma_l (|o| + e2 A) + (u_b + eps_O (1 + u_b)) (1 + e2) A] / (1 - gamma_l)   (4, 5: P rounding, sums)
               + gamma(3) (|o| + ...)                                          (6)
               + n 2^-125 (1 + max|v|)                                         (7)
    |got - o| <= u_b |o| + (1 + u_b) |o_k - o| + 2^-134                        (8)

To first order this is u_b |o| + (u_b + eps_O + 2 Delta') A + gamma_l |o|.  `bound` computes it elementwise.

Probes with exact answers (q = 0 makes every score the bias alone; needles make one score 60 nats above all others)
and their expected outputs are built below; `MUTANTS` lists kernel bugs the reference can reproduce, so that a test
on this machine's CPU shows that the GPU probes would see them.
"""
from __future__ import annotations

import math

import torch

U = 2.0 ** -24          # fp32 unit roundoff
U_BF16 = 2.0 ** -8      # bf16 unit roundoff (8-bit significand, round to nearest)
E_STEP = 48 * 2.0 ** -23
EX2 = 2.0 ** -22        # ex2.approx.f32: 2 ulp
AK = 64                 # keys per block
BLOCK_BYTES = 256 << 20  # largest float64 score block the reference materialises

# The probe sweeps.  A warp's block offset lo = 64 j - qw - 15 is always 1 mod 16, so at sat = 1 mod 16 the one-value
# test holds with equality and at sat = 2 mod 16 a test loosened by one would misfire; T = 768 >= 2 sat + 80 reaches
# the one-value blocks on both sides for every sat.
BIAS_SATS = (1, 2, 16, 17, 18, 64, 91, 97, 98, 113, 114, 127, 128)
BIAS_TS = (3, 64, 65, 200, 575, 768)
NEEDLE_SHAPES = ((2, 1, 2), (2, 3, 2), (2, 64, 2), (2, 65, 2), (2, 129, 2), (2, 1000, 2), (2, 3072, 2), (1, 575, 20))
NEEDLE_RAGGED_T = 768
NEEDLE_RAGGED = (1, 63, 64, 65, 127, 128, 129, 200, NEEDLE_RAGGED_T)

# Kernel bugs the reference can reproduce (test_attention_ref_cpu's power checks; DESIGN §6 lists the GPU mutants).
MUTANTS = (
    "key_gt_len",          # the ragged last block's mask is key > len: key len takes part (its k row / v^T column)
    "edge_sat_minus_1",    # the one-value branch reads bias[+-(sat - 1)]
    "one_value_loose",     # the one-value condition loosened by one: lo >= sat - 1, lo + 78 <= -sat + 1
    "head_plus_1",         # the bias is read from head (h + 1) % H
    "no_l_rescale",        # l[r] *= alpha[r] removed
    "left_edge_entry1",    # the table fill clamps to entry 1 on the left: bias[-sat] and its copies hold bias[-sat+1]
)


def gamma(k):
    return k * U / (1.0 - k * U)


def _keys(qk, vT, b, n, T, d, extra):
    """k (nk, d) and v (nk, d) float64 of batch row b: its n keys, plus key n if extra (the kernel's TMA reads k rows
    past T and v^T columns past Tpad as zeros)."""
    k = qk[b, :n, d:].double()
    v = vT[b, :, :n].double().t()
    if extra:
        zk = qk.new_zeros(1, d, dtype=torch.float64)
        k = torch.cat([k, qk[b, n:n + 1, d:].double() if n < T else zk])
        v = torch.cat([v, vT[b, :, n:n + 1].double().t() if n < vT.shape[2] else zk])
    return k, v


def _bias_index(qi, ki, sat, n, mutant):
    """Table entry (rows, keys) read for queries qi and keys ki, with the kernel's branch structure where a mutant
    needs it: a warp's 16 rows against a 64-key block take the one-value branch when the block is wholly beyond
    +-sat (lo = 64 j - qw - 15, qw the warp's first row), unless it is the ragged last block."""
    r = ki[None, :] - qi[:, None]
    idx = r.clamp(-sat, sat) + sat
    if mutant in ("edge_sat_minus_1", "one_value_loose"):
        nblk = (n + AK - 1) // AK
        j = ki[None, :] // AK
        lo = AK * j - (qi[:, None] - qi[:, None] % 16) - 15
        slack = 1 if mutant == "one_value_loose" else 0
        plain = ~((n % AK != 0) & (j == nblk - 1))
        hi = plain & (lo >= sat - slack)
        lw = plain & (lo + 78 <= -sat + slack)
        if mutant == "edge_sat_minus_1":
            idx = torch.where(hi, torch.full_like(idx, 2 * sat - 1), torch.where(lw, torch.full_like(idx, 1), idx))
        else:
            idx = torch.where(hi, torch.full_like(idx, 2 * sat), torch.where(lw, torch.zeros_like(idx), idx))
    return idx


def attention_ref(qk, vT, rel, sat, frames=None, mutant=None):
    """o, A (B, T, d) float64 on qk's device (rows q >= frames[b] are 0), D (B, T, H) = max_k D_k, and the per-row
    key counts n (B,).  mutant: one of MUTANTS, to reproduce that kernel bug instead."""
    assert mutant is None or mutant in MUTANTS, mutant
    B, T, d2 = qk.shape
    d = d2 // 2
    H = d // 64
    dev = qk.device
    lens = [T] * B if frames is None else [int(x) for x in frames]
    tab = rel.double().to(dev)
    if mutant == "left_edge_entry1":
        tab = tab.clone()
        tab[0] = tab[1]
    heads = torch.arange(H, device=dev)
    if mutant == "head_plus_1":
        heads = (heads + 1) % H
    o = torch.zeros(B, T, d, dtype=torch.float64, device=dev)
    A = torch.zeros_like(o)
    D = torch.zeros(B, T, H, dtype=torch.float64, device=dev)
    for b, n in enumerate(lens):
        extra = mutant == "key_gt_len" and n % AK != 0
        k, v = _keys(qk, vT, b, n, T, d, extra)
        nk = k.shape[0]
        kh, vh = k.view(nk, H, 64).transpose(0, 1), v.view(nk, H, 64).transpose(0, 1)   # (H, nk, 64)
        ki = torch.arange(nk, device=dev)
        rows = max(1, BLOCK_BYTES // (8 * H * nk))
        for q0 in range(0, n, rows):
            q1 = min(n, q0 + rows)
            qh = qk[b, q0:q1, :d].double().view(q1 - q0, H, 64).transpose(0, 1)
            qi = torch.arange(q0, q1, device=dev)
            bias = tab[_bias_index(qi, ki, sat, n, mutant)][..., heads].permute(2, 0, 1)   # (H, rows, nk)
            x = qh @ kh.transpose(1, 2) / 8 + bias
            Dk = (qh.abs() @ kh.abs().transpose(1, 2) / 8 + bias.abs())
            D[b, q0:q1] = Dk.amax(-1).t()
            del Dk
            m = x.amax(-1, keepdim=True)
            w = torch.exp(x - m)
            if mutant == "no_l_rescale":
                nb = (nk + AK - 1) // AK
                xb = torch.nn.functional.pad(x, (0, nb * AK - nk), value=-math.inf).view(H, q1 - q0, nb, AK)
                mj = xb.amax(-1).cummax(-1).values
                l = torch.exp(xb - mj[..., None]).sum((-1, -2))
                del xb
            else:
                l = w.sum(-1)
            o[b, q0:q1] = ((w @ vh) / l[..., None]).transpose(0, 1).reshape(q1 - q0, d)
            A[b, q0:q1] = ((w @ vh.abs()) / w.sum(-1)[..., None]).transpose(0, 1).reshape(q1 - q0, d)
            del x, w, bias
    return o, A, D, torch.tensor(lens)


def bound(o, A, D, lens, vT, exps=True):
    """Elementwise bound (B, T, d) on |kernel - o| (module docstring).  exps=False: every weight is exactly 1 or 0 in
    fp32 and bf16 (the bias probes' rows), so only the sums, the division and the output round."""
    B, T, d = o.shape
    H = d // 64
    dev = o.device
    n = lens.to(dev, torch.float64)[:, None, None]
    nblk = torch.ceil(n / AK)
    vmax = torch.stack([vT[b, :, :int(lens[b])].double().abs().amax() for b in range(B)]).to(dev)[:, None, None]
    eps_o = nblk * (4 * E_STEP + U)
    g_l = gamma(17 * nblk + 2)
    if exps:
        delta = (4 * E_STEP + 3 * 2.0 ** -23 + 2.0 ** -22) * D.repeat_interleave(64, dim=2) \
            - (nblk + 1) * math.log1p(-EX2)
        e2 = torch.expm1(2 * delta)
        p_round = U_BF16
    else:
        e2 = torch.zeros_like(o)
        p_round = 0.0
    dev_w = e2 * A
    o_t = o.abs() + dev_w
    dev_s = (g_l * o_t + (p_round + eps_o * (1 + p_round)) * (A + dev_w)) / (1 - g_l)
    dev_k = dev_w + dev_s + gamma(3) * (o_t + dev_s) + n * 2.0 ** -125 * (1 + vmax)
    return U_BF16 * o.abs() + (1 + U_BF16) * dev_k + 2.0 ** -134


def vT_of(v, Tpad):
    """v (B, T, d) -> the kernel's v^T operand (B, d, Tpad), zero-padded."""
    B, T, d = v.shape
    vT = v.new_zeros(B, d, Tpad)
    vT[:, :, :T] = v.transpose(1, 2)
    return vT


def pad_with(vT, lens, T, value):
    """A copy of vT with `value` in every column the mask must exclude: [lens[b], Tpad) of each batch row (lens None:
    [T, Tpad))."""
    vT = vT.clone()
    for b in range(vT.shape[0]):
        vT[b, :, (T if lens is None else lens[b]):] = value
    return vT


def padding_probe(lens, T, H=2):
    """Random qk, rel (sat 128) and a vT with 1e4 in every column the mask must exclude (pad_with): an extra key would
    move the output by about 1e4 / n.  lens None: one batch row at T (columns [T, Tpad) only)."""
    B = 1 if lens is None else len(lens)
    d = 64 * H
    g = torch.Generator().manual_seed(T + B)
    qk = torch.randn(B, T, 2 * d, generator=g).bfloat16()
    vT = vT_of(torch.randn(B, T, d, generator=g).bfloat16(), (T + 7) // 8 * 8)
    rel = torch.randn(2 * 128 + 1, H, generator=g) * 0.5
    return qk, pad_with(vT, lens, T, 1e4), rel


def values(shape, g):
    """+-(0.5 + |N(0,1)|) in bf16: no value near 0, so a missing or extra weight moves the output."""
    x = torch.randn(shape, generator=g)
    sign = torch.randint(0, 2, shape, generator=g) * 2 - 1
    return (sign * (0.5 + x.abs())).bfloat16()


# ------------------------------------------------------------------------------------------------------ bias probes
def rstars(sat):
    """The peak offsets of the bias probe: both one-value edges, the entries next to them, and the centre."""
    return sorted({-sat, -sat + 1, -1, 0, 1, sat - 1, sat})


def bias_probe(B, T, sat, seed):
    """q = 0, so every score is the bias alone.  Head h's table is 0 except entry r*_h = rstars(sat)[h], which holds
    +100.  k random, v = values().  Returns qk, vT (CPU, bf16), rel (fp32) and the offsets."""
    rs = rstars(sat)
    H = len(rs)
    d = 64 * H
    g = torch.Generator().manual_seed(seed)
    qk = torch.zeros(B, T, 2 * d, dtype=torch.bfloat16)
    qk[..., d:] = torch.randn(B, T, d, generator=g).bfloat16()
    vT = vT_of(values((B, T, d), g), (T + 7) // 8 * 8)
    rel = torch.zeros(2 * sat + 1, H)
    for h, r in enumerate(rs):
        rel[r + sat, h] = 100.0
    return qk, vT, rel, rs


def bias_probe_expect(vT, T, sat, rs, lens=None):
    """Closed form of the bias probe: (expected (B, T, d) float64, exact (B, T, d) bool, A (B, T, d)).  A row whose
    peak offset |r*| < sat lands on a valid key is exactly that key's v (every other weight is below e^-100); a row with
    r* = +-sat averages v over the keys at distance >= sat on that side; a row with no key at the peak averages all
    its valid keys."""
    B, d, _ = vT.shape
    lens = [T] * B if lens is None else list(lens)
    exp = torch.zeros(B, T, d, dtype=torch.float64)
    A = torch.zeros_like(exp)
    exact = torch.zeros(B, T, d, dtype=torch.bool)
    for b, n in enumerate(lens):
        v = vT[b, :, :n].double().t()                                  # (n, d)
        cs = torch.cat([torch.zeros(1, d, dtype=torch.float64), v.cumsum(0)])
        ca = torch.cat([torch.zeros(1, d, dtype=torch.float64), v.abs().cumsum(0)])
        q = torch.arange(n)
        for h, r in enumerate(rs):
            cols = slice(64 * h, 64 * h + 64)
            lo, hi = torch.zeros_like(q), torch.full_like(q, n)          # key range averaged: all valid keys
            if abs(r) < sat:
                key = q + r
                hit = (key >= 0) & (key < n)
                exp[b, q[hit], cols] = v[key[hit], cols]
                A[b, q[hit], cols] = v[key[hit], cols].abs()
                exact[b, q[hit], cols] = True
                q_mean = q[~hit]
                lo, hi = lo[~hit], hi[~hit]
            else:
                q_mean = q
                if r == sat:
                    side = q + sat < n
                    lo = torch.where(side, q + sat, lo)
                else:
                    side = q - sat >= 0
                    hi = torch.where(side, q - sat + 1, hi)
            cnt = (hi - lo).double()[:, None]
            exp[b, q_mean, cols] = (cs[hi, cols] - cs[lo, cols]) / cnt
            A[b, q_mean, cols] = (ca[hi, cols] - ca[lo, cols]) / cnt
    return exp, exact, A


# ---------------------------------------------------------------------------------------------------- needle probes
def needle_pairs(n):
    """Transpositions the permutation must contain: 0 <-> n-1, and where the row reaches them the block edges
    63 <-> 64 and 127 <-> 128 and the 3-stage K/V ring's wrap 191 <-> 192 (block 2 -> block 3, stage 2 -> stage 0)."""
    pairs, used = [], set()
    for a, c in ((0, n - 1), (63, 64), (127, 128), (191, 192)):
        if c < n and a != c and a not in used and c not in used:
            pairs.append((a, c))
            used |= {a, c}
    return pairs


def needle_probe(lens, T, H, seed):
    """Keys are +-1 vectors; query i of batch row b is 32 k_{pi_b(i)} for a permutation pi_b of the row's valid keys
    (needle_pairs forced, the rest random), so the needle's score is 256 + rel.  The table is random with |rel| <= 2.
    Padded q / k rows (i >= lens[b]) hold NaN, padded v^T columns 0.  Returns qk, vT (CPU bf16), rel, pi (B, T) with
    pi[b, i] = -1 past the row's length."""
    B, d = len(lens), 64 * H
    g = torch.Generator().manual_seed(seed)
    k = (torch.randint(0, 2, (B, T, d), generator=g) * 2 - 1).float()
    v = values((B, T, d), g)
    rel = torch.rand(2 * 128 + 1, H, generator=g) * 4 - 2
    pi = torch.full((B, T), -1, dtype=torch.long)
    qk = torch.full((B, T, 2 * d), float("nan"))
    for b, n in enumerate(lens):
        p = torch.full((n,), -1, dtype=torch.long)
        for a, c in needle_pairs(n):
            p[a], p[c] = c, a
        free = (p < 0).nonzero().flatten()
        p[free] = free[torch.randperm(free.numel(), generator=g)]
        pi[b, :n] = p
        qk[b, :n, :d] = 32 * k[b, p]
        qk[b, :n, d:] = k[b, :n]
    vT = vT_of(v, (T + 7) // 8 * 8)
    for b, n in enumerate(lens):
        vT[b, :, n:] = 0
    return qk.bfloat16(), vT, rel, pi


def needle_gap(qk, rel, pi, sat=128):
    """Smallest float64 margin (nats) between a row's needle score and its other scores, over every (b, h, row)."""
    B, T, d2 = qk.shape
    d = d2 // 2
    H = d // 64
    gap = math.inf
    tab = rel.double().to(qk.device)
    for b in range(B):
        n = int((pi[b] >= 0).sum())
        q = qk[b, :n, :d].double().view(n, H, 64).transpose(0, 1)
        k = qk[b, :n, d:].double().view(n, H, 64).transpose(0, 1)
        ar = torch.arange(n, device=qk.device)
        x = q @ k.transpose(1, 2) / 8 + tab[(ar[None, :] - ar[:, None]).clamp(-sat, sat) + sat].permute(2, 0, 1)
        p = pi[b, :n].to(qk.device)
        needle = x[:, ar, p]
        x[:, ar, p] = -math.inf
        gap = min(gap, float((needle - x.amax(-1)).min()))
    return gap


def needle_expect(vT, pi):
    """out[b, i] = v[b, pi(i)] (B, T, d) float64; rows past the length are 0."""
    B, d, _ = vT.shape
    T = pi.shape[1]
    exp = torch.zeros(B, T, d, dtype=torch.float64)
    for b in range(B):
        n = int((pi[b] >= 0).sum())
        exp[b, :n] = vT[b, :, :n].double().t()[pi[b, :n]]
    return exp
