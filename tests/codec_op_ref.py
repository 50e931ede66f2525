"""Float64 references of the codec kernels at the level of their C ABI (vnb_codec_conv_tc, vnb_codec_conv_in,
vnb_codec_conv_out, vnb_codec_rvq, vnb_codec_conv1d): channels-last activations, packed split-bf16 weights and the
offset / limit / batch-stride store, exactly as the entry points take them.  tests/test_codec_op_ref_cpu.py ties each
of them to the layers of oracle/dac_oracle.py; tests/test_gpu_codec_ops.py holds the kernels to them.

Every function works on the device of its inputs and returns float64 tensors."""
from __future__ import annotations

import torch

HH_HL_LH = ("hh", "hl", "lh")   # the three products the tensor-core kernel forms (lo * lo is below fp32 grade)
ALL_PRODUCTS = HH_HL_LH + ("ll",)


def snake(v, alpha):
    """Snake with alpha broadcast over the last dimension: v + sin^2(alpha v) / (alpha + 1e-9)."""
    a = alpha.double()
    return v + torch.sin(a * v).pow(2) / (a + 1e-9)


def conv_tc_acc(a_hi, a_lo, w_hi, w_lo, s, N, taps, dil, pad, Tq, products=HH_HL_LH):
    """The accumulator of the tensor-core convolution before its epilogue:
        y[b, q, n] = sum_tap sum_ci sum_(products) W[n, tap, ci] * a[b, q*s + tap*dil - pad, ci]
    with a = (B, Tin, Cin) channels-last (zero outside [0, Tin)) and W the packed (N, taps * cblocks * 64) weights.
    Returns y (B, Tq, N) and the root-sum-square of the per-term products (the scale of fp32 accumulation error)."""
    B, Tin, Cin = a_hi.shape
    cb = (Cin + 63) // 64
    W = {"h": w_hi.double().view(N, taps, cb * 64)[:, :, :Cin], "l": w_lo.double().view(N, taps, cb * 64)[:, :, :Cin]}
    dev = a_hi.device
    y = torch.zeros(B, Tq, N, dtype=torch.float64, device=dev)
    r2 = torch.zeros_like(y)
    q = torch.arange(Tq, device=dev)
    for tap in range(taps):
        idx = q * s + tap * dil - pad
        ok = ((idx >= 0) & (idx < Tin)).double()[None, :, None]
        ic = idx.clamp(0, Tin - 1)
        A = {"h": a_hi[:, ic].double() * ok, "l": a_lo[:, ic].double() * ok}
        for p in products:
            a, w = A[p[0]], W[p[1]][:, tap].t()
            y += a @ w
            r2 += (a * a) @ (w * w)
    return y, r2.sqrt()


def conv_tc_store(y, rss, bias, bias_mod, alpha, alpha_mod, resid, out_batch_stride, out_offset, out_limit, do_tanh):
    """The epilogue and store of the tensor-core convolution.  Element (q, n) of y goes to flat position
    q*N + n + out_offset of each batch item when that lies in [0, out_limit).  Returns (pos, f32, act, rss, skip):
    the written flat positions (P,), the fp32-stream value (B, P) (bias, skip, tanh applied), the split output's value
    (B, P) (= snake_next(f32) when alpha is given), the accumulator's rss and |skip| at those positions."""
    B, Tq, N = y.shape
    dev = y.device
    n = torch.arange(N, device=dev)
    flat = torch.arange(Tq, device=dev)[:, None] * N + n[None, :] + out_offset
    ok = (flat >= 0) & (flat < out_limit)
    pos, nn = flat[ok], n.expand(Tq, N)[ok]
    v = y[:, ok]
    if bias is not None:
        v = v + bias.double()[nn % bias_mod]
    skip = torch.zeros_like(v)
    if resid is not None:
        skip = resid.double().reshape(B, out_batch_stride)[:, pos]
        v = v + skip
    if do_tanh:
        v = torch.tanh(v)
    act = snake(v, alpha[nn % alpha_mod]) if alpha is not None else v
    return pos, v, act, rss[:, ok], skip.abs()


def conv_in(x, w, bias, pad):
    """encoder.conv1 at the ABI of vnb_codec_conv_in: x (B, T) -> y (B, T, C) channels-last, and sum |terms|."""
    B, T = x.shape
    C, _, K = w.shape
    xp = torch.nn.functional.pad(x.double(), (pad, K - 1 - pad))
    cols = xp.unfold(1, K, 1)                        # (B, T, K): x[t + k - pad]
    wk = w.double().reshape(C, K).t()                # (K, C)
    y = cols @ wk + bias.double()
    return y, cols.abs() @ wk.abs() + bias.double().abs()


def conv_out(a_hi, a_lo, w, bias, pad):
    """decoder.conv2 at the ABI of vnb_codec_conv_out: a = hi + lo (B, T, C) -> audio (B, T) = tanh(bias + conv),
    and the sum |terms| of the convolution."""
    B, T, C = a_hi.shape
    K = w.shape[-1]
    a = a_hi.double() + a_lo.double()
    ap = torch.nn.functional.pad(a, (0, 0, pad, K - 1 - pad))
    cols = ap.unfold(1, K, 1)                        # (B, T, C, K)
    wk = w.double().reshape(C, K)
    y = torch.einsum("btck,ck->bt", cols, wk) + bias.double()
    return torch.tanh(y), torch.einsum("btck,ck->bt", cols.abs(), wk.abs())


def conv1d(x, w, bias, alpha, resid, Tout, stride, dil, pad, out_stride, out_off, nq, do_tanh, y_init):
    """vnb_codec_conv1d (channels-first, fp32 CUDA-core path):
        y[b, co, q*out_stride + out_off] = bias[co] + sum_ci sum_j W[co, ci, j] * act(x[b, ci, q*stride + j*dil - pad])
    (+ resid at the same index, tanh optional) for q < nq and 0 <= index < Tout; act = snake_alpha or identity, applied
    before the zero padding.  Positions not written keep y_init.  Returns (y, written mask (Tout,), rss of the terms,
    and the error scale sum |W| (|x| + 1/alpha) + |bias| + |resid| that covers the fp32 Snake's rounding)."""
    B, Cin, Tin = x.shape
    Cout, _, K = w.shape
    dev = x.device
    a = x.double()
    mag = a.abs()
    if alpha is not None:
        a = snake(a.transpose(1, 2), alpha).transpose(1, 2)
        mag = mag + 1.0 / alpha.double()[None, :, None]
    q = torch.arange(nq, device=dev)
    acc = torch.zeros(B, Cout, nq, dtype=torch.float64, device=dev)
    r2 = torch.zeros_like(acc)
    ab = torch.zeros_like(acc)
    for j in range(K):
        idx = q * stride + j * dil - pad
        ok = ((idx >= 0) & (idx < Tin)).double()
        ic = idx.clamp(0, Tin - 1)
        xs = a[:, :, ic] * ok
        wj = w[:, :, j].double()
        acc += torch.einsum("oc,bct->bot", wj, xs)
        r2 += torch.einsum("oc,bct->bot", wj * wj, xs * xs)
        ab += torch.einsum("oc,bct->bot", wj.abs(), mag[:, :, ic] * ok)
    if bias is not None:
        acc += bias.double()[None, :, None]
        ab += bias.double().abs()[None, :, None]
    yo = q * out_stride + out_off
    keep = (yo >= 0) & (yo < Tout)
    y = y_init.double().clone()
    cols = yo[keep]
    v = acc[:, :, keep]
    if resid is not None:
        v = v + resid.double()[:, :, cols]
    if do_tanh:
        v = torch.tanh(v)
    y[:, :, cols] = v
    written = torch.zeros(Tout, dtype=torch.bool, device=dev)
    written[cols] = True
    rss, scale = torch.zeros_like(y), torch.zeros_like(y)
    rss[:, :, cols] = r2[:, :, keep].sqrt()
    scale[:, :, cols] = ab[:, :, keep] + (resid.double()[:, :, cols].abs() if resid is not None else 0.0)
    return y, written, rss, scale


def code_divergence(codes, latents, ref):
    """Where the kernel's codes leave the float64 reference's.  codes (B, L, T) and latents (B, 8L, T) are the
    kernel's, ref is rvq(...) of the same input.  For each frame, `first` is the first level whose code differs (L if
    none); later levels of that frame see a different residual and are not comparable.  err_en is the largest L2 error
    of the normalised latent on the comparable levels (up to and including `first`); a score difference between two
    unit codebook vectors moves by at most 4 err_en, so delta = 4 err_en + 2^-20 (fp32 rounding of the score itself)
    bounds a legitimate near-tie.  gap is the float64 score of the reference's pick minus that of the kernel's pick at
    level `first` (0 where the frame agrees throughout)."""
    B, L, T = codes.shape
    dev = ref["codes"].device
    codes = codes.to(dev)
    diff = codes != ref["codes"]
    anyd = diff.any(1)
    first = torch.where(anyd, diff.int().argmax(1), torch.full((B, T), L, device=dev, dtype=torch.int64))
    lv = torch.arange(L, device=dev)[None, :, None]
    comparable = lv <= first[:, None, :]
    e = latents.to(dev).double().view(B, L, 8, T).permute(0, 1, 3, 2)
    en = e / e.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    err_en = (en - ref["en"]).norm(dim=-1)[comparable].max().item()
    gap = torch.zeros(B, T, dtype=torch.float64, device=dev)
    b, t = anyd.nonzero(as_tuple=True)
    if b.numel():
        l = first[b, t]
        sc = ref["scores"][b, l, t]
        gap[b, t] = sc.gather(1, ref["codes"][b, l, t][:, None])[:, 0] - sc.gather(1, codes[b, l, t][:, None])[:, 0]
    return dict(first=first, err_en=err_en, delta=4 * err_en + 2.0 ** -20, gap=gap, comparable=comparable)


def rvq(mode, in_f, in_codes, win, bin_, wout, bout, cb, cbn, L, channels_last=False):
    """vnb_codec_rvq in float64.  mode 0 encodes z, 1 re-quantises latents, 2 decodes codes.  Nearest code per level:
    argmax_v of the oracle's score -(|en|^2 - 2 en.cbn_v) + |cbn_v|^2 with en = e / max(|e|, 1e-12), first index on
    ties (torch.max).  Returns a dict: codes (B, L, T) int64, latents (B, 8L, T), zq (B, D, T) channels-first,
    scores (B, L, T, V), en (B, L, T, 8), and the error scales zq_scale (B, D, T) = |z| + sum_l |out_l| and
    lat_scale (B, L, 8, T) = sum_d |win x res| + |bin|."""
    f64 = torch.float64
    if mode == 2:
        B, _, T = in_codes.shape
    elif mode == 1:
        B, _, T = in_f.shape
    else:
        B = in_f.shape[0]
        T = in_f.shape[1] if channels_last else in_f.shape[2]
    D = wout.shape[1]
    win, bin_, wout, bout, cb, cbn = (t.double() for t in (win, bin_, wout, bout, cb, cbn))
    dev = wout.device
    z = None
    if mode == 0:
        z = in_f.double().transpose(1, 2) if channels_last else in_f.double()
        res = z.clone()
        zscale = z.abs()
    else:
        res = torch.zeros(B, D, T, dtype=f64, device=dev)
        zscale = torch.zeros_like(res)
    codes, lats, scores, ens, lscale = [], [], [], [], []
    for l in range(L):
        if mode == 0:
            e = torch.einsum("jd,bdt->bjt", win[l], res) + bin_[l][:, None]
            lscale.append(torch.einsum("jd,bdt->bjt", win[l].abs(), res.abs()) + bin_[l].abs()[:, None])
        elif mode == 1:
            e = in_f[:, 8 * l:8 * l + 8].double()
        if mode != 2:
            en = e / e.norm(dim=1, keepdim=True).clamp_min(1e-12)
            sc = -(en.pow(2).sum(1)[:, :, None] - 2 * torch.einsum("bjt,vj->btv", en, cbn[l])) + cbn[l].pow(2).sum(1)
            idx = sc.max(-1)[1]
            scores.append(sc)
            ens.append(en.transpose(1, 2))
        else:
            idx = in_codes[:, l].long()
        qv = cb[l][idx].transpose(1, 2)            # (B, 8, T)
        if mode == 1:
            qv = e + (qv - e)
        out = torch.einsum("dj,bjt->bdt", wout[l], qv) + bout[l][:, None]
        zscale = zscale + out.abs()
        if mode == 0:
            res = res - out
            lats.append(e)
        else:
            res = res + out
        codes.append(idx)
    r = dict(codes=torch.stack(codes, 1), zq=(z - res) if mode == 0 else res, zq_scale=zscale)
    if mode == 0:
        r["latents"] = torch.cat(lats, 1)
        r["lat_scale"] = torch.stack(lscale, 1)
    if mode != 2:
        r["scores"] = torch.stack(scores, 1)
        r["en"] = torch.stack(ens, 1)
    return r
