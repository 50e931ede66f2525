"""GPU: the validation-metric kernels (csrc/validate.cu) through the C ABI on seeded fp32 logits, against the float64
oracle (oracle/validate_oracle.py):
* per-row nll / smooth within 1e-12 relative, gt / eq exact, planted ties at the top-1 and top-25 boundaries counted as
  ambiguous (neither correct nor wrong);
* the 9 outputs: loss within 1e-6 relative, accuracies bit for bit (NaN where the oracle's is NaN);
* a B = 8 launch's records equal each item run alone, and two launches give the same bits;
* the reference's validation shape (B = 8, T = 575, coarse Cp = 4 and c2f Cp = 10);
* every refusal, with the library working afterwards; an out-of-range code gives NaN without an error."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import validate_oracle as vor

pytestmark = pytest.mark.gpu

ROW = np.dtype([("nll", "<f8"), ("smooth", "<f8"), ("gt", "<i4"), ("eq", "<i4")])


def lib():
    from vampnet_b200 import _lib
    return _lib


def rows_of(logits, z, ncc):
    """vnb_dbg_xent_rows: the per-row records as a numpy structured array (B * S,)."""
    L = lib()
    B, Cb, T = z.shape
    out = torch.empty(B * T * (Cb - ncc) * ROW.itemsize, dtype=torch.uint8, device="cuda")
    L.check(L.lib().vnb_dbg_xent_rows(L.ptr(logits), L.ptr(z), B, Cb, T, ncc, logits.shape[-1], L.ptr(out),
                                      L.stream_ptr()))
    return out.cpu().numpy().view(ROW)


def metrics(logits, z, mask, r, ncc, eps=0.1):
    from vampnet_b200.metrics import xent_metrics
    out, amb = xent_metrics(logits, z, mask, r, ncc, eps, return_ambiguous=True)
    return out.cpu().numpy(), amb.cpu().numpy()


def case(B, Cb, ncc, T, V, seed, plant=True):
    """Seeded logits (B, S, V) fp32, codes, a random binary mask and r on the device, with ties planted: row 3k + 1 has
    its target tied with another column at the top (top-1 ambiguous), row 3k + 2 its target tied with the 25th largest
    other (top-25 ambiguous), every 5th row its target strictly on top."""
    g = torch.Generator().manual_seed(seed)
    S = T * (Cb - ncc)
    z = torch.randint(0, V, (B, Cb, T), generator=g)
    mask = (torch.rand(B, Cb, T, generator=g) < 0.6).long()
    x = torch.randn(B, S, V, generator=g) * 2
    target, _ = vor.targets(z.numpy(), mask.numpy(), ncc)
    target = torch.from_numpy(target)
    if plant:
        for b in range(B):
            for s in range(S):
                t = int(target[b, s])
                row = x[b, s]
                if s % 3 == 1 and V > 1:
                    other = (t + 1 + s % (V - 1)) % V
                    row[t] = row[other] = row.max() + 0.5
                elif s % 3 == 2 and V > 25:
                    others = torch.cat([row[:t], row[t + 1:]])
                    row[t] = others.sort(descending=True).values[24]
                elif s % 5 == 0:
                    row[t] = row.max() + 1.0
    r = torch.rand(B, generator=g, dtype=torch.float64)
    return [v.cuda() for v in (x, z, mask, r)]


def check_against_oracle(x, z, mask, r, ncc, eps=0.1, want_ties=True):
    rec = rows_of(x, z, ncc)
    target, flat_mask = vor.targets(z.cpu().numpy(), mask.cpu().numpy(), ncc)
    vals, amb, st = vor.metrics(x.cpu().numpy(), target, flat_mask, r.cpu().numpy(), eps)
    assert np.array_equal(rec["gt"], st["gt"]) and np.array_equal(rec["eq"], st["eq"])
    for f in ("nll", "smooth"):
        err = np.abs(rec[f] - st[f]) / np.maximum(np.abs(st[f]), 1e-300)
        assert err.max() <= 1e-12, (f, err.max())
    out, got_amb = metrics(x, z, mask, r, ncc, eps)
    want = np.array([vals[k] for k in vor.KEYS])
    assert (np.isnan(out[0]) and np.isnan(want[0])) or abs(out[0] - want[0]) <= 1e-6 * abs(want[0]), (out[0], want[0])
    assert np.array_equal(out[1:], want[1:].astype(np.float32), equal_nan=True), (out, want)
    assert list(got_amb) == [amb[k] for k in vor.KEYS]
    if want_ties:
        assert got_amb[1:].sum() > 0
    return out


@pytest.mark.parametrize("B,Cb,ncc,T,V", [(3, 4, 0, 7, 1024), (2, 14, 4, 3, 1024), (3, 5, 2, 9, 100), (2, 3, 1, 5, 4),
                                          (2, 4, 0, 6, 132)])
def test_rows_and_metrics_match_oracle(B, Cb, ncc, T, V):
    x, z, mask, r = case(B, Cb, ncc, T, V, seed=B * 100 + V)
    r[0] = 0.25
    r[1] = 0.75  # both ranges populated
    check_against_oracle(x, z, mask, r, ncc, want_ties=V > 25)
    for eps in (0.0, 1.0, 0.37):
        check_against_oracle(x, z, mask, r, ncc, eps, want_ties=V > 25)


def test_ratio_edges_and_empty_selections():
    """r = 1.0 and r < 0 are in neither range, r = 0.5 is in the second, r = 0 in the first; empty selections and a mask
    with nothing masked give NaN."""
    x, z, mask, r = case(4, 4, 0, 5, 1024, seed=7)
    r[:] = torch.tensor([0.0, 0.5, 1.0, -0.1], dtype=torch.float64)
    out = check_against_oracle(x, z, mask, r, 0)
    assert not np.isnan(out[1:]).any()
    r[:] = torch.tensor([1.0, 1.0, 0.2, 0.3], dtype=torch.float64)
    out = check_against_oracle(x, z, mask, r, 0)
    assert np.isnan(out[5:]).all() and not np.isnan(out[1:5]).any()
    out = check_against_oracle(x, z, torch.zeros_like(mask), r, 0)
    assert np.isnan(out[0]) and np.isnan(out[[2, 4]]).all() and not np.isnan(out[[1, 3]]).any()


def test_batch_rows_equal_rows_alone_and_runs_repeat():
    B, Cb, ncc, T, V = 8, 14, 4, 11, 1024
    x, z, mask, r = case(B, Cb, ncc, T, V, seed=3)
    rec = rows_of(x, z, ncc)
    S = T * (Cb - ncc)
    for b in range(B):
        alone = rows_of(x[b:b + 1].contiguous(), z[b:b + 1].contiguous(), ncc)
        assert alone.tobytes() == rec[b * S:(b + 1) * S].tobytes(), b
    assert rows_of(x, z, ncc).tobytes() == rec.tobytes()
    a, amb_a = metrics(x, z, mask, r, ncc)
    b_, amb_b = metrics(x, z, mask, r, ncc)
    assert a.tobytes() == b_.tobytes() and np.array_equal(amb_a, amb_b)


@pytest.mark.parametrize("Cb,ncc", [(4, 0), (14, 4)])
def test_reference_validation_shape(Cb, ncc):
    """B = 8 ten-second clips (T = 575): coarse (S = 2300) and c2f (S = 5750) rows of V = 1024."""
    x, z, mask, r = case(8, Cb, ncc, 575, 1024, seed=Cb, plant=False)
    r[:] = torch.linspace(0.05, 0.95, 8, dtype=torch.float64)
    check_against_oracle(x, z, mask, r, ncc, want_ties=False)


def test_out_of_range_code_gives_nan_without_error():
    x, z, mask, r = case(2, 4, 0, 5, 1024, seed=9, plant=False)
    r[:] = torch.tensor([0.2, 0.7], dtype=torch.float64)
    ok, _ = metrics(x, z, mask, r, 0)
    assert not np.isnan(ok).any()
    zb = z.clone()
    zb[1, 2, 3] = 1024  # the mask token: a masked-input code, never a target
    mask[1, 2, 3] = 1
    out, _ = metrics(x, zb, mask, r, 0)
    assert np.isnan(out[0]) and np.isnan(out[[6, 8]]).all()    # the loss, the second range's masked accuracies
    assert np.array_equal(out[1:5], ok[1:5])                    # the first range does not hold the row
    rec = rows_of(x, zb, 0)
    bad = 1 * 20 + 3 * 4 + 2
    assert np.isnan(rec["nll"][bad]) and rec["gt"][bad] == -1
    zb[1, 2, 3] = -5
    out, _ = metrics(x, zb, mask, r, 0)
    assert np.isnan(out[0])


def test_refusals_leave_the_library_working():
    L = lib()
    F = L.lib().vnb_xent_metrics
    x, z, mask, r = case(2, 4, 0, 5, 1024, seed=11, plant=False)
    need = C.c_uint64()
    L.check(L.lib().vnb_xent_metrics_workspace_bytes(2, 20, C.byref(need)))
    ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    out = torch.empty(9, device="cuda")
    p = L.ptr
    base = dict(logits=p(x), z=p(z), mask=p(mask), r=p(r), B=2, C=4, T=5, ncc=0, V=1024, ls=0.1, ws=p(ws),
                wsb=need.value, out=p(out))

    def call(**kw):
        a = dict(base, **kw)
        return F(a["logits"], a["z"], a["mask"], a["r"], a["B"], a["C"], a["T"], a["ncc"], a["V"], a["ls"], a["ws"],
                 a["wsb"], a["out"], None, L.stream_ptr())

    odd = torch.empty(2 * 20 * 1024 + 1, device="cuda")
    bad = [dict(logits=None), dict(z=None), dict(mask=None), dict(r=None), dict(ws=None), dict(out=None), dict(B=0),
           dict(C=0), dict(T=0), dict(ncc=-1), dict(ncc=4), dict(V=0), dict(V=1028), dict(V=1022), dict(ls=-0.01),
           dict(ls=1.01), dict(ls=float("nan")), dict(wsb=need.value - 1), dict(logits=C.c_void_p(odd.data_ptr() + 4))]
    for kw in bad:
        assert call(**kw) != 0, kw
        assert L.lib().vnb_last_error(), kw
    with pytest.raises(RuntimeError):
        L.check(L.lib().vnb_xent_metrics_workspace_bytes(0, 20, C.byref(need)))
    with pytest.raises(RuntimeError):
        L.check(L.lib().vnb_dbg_xent_rows(p(x), p(z), 2, 4, 5, 0, 1022, p(out), L.stream_ptr()))
    assert call() == 0
    want, _ = metrics(x, z, mask, r, 0)
    assert np.array_equal(out.cpu().numpy(), want, equal_nan=True)
