"""CPU: Interface orchestration (SURVEY.md §8 rows A1-A3 + build_mask) pinned against the ORIGINAL project's own code.

The original's vampnet/interface.py was run by oracle/gen_reference_golden.py with the same stand-in models as here
(`generate` is a deterministic pure function of (start_tokens, mask)); its outputs and the generate calls its models
saw are stored in tests/golden/reference_interface.npz.  Our `coarse_vamp`, `coarse_to_fine`, `vamp` and
`build_mask` must reproduce them exactly: chunking, edge anchors, padding, codebook stacking, time stretch, feedback
passes, mask composition and RNG consumption.  The oracle's restatement (oracle/vampnet_oracle.py) is checked in the
same breath, which is what lets the GPU tests rely on it."""
import os

import numpy as np
import pytest
import torch

from oracle import vampnet_oracle as vo
from oracle.gen_reference_golden import BUILD_MASK_KWS, UNIT_SECONDS, calls_signature
from tests.test_interface_cpu import MASK_TOKEN, StubCodec, StubModel, fake_generate, rand_case


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "reference_interface.npz"))


def g(golden, key):
    return torch.from_numpy(golden[key]).long()


def make_iface(coarse_s=0.6, c2f_s=0.25):
    from vampnet_b200.interface import Interface
    coarse, c2f = StubModel(4, 0, salt=5), StubModel(14, 4, salt=9)
    coarse.chunk_size_s, c2f.chunk_size_s = coarse_s, c2f_s
    return Interface.from_models(StubCodec(), coarse, c2f, device="cpu", coarse_chunk_size_s=coarse_s,
                                 coarse2fine_chunk_size_s=c2f_s)


@pytest.mark.parametrize("T", [1, 34, 35, 36, 83, 140])
def test_coarse_vamp(golden, T):
    ours = make_iface()
    z, mask = rand_case(2, T, seed=T)
    if T > 70:
        mask[:, :, 70:] = 1
    want, want_start = g(golden, f"coarse_vamp_T{T}"), g(golden, f"coarse_vamp_T{T}_start")
    got, got_start = ours.coarse_vamp(z, mask, return_mask=True, temperature=0.7)
    assert torch.equal(got, want) and torch.equal(got_start, want_start)
    o, o_start = vo.coarse_vamp(z, mask, 4, ours.s2t(0.6), MASK_TOKEN, lambda s, m: fake_generate(s, m, 5))
    assert torch.equal(o, want) and torch.equal(o_start, want_start)
    assert calls_signature(ours.coarse.calls, ("shape", "kwargs")) == str(golden[f"coarse_vamp_T{T}_calls"])


@pytest.mark.parametrize("T,n_in", [(15, 14), (29, 14), (30, 4), (47, 14), (1, 4)])
def test_coarse_to_fine(golden, T, n_in):
    ours = make_iface()
    z, mask = rand_case(2, T, seed=100 + T)
    z = z[:, :n_in]
    key = f"c2f_T{T}_n{n_in}"
    want, want_start = g(golden, key), g(golden, key + "_start")
    got, got_start = ours.coarse_to_fine(z, mask=mask, return_mask=True)
    assert torch.equal(got, want) and torch.equal(got_start, want_start)
    o, o_start = vo.coarse_to_fine(z, mask, 14, 4, ours.s2t(0.25), MASK_TOKEN, lambda s, m: fake_generate(s, m, 9))
    assert torch.equal(o, want) and torch.equal(o_start, want_start)
    assert torch.equal(ours.coarse_to_fine(z, mask=None), g(golden, key + "_nomask"))
    assert calls_signature(ours.c2f.calls, ("time_steps", "shape", "kwargs")) == str(golden[key + "_calls"])


@pytest.mark.parametrize("batch,feedback,stretch,T", [(1, 1, 1, 83), (3, 1, 1, 40), (2, 2, 1, 61), (2, 3, 2, 37),
                                                       (1, 1, 3, 20)])
def test_vamp(golden, batch, feedback, stretch, T):
    ours = make_iface()
    z, mask = rand_case(1, T, seed=7 * T + batch)
    kw = dict(batch_size=batch, feedback_steps=feedback, time_stretch_factor=stretch, return_mask=True, temperature=1.3)
    key = f"vamp_{batch}_{feedback}_{stretch}_{T}"
    want, want_mask = g(golden, key), g(golden, key + "_mask")
    got, got_mask = ours.vamp(z, mask, **kw)
    assert torch.equal(got, want) and torch.equal(got_mask, want_mask)
    o, o_mask = vo.vamp(z, mask, batch, feedback, stretch, 4, 14, 4, ours.s2t(0.6), ours.s2t(0.25), MASK_TOKEN,
                        lambda s, m: fake_generate(s, m, 5), lambda s, m: fake_generate(s, m, 9))
    assert torch.equal(o, want) and torch.equal(o_mask, want_mask)
    assert calls_signature(ours.c2f.calls, ("kwargs",)) == str(golden[key + "_calls"])


@pytest.mark.parametrize("i", range(len(BUILD_MASK_KWS)), ids=lambda i: f"kw{i}")
def test_build_mask(golden, i):
    ours = make_iface()
    z, _ = rand_case(2, 97, seed=3)
    torch.manual_seed(11)
    got = ours.build_mask(z, **BUILD_MASK_KWS[i])
    assert torch.equal(got, g(golden, f"build_mask{i}"))
    # the same draws were consumed in the same order: the global stream continues identically
    assert torch.equal(torch.rand(4), torch.from_numpy(golden[f"build_mask{i}_next_draws"]))


def test_units(golden):
    ours = make_iface()
    assert [ours.s2t(s) for s in UNIT_SECONDS] == golden["units_s2t"].tolist()
    assert [ours.s2t2s(s) for s in UNIT_SECONDS] == golden["units_s2t2s"].tolist()
    assert ours.t2s(575) == float(golden["units_t2s_575"])
