"""GPU: per-request LoRA adapters end to end (VampNet.add_adapter, generate(adapter=), generate_many, forward_codes,
Interface.add_finetuned / vamp_many).

* forward_codes(adapter=X) on the base model meets the criteria the folded fine-tune meets (tests/test_gpu_parity.py
  test_forward_vs_oracle_and_golden, case coarse_lora) against the same golden and the fp32 / bf16 oracle; at the
  full-size coarse shape it stays within the measured bf16 floor of the folded model (tests/test_gpu_parity_shapes.py).
* generate_many with base, X and Y calls mixed equals the sequential generate(adapter=...) calls bit for bit and leaves
  the same RNG state (both sampler paths, tiny coarse and c2f); vamp_many with mixed adapter= requests equals the
  sequential vamp calls.
* Graphs: regrouping adapters across replays captures nothing new after the first adapted capture; a base-only launch
  with adapters registered launches no adapter kernel.  Unknown and removed ids are refused and the library keeps
  working."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import vampnet_oracle as vo
from tests.test_gpu_generate_many import assert_same_rng, mix, rng_state, reseed_globals, set_fused
from tests.test_gpu_parity import TINY_C2F, TINY_COARSE, StubCodec
from tests.test_gpu_parity_shapes import FULL_COARSE

pytestmark = pytest.mark.gpu


def base_with_adapters(cfgd, seed=0, n=2, cb_seed=1):
    """The base model of `n` LoRA fine-tunes (the fine-tunes of make_state_dict(seed, lora=True) without their LoRA
    tensors), with fine-tune i registered as adapter 'ft{i}' (its LoRA tensors redrawn from seed 100 + i, except ft0,
    which is the make_state_dict one).  Returns (cfg, fine-tune 0 state dict, model, codebooks, codec)."""
    from vampnet_b200.modules.transformer import VampNet
    cfg = vo.OracleConfig(**cfgd)
    sd = vo.make_state_dict(cfg, seed=seed, lora=True)
    model = VampNet(**cfgd)
    model.load_state_dict({k: v for k, v in sd.items() if ".lora_" not in k}, strict=False)
    model = model.to("cuda")
    model.add_adapter("ft0", sd)
    for i in range(1, n):
        g = torch.Generator().manual_seed(100 + i)
        other = {k: (torch.randn(v.shape, generator=g) * v.std() if ".lora_" in k else v) for k, v in sd.items()}
        model.add_adapter(f"ft{i}", other)
    cb = vo.make_codebooks(cfg.n_codebooks, seed=cb_seed)
    return cfg, sd, model, cb, StubCodec(cb.cuda())


def folded_model(cfgd, sd):
    from vampnet_b200.modules.transformer import VampNet
    m = VampNet(**cfgd)
    m.load_state_dict(sd)
    return m.to("cuda")


def test_forward_adapted_vs_oracle_and_golden(golden_dir):
    """Against the fp32 golden under the folded case's criteria (mean < 1.2e-2, max < 0.09), and no farther from the
    fp32 oracle than the folded model is (x 1.25).  The bf16-oracle bound of the folded case does not apply: that oracle
    rounds W + BA to bf16 as the folded model does, while an adapter adds B A x in fp32 to bf16(W) x, a different
    rounding of the same function (DESIGN.md §2)."""
    g = np.load(os.path.join(golden_dir, "forward_tiny_coarse_lora.npz"))
    cfg, sd, model, cb, codec = base_with_adapters(TINY_COARSE, seed=int(g["weight_seed"]), cb_seed=int(g["codebook_seed"]))
    codes = torch.from_numpy(g["codes"]).cuda()
    got = model.forward_codes(codes, codec, adapter="ft0").permute(0, 2, 1).cpu()
    folded = folded_model(TINY_COARSE, sd).forward_codes(codes, codec).permute(0, 2, 1).cpu()
    nref = g["logits"].shape[0]
    gold = torch.from_numpy(g["logits"])
    e32, f32 = (got[:nref] - gold).abs(), (folded[:nref] - gold).abs()
    ref32 = vo.OracleVampNet(cfg, sd, "fp32").forward(torch.from_numpy(g["latents"]))
    o32, of32 = (got - ref32).abs(), (folded - ref32).abs()
    print(f"[adapter] vs fp32 golden: max {e32.max():.3e} mean {e32.mean():.3e} (folded: max {f32.max():.3e} mean "
          f"{f32.mean():.3e}); vs fp32 oracle: mean {o32.mean():.3e} (folded {of32.mean():.3e})")
    assert e32.mean() < 1.2e-2 and e32.max() < 0.09
    assert o32.mean() <= 1.25 * of32.mean() and o32.max() <= 1.25 * of32.max()
    # the base rows of the same model are the plain forward; an adapter changes them
    base = model.forward_codes(codes, codec).permute(0, 2, 1).cpu()
    assert (base - got).abs().max() > 1e-2
    # per-row adapters in one launch equal one launch per adapter
    from vampnet_b200 import _lib as L
    B, T = codes.shape[0], codes.shape[-1]
    ids = [model._adapter_id(n) for n in (["ft0", None, "ft1"] * B)[:B]]
    logits = torch.empty(B, T * model.n_predict_codebooks, 1024, device="cuda")
    L.check(L.lib().vnb_forward_codes_adapted(model._handle, L.ptr(codes), B, T, (C.c_int32 * B)(*ids), L.ptr(logits),
                                              L.stream_ptr()))
    for b, name in enumerate((["ft0", None, "ft1"] * B)[:B]):
        alone = model.forward_codes(codes[b:b + 1], codec, adapter=name)
        assert torch.equal(logits[b:b + 1], alone), f"row {b} ({name}) differs from its own launch"


def test_full_coarse_adapted_vs_folded_within_bf16_floor():
    """Full-size coarse (d = 1280, 20 layers), B = 2, T = 768 (every 3rd frame masked): the adapted base and the folded
    fine-tune are two bf16 implementations of the same fp32 function.  The folded model's distance to the fp32 oracle
    on the last row is the bf16 floor of this shape; the adapted model must stay within 1.25x of it (max and mean), and
    its greedy decisions must be the oracle's wherever the fp32 margin allows (tests/test_gpu_parity_shapes.py)."""
    from tests.test_gpu_parity_shapes import assert_decisions_exact_where_margin_allows
    cfg, sd, model, cb, codec = base_with_adapters(FULL_COARSE, seed=0, n=1)
    g = torch.Generator().manual_seed(4)
    z = torch.randint(0, 1024, (2, 4, 768), generator=g)
    z[:, :, ::3] = 1024
    a = model.forward_codes(z.cuda(), codec, adapter="ft0")[1].cpu()
    del model
    f = folded_model(FULL_COARSE, sd).forward_codes(z.cuda(), codec)[1].cpu()
    orc = vo.OracleVampNet(cfg, sd, "fp32")
    ref32 = orc.forward(orc.from_codes(z[1:2], cb))[0].t()          # (S, V)
    ea, ef = (a - ref32).abs(), (f - ref32).abs()
    print(f"[full coarse] vs fp32 oracle: adapted max {ea.max():.3e} mean {ea.mean():.3e}; folded max {ef.max():.3e} "
          f"mean {ef.mean():.3e}; adapted vs folded max {(a - f).abs().max():.3e}")
    assert ea.mean() <= 1.25 * ef.mean() and ea.max() <= 1.25 * ef.max()
    assert_decisions_exact_where_margin_allows(a[None], ref32[None], "full coarse adapted")


def adapter_mix(cfgd, seed):
    """The generate_many mix of tests/test_gpu_generate_many.py with the calls spread over base, ft0 and ft1."""
    calls = mix(cfgd, seed)
    for i, c in enumerate(calls):
        name = (None, "ft0", "ft1")[i % 3]
        if name is not None:
            c["adapter"] = name
    return calls


@pytest.mark.parametrize("fused", [1, 0])
@pytest.mark.parametrize("tag,cfgd", [("coarse", TINY_COARSE), ("c2f", TINY_C2F)])
def test_generate_many_with_adapters_equals_sequential_calls(tag, cfgd, fused):
    _, _, model, _, codec = base_with_adapters(cfgd, seed=2)
    prev = set_fused(fused)
    try:
        calls = adapter_mix(cfgd, seed=31)
        reseed_globals(123)
        want = [model.generate(codec, **c) for c in calls]
        want_rng = rng_state()
        reseed_globals(123)
        got = model.generate_many(codec, calls)
        got_rng = rng_state()
        # the adapter matters: the same call on the base gives other tokens
        c = dict(calls[1], seed=11)
        c.pop("adapter")
        other = model.generate(codec, **c)
    finally:
        set_fused(prev)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape and torch.equal(a, b), f"[{tag}] call {i} ({calls[i].get('adapter')}) differs"
    assert_same_rng(got_rng, want_rng)
    assert not torch.equal(other, model.generate(codec, **dict(calls[1], seed=11)))


def profile(model, fn):
    from vampnet_b200 import _lib as L
    lib = L.lib()
    L.check(lib.vnb_profile_begin(model._handle))
    fn()
    ms, n = (C.c_float * 11)(), (C.c_int32 * 11)()
    L.check(lib.vnb_profile_end(model._handle, ms, n, 11))
    return list(n)


def test_graphs_launches_and_refusals():
    from vampnet_b200 import _lib as L
    lib = L.lib()
    _, _, model, _, codec = base_with_adapters(TINY_COARSE, seed=2, n=3)
    g = torch.Generator().manual_seed(0)
    z = torch.randint(0, 1024, (4, 4, 30), generator=g).cuda()

    def calls(names):
        return [dict(start_tokens=z[i:i + 1], _sampling_steps=3, seed=i, return_signal=False, adapter=n)
                for i, n in enumerate(names)]
    model.generate_many(codec, calls([None, "ft0", "ft1", None]))
    before = lib.vnb_graph_capture_count()
    for names in (["ft2", None, "ft0", "ft0"], ["ft1", "ft1", "ft1", "ft1"], [None, "ft2", None, "ft1"]):
        model.generate_many(codec, calls(names))
    assert lib.vnb_graph_capture_count() == before, "regrouping adapters captured a new graph"
    # a base-only launch runs the plain kernels: no down-projection, one GEMM per LoRA'd projection and layer
    n = profile(model, lambda: model.generate_many(codec, calls([None] * 4)))
    assert n[L.LORA_DOWN_FAMILY] == 0 and n[2] == 3 * model.n_layers
    n = profile(model, lambda: model.generate_many(codec, calls([None, "ft0", None, None])))
    assert n[L.LORA_DOWN_FAMILY] == 3 * 4 * model.n_layers and n[2] == 3 * model.n_layers
    torch.cuda.synchronize()
    # malformed ids, a removed adapter, a NULL weight pointer and a full table are refused; the library still works
    grp = _lib_group(L, 1)
    out = torch.empty_like(z[:1])
    gam = (C.c_float * 3)(0.5, 0.3, 0.0)
    for bad in (99, -2, model._adapter_id("ft2")):
        if bad == model._adapter_id("ft2"):
            model.remove_adapter("ft2")
        rc = lib.vnb_generate_many_adapted(model._handle, L.ptr(z[:1]), None, 1, 30, 3, gam, grp, 1,
                                           (C.c_int32 * 1)(bad), 1, L.ptr(out), L.stream_ptr())
        assert rc != 0 and b"not registered" in lib.vnb_last_error()
    with pytest.raises(KeyError):
        model.generate(codec, start_tokens=z[:1], _sampling_steps=3, adapter="ft2", return_signal=False)
    assert lib.vnb_adapter_remove(model._handle, 99) != 0
    w = L.AdapterWeights()
    i = C.c_int32()
    assert lib.vnb_adapter_add(model._handle, C.byref(w), C.byref(i)) != 0 and b"NULL" in lib.vnb_last_error()
    p = model._adapters["ft0"]
    full = L.AdapterWeights(**{k: v.data_ptr() for k, v in p.items()})
    added = []
    while lib.vnb_adapter_add(model._handle, C.byref(full), C.byref(i)) == 0:
        added.append(i.value)
    assert len(added) == L.MAX_ADAPTERS - 2 and b"full" in lib.vnb_last_error()
    for a in added:
        L.check(lib.vnb_adapter_remove(model._handle, a))
    a = model.generate(codec, start_tokens=z[:1], _sampling_steps=3, seed=1, adapter="ft1", return_signal=False)
    b = model.generate_many(codec, calls([None, "ft1"]))[1]
    assert a.shape == b.shape


def _lib_group(L, rows):
    tef = (C.c_float * 3)(10.0, 5.0, 0.0)
    dos = (C.c_int32 * 3)(1, 1, 1)
    grp = (L.GenGroup * 1)()
    grp[0].rows, grp[0].temperature, grp[0].temp_eff, grp[0].do_sample = rows, 1.0, tef, dos
    grp[0].seed_lo, grp[0].seed_hi, grp[0].top_p = 1, 0, 0.0
    _lib_group.keep = (tef, dos)
    return grp


def test_vamp_many_with_adapters_equals_sequential_vamp(tmp_path, monkeypatch):
    from tests.test_gpu_interface import C2F, CODEC, COARSE
    from oracle import dac_oracle as do
    from vampnet_b200.codec import DAC
    from vampnet_b200.interface import Interface
    from vampnet_b200.modules.transformer import VampNet
    codec = DAC(encoder_dim=CODEC.encoder_dim, encoder_rates=CODEC.encoder_rates, decoder_dim=CODEC.decoder_dim)
    codec.load_flat(do.make_codec_weights(CODEC, seed=0))
    models = {}
    for tag, cfgd, seed in (("coarse", COARSE, 0), ("c2f", C2F, 1)):
        sd = vo.make_state_dict(vo.OracleConfig(**cfgd), seed=seed, lora=True)
        m = VampNet(**cfgd)
        m.load_state_dict({k: v for k, v in sd.items() if ".lora_" not in k}, strict=False)
        models[tag] = m
        for name, s in (("x", 1), ("y", 2)):
            g = torch.Generator().manual_seed(s)
            ft = {k: (torch.randn(v.shape, generator=g) * v.std() if ".lora_" in k else v) for k, v in sd.items()}
            os.makedirs(tmp_path / "loras" / name, exist_ok=True)
            torch.save({"state_dict": ft, "metadata": {"kwargs": cfgd}}, tmp_path / "loras" / name / f"{tag}.pth")
    monkeypatch.setenv("VAMPNET_MODELS_DIR", str(tmp_path))
    iface = Interface.from_models(codec, models["coarse"], models["c2f"], device="cuda", coarse_chunk_size_s=0.6,
                                  coarse2fine_chunk_size_s=0.25)
    iface.add_finetuned("x")
    iface.add_finetuned("y")
    with pytest.raises(RuntimeError, match="not in the local model cache"):
        iface.add_finetuned("missing")
    g = torch.Generator().manual_seed(12)
    reqs = []
    for T, bs, fb, ad in [(83, 2, 1, "x"), (50, 1, 2, None), (61, 1, 1, "y"), (40, 2, 1, "x")]:
        z = torch.randint(0, 1024, (1, 14, T), generator=g).cuda()
        mask = (torch.rand(1, 14, T, generator=g) < 0.7).long().cuda()
        reqs.append(dict(codes=z, mask=mask, batch_size=bs, feedback_steps=fb, _sampling_steps=3, adapter=ad))
    reseed_globals(21)
    want = [iface.vamp(**r) for r in reqs]
    want_rng = rng_state()
    reseed_globals(21)
    got = iface.vamp_many(reqs)
    assert_same_rng(rng_state(), want_rng)
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), f"request {i} differs"
    reseed_globals(21)
    plain = iface.vamp(**dict(reqs[0], adapter=None))
    assert not torch.equal(plain, want[0])
