"""GPU: the forward, the sampling epilogue and generate at model geometries other than the shipped two.

vnb_model_create accepts d_model = 64 * n_heads for any multiple of 256, vocab_size 256, 512, 768 or 1024, 1 to 16
codebooks with any number of conditioning codebooks below that, and a relative-bias table saturating anywhere in
1 .. 128.  Every shipped model has V = 1024 (so the mask token is 1024, a codebook spans 8 sampling strips) and
d = 1280 or 256, Cp = 4 or 10.  The configurations below reach the geometry-dependent paths those never do:

  tag  d / H      V     C / ncc  what it reaches
  A    512 / 8    256   1 / 0    Cp = 1, 2 strips per codebook, embedding K = 8 of Kp = 64
  B    768 / 12   512   16 / 0   K = Kp = 128, d/256 = 3 embedding partials of 6, the largest Cp
  C    1024 / 16  768   9 / 2    6 strips, odd Cp = 7, K = 72 of Kp = 128
  D    256 / 4    1024  8 / 7    Cp = 1 with conditioning, K = Kp = 64
  E    1536 / 24  1024  14 / 4   wider than production: q/k columns up to 2d = 3072, 12 residual partials
  F    256 / 4    256   2 / 1    a bias table whose buckets beyond distance 3 are equal, cut to rel_sat = 3

The criteria are the shipped shapes' own (tests/test_gpu_parity.py, tests/test_gpu_parity_shapes.py,
tests/test_gpu_adapters.py, tests/test_gpu_generate_many.py); the oracle is pinned to the reference at V = 256 and 768
by tests/test_oracle_configs_vs_reference.py."""
import ctypes as C

import pytest
import torch

from oracle import vampnet_oracle as vo
from tests.test_gpu_generate_many import assert_same_rng, mix, rng_state, reseed_globals, set_fused
from tests.test_gpu_parity import StubCodec, _teacher_forced
from tests.test_gpu_parity_shapes import _calibrated_compare

pytestmark = pytest.mark.gpu


def _cfg(H, V, Cn, ncc, layers=2):
    return dict(n_heads=H, n_layers=layers, n_codebooks=Cn, n_conditioning_codebooks=ncc, embedding_dim=64 * H,
                vocab_size=V)


CONFIGS = {
    "A": _cfg(8, 256, 1, 0),
    "B": _cfg(12, 512, 16, 0),
    "C": _cfg(16, 768, 9, 2),
    "D": _cfg(4, 1024, 8, 7),
    "E": _cfg(24, 1024, 14, 4),
    "F": _cfg(4, 256, 2, 1),
}
TAGS = sorted(CONFIGS)
F_SAT = 3   # configuration F: relative-attention buckets of distance >= F_SAT share one weight per head and side


def _equal_tail_buckets(sd, sat):
    """The bucket weights of distance >= sat (buckets sat..15 for key < query, 16+sat..31 for key > query) made equal
    per head, so the bias is constant beyond distance sat - 1 on each side."""
    key = "transformer.layers.0.self_attn.relative_attention_bias.weight"
    w = sd[key].clone()
    w[sat:16] = w[sat]
    w[16 + sat:32] = w[16 + sat]
    sd[key] = w


def _trim_equal_ends(rel_bias_table):
    """rel_bias_table, then the table cut while both of its end rows equal their neighbours: the bias at every distance
    is unchanged (the kernel extends the end rows outwards), only rel_sat shrinks."""
    def table(weight):
        t, sat = rel_bias_table(weight)
        while sat > 1 and torch.equal(t[0], t[1]) and torch.equal(t[-1], t[-2]):
            t, sat = t[1:-1], sat - 1
        return t.contiguous(), sat
    return table


@pytest.fixture
def build_config(monkeypatch):
    """build_config(tag, seed=0, lora=False, base_only=False) -> (cfg, state dict, model on cuda:0, codebooks, codec),
    with vocab_size-entry codebooks.  base_only: the model gets the state dict without its LoRA tensors (an adapter's
    base).  For F the library's relative-bias table is cut to the smallest rel_sat that leaves the bias unchanged."""
    from vampnet_b200.modules import transformer as TR

    def make(tag, seed=0, lora=False, base_only=False, cb_seed=1):
        cfgd = CONFIGS[tag]
        cfg = vo.OracleConfig(**cfgd)
        sd = vo.make_state_dict(cfg, seed=seed, lora=lora)
        if tag == "F":
            _equal_tail_buckets(sd, F_SAT)
            monkeypatch.setattr(TR, "rel_bias_table", _trim_equal_ends(TR.rel_bias_table))
        model = TR.VampNet(**cfgd)
        res = model.load_state_dict({k: v for k, v in sd.items() if not (base_only and ".lora_" in k)}, strict=False)
        assert not res.unexpected_keys, res.unexpected_keys
        assert all("lora" in k for k in res.missing_keys), res.missing_keys
        model = model.to("cuda")
        cb = vo.make_codebooks(cfg.n_codebooks, vocab_size=cfg.vocab_size, seed=cb_seed)
        codec = StubCodec(cb.cuda())
        model._ensure_handle(codec)
        assert model._rel_sat == (F_SAT if tag == "F" else 91)
        return cfg, sd, model, cb, codec
    return make


def codes(cfg, B, T, seed, mask_every=3):
    """Random codes in [0, V] (the mask token included) with every `mask_every`-th frame masked in every codebook."""
    z = torch.randint(0, cfg.vocab_size + 1, (B, cfg.n_codebooks, T), generator=torch.Generator().manual_seed(seed))
    z[:, :, ::mask_every] = cfg.mask_token
    return z


def gen_inputs(cfg, B, T, seed, every):
    g = torch.Generator().manual_seed(seed)
    z = torch.randint(0, cfg.vocab_size, (B, cfg.n_codebooks, T), generator=g)
    mask = torch.ones_like(z)
    mask[:, :, ::every] = 0
    mask[:, :cfg.n_conditioning_codebooks, :] = 0
    return z, mask


# ---------------------------------------------------------------------------------------------------- 1. embedding
@pytest.mark.parametrize("tag", TAGS)
def test_embedding_is_fp32_grade(build_config, tag):
    """With every projection that feeds the residual stream zeroed, the final residual stream is the embedding: within
    3e-5 relative of the float64 einsum, with the mask token in every codebook; the latents entry point is identical."""
    cfg, sd, model, cb, codec = build_config(tag, seed=4)
    sd = dict(sd)
    for k in list(sd):
        if k.endswith("self_attn.fc.weight") or k.endswith("feed_forward.w_2.weight"):
            sd[k] = torch.zeros_like(sd[k])
    model.load_state_dict(sd, strict=False)
    B, T = 2, 37
    z = codes(cfg, B, T, seed=8, mask_every=5)
    z[:, :, 1] = cfg.mask_token
    assert all(bool((z[:, c] == cfg.vocab_size).any()) for c in range(cfg.n_codebooks))
    model.forward_codes(z.cuda(), codec)
    x = model.hidden_state(B, T).cpu()
    orc = vo.OracleVampNet(cfg, sd, "fp32")
    lat = orc.from_codes(z, cb)
    want = torch.einsum("bkt,nk->btn", lat.double(), orc.emb_w.double()) + orc.emb_b.double()
    err = (x.double() - want).abs().max().item()
    bound = 3e-5 * max(1.0, want.abs().max().item())
    print(f"[{tag}] embedding: max err {err:.2e}, ratio to bound {err / bound:.3f}")
    assert err < bound
    model(lat.cuda())
    assert torch.equal(model.hidden_state(B, T).cpu(), x)


# ---------------------------------------------------------------------------------------------------- 2. forward
FORWARD = [(t, T) for t in TAGS for T in (37, 131)] + [("E", 575)]


@pytest.mark.parametrize("tag,T", FORWARD, ids=[f"{t}_T{T}" for t, T in FORWARD])
def test_forward_calibrated(build_config, tag, T):
    """B = 3, so batch boundaries fall inside a 128-row tile: every row equals its own B = 1 run and a repeated call
    on the same workspace, bit for bit; the first and last rows meet the calibrated criteria of
    tests/test_gpu_parity_shapes.py (within 1.5x of the bf16 oracle's jitter floor, decisions exact where the fp32
    margin is safe)."""
    cfg, sd, model, cb, codec = build_config(tag, seed=1)
    B = 3
    z = codes(cfg, B, T, seed=100 + T)
    got = model.forward_codes(z.cuda(), codec).clone()
    again = model.forward_codes(z.cuda(), codec)
    assert torch.equal(got, again), "a second call on the same workspace differs"
    for b in range(B):
        alone = model.forward_codes(z[b:b + 1].cuda(), codec)
        assert torch.equal(alone[0], got[b]), f"row {b} of the batch differs from its B=1 run"
    assert got.shape == (B, T * cfg.n_predict_codebooks, cfg.vocab_size)
    orc = vo.OracleVampNet(cfg, sd, "fp32")
    rows = (0, B - 1) if T < 575 else (B - 1,)
    _calibrated_compare(cfg, sd, [got[b].t().cpu() for b in rows], [orc.from_codes(z[b:b + 1], cb) for b in rows],
                        f"{tag} T={T}")


# ---------------------------------------------------------------------------------------------------- 3. greedy generate
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("steps", [1, 6])
@pytest.mark.parametrize("tag", TAGS)
def test_generate_greedy_bit_exact_given_logits(build_config, tag, steps, graph):
    cfg, sd, model, cb, codec = build_config(tag)
    model.use_cuda_graph = graph
    orc = vo.OracleVampNet(cfg, sd, "bf16")
    z, mask = gen_inputs(cfg, 3, 40, seed=11, every=7)
    kw = dict(sample_cutoff=-1.0, mask_temperature=0.0)
    want = orc.generate(cb, z.clone(), mask.clone(), _sampling_steps=steps, rng="philox", philox_key=(5, 0),
                        logits_fn=_teacher_forced(model, codec), **kw)
    for _ in range(2):  # the second call replays the captured graph
        got = model.generate(codec, start_tokens=z.cuda(), mask=mask.cuda(), _sampling_steps=steps, seed=5,
                             return_signal=False, **kw).cpu()
        assert torch.equal(got, want), f"{(got != want).sum().item()} of {got.numel()} tokens differ"
    assert not (got == cfg.mask_token).any() and int(got.max()) < cfg.vocab_size
    assert torch.equal(got[mask == 0], z[mask == 0])


# ---------------------------------------------------------------------------------------------------- 4. sampled generate
SAMPLED = [dict(), dict(temperature=0.9, top_p=0.85), dict(top_p=0.5, sample_cutoff=-1.0, mask_temperature=0.0)]
SAMPLED_IDS = ["sample", "sample_top_p", "greedy_top_p"]


@pytest.mark.parametrize("kw", SAMPLED, ids=SAMPLED_IDS)
@pytest.mark.parametrize("tag", TAGS)
def test_generate_sampled_matches_oracle_with_shared_noise(build_config, tag, kw):
    """Under the shared Philox stream the tokens are the oracle's except at its numerical near-ties (libm vs CUDA
    logf / expf), at most 0.2 % of them, as at the shipped shapes."""
    cfg, sd, model, cb, codec = build_config(tag)
    orc = vo.OracleVampNet(cfg, sd, "bf16")
    z, mask = gen_inputs(cfg, 2, 33, seed=12, every=5)
    seed = 1234567
    want = orc.generate(cb, z.clone(), mask.clone(), _sampling_steps=6, rng="philox", philox_key=(seed, 0),
                        logits_fn=_teacher_forced(model, codec), **kw)
    got = model.generate(codec, start_tokens=z.cuda(), mask=mask.cuda(), _sampling_steps=6, seed=seed,
                         return_signal=False, **kw).cpu()
    diff = (got != want).float().mean().item()
    print(f"[{tag} {kw}] sampled-token mismatch fraction {diff:.5f} (ratio to bound {diff / 0.002:.3f})")
    assert diff <= 0.002
    assert torch.equal(got[mask == 0], z[mask == 0])
    assert not (got == cfg.mask_token).any()


@pytest.mark.parametrize("kw", SAMPLED[:2] + [dict(sample_cutoff=-1.0, mask_temperature=0.0)],
                         ids=["sample", "sample_top_p", "greedy"])
@pytest.mark.parametrize("tag", TAGS)
def test_fused_sampler_equals_materialised_sampler(build_config, tag, kw):
    """Sampling inside the classifier GEMM's epilogue and from the materialised logits give the same tokens, eager
    and graph-replayed.  T = 150: two row tiles with a ragged tail."""
    from vampnet_b200 import _lib as L
    cfg, sd, model, cb, codec = build_config(tag)
    z, mask = gen_inputs(cfg, 3, 150, seed=23, every=5)
    prev = set_fused(1)
    outs = []
    try:
        for fused in (1, 0):
            L.check(L.lib().vnb_set_option(b"fused_sampler", fused))
            for graph in (False, True):
                model.use_cuda_graph = graph
                outs.append(model.generate(codec, start_tokens=z.cuda(), mask=mask.cuda(), _sampling_steps=5, seed=17,
                                           return_signal=False, **kw).cpu())
    finally:
        set_fused(prev)
    assert not (outs[0] == cfg.mask_token).any() and int(outs[0].max()) < cfg.vocab_size
    for o in outs[1:]:
        assert torch.equal(outs[0], o), f"{(outs[0] != o).sum().item()} of {o.numel()} tokens differ"


# ---------------------------------------------------------------------------------------------------- 5. generate_many
@pytest.mark.parametrize("fused", [1, 0])
@pytest.mark.parametrize("tag", ["A", "D"])
def test_generate_many_equals_sequential_calls(build_config, tag, fused):
    """A (V = 256, Cp = 1) and D (Cp = 1 under 7 conditioning codebooks): the mix of tests/test_gpu_generate_many.py
    (two lengths, two step counts, a top-p bucket) batched equals the calls one by one, and the RNG state after."""
    cfg, sd, model, cb, codec = build_config(tag)
    prev = set_fused(fused)
    try:
        calls = mix(CONFIGS[tag], seed=31)
        reseed_globals(123)
        want = [model.generate(codec, **c) for c in calls]
        want_rng = rng_state()
        reseed_globals(123)
        got = model.generate_many(codec, calls)
        got_rng = rng_state()
    finally:
        set_fused(prev)
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape and torch.equal(a, b), f"[{tag}] call {i} differs"
        assert int(a[:, cfg.n_conditioning_codebooks:].max()) < cfg.vocab_size  # a call without start tokens keeps
        # its conditioning codebooks at the mask token
    assert_same_rng(got_rng, want_rng)


# ---------------------------------------------------------------------------------------------------- 6. adapters
def test_adapters_off_the_shipped_width(build_config):
    """C (d = 1024, V = 768, Cp = 7): the adapted base against the oracle of the folded fine-tune, under the criteria of
    tests/test_gpu_adapters.py (fp32 caps; no farther from the fp32 oracle than the folded model, x 1.25); per-row
    adapters in one launch equal one launch per adapter."""
    from vampnet_b200 import _lib as L
    cfg, sd, model, cb, codec = build_config("C", seed=2, lora=True, base_only=True)
    model.add_adapter("ft0", sd)
    g = torch.Generator().manual_seed(101)
    other = {k: (torch.randn(v.shape, generator=g) * v.std() if ".lora_" in k else v) for k, v in sd.items()}
    model.add_adapter("ft1", other)
    B, T = 3, 37
    z = codes(cfg, B, T, seed=5)
    got = model.forward_codes(z.cuda(), codec, adapter="ft0").cpu()            # (B, S, V)
    _, _, folded, _, fcodec = build_config("C", seed=2, lora=True)
    fgot = folded.forward_codes(z.cuda(), fcodec).cpu()
    del folded
    orc = vo.OracleVampNet(cfg, sd, "fp32")
    ref32 = orc.forward(orc.from_codes(z, cb)).permute(0, 2, 1)
    o32, of32 = (got - ref32).abs(), (fgot - ref32).abs()
    print(f"[C adapter] vs fp32 oracle: max {o32.max():.3e} mean {o32.mean():.3e} (folded max {of32.max():.3e} mean "
          f"{of32.mean():.3e}); ratios {o32.mean() / (1.25 * of32.mean()):.3f} mean, "
          f"{o32.max() / (1.25 * of32.max()):.3f} max")
    assert o32.mean() < 1.2e-2 and o32.max() < 0.09
    assert o32.mean() <= 1.25 * of32.mean() and o32.max() <= 1.25 * of32.max()
    base = model.forward_codes(z.cuda(), codec).cpu()
    assert (base - got).abs().max() > 1e-2
    names = ["ft0", None, "ft1"]
    ids = [model._adapter_id(n) for n in names]
    zc = z.cuda().contiguous()
    logits = torch.empty(B, T * cfg.n_predict_codebooks, cfg.vocab_size, device="cuda")
    L.check(L.lib().vnb_forward_codes_adapted(model._handle, L.ptr(zc), B, T, (C.c_int32 * B)(*ids), L.ptr(logits),
                                              L.stream_ptr()))
    for b, name in enumerate(names):
        alone = model.forward_codes(z[b:b + 1].cuda(), codec, adapter=name)
        assert torch.equal(logits[b:b + 1], alone), f"row {b} ({name}) differs from its own launch"


# ---------------------------------------------------------------------------------------------------- 7. refusals
REFUSED = [
    ("d384", dict(n_heads=6, embedding_dim=384), "multiple of 256"),
    ("d512_h4", dict(n_heads=4, embedding_dim=512), "n_heads\\*64"),
    ("v128", dict(vocab_size=128), "vocab_size"),
    ("v300", dict(vocab_size=300), "vocab_size"),
    ("v1280", dict(vocab_size=1280), "vocab_size"),
    ("c17", dict(n_codebooks=17), "n_codebooks"),
]


@pytest.mark.parametrize("what,change,message", REFUSED, ids=[r[0] for r in REFUSED])
def test_refused_configurations(build_config, what, change, message):
    """A geometry the kernels do not cover is refused by vnb_model_create with its message, before any kernel of the
    library runs; the library works afterwards."""
    from vampnet_b200 import _lib as L
    from vampnet_b200.modules.transformer import VampNet
    cfgd = {**CONFIGS["A"], "n_layers": 1, **change}
    cfg = vo.OracleConfig(**cfgd)
    model = VampNet(**cfgd)
    model.load_state_dict(vo.make_state_dict(cfg, seed=0), strict=False)
    model = model.to("cuda")
    codec = StubCodec(vo.make_codebooks(cfg.n_codebooks, vocab_size=cfg.vocab_size).cuda())
    z = torch.randint(0, cfg.vocab_size, (1, cfg.n_codebooks, 16)).cuda()
    before = L.lib().vnb_launch_count()
    with pytest.raises(RuntimeError, match=message):
        model.forward_codes(z, codec)
    assert L.lib().vnb_launch_count() == before
    assert model._handle is None
    cfg2, sd2, good, cb2, codec2 = build_config("A")
    out = good.generate(codec2, start_tokens=torch.randint(0, 256, (1, 1, 16)).cuda(), _sampling_steps=2, seed=1,
                        return_signal=False, sample_cutoff=-1.0, mask_temperature=0.0)
    assert L.lib().vnb_launch_count() > before and int(out.max()) < 256
