"""Run the ORIGINAL project's code once and store what the reference-comparison tests compare against.

    VAMPNET_REFERENCE_ROOT=<checkout of the original vampnet> python -m oracle.gen_reference_golden

Writes tests/golden/reference_{mask,vampnet,vampnet_configs,interface}.npz.  The tests (test_mask_cpu,
test_oracle_vs_reference, test_oracle_configs_vs_reference, test_interface_vs_reference) recompute their side with the same seeds and compare with these arrays, so they need
no checkout of the original.  Kept small: token ids and masks as int16, and where a test compared large fp32 tensors
a fixed seeded sample of their entries (``sample_idx``).
"""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_shims  # noqa: E402
from oracle import vampnet_oracle as vo  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
N_SAMPLE = 512


def sample_idx(numel: int, seed: int, n: int = N_SAMPLE) -> np.ndarray:
    """Fixed flat indices into a tensor of `numel` entries (shared by the generator and the tests)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randperm(numel, generator=g)[:min(n, numel)].numpy()


def i16(t) -> np.ndarray:
    return t.numpy().astype(np.int16)


# ------------------------------------------------------------------------------------------------ mask.py
MASK_X_SHAPE, MASK_X_SEED = (3, 9, 57), 0


def mask_cases(M, x):
    return [
        lambda: M.linear_random(x, 0.7),
        lambda: M.random(x, 0.3),
        lambda: M.inpaint(x, 4, 9),
        lambda: M.inpaint(x, 0, 0),
        lambda: M.periodic_mask(x, 7, 1, random_roll=True),
        lambda: M.periodic_mask(x, 5, 3, random_roll=True),
        lambda: M.periodic_mask(x, 0, 1),
        lambda: M.codebook_mask(M.codebook_unmask(M.full_mask(x), 2), 5),
        lambda: M.dropout(M.periodic_mask(x, 3, 1), 0.3),
        lambda: M.mask_or(M.inpaint(x, 2, 2), M.periodic_mask(x, 4, 1)),
        lambda: M.time_stretch_mask(x, 3),
        lambda: M.apply_mask(x, M.periodic_mask(x, 7, 1), 1024)[0],
        lambda: M._gamma(torch.linspace(0, 1, 13)),
    ]


def build_mask_chain(M, x):
    m = M.linear_random(x, 1.0)
    m = M.mask_and(m, M.inpaint(x, 0, 0))
    m = M.mask_and(m, M.periodic_mask(x, 7, 1, random_roll=True))
    m = M.dropout(m, 0.1)
    m = M.codebook_unmask(m, 0)
    return M.codebook_mask(m, 3, None)


def gen_mask(rm):
    out = {}
    x = torch.randint(0, 1024, MASK_X_SHAPE, generator=torch.Generator().manual_seed(MASK_X_SEED))
    for i, fn in enumerate(mask_cases(rm, x)):
        torch.manual_seed(123 + i)
        want = fn()
        out[f"case{i}"] = want.numpy() if want.is_floating_point() else i16(want)
    x = torch.randint(0, 1024, (2, 14, 100), generator=torch.Generator().manual_seed(1))
    torch.manual_seed(7)
    out["chain"] = i16(build_mask_chain(rm, x))
    out["chain_next_draws"] = torch.rand(4).numpy()
    return out


# ------------------------------------------------------------------------------------------------ VampNet
CFGS = {
    "coarse": dict(n_heads=4, n_layers=2, n_codebooks=4, n_conditioning_codebooks=0, embedding_dim=256),
    "c2f": dict(n_heads=2, n_layers=1, n_codebooks=14, n_conditioning_codebooks=4, embedding_dim=128),
}
GEN_KWS = [dict(sample_cutoff=-1.0, mask_temperature=0.0), dict(), dict(temperature=1.3, top_p=0.8),
           dict(sample_cutoff=0.4)]
GEN_STEPS = (1, 2, 7)
# off the shipped geometry (vocab_size != 1024, a single predicted codebook, an odd number of them): configurations A and
# C of tests/test_gpu_model_configs.py, at fewer layers
CONFIG_CFGS = {
    "v256_cp1": dict(n_heads=8, n_layers=1, n_codebooks=1, n_conditioning_codebooks=0, embedding_dim=512,
                     vocab_size=256),
    "v768_cp7": dict(n_heads=16, n_layers=1, n_codebooks=9, n_conditioning_codebooks=2, embedding_dim=1024,
                     vocab_size=768),
}


def vampnet_case(tag, lora, cfgs=CFGS):
    """Inputs of one forward / generate case (everything seeded)."""
    cfgd = cfgs[tag]
    cfg = vo.OracleConfig(**cfgd)
    V = cfg.vocab_size
    sd = vo.make_state_dict(cfg, seed=7, lora=lora)
    cb = vo.make_codebooks(cfg.n_codebooks, vocab_size=V, seed=2)
    g = torch.Generator().manual_seed(3)
    z = torch.randint(0, V, (3, cfg.n_codebooks, 31), generator=g)
    zm = z.clone()
    zm[:, cfg.n_conditioning_codebooks:, ::2] = cfg.mask_token
    mask = torch.ones_like(z)
    mask[:, :, ::5] = 0
    return cfgd, cfg, sd, cb, z, zm, mask


def gen_vampnet(tr, cfgs=CFGS, loras=(False, True), extras=True):
    out = {}
    for tag in cfgs:
        for lora in loras:
            key = f"{tag}_lora{int(lora)}"
            cfgd, cfg, sd, cb, z, zm, mask = vampnet_case(tag, lora, cfgs)
            ref = tr.VampNet(flash_attn=False, **cfgd)
            res = ref.load_state_dict(sd, strict=False)
            assert not res.unexpected_keys
            ref.eval()
            codec = ref_shims.StubCodec(cb)
            with torch.no_grad():
                lat = ref.embedding.from_codes(zm, codec)
                logits = ref(lat)
                logits2, acts = ref(lat, return_activations=True)
            assert torch.equal(logits2, logits)
            out[f"{key}_latents"] = lat.flatten()[sample_idx(lat.numel(), 1)].numpy()
            out[f"{key}_logits"] = logits.flatten()[sample_idx(logits.numel(), 2)].numpy()
            out[f"{key}_acts_shape"] = np.array(acts.shape)
            out[f"{key}_acts"] = acts.flatten()[sample_idx(acts.numel(), 3)].numpy()
            out[f"{key}_acts_absmax"] = np.float32(acts.abs().max().item())
            for ki, kw in enumerate(GEN_KWS):
                for steps in GEN_STEPS:
                    zr = ref.generate(codec, start_tokens=z.clone(), mask=mask.clone(), _sampling_steps=steps, seed=9,
                                      return_signal=False, **kw)
                    out[f"{key}_gen{ki}_s{steps}"] = i16(zr)
    if not extras:
        return out
    # typical_filter: the reference discards its result (transformer.py:989-993)
    logits = torch.randn(2, 9, 1024, generator=torch.Generator().manual_seed(0))
    torch.manual_seed(1)
    a = tr.sample_from_logits(logits.clone(), typical_filtering=True, typical_mass=0.15, typical_min_tokens=64)
    torch.manual_seed(1)
    b = tr.sample_from_logits(logits.clone(), typical_filtering=False)
    for name, v in (("typical_on", a), ("typical_off", b)):
        v = v if isinstance(v, (tuple, list)) else (v,)
        for j, t in enumerate(v):
            out[f"{name}_{j}"] = t.numpy()
    # 2-d and default masks
    cfgd = CFGS["c2f"]
    cfg = vo.OracleConfig(**cfgd)
    sd = vo.make_state_dict(cfg, seed=4)
    ref = tr.VampNet(flash_attn=False, **cfgd)
    ref.load_state_dict(sd, strict=False)
    ref.eval()
    codec = ref_shims.StubCodec(vo.make_codebooks(cfg.n_codebooks, seed=2))
    z = torch.randint(0, 1024, (2, 14, 12), generator=torch.Generator().manual_seed(1))
    m2 = torch.ones(2, 12, dtype=torch.long)
    m2[:, ::3] = 0
    for name, mask in (("mask_default", None), ("mask_2d", m2)):
        zr = ref.generate(codec, start_tokens=z.clone(), mask=None if mask is None else mask.clone(), _sampling_steps=3,
                          seed=1, return_signal=False)
        out[name] = i16(zr)
    return out


def gen_vampnet_configs(tr):
    """The reference at CONFIG_CFGS: forward and generate with a vocabulary, and so a mask token, other than 1024."""
    return gen_vampnet(tr, CONFIG_CFGS, loras=(False,), extras=False)


# ------------------------------------------------------------------------------------------------ Interface
COARSE_VAMP_T = [1, 34, 35, 36, 83, 140]
C2F_CASES = [(15, 14), (29, 14), (30, 4), (47, 14), (1, 4)]
VAMP_CASES = [(1, 1, 1, 83), (3, 1, 1, 40), (2, 2, 1, 61), (2, 3, 2, 37), (1, 1, 3, 20)]
BUILD_MASK_KWS = [
    dict(),
    dict(rand_mask_intensity=0.7, periodic_prompt=5, periodic_prompt_width=2, upper_codebook_mask=4),
    dict(prefix_s=0.3, suffix_s=0.2, periodic_prompt=0, _dropout=0.3, ncc=1),
    dict(rand_mask_intensity=0.0, periodic_prompt=3, upper_codebook_mask=14),
]
UNIT_SECONDS = (0.0, 0.1, 1.0, 3.0, 10.0, 13.37)


def stub_models(coarse_s=0.6, c2f_s=0.25):
    from tests.test_interface_cpu import StubModel
    coarse, c2f = StubModel(4, 0, salt=5), StubModel(14, 4, salt=9)
    coarse.chunk_size_s, c2f.chunk_size_s = coarse_s, c2f_s
    return coarse, c2f


def calls_signature(calls, fields):
    """The generate calls a stub model saw, as a string (compared verbatim by the tests)."""
    return repr([tuple(c[f] for f in fields) for c in calls])


def gen_interface(ref_mod):
    from tests.test_interface_cpu import StubCodec, rand_case

    def make_ref():
        ref = ref_mod.Interface.__new__(ref_mod.Interface)   # the reference constructor loads checkpoints from disk
        torch.nn.Module.__init__(ref)
        ref.codec = StubCodec()
        ref.coarse, ref.c2f = stub_models()
        ref.device = "cpu"
        return ref

    def quiet(fn, *a, **k):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return fn(*a, **k)

    out = {}
    for T in COARSE_VAMP_T:
        ref = make_ref()
        z, mask = rand_case(2, T, seed=T)
        if T > 70:
            mask[:, :, 70:] = 1
        want, start = quiet(ref.coarse_vamp, z, mask, return_mask=True, temperature=0.7)
        out[f"coarse_vamp_T{T}"], out[f"coarse_vamp_T{T}_start"] = i16(want), i16(start)
        out[f"coarse_vamp_T{T}_calls"] = np.array(calls_signature(ref.coarse.calls, ("shape", "kwargs")))
    for T, n_in in C2F_CASES:
        ref = make_ref()
        z, mask = rand_case(2, T, seed=100 + T)
        z = z[:, :n_in]
        want, start = quiet(ref.coarse_to_fine, z, mask=mask, return_mask=True)
        out[f"c2f_T{T}_n{n_in}"], out[f"c2f_T{T}_n{n_in}_start"] = i16(want), i16(start)
        out[f"c2f_T{T}_n{n_in}_nomask"] = i16(quiet(ref.coarse_to_fine, z, mask=None))
        out[f"c2f_T{T}_n{n_in}_calls"] = np.array(calls_signature(ref.c2f.calls, ("time_steps", "shape", "kwargs")))
    for batch, feedback, stretch, T in VAMP_CASES:
        ref = make_ref()
        z, mask = rand_case(1, T, seed=7 * T + batch)
        kw = dict(batch_size=batch, feedback_steps=feedback, time_stretch_factor=stretch, return_mask=True,
                  temperature=1.3)
        want, wmask = quiet(ref.vamp, z, mask, **kw)
        key = f"vamp_{batch}_{feedback}_{stretch}_{T}"
        out[key], out[key + "_mask"] = i16(want), i16(wmask)
        out[key + "_calls"] = np.array(calls_signature(ref.c2f.calls, ("kwargs",)))
    for i, kw in enumerate(BUILD_MASK_KWS):
        ref = make_ref()
        z, _ = rand_case(2, 97, seed=3)
        torch.manual_seed(11)
        out[f"build_mask{i}"] = i16(ref.build_mask(z, **kw))
        out[f"build_mask{i}_next_draws"] = torch.rand(4).numpy()
    ref = make_ref()
    out["units_s2t"] = np.array([ref.s2t(s) for s in UNIT_SECONDS])
    out["units_s2t2s"] = np.array([ref.s2t2s(s) for s in UNIT_SECONDS], dtype=np.float64)
    out["units_t2s_575"] = np.float64(ref.t2s(575))
    return out


def main():
    if not ref_shims.available():
        raise SystemExit(f"the original project is not at {ref_shims.REFERENCE_ROOT} (set VAMPNET_REFERENCE_ROOT)")
    tr, rm, _ = ref_shims.load_reference()
    try:
        np.savez_compressed(os.path.join(GOLDEN, "reference_mask.npz"), **gen_mask(rm))
        np.savez_compressed(os.path.join(GOLDEN, "reference_vampnet.npz"), **gen_vampnet(tr))
        np.savez_compressed(os.path.join(GOLDEN, "reference_vampnet_configs.npz"), **gen_vampnet_configs(tr))
        np.savez_compressed(os.path.join(GOLDEN, "reference_interface.npz"),
                            **gen_interface(ref_shims.load_reference_interface()))
    finally:
        ref_shims.uninstall()
    for n in ("mask", "vampnet", "vampnet_configs", "interface"):
        p = os.path.join(GOLDEN, f"reference_{n}.npz")
        print(p, os.path.getsize(p), "bytes")


if __name__ == "__main__":
    main()
