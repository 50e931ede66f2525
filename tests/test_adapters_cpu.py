"""CPU: packing and validation of per-request LoRA adapters (VampNet.add_adapter, pack_adapter).

The packed A' / B', applied in float64 in the packed row order the kernels use (include/vampnet_b200.h:
vnb_adapter_weights), must reproduce the reference LoRA delta (x * norm) . (B . A . alpha / r)^T of each LoRA'd
projection on the corresponding rows of the packed wqkv / wo / w1 / w2."""
import os
import tempfile

import pytest
import torch

from oracle import vampnet_oracle as vo
from vampnet_b200.modules.transformer import LORA_MODULES, VampNet

TINY_COARSE = dict(n_heads=4, n_layers=2, n_codebooks=4, n_conditioning_codebooks=0, embedding_dim=256)
TINY_C2F = dict(n_heads=4, n_layers=2, n_codebooks=14, n_conditioning_codebooks=4, embedding_dim=256)


def base_and_lora(cfgd, seed=0):
    """(base model, LoRA fine-tune state dict of that base): the base is the fine-tune without its LoRA tensors."""
    sd = vo.make_state_dict(vo.OracleConfig(**cfgd), seed=seed, lora=True)
    model = VampNet(**cfgd)
    model.load_state_dict({k: v for k, v in sd.items() if ".lora_" not in k}, strict=False)
    return model, sd


def w1_packed_rows(d):
    """Original w_1 row of every packed w1 row: per 256-row tile j, 128 value rows then 128 gate rows."""
    rows = []
    for p in range(4 * d):
        j, r = divmod(p, 256)
        rows.append(j * 128 + r if r < 128 else 2 * d + j * 128 + (r - 128))
    return torch.tensor(rows)


@pytest.mark.parametrize("cfgd", [TINY_COARSE, TINY_C2F], ids=["coarse", "c2f"])
def test_packed_adapter_reproduces_reference_lora_delta(cfgd):
    model, sd = base_and_lora(cfgd, seed=3)
    model.add_adapter("x", sd)
    p = {k: v.double() for k, v in model._adapters["x"].items()}
    d, s = cfgd["embedding_dim"], 1.0 / 8
    g = torch.Generator().manual_seed(0)
    x = torch.randn(37, d, generator=g, dtype=torch.float64)
    h = torch.randn(37, 2 * d, generator=g, dtype=torch.float64)
    kperm = w1_packed_rows(d)
    for l in range(cfgd["n_layers"]):
        pre = f"transformer.layers.{l}."
        A = {m: sd[pre + m + ".lora_A"].double() for m in LORA_MODULES}
        Bm = {m: sd[pre + m + ".lora_B"].double() for m in LORA_MODULES}
        n1, n3 = sd[pre + "norm_1.weight"].double(), sd[pre + "norm_3.weight"].double()

        def ref(m, inp, norm=None):
            xin = inp * norm[None, :] if norm is not None else inp
            return xin @ (Bm[m] @ A[m] * s).t()
        # wqkv rows [q | k | v]: k rows carry no LoRA
        u = x @ p["a_qkv"][l]                                                        # (M, 16)
        got = torch.cat([u[:, :8] @ p["b_qkv"][l][:d].t(), torch.zeros(37, d, dtype=torch.float64),
                         u[:, 8:] @ p["b_qkv"][l][d:].t()], 1)
        want = torch.cat([ref("self_attn.w_qs", x, n1), torch.zeros(37, d, dtype=torch.float64),
                          ref("self_attn.w_vs", x, n1)], 1)
        torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-7)
        torch.testing.assert_close((x @ p["a_wo"][l]) @ p["b_wo"][l].t(), ref("self_attn.fc", x), rtol=1e-5, atol=1e-7)
        torch.testing.assert_close((x @ p["a_w1"][l]) @ p["b_w1"][l].t(), ref("feed_forward.w_1", x, n3)[:, kperm],
                                   rtol=1e-5, atol=1e-7)
        torch.testing.assert_close((h @ p["a_w2"][l]) @ p["b_w2"][l].t(), ref("feed_forward.w_2", h), rtol=1e-5,
                                   atol=1e-7)
    assert model.adapters() == ["x"]
    model.remove_adapter("x")
    assert model.adapters() == []


def test_mismatched_base_is_refused_naming_a_tensor():
    model, _ = base_and_lora(TINY_COARSE, seed=3)
    other = vo.make_state_dict(vo.OracleConfig(**TINY_COARSE), seed=4, lora=True)
    with pytest.raises(ValueError, match=r"transformer\.|embedding\.|classifier\."):
        model.add_adapter("other", other)
    assert model.adapters() == []


def test_wrong_rank_is_refused():
    model, sd = base_and_lora(TINY_COARSE, seed=3)
    bad = dict(sd)
    key = "transformer.layers.1.feed_forward.w_2"
    bad[key + ".lora_A"] = sd[key + ".lora_A"][:4]
    bad[key + ".lora_B"] = sd[key + ".lora_B"][:, :4]
    with pytest.raises(ValueError, match="rank 4"):
        model.add_adapter("r4", bad)


def test_wrong_architecture_is_refused():
    model, sd = base_and_lora(TINY_COARSE, seed=3)
    blob = {"state_dict": sd, "metadata": {"kwargs": dict(TINY_COARSE, n_layers=3)}}
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "coarse.pth")
        torch.save(blob, path)
        with pytest.raises(ValueError, match="architecture"):
            model.add_adapter("deep", path)
        # the same checkpoint with matching metadata is accepted from a path
        torch.save({"state_dict": sd, "metadata": {"kwargs": dict(TINY_COARSE)}}, path)
        model.add_adapter("ok", path)
    assert model.adapters() == ["ok"]


def test_folded_live_model_is_refused():
    _, sd = base_and_lora(TINY_COARSE, seed=3)
    folded = VampNet(**TINY_COARSE)
    folded.load_state_dict(sd)
    with pytest.raises(ValueError, match="folded"):
        folded.add_adapter("x", sd)


def test_missing_lora_tensors_are_refused():
    model, sd = base_and_lora(TINY_COARSE, seed=3)
    with pytest.raises(ValueError, match="missing"):
        model.add_adapter("base", {k: v for k, v in sd.items() if ".lora_" not in k})


def test_new_base_drops_adapters_and_names_then_raise():
    model, sd = base_and_lora(TINY_COARSE, seed=3)
    model.add_adapter("x", sd)
    # the same base again keeps them
    model.load_state_dict({k: v for k, v in sd.items() if ".lora_" not in k}, strict=False)
    assert model.adapters() == ["x"]
    other = vo.make_state_dict(vo.OracleConfig(**TINY_COARSE), seed=4)
    model.load_state_dict(other, strict=False)
    assert model.adapters() == []
    with pytest.raises(KeyError, match="not registered"):
        model.generate(None, time_steps=8, adapter="x")
