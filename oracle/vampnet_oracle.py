"""TEST INFRASTRUCTURE — CPU oracle for the VampNet masked-token generation hot path.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
leg may import this file.  The product (vampnet_b200/) never does.

This is a *restatement* (plain torch ops on CPU tensors, functional style over a
state_dict with the reference's key names) of the algorithm in the reference
files below; every function cites the lines it follows.  It is pinned against the
reference's own code (imported through oracle/ref_shims.py) by
tests/test_oracle_vs_reference.py (live, authoring container only) and by the
committed fixtures in tests/golden/ (made by oracle/gen_golden.py).
The reference ships no tests or golden vectors of its own (SURVEY.md §4), so the
reference code executed here is the only pin there is.

Two numeric modes:
  * "fp32"  — what the reference computes on CPU (torch.autocast("cuda") is inert
              there): every op in fp32.
  * "bf16"  — same algorithm with GEMM operands rounded to bf16 at the points
              where the CUDA path rounds (RMSNorm output, q/k/v, softmax
              numerators, attention output, GEGLU output; weights once at pack
              time), fp32 accumulation, fp32 residual stream and fp32 logits.
              This is the parity target for the kernels; its distance from the
              "fp32" mode is the bf16 quantisation error and is reported, not hidden.

Two RNG modes for sampling:
  * "torch"  — the reference's calls (torch.multinomial, Tensor.uniform_) in the
               reference's order: bit-identical to the reference under a seed.
  * "philox" — the counter-based Philox4x32-10 stream the CUDA sampler uses
               (oracle/philox.py), so kernel and oracle share noise exactly.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from . import philox

MASK_TOKEN_OFFSET = 0  # mask token id == vocab_size (layers.py:128-130)


@dataclass
class OracleConfig:
    n_heads: int = 20
    n_layers: int = 16
    n_codebooks: int = 9
    n_conditioning_codebooks: int = 0
    latent_dim: int = 8
    embedding_dim: int = 1280
    vocab_size: int = 1024

    @property
    def n_predict_codebooks(self):
        return self.n_codebooks - self.n_conditioning_codebooks

    @property
    def mask_token(self):
        return self.vocab_size


# --------------------------------------------------------------------------------------
# synthetic weights (seeded; the same function feeds the reference model, the oracle
# and the CUDA path, so fixtures only need to carry a seed)
# --------------------------------------------------------------------------------------
def make_state_dict(cfg: OracleConfig, seed: int = 0, lora: bool = False) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    d, C, Cp, V, H = cfg.embedding_dim, cfg.n_codebooks, cfg.n_predict_codebooks, cfg.vocab_size, cfg.n_heads

    def rn(*shape, scale=1.0):
        return torch.randn(*shape, generator=g) * scale

    sd: Dict[str, torch.Tensor] = {}
    sd["embedding.special.MASK"] = rn(C, cfg.latent_dim)
    sd["embedding.out_proj.weight"] = rn(d, C * cfg.latent_dim, 1, scale=1.0 / math.sqrt(C * cfg.latent_dim))
    sd["embedding.out_proj.bias"] = rn(d, scale=0.1)
    for i in range(cfg.n_layers):
        p = f"transformer.layers.{i}."
        sd[p + "norm_1.weight"] = 1.0 + rn(d, scale=0.1)
        for w in ("w_qs", "w_ks", "w_vs", "fc"):
            sd[p + f"self_attn.{w}.weight"] = rn(d, d, scale=1.0 / math.sqrt(d))
        if i == 0:
            sd[p + "self_attn.relative_attention_bias.weight"] = rn(32, H, scale=0.5)
        sd[p + "norm_3.weight"] = 1.0 + rn(d, scale=0.1)
        sd[p + "feed_forward.w_1.weight"] = rn(4 * d, d, scale=1.0 / math.sqrt(d))
        sd[p + "feed_forward.w_2.weight"] = rn(d, 2 * d, scale=1.0 / math.sqrt(2 * d))
        if lora:
            r = 8
            for name, (o, k) in {
                "self_attn.w_qs": (d, d), "self_attn.w_vs": (d, d), "self_attn.fc": (d, d),
                "feed_forward.w_1": (4 * d, d), "feed_forward.w_2": (d, 2 * d),
            }.items():
                sd[p + name + ".lora_A"] = rn(r, k, scale=1.0 / math.sqrt(k))
                sd[p + name + ".lora_B"] = rn(o, r, scale=0.05)
    sd["transformer.norm.weight"] = 1.0 + rn(d, scale=0.1)
    v = rn(V * Cp, d, 1, scale=1.0 / math.sqrt(d))
    sd["classifier.layers.0.weight_v"] = v
    sd["classifier.layers.0.weight_g"] = v.flatten(1).norm(dim=1).view(-1, 1, 1) * (1.0 + rn(V * Cp, 1, 1, scale=0.1))
    sd["classifier.layers.0.bias"] = rn(V * Cp, scale=0.1)
    return sd


def make_codebooks(n_codebooks: int, vocab_size: int = 1024, latent_dim: int = 8, seed: int = 1) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n_codebooks, vocab_size, latent_dim, generator=g)


# --------------------------------------------------------------------------------------
# helpers
# --------------------------------------------------------------------------------------
def _bf16(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16).to(torch.float32)


def fold_lora(sd: Dict[str, torch.Tensor], name: str, lora_r: int = 8, lora_alpha: float = 1.0) -> torch.Tensor:
    """W_eff = W + (alpha/r) * B @ A  (loralib.Linear, merged form; reference builds
    w_qs/w_vs/fc/w_1/w_2 as lora.Linear(r=LORA_R=8): transformer.py:22, 67-68, 109-114)."""
    w = sd[name + ".weight"].float()
    if name + ".lora_A" in sd:
        w = w + (sd[name + ".lora_B"].float() @ sd[name + ".lora_A"].float()) * (lora_alpha / lora_r)
    return w


def weight_norm_fold(g: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """torch.nn.utils.weight_norm with dim=0: w = g * v / ||v|| per output channel
    (layers.py:47-48; recomputed on every call in the reference)."""
    norm = v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1)))
    return v * (g / norm)


def relative_position_bucket_lut(T: int, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """Bucket index for rel = key - query in [-(T-1), T-1]; entry [rel + T - 1].
    Restates transformer.py:123-181 (bidirectional branch), same torch expressions so
    the fp32 log boundaries fall identically."""
    rel = torch.arange(-(T - 1), T, dtype=torch.long)
    nb = num_buckets // 2
    out = (rel > 0).to(torch.long) * nb
    a = rel.abs()
    max_exact = nb // 2
    small = a < max_exact
    large = max_exact + (
        torch.log(a.float() / max_exact) / math.log(max_distance / max_exact) * (nb - max_exact)
    ).to(torch.long)
    large = torch.minimum(large, torch.full_like(large, nb - 1))
    return out + torch.where(small, a, large)


def gamma(r: torch.Tensor) -> torch.Tensor:
    """Cosine schedule, mask.py:8-9."""
    return (r * torch.pi / 2).cos().clamp(1e-10, 1.0)


def codebook_flatten(t: torch.Tensor) -> torch.Tensor:
    """(B, C, T) -> (B, T*C) with s = t*C + c (util.py:35-39)."""
    return t.permute(0, 2, 1).reshape(t.shape[0], -1)


def codebook_unflatten(t: torch.Tensor, n_c: int) -> torch.Tensor:
    """(B, T*C) -> (B, C, T) (util.py:41-46)."""
    B = t.shape[0]
    return t.reshape(B, -1, n_c).permute(0, 2, 1)


# --------------------------------------------------------------------------------------
# the model
# --------------------------------------------------------------------------------------
class OracleVampNet:
    def __init__(self, cfg: OracleConfig, state_dict: Dict[str, torch.Tensor], mode: str = "fp32",
                 jitter: float = 0.0, jitter_seed: int = 0):
        """jitter (bf16 mode only) is a CONDITIONING PROBE, not a numeric mode: every activation is multiplied by
        (1 + jitter * N(0,1)) right before it is rounded to bf16.  With jitter ~1e-7..1e-6 (the size of fp32
        accumulation-order differences) the logits move by as much as two correct bf16 implementations differ
        (tests/test_oracle_conditioning_cpu.py): a relative 1e-7 nudge flips the bf16 rounding of a fraction of the
        activations, each flip is a 2^-9 relative change, and 20 layers amplify them.  The distance between the
        probe and the unperturbed oracle is therefore the floor for ANY bf16 implementation that does not share the
        oracle's exact summation order, and the GPU parity tests are calibrated against it."""
        assert mode in ("fp32", "bf16")
        assert jitter == 0.0 or mode == "bf16"
        self.cfg = cfg
        self.mode = mode
        self.sd = {k: v.detach().float().cpu() for k, v in state_dict.items()}
        q = _bf16 if mode == "bf16" else (lambda x: x)
        self.qa = q  # activation rounding at GEMM inputs
        if jitter > 0.0:
            gen = torch.Generator().manual_seed(jitter_seed)
            self.qa = lambda x: _bf16(x * (1.0 + jitter * torch.randn(x.shape, generator=gen)))
        L = cfg.n_layers
        self.layers = []
        for i in range(L):
            p = f"transformer.layers.{i}."
            n1, n3 = self.sd[p + "norm_1.weight"], self.sd[p + "norm_3.weight"]
            # bf16 mode mirrors the kernels: the RMSNorm weight is folded into the following projection
            # (W * w[None, :], then rounded to bf16) and the 1/rms factor is applied to the GEMM result.
            f1 = n1[None, :] if mode == "bf16" else 1.0
            f3 = n3[None, :] if mode == "bf16" else 1.0
            self.layers.append(dict(
                norm_1=n1,
                wq=q(fold_lora(self.sd, p + "self_attn.w_qs") * f1),
                wk=q(self.sd[p + "self_attn.w_ks.weight"] * f1),
                wv=q(fold_lora(self.sd, p + "self_attn.w_vs") * f1),
                wo=q(fold_lora(self.sd, p + "self_attn.fc")),
                norm_3=n3,
                w1=q(fold_lora(self.sd, p + "feed_forward.w_1") * f3),
                w2=q(fold_lora(self.sd, p + "feed_forward.w_2")),
            ))
        self.rel_bias = self.sd["transformer.layers.0.self_attn.relative_attention_bias.weight"]  # (32, H)
        self.final_norm = self.sd["transformer.norm.weight"]
        fc = self.final_norm[None, :] if mode == "bf16" else 1.0
        self.cls_w = q(weight_norm_fold(self.sd["classifier.layers.0.weight_g"],
                                        self.sd["classifier.layers.0.weight_v"]).squeeze(-1) * fc)
        self.cls_b = self.sd["classifier.layers.0.bias"]
        self.emb_w = self.sd["embedding.out_proj.weight"].squeeze(-1)  # (d, C*8), stays fp32 in both modes
        self.emb_b = self.sd["embedding.out_proj.bias"]
        self.mask_rows = self.sd["embedding.special.MASK"]  # (C, 8)

    # ---- A6: CodebookEmbedding.from_codes (layers.py:134-156) -------------------------
    def from_codes(self, codes: torch.Tensor, codebooks: torch.Tensor) -> torch.Tensor:
        """codes (B, C', T) int64, codebooks (>=C', V, 8) -> latents (B, C'*8, T), channel = c*8 + j.
        Token id V selects the learned MASK row of that codebook."""
        B, Cn, T = codes.shape
        outs = []
        for c in range(Cn):
            table = torch.cat([codebooks[c].float(), self.mask_rows[c:c + 1]], dim=0)  # (V+1, 8)
            outs.append(table[codes[:, c, :]].permute(0, 2, 1))  # (B, 8, T)
        return torch.cat(outs, dim=1)

    # ---- A8: RMSNorm (transformer.py:43-58) ---------------------------------------------
    @staticmethod
    def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
        var = x.pow(2).mean(-1, keepdim=True)
        return w * (x * torch.rsqrt(var + eps))

    # ---- A11: position bias (transformer.py:183-209) ------------------------------------
    def position_bias(self, T: int) -> torch.Tensor:
        """(H, T, T) with [h, q, k] = E[bucket(k - q), h]."""
        lut = relative_position_bucket_lut(T)
        idx = torch.arange(T)[None, :] - torch.arange(T)[:, None] + (T - 1)  # k - q + T - 1
        buckets = lut[idx]  # (T, T)
        return self.rel_bias[buckets].permute(2, 0, 1)

    # ---- A10: MultiHeadRelativeAttention.forward (transformer.py:211-257) ---------------
    def attention(self, y: torch.Tensor, lw: dict, bias: torch.Tensor, rs=1.0) -> torch.Tensor:
        """y: normed input (fp32 mode) or the raw residual stream with rs = 1/rms per row (bf16 mode)."""
        B, T, d = y.shape
        H = self.cfg.n_heads
        dh = d // H
        ya = self.qa(y)
        q = self.qa((ya @ lw["wq"].t()) * rs).view(B, T, H, dh).permute(2, 0, 1, 3)  # (H, B, T, dh)
        k = self.qa((ya @ lw["wk"].t()) * rs).view(B, T, H, dh).permute(2, 0, 1, 3)
        v = self.qa((ya @ lw["wv"].t()) * rs).view(B, T, H, dh).permute(2, 0, 1, 3)
        s = torch.matmul(q, k.transpose(-1, -2)) / np.sqrt(dh)  # (H, B, T, T)
        s = s + bias[:, None]
        # x_mask is all ones on this path (transformer.py:619) -> masked_fill is a no-op
        if self.mode == "fp32":
            p = torch.softmax(s, dim=3)
            o = torch.matmul(p, v)
        else:
            m = s.amax(dim=3, keepdim=True)
            e = torch.exp(s - m)
            l = e.sum(dim=3, keepdim=True)
            o = torch.matmul(_bf16(e), v) / l
        o = o.permute(1, 2, 0, 3).reshape(B, T, d)
        return self.qa(o) @ lw["wo"].t()

    # ---- A12: FeedForward + GatedGELU (transformer.py:72-85, activations.py:16-35) ------
    def ffn(self, y: torch.Tensor, lw: dict, rs=1.0) -> torch.Tensor:
        h = (self.qa(y) @ lw["w1"].t()) * rs
        p1, p2 = h.chunk(2, dim=-1)  # gate is the second half
        gelu = 0.5 * p2 * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (p2 + 0.044715 * torch.pow(p2, 3.0))))
        return self.qa(p1 * gelu) @ lw["w2"].t()

    # ---- A7/A13/A14: VampNet.forward (transformer.py:617-639) ---------------------------
    def forward(self, latents: torch.Tensor, return_hidden: bool = False, return_activations: bool = False):
        """latents (B, C*8, T) -> logits (B, V, T*Cp).  return_activations: also the residual stream after every
        layer, stacked (L, B, T, d) (transformer.py:443-461, 626-637)."""
        cfg = self.cfg
        B, _, T = latents.shape
        x = torch.einsum("bkt,nk->btn", latents.float(), self.emb_w) + self.emb_b  # Conv1d k=1 (layers.py:162)
        bias = self.position_bias(T)
        acts = []
        if self.mode == "fp32":
            for lw in self.layers:  # TransformerLayer.forward (transformer.py:314-369); FiLM is identity (d_cond=0)
                x = x + self.attention(self.rmsnorm(x, lw["norm_1"]), lw, bias)
                x = x + self.ffn(self.rmsnorm(x, lw["norm_3"]), lw)
                acts.append(x)
            out = self.rmsnorm(x, self.final_norm) @ self.cls_w.t() + self.cls_b  # (B, T, V*Cp), channel = p*Cp + c
        else:
            inv_rms = lambda t: torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-6)
            for lw in self.layers:
                x = x + self.attention(x, lw, bias, inv_rms(x))
                x = x + self.ffn(x, lw, inv_rms(x))
                acts.append(x)
            out = (self.qa(x) @ self.cls_w.t()) * inv_rms(x) + self.cls_b
        Cp, V = cfg.n_predict_codebooks, cfg.vocab_size
        # "b (p c) t -> b p (t c)" (transformer.py:634)
        logits = out.view(B, T, V, Cp).permute(0, 2, 1, 3).reshape(B, V, T * Cp)
        if return_activations:
            return logits, torch.stack(acts)
        if return_hidden:
            return logits, x
        return logits

    # ---- A15: sample_from_logits (transformer.py:952-1034) ------------------------------
    def sample_from_logits(self, logits, sample, temperature, top_p=None, rng="torch",
                           philox_key=(0, 0), step=0):
        """logits (B, S, V) -> token (B, S) int64, prob-of-token (B, S) fp32.
        typical_filter (transformer.py:989-993) discards its result in the reference and is
        therefore absent here.  top_k is always None on this path (transformer.py:858)."""
        B, S, V = logits.shape
        if top_p is not None and top_p < 1.0:  # transformer.py:1001-1016, modifies logits in place
            v, si = logits.sort(descending=True)
            cum = v.softmax(dim=-1).cumsum(dim=-1)
            rm = cum > top_p
            rm = F.pad(rm, (1, 0), value=False)[..., :-1]
            rm = rm.scatter(-1, si, rm)
            logits = logits.masked_fill(rm, -float("inf"))
        scaled = logits / temperature if temperature > 0 else logits
        probs = F.softmax(scaled, dim=-1)
        if not sample:
            token = logits.argmax(-1)
        elif rng == "torch":
            token = probs.view(-1, V).multinomial(1).squeeze(1).view(B, S)
        else:
            # the CUDA sampler's draw (same distribution as multinomial): a two-level inverse CDF in natural
            # vocabulary order.  The vocabulary is cut into tiles of 128 entries (what one epilogue thread of the
            # classifier GEMM holds, csrc/gemm_wgmma.cu EPI_SAMPLE); uniform 1 picks the tile by its probability
            # mass, uniform 2 the entry inside it: token = first v in the tile with cumsum(e)[v] > u2 * mass(tile).
            u1 = philox.uniform_bs(philox_key, step, B, S, stream=0, word=0)  # (B, S) fp32 in (0,1)
            u2 = philox.uniform_bs(philox_key, step, B, S, stream=0, word=1)
            inv_t = np.float32(1.0 / temperature) if temperature > 0 else np.float32(1.0)
            TILE = 128
            assert V % TILE == 0
            xs = (logits.numpy().astype(np.float32) * inv_t).reshape(B, S, V // TILE, TILE)
            m_k = xs.max(-1)                                                        # tile maxima
            # a tile the nucleus filter emptied (all -inf) has mass 0, not exp(-inf - -inf) = NaN
            e = np.exp(xs - np.where(np.isfinite(m_k), m_k, 0.0)[..., None], dtype=np.float32)
            cdf_in = np.cumsum(e, axis=-1, dtype=np.float32)                        # within-tile, sequential fp32
            mass = cdf_in[..., -1] * np.exp(m_k - m_k.max(-1, keepdims=True), dtype=np.float32)
            cdf_t = np.cumsum(mass, axis=-1, dtype=np.float32)
            hit_t = cdf_t > (u1 * cdf_t[..., -1])[..., None]
            k = np.where(hit_t.any(-1), hit_t.argmax(-1), m_k.argmax(-1))           # fallback: tile of the arg-max
            cdf_k = np.take_along_axis(cdf_in, k[..., None, None], axis=2)[:, :, 0, :]
            xs_k = np.take_along_axis(xs, k[..., None, None], axis=2)[:, :, 0, :]
            hit_v = cdf_k > (u2 * cdf_k[..., -1])[..., None]
            idx = np.where(hit_v.any(-1), hit_v.argmax(-1), xs_k.argmax(-1))        # fallback: arg-max of the tile
            token = torch.from_numpy((k * TILE + idx).astype(np.int64))
        token_probs = probs.take_along_dim(token.unsqueeze(-1), dim=-1).squeeze(-1)
        return token, token_probs

    # ---- A17: mask_by_random_topk (transformer.py:1038-1074) ----------------------------
    @staticmethod
    def mask_by_random_topk(num_to_mask, probs, temperature, rng="torch", philox_key=(0, 0), step=0):
        B, S = probs.shape
        if rng == "torch":
            u = torch.zeros_like(probs).uniform_(1e-20, 1)  # gumbel_noise_like, transformer.py:28-30
            noise = -torch.log(-torch.log(u))
        else:
            u = philox.uniform_bs(philox_key, step, B, S)
            noise = torch.from_numpy(-np.log(-np.log(u, dtype=np.float32), dtype=np.float32))
        conf = torch.log(probs) + temperature.unsqueeze(-1) * noise
        sorted_conf, _ = conf.sort(dim=-1)
        cut = torch.take_along_dim(sorted_conf, num_to_mask, dim=-1)
        return conf < cut, conf

    # ---- A5: VampNet.generate (transformer.py:686-946) ----------------------------------
    @torch.inference_mode()
    def generate(self, codebooks, start_tokens, mask=None, _sampling_steps=12, temperature=1.0,
                 mask_temperature=10.5, top_p=None, seed=None, sample_cutoff=1.0,
                 rng="torch", philox_key=(0, 0), trace: Optional[List[dict]] = None,
                 logits_fn=None):
        """Returns sampled_z (B, C, T) int64.  cfg/ctrls/causal_weight/cond/time_steps/typical_* are
        dead on this path (SURVEY.md §A.6) and therefore not parameters here."""
        cfg = self.cfg
        if seed is not None and rng == "torch":
            import random
            random.seed(seed); np.random.seed(seed); torch.manual_seed(seed)  # at.util.seed, transformer.py:711
        z = start_tokens
        B = z.shape[0]
        ncc, Cp, MT = cfg.n_conditioning_codebooks, cfg.n_predict_codebooks, cfg.mask_token
        if mask is None:  # transformer.py:749-753
            mask = torch.ones_like(z).int()
            mask[:, :ncc, :] = 0
        if mask.ndim == 2:
            mask = mask[:, None, :].repeat(1, z.shape[1], 1)
        z_masked = z.masked_fill(mask.bool(), MT)  # :762
        n0 = (z_masked == MT).sum()  # whole-batch scalar, :766
        sampled_z = None
        for i in range(_sampling_steps):
            r = torch.tensor((i + 1) / _sampling_steps).repeat(B)  # util.py:6-7, fp32
            if logits_fn is None:
                logits = self.forward(self.from_codes(z_masked, codebooks))  # (B, V, S)
            else:
                logits = logits_fn(i, z_masked)
            logits = logits.permute(0, 2, 1)  # (B, S, V)  :849
            do_sample = (i / _sampling_steps) <= sample_cutoff
            sampled_z, sel_p = self.sample_from_logits(logits, do_sample, temperature, top_p,
                                                       rng=rng, philox_key=philox_key, step=i)
            zf = codebook_flatten(z_masked[:, ncc:, :])  # :879
            m = zf == MT
            sampled_z = torch.where(m, sampled_z, zf)  # :893-895
            sel_p = torch.where(m, sel_p, torch.inf)  # :898-900
            num_to_mask = torch.floor(gamma(r) * n0).unsqueeze(1).long()  # :903
            if i != _sampling_steps - 1:  # :906-913
                num_to_mask = torch.maximum(torch.tensor(1),
                                            torch.minimum(m.sum(dim=-1, keepdim=True) - 1, num_to_mask))
            new_mask, conf = self.mask_by_random_topk(num_to_mask, sel_p, mask_temperature * (1 - r),
                                                      rng=rng, philox_key=philox_key, step=i)  # :917-919
            zf_next = torch.where(new_mask, MT, sampled_z)  # :922-924
            z_masked = torch.cat((z[:, :ncc, :], codebook_unflatten(zf_next, Cp)), dim=1)  # :926-932
            if trace is not None:
                trace.append(dict(logits=logits.clone(), tokens=sampled_z.clone(), conf=conf.clone(),
                                  num_to_mask=num_to_mask.clone(), z_masked=z_masked.clone()))
        out = codebook_unflatten(sampled_z, Cp)  # :935-938
        return torch.cat((z[:, :ncc, :], out), dim=1)


# --------------------------------------------------------------------------------------
# Interface-level orchestration (A1-A4), restated from interface.py:328-562 and mask.py:24-38
# with the generate call abstracted so it can be driven by the oracle or compared with the product.
# --------------------------------------------------------------------------------------
def apply_mask(x, mask, mask_token):
    """mask.py:24-38."""
    assert mask.ndim == 3 and mask.shape == x.shape and mask.dtype == torch.long
    assert not torch.any(mask > 1) and not torch.any(mask < 0)
    return x * (1 - mask) + mask_token * mask, mask


def s2t(seconds: float, sample_rate: int = 44100, hop_length: int = 768) -> int:
    """interface.py:176-181."""
    return math.ceil(seconds * sample_rate / hop_length)


def coarse_vamp(z, mask, n_coarse, chunk_len, mask_token, gen_fn):
    """interface.py:383-452.  gen_fn(start_tokens, mask) -> tokens."""
    cz = z[:, :n_coarse, :].clone()
    mask = mask[:, :n_coarse, :]
    n_chunks = math.ceil(cz.shape[-1] / chunk_len)
    masked_chunks, vamped = [], []
    for i in range(n_chunks):
        chunk = cz[:, :, i * chunk_len:(i + 1) * chunk_len]
        mc = mask[:, :, i * chunk_len:(i + 1) * chunk_len]
        if torch.any(mc == 0):  # edge frames force-unmasked, :410-413
            mc = mc.clone()
            mc[:, :, 0] = 0
            mc[:, :, -1] = 0
        cm, mc = apply_mask(chunk, mc, mask_token)
        masked_chunks.append(cm)
        vamped.append(gen_fn(cm, mc))
    c_vamp = torch.cat(vamped, dim=-1)
    c_vamp = torch.cat([c_vamp, z[:, n_coarse:, :]], dim=1)
    return c_vamp, torch.cat(masked_chunks, dim=-1)


def coarse_to_fine(z, mask, n_c2f, n_cond, chunk_len, mask_token, gen_fn):
    """interface.py:328-380."""
    length = z.shape[-1]
    n_chunks = math.ceil(length / chunk_len)
    if length % chunk_len != 0:
        pad = chunk_len - (length % chunk_len)
        z = F.pad(z, (0, pad))
        mask = F.pad(mask, (0, pad), value=1) if mask is not None else None
    if n_c2f - z.shape[1] > 0:
        z = torch.cat([z, torch.zeros(z.shape[0], n_c2f - z.shape[1], z.shape[-1]).long()], dim=1)
    if mask is not None:
        mask = mask.clone()
        mask[:, :n_cond, :] = 0
    fine = []
    for i in range(n_chunks):
        chunk = z[:, :, i * chunk_len:(i + 1) * chunk_len]
        mc = mask[:, :, i * chunk_len:(i + 1) * chunk_len] if mask is not None else None
        fine.append(gen_fn(chunk, mc))
    fine = torch.cat(fine, dim=-1)
    return fine[:, :, :length].clone(), apply_mask(fine, mask, mask_token)[0][:, :, :length].clone()


def vamp(codes, mask, batch_size, feedback_steps, time_stretch_factor, n_coarse, n_c2f, n_cond, coarse_chunk_len,
         c2f_chunk_len, mask_token, coarse_gen, c2f_gen):
    """interface.py:491-562.  coarse_gen / c2f_gen(start_tokens, mask) -> tokens stand in for the two generate()
    calls (the reference forwards **kwargs to the coarse one and pins the fine one to 2 steps, :545-551).
    Returns (z, mask_z) like return_mask=True."""
    z = codes.expand(batch_size, -1, -1)
    mask = mask.expand(batch_size, -1, -1)
    if time_stretch_factor > 1:  # :510-516
        z = z.repeat_interleave(time_stretch_factor, dim=-1)
        mask = mask.repeat_interleave(time_stretch_factor, dim=-1)
        added = torch.ones_like(mask)
        added[:, :, ::time_stretch_factor] = 0
        mask = (mask.bool() | added.bool()).long()
    zv = z
    for i in range(feedback_steps):  # :522-532
        zv, mask_z = coarse_vamp(zv, mask, n_coarse, coarse_chunk_len, mask_token, coarse_gen)
        mask_z = mask_z.roll(shifts=(i + 1) % feedback_steps, dims=-1)
    if zv.shape[1] < z.shape[1]:  # :536-541
        zv = torch.cat([zv, z[:, n_coarse:, :]], dim=1)
    zv, fine_mask = coarse_to_fine(zv, mask, n_c2f, n_cond, c2f_chunk_len, mask_token, c2f_gen)
    mask_z = torch.cat([mask_z[:, :n_coarse, :], fine_mask[:, n_coarse:, :]], dim=1)
    return zv, mask_z
