"""VampNet — drop-in for the reference's ``vampnet.modules.transformer.VampNet`` surface
(reference vampnet/modules/transformer.py:535-946) whose compute runs in hand-written sm_90a
CUDA behind the C ABI (include/vampnet_b200.h).

The nn.Module tree below only *holds parameters* under the reference's state_dict key names
(SURVEY.md §8b) so that reference checkpoints and LoRA overlays load unchanged
(interface.py:27-50); no torch op of the forward pass is ever executed.  There is no CPU path:
calling forward/generate on a CPU-resident model raises.
"""
from __future__ import annotations

import ctypes as C
import math
import random
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from .. import _lib

LORA_R = 8          # reference transformer.py:22
LORA_ALPHA = 1.0    # loralib default (lora.Linear(..., r=LORA_R) never overrides it)
REL_SAT = 128       # attention_max_distance: every |key-query| >= 128 shares the last bucket


# ------------------------------------------------------------------------------------------------
# parameter containers (names mirror the reference module tree; no forward methods)
# ------------------------------------------------------------------------------------------------
class _Weight(nn.Module):
    def __init__(self, *shape, init=None):
        super().__init__()
        w = torch.empty(*shape)
        if init == "ones":
            nn.init.ones_(w)
        elif init == "normal":
            nn.init.normal_(w)
        else:
            nn.init.kaiming_uniform_(w.view(shape[0], -1), a=math.sqrt(5))
        self.weight = nn.Parameter(w)


class _LoraLinear(_Weight):
    """lora.Linear(in, out, bias=False, r=8): weight + lora_A (r,in) + lora_B (out,r)."""

    def __init__(self, out_f, in_f):
        super().__init__(out_f, in_f)
        a = torch.empty(LORA_R, in_f)
        nn.init.kaiming_uniform_(a, a=math.sqrt(5))
        self.lora_A = nn.Parameter(a)
        self.lora_B = nn.Parameter(torch.zeros(out_f, LORA_R))

    def folded(self) -> torch.Tensor:
        return self.weight.float() + (self.lora_B.float() @ self.lora_A.float()) * (LORA_ALPHA / LORA_R)


class _Attention(nn.Module):
    def __init__(self, d, n_heads, has_bias_table):
        super().__init__()
        self.w_qs = _LoraLinear(d, d)
        self.w_ks = _Weight(d, d)
        self.w_vs = _LoraLinear(d, d)
        self.fc = _LoraLinear(d, d)
        if has_bias_table:
            self.relative_attention_bias = _Weight(32, n_heads, init="normal")


class _FeedForward(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.w_1 = _LoraLinear(4 * d, d)
        self.w_2 = _LoraLinear(d, 2 * d)


class _Layer(nn.Module):
    def __init__(self, d, n_heads, first):
        super().__init__()
        self.norm_1 = _Weight(d, init="ones")
        self.self_attn = _Attention(d, n_heads, first)
        self.norm_3 = _Weight(d, init="ones")
        self.feed_forward = _FeedForward(d)


class _Stack(nn.Module):
    def __init__(self, d, n_heads, n_layers):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(d, n_heads, i == 0) for i in range(n_layers)])
        self.norm = _Weight(d, init="ones")


class _WNConv(nn.Module):
    """weight_norm(Conv1d(in, out, 1)): weight_g (out,1,1), weight_v (out,in,1), bias."""

    def __init__(self, in_c, out_c):
        super().__init__()
        v = torch.empty(out_c, in_c, 1)
        nn.init.kaiming_uniform_(v.view(out_c, in_c), a=math.sqrt(5))
        self.weight_v = nn.Parameter(v)
        self.weight_g = nn.Parameter(v.flatten(1).norm(dim=1).view(-1, 1, 1).clone())
        self.bias = nn.Parameter(torch.zeros(out_c))


class _Classifier(nn.Module):
    def __init__(self, in_c, out_c):
        super().__init__()
        self.layers = nn.ModuleList([_WNConv(in_c, out_c)])


class _OutProj(nn.Module):
    def __init__(self, in_c, out_c):
        super().__init__()
        w = torch.empty(out_c, in_c, 1)
        nn.init.kaiming_uniform_(w.view(out_c, in_c), a=math.sqrt(5))
        self.weight = nn.Parameter(w)
        self.bias = nn.Parameter(torch.zeros(out_c))


class CodebookEmbedding(nn.Module):
    """Parameter holder + from_codes for reference layers.py:105-164."""

    def __init__(self, vocab_size, latent_dim, n_codebooks, emb_dim, special_tokens=("MASK",)):
        super().__init__()
        self.n_codebooks = n_codebooks
        self.emb_dim = emb_dim
        self.latent_dim = latent_dim
        self.vocab_size = vocab_size
        self.special = nn.ParameterDict({t: nn.Parameter(torch.randn(n_codebooks, latent_dim)) for t in special_tokens})
        self.special_idxs = {t: i + vocab_size for i, t in enumerate(special_tokens)}
        self.out_proj = _OutProj(n_codebooks * latent_dim, emb_dim)

    def lookup_tables(self, codec, n: Optional[int] = None) -> torch.Tensor:
        """(n, V+1, latent_dim): codec codebook i with this model's MASK row appended (layers.py:145-150)."""
        n = self.n_codebooks if n is None else n
        tabs = []
        for i in range(n):
            cb = codec.quantizer.quantizers[i].codebook.weight.to(self.special["MASK"].device, torch.float32)
            # MASK rows exist only for this model's own codebooks; decode() of more codebooks than that
            # (reference transformer.py:672 with the 4-codebook coarse model and 14-codebook z) never indexes them
            extra = self.special["MASK"][i:i + 1].float() if i < self.n_codebooks else torch.zeros_like(cb[:1])
            tabs.append(torch.cat([cb, extra], dim=0))
        return torch.stack(tabs, 0)

    def from_codes(self, codes: torch.Tensor, codec) -> torch.Tensor:
        """codes (B, C', T) -> latents (B, C'*latent_dim, T).  Pure gather (index_select on the device
        the codes live on); kept for API compatibility (scripts call it), not on the generate() path."""
        tables = self.lookup_tables(codec, codes.shape[1])
        outs = [tables[i][codes[:, i, :]].transpose(1, 2) for i in range(codes.shape[1])]
        return torch.cat(outs, dim=1)


# ------------------------------------------------------------------------------------------------
def relative_position_bucket(rel: torch.Tensor, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """T5 bidirectional buckets for rel = key - query (reference transformer.py:123-181), evaluated with
    the same fp32 torch expressions so the log-spaced boundaries coincide."""
    nb = num_buckets // 2
    ret = (rel > 0).long() * nb
    n = rel.abs()
    exact = nb // 2
    big = exact + (torch.log(n.float() / exact) / math.log(max_distance / exact) * (nb - exact)).long()
    big = big.clamp(max=nb - 1)
    return ret + torch.where(n < exact, n, big)


def gamma_schedule(steps: int):
    """Per-step fp32 schedule values computed exactly as the reference does on CPU
    (util.py:6-7 -> fp32 tensor; mask.py:8-9; transformer.py:831-834, 917-919)."""
    r = torch.tensor([(i + 1) / steps for i in range(steps)], dtype=torch.float64).to(torch.float32)
    g = (r * torch.pi / 2).cos().clamp(1e-10, 1.0)
    return r, g


def draw_philox_key(seed=None) -> int:
    """The sampler's 64-bit Philox key of one generate() call.  A seed reseeds random, numpy and torch (at.util.seed,
    reference transformer.py:711), a process-global side effect callers rely on, and is the key; without a seed the key
    is drawn from torch's (possibly user-seeded) global generator.  Batched callers draw their keys with this in the
    order the sequential calls would, so keys and RNG state afterwards are the same."""
    if seed is not None:
        random.seed(seed)
        np.random.seed(seed)
        torch.manual_seed(seed)
        return int(seed) & 0xFFFFFFFFFFFFFFFF
    return int(torch.randint(0, 2 ** 62, (1,)).item())


# generate_many() splits a launch whose B*T would exceed this many rows: M = 24576 is the largest GEMM height the
# benchmarks measure (BASELINE.json configs[4], B = 8 at T = 3072)
MANY_MAX_ROWS = 24576


class VampNet(nn.Module):
    def __init__(
        self,
        n_heads: int = 20,
        n_layers: int = 16,
        r_cond_dim: int = 0,
        n_codebooks: int = 9,
        n_conditioning_codebooks: int = 0,
        latent_dim: int = 8,
        embedding_dim: int = 1280,
        vocab_size: int = 1024,
        flash_attn: bool = True,
        noise_mode: str = "mask",
        dropout: float = 0.1,
        ctrl_dims: Optional[dict] = None,
        cfg_dropout_prob: float = 0.2,
        cond_dim: int = 0,
    ):
        super().__init__()
        assert r_cond_dim == 0, f"r_cond_dim must be 0 (not supported), but got {r_cond_dim}"
        assert noise_mode == "mask", "deprecated"
        if ctrl_dims is not None:
            raise NotImplementedError("ctrl_dims / ControlEncoder is outside the hot path (SURVEY.md §8)")
        self.n_heads = n_heads
        self.n_layers = n_layers
        self.r_cond_dim = r_cond_dim
        self.n_codebooks = n_codebooks
        self.n_conditioning_codebooks = n_conditioning_codebooks
        self.embedding_dim = embedding_dim
        self.vocab_size = vocab_size
        self.latent_dim = latent_dim
        self.flash_attn = flash_attn  # accepted and ignored: attention is always the fused sm_90a kernel
        self.noise_mode = noise_mode
        self.cond_dim = cond_dim
        self.dropout = dropout
        self.cfg_dropout_prob = cfg_dropout_prob
        self.ctrl_dims = ctrl_dims
        self.n_predict_codebooks = n_codebooks - n_conditioning_codebooks

        self.embedding = CodebookEmbedding(vocab_size=vocab_size, latent_dim=latent_dim, n_codebooks=n_codebooks,
                                           emb_dim=embedding_dim, special_tokens=("MASK",))
        self.mask_token = self.embedding.special_idxs["MASK"]
        self.transformer = _Stack(embedding_dim, n_heads, n_layers)
        self.classifier = _Classifier(embedding_dim, vocab_size * self.n_predict_codebooks)

        self._handle = None       # vnb_model*
        self._packed = None       # dict of device tensors kept alive for the handle
        self._packed_key = None
        self._packed_codec = None
        self.use_cuda_graph = True
        self.eval()

    # ------------------------------------------------------------------ housekeeping
    @property
    def device(self):
        return self.embedding.out_proj.weight.device

    def _invalidate(self):
        if getattr(self, "_handle", None) is not None:
            _lib.lib().vnb_model_destroy(self._handle)
        self._handle = None
        self._packed = None
        self._packed_key = None
        self._packed_codec = None

    def _apply(self, fn, *a, **k):
        self._invalidate()
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, *a, **k):
        """Cold model: plain nn.Module load.  Live model (a device handle exists): hot swap — parameters are
        overwritten in place and the packed device buffers the handle, its tensor maps and its captured generate
        graphs point at are rewritten in place, so no workspace, tensor map or graph is rebuilt (SURVEY.md §8 f-4)."""
        flash = [k for k in state_dict if ".self_attn.Wqkv." in k or ".self_attn.out_proj." in k]
        if flash:
            raise RuntimeError(
                f"state_dict holds FlashMHA tensors ({flash[0]} ...): a flash_attn=True checkpoint has no relative "
                "position bias and different projection names; this implementation covers the flash_attn=False "
                "architecture the released VampNet checkpoints use (conf/vampnet.yml:33)")
        live = self._handle is not None and getattr(self, "_packed_codec", None) is not None
        if not live:
            self._invalidate()
            return super().load_state_dict(state_dict, *a, **k)
        result = super().load_state_dict(state_dict, *a, **k)
        self.repack()
        return result

    @torch.no_grad()
    def repack(self):
        """Re-fold the current parameters into the live handle's packed buffers (same addresses, same shapes)."""
        if self._handle is None:
            return
        # the packed tensors may have been created under generate()'s inference_mode: update them in the same mode
        with torch.inference_mode(), torch.cuda.device(self.device):
            fresh = self.pack_weights(self._packed_codec)
            for name, dst in self._packed.items():
                src = fresh[name]
                if src.shape != dst.shape or src.dtype != dst.dtype:
                    raise RuntimeError(f"packed tensor {name} changed layout {tuple(dst.shape)} -> {tuple(src.shape)}")
                dst.copy_(src)

    def architecture(self) -> dict:
        """The constructor arguments that fix the packed layout (what two checkpoints must share to be hot-swappable)."""
        return dict(n_heads=self.n_heads, n_layers=self.n_layers, n_codebooks=self.n_codebooks,
                    n_conditioning_codebooks=self.n_conditioning_codebooks, latent_dim=self.latent_dim,
                    embedding_dim=self.embedding_dim, vocab_size=self.vocab_size)

    @torch.no_grad()
    def swap_checkpoint(self, location, map_location="cpu") -> bool:
        """Load another checkpoint of the SAME architecture into this model in place (LoRA checkpoints included).
        Tensors the checkpoint does not carry go back to their constructor state where that matters for the result
        (lora_B = 0, i.e. no adapter), which is what the reference gets by building a fresh model in reload()
        (interface.py:146-174).  Returns False — and changes nothing — when the architecture differs."""
        blob = torch.load(str(location), map_location=map_location, weights_only=False)
        import inspect
        defaults = {k: v.default for k, v in inspect.signature(type(self).__init__).parameters.items()}
        want = dict(blob.get("metadata", {}).get("kwargs", {}))
        if any(want.get(k, defaults[k]) != v for k, v in self.architecture().items()):
            return False
        sd = blob["state_dict"]
        for name, prm in self.named_parameters():
            if name.endswith("lora_B") and name not in sd:
                prm.zero_()
        self.load_state_dict(sd, strict=False)
        return True

    def __del__(self):
        try:
            self._invalidate()
        except Exception:
            pass

    @classmethod
    def load(cls, location, map_location="cpu", strict: bool = False, **kwargs):
        """audiotools BaseModel.load: a torch-saved dict with 'state_dict' and 'metadata'['kwargs']
        (interface.py:34)."""
        blob = torch.load(str(location), map_location=map_location, weights_only=False)
        ctor = dict(blob.get("metadata", {}).get("kwargs", {}))
        ctor.update(kwargs)
        import inspect
        ok = set(inspect.signature(cls.__init__).parameters)
        model = cls(**{k: v for k, v in ctor.items() if k in ok})
        res = model.load_state_dict(blob["state_dict"], strict=strict)
        # strict=False (how the reference loads, interface.py:34) tolerates absent LoRA adapters, nothing else: a
        # checkpoint of another architecture would otherwise leave projections at their random initialisation
        missing = [k for k in getattr(res, "missing_keys", []) if ".lora_" not in k]
        if missing:
            raise RuntimeError(f"checkpoint {location} lacks {len(missing)} tensors of this architecture, e.g. {missing[:3]}")
        return model

    # ------------------------------------------------------------------ weight packing
    @torch.no_grad()
    def pack_weights(self, codec) -> dict:
        """Fold LoRA (W + B.A*alpha/r) and weight-norm (g*v/|v|), round GEMM weights to bf16 once, and lay
        them out as include/vampnet_b200.h: vnb_weights documents."""
        dev = self.device
        d, L, C_, Cp, V, H = (self.embedding_dim, self.n_layers, self.n_codebooks, self.n_predict_codebooks,
                              self.vocab_size, self.n_heads)
        bf = torch.bfloat16
        p = {}
        p["emb_table"] = self.embedding.lookup_tables(codec).to(dev).contiguous()
        # out_proj as a tensor-core contraction with fp32-grade accuracy: w = hi + lo in bf16, K padded to a multiple of
        # 64, rows [hi | lo | hi] against the gathered latents [a_hi | a_hi | a_lo] (vnb_weights.emb_w3)
        w = self.embedding.out_proj.weight.float().squeeze(-1)                      # (d, 8C)
        kp = (w.shape[1] + 63) // 64 * 64
        wp = torch.zeros(d, kp, device=w.device, dtype=torch.float32)
        wp[:, :w.shape[1]] = w
        hi = wp.to(bf)
        lo = (wp - hi.float()).to(bf)
        p["emb_w3"] = torch.cat([hi, lo, hi], dim=1).contiguous()                   # (d, 3*Kp)
        p["emb_b"] = self.embedding.out_proj.bias.float().contiguous()
        lay = self.transformer.layers
        p["norm1"] = torch.stack([l.norm_1.weight.float() for l in lay]).contiguous()
        p["norm3"] = torch.stack([l.norm_3.weight.float() for l in lay]).contiguous()
        # RMSNorm is fused into the consuming GEMMs: norm weights are folded into the K axis of wqkv / w1 / wcls here,
        # the kernels apply rsqrt(mean(x^2) + eps) as a row scale in their epilogues (DESIGN.md §4)
        p["wqkv"] = torch.stack([torch.cat([l.self_attn.w_qs.folded(), l.self_attn.w_ks.weight.float(),
                                            l.self_attn.w_vs.folded()], 0) * l.norm_1.weight.float()[None, :]
                                 for l in lay]).to(bf).contiguous()
        p["wo"] = torch.stack([l.self_attn.fc.folded() for l in lay]).to(bf).contiguous()
        w1 = torch.stack([l.feed_forward.w_1.folded() * l.norm_3.weight.float()[None, :] for l in lay])  # (L, 4d, d): [value 2d | gate 2d]
        nt = (2 * d) // 128
        val = w1[:, :2 * d].view(L, nt, 128, d)
        gate = w1[:, 2 * d:].view(L, nt, 128, d)
        p["w1"] = torch.cat([val, gate], dim=2).reshape(L, 4 * d, d).to(bf).contiguous()
        p["w2"] = torch.stack([l.feed_forward.w_2.folded() for l in lay]).to(bf).contiguous()
        p["norm_f"] = self.transformer.norm.weight.float().contiguous()
        wn = self.classifier.layers[0]
        v = wn.weight_v.float().squeeze(-1)
        w = v * (wn.weight_g.float().view(-1, 1) / v.norm(dim=1, keepdim=True))
        w = w * self.transformer.norm.weight.float()[None, :]
        # channel r = p*Cp + c  ->  row c*V + p, so a row-major (M, Cp*V) store IS (B, S = t*Cp + c, V)
        p["wcls"] = w.view(V, Cp, d).permute(1, 0, 2).reshape(Cp * V, d).to(bf).contiguous()
        p["bcls"] = wn.bias.float().view(V, Cp).t().reshape(-1).contiguous()
        # Toeplitz bias table over key-query in [-sat, sat]; sat = the distance beyond which the bucket no longer
        # changes (91 for the reference's 32 buckets / max_distance 128), found from the bucket function itself
        probe = relative_position_bucket(torch.arange(-REL_SAT, REL_SAT + 1))
        sat = REL_SAT
        while sat > 1 and probe[REL_SAT + sat - 1] == probe[-1] and probe[REL_SAT - (sat - 1)] == probe[0]:
            sat -= 1
        self._rel_sat = sat
        rel = torch.arange(-sat, sat + 1)
        buckets = relative_position_bucket(rel).to(dev)
        p["rel_bias"] = lay[0].self_attn.relative_attention_bias.weight.float()[buckets].contiguous()  # (2*sat+1, H)
        return p

    def _ensure_handle(self, codec):
        if self.device.type != "cuda":
            raise RuntimeError("vampnet_b200.VampNet runs only on a CUDA (sm_90a) device; there is no CPU fallback. "
                               "Move the model with .to('cuda').")
        key = (id(codec), str(self.device))
        if self._handle is not None and self._packed_key == key:
            return
        self._invalidate()
        lib = _lib.lib()
        with torch.cuda.device(self.device):
            p = self.pack_weights(codec)
            cfg = _lib.Config(self.n_heads, self.n_layers, self.n_codebooks, self.n_conditioning_codebooks,
                              self.latent_dim, self.embedding_dim, self.vocab_size)
            w = _lib.Weights()
            for name in ("emb_table", "emb_w3", "emb_b", "norm1", "wqkv", "wo", "norm3", "w1", "w2", "norm_f", "wcls",
                         "bcls", "rel_bias"):
                setattr(w, name, p[name].data_ptr())
            w.rel_sat = self._rel_sat
            h = C.c_void_p()
            torch.cuda.synchronize(self.device)
            _lib.check(lib.vnb_model_create(C.byref(cfg), C.byref(w), C.byref(h)))
        self._handle, self._packed, self._packed_key = h, p, key
        self._packed_codec = codec

    # ------------------------------------------------------------------ forward
    class _NoCodec:
        """forward() takes latents, so the gather tables are unused; pack with zero codebooks."""

        def __init__(self, n, V, ld, dev):
            q = [type("Q", (), {"codebook": type("CB", (), {"weight": torch.zeros(V, ld, device=dev)})()})()
                 for _ in range(n)]
            self.quantizer = type("QZ", (), {"quantizers": q})()

    @torch.no_grad()
    def forward(self, x, ctrls=None, ctrl_masks=None, return_activations: bool = False):
        """x: latents (B, n_codebooks*latent_dim, T) -> logits (B, vocab, T*n_predict_codebooks)
        (reference transformer.py:617-639).  Returned as a permuted view of the kernel's (B, S, V) buffer."""
        if ctrls is not None or ctrl_masks is not None:
            raise NotImplementedError("controls are outside the hot path (SURVEY.md §8)")
        if self._handle is None:
            self._codec_stub = self._NoCodec(self.n_codebooks, self.vocab_size, self.latent_dim, self.device)
            self._ensure_handle(self._codec_stub)
        B, K, T = x.shape
        assert K == self.n_codebooks * self.latent_dim, (K, self.n_codebooks, self.latent_dim)
        x = x.to(self.device, torch.float32).contiguous()
        S = T * self.n_predict_codebooks
        logits = torch.empty(B, S, self.vocab_size, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            if return_activations:  # the residual stream after every layer (reference :443-461, :626-637)
                acts = torch.empty(self.n_layers, B, T, self.embedding_dim, device=self.device, dtype=torch.float32)
                _lib.check(_lib.lib().vnb_forward_latents_acts(self._handle, _lib.ptr(x), B, T, _lib.ptr(logits),
                                                               _lib.ptr(acts), _lib.stream_ptr(self.device)))
                return logits.permute(0, 2, 1), acts
            _lib.check(_lib.lib().vnb_forward_latents(self._handle, _lib.ptr(x), B, T, _lib.ptr(logits),
                                                      _lib.stream_ptr(self.device)))
        return logits.permute(0, 2, 1)

    @torch.no_grad()
    def forward_codes(self, codes: torch.Tensor, codec) -> torch.Tensor:
        """embedding.from_codes + forward fused: codes (B, C, T) int64 (mask token allowed) -> (B, S, V) fp32."""
        self._ensure_handle(codec)
        B, C_, T = codes.shape
        assert C_ == self.n_codebooks
        codes = codes.to(self.device, torch.int64).contiguous()
        logits = torch.empty(B, T * self.n_predict_codebooks, self.vocab_size, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().vnb_forward_codes(self._handle, _lib.ptr(codes), B, T, _lib.ptr(logits),
                                                    _lib.stream_ptr(self.device)))
        return logits

    def hidden_state(self, B: int, T: int) -> torch.Tensor:
        """fp32 residual stream (B, T, d) after the last layer of the most recent forward of that shape (debug tap)."""
        out = torch.empty(B, T, self.embedding_dim, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().vnb_get_hidden(self._handle, _lib.ptr(out), _lib.stream_ptr(self.device)))
        return out

    # ------------------------------------------------------------------ generate
    @torch.inference_mode()
    def generate(
        self,
        codec,
        time_steps: int = 300,
        _sampling_steps: int = 12,
        start_tokens: Optional[torch.Tensor] = None,
        temperature: float = 1.0,
        mask: Optional[torch.Tensor] = None,
        mask_temperature: float = 10.5,
        ctrls: dict = None,
        ctrl_masks: dict = None,
        typical_filtering=True,
        typical_mass=0.15,
        typical_min_tokens=64,
        top_p=None,
        seed: int = None,
        sample_cutoff: float = 1.0,
        return_signal=True,
        debug=False,
        causal_weight: float = 0.0,
        cfg_scale: float = 3.0,
        cfg_guidance: float = None,
        cond=None,
        philox_key: int = None,
    ):
        """Iterative parallel decoding, reference transformer.py:686-946.

        Accepted-and-ignored exactly as the reference ignores them (SURVEY.md §A.6): typical_filtering /
        typical_mass / typical_min_tokens (its result is discarded at :989-993), causal_weight, cond,
        cfg_scale, debug.  cfg_guidance only computes an unused tensor in the reference (:845-847) but also
        doubles the batch; it is None on every call path of Interface and is rejected here.
        philox_key (not in the reference): a key already drawn with draw_philox_key(); the global RNGs are then left
        alone, and `seed` must be None.
        """
        call = self._prepare_call(codec, time_steps, _sampling_steps, start_tokens, temperature, mask,
                                  mask_temperature, ctrls, ctrl_masks, top_p, seed, sample_cutoff, cfg_guidance,
                                  philox_key)
        out = self._launch_calls([call])[0]
        if return_signal:
            return self.decode(out, codec)
        return out

    @torch.inference_mode()
    def generate_many(self, codec, calls):
        """Run many independent generate() calls, batched into as few launches as the shapes allow.

        `calls` is a list of dicts of generate() keyword arguments.  The result equals
        [self.generate(codec, **c) for c in calls] bit for bit, return_signal included, and the random, numpy and torch
        global RNG states afterwards are those the sequential calls leave: keys are drawn (draw_philox_key) in list
        order.  Calls with the same T, sampling steps and top-p on/off share one vnb_generate_many launch, in which
        each keeps its own N0, temperatures, schedules, top_p and key; a launch whose B*T would exceed MANY_MAX_ROWS is
        split."""
        import inspect
        sig = inspect.signature(VampNet.generate)
        prepared, want_signal = [], []
        for kw in calls:
            a = sig.bind(self, codec, **kw)
            a.apply_defaults()
            a = a.arguments
            prepared.append(self._prepare_call(codec, a["time_steps"], a["_sampling_steps"], a["start_tokens"],
                                               a["temperature"], a["mask"], a["mask_temperature"], a["ctrls"],
                                               a["ctrl_masks"], a["top_p"], a["seed"], a["sample_cutoff"],
                                               a["cfg_guidance"], a["philox_key"]))
            want_signal.append(bool(a["return_signal"]))
        outs = self._launch_calls(prepared)
        return [self.decode(o, codec) if sig_ else o for o, sig_ in zip(outs, want_signal)]

    def _prepare_call(self, codec, time_steps, steps, start_tokens, temperature, mask, mask_temperature, ctrls,
                      ctrl_masks, top_p, seed, sample_cutoff, cfg_guidance, philox_key) -> dict:
        """Validate one generate() call, draw its key and stage its device inputs and per-step host schedules."""
        if ctrls is not None or ctrl_masks is not None:
            raise NotImplementedError("ctrls/ctrl_masks: ControlEncoder is outside the hot path")
        if cfg_guidance is not None:
            raise NotImplementedError("cfg_guidance is dead code in the reference (transformer.py:845-847)")
        if philox_key is not None:
            if seed is not None:
                raise ValueError("generate: pass either seed or philox_key, not both")
            k = int(philox_key) & 0xFFFFFFFFFFFFFFFF
        else:
            k = draw_philox_key(seed)
        self._ensure_handle(codec)
        dev = self.device
        steps = int(steps)
        if start_tokens is None:
            z = torch.full((1, self.n_codebooks, time_steps), self.mask_token, device=dev, dtype=torch.int64)
        else:
            z = start_tokens.to(dev, torch.int64).contiguous()
        B, C_, T = z.shape
        assert C_ == self.n_codebooks, f"expected {self.n_codebooks} codebooks, got {C_}"
        m32 = None
        if mask is not None:
            if mask.ndim == 2:
                mask = mask[:, None, :].repeat(1, C_, 1)
            # the reference applies the mask with z.masked_fill(mask.bool(), ...) (:762): broadcastable masks are legal
            m32 = (mask.to(dev) != 0).expand_as(z).to(torch.int32).contiguous()
        r, g = gamma_schedule(steps)
        temp_eff = (mask_temperature * (1 - r)).to(torch.float32)
        return dict(z=z, mask=m32, steps=steps, temperature=float(temperature), gamma=[float(v) for v in g],
                    temp_eff=[float(v) for v in temp_eff],
                    do_sample=[1 if (i / steps) <= sample_cutoff else 0 for i in range(steps)], key=k,
                    top_p=float(top_p) if (top_p is not None and top_p < 1.0) else 0.0)

    def _launch_calls(self, calls: list) -> list:
        """Launch prepared calls, one vnb_generate_many per (T, steps, top-p on) bucket of at most MANY_MAX_ROWS rows
        (a single larger call runs alone); returns each call's (B, C, T) int64 tokens in list order."""
        buckets = {}
        for i, c in enumerate(calls):
            top_p_on = 0.0 < c["top_p"] < 1.0
            buckets.setdefault((c["z"].shape[-1], c["steps"], top_p_on), []).append(i)
        launches = []
        for (T, _, _), idx in buckets.items():
            cur, rows = [], 0
            for i in idx:
                B = calls[i]["z"].shape[0]
                if cur and (rows + B) * T > MANY_MAX_ROWS:
                    launches.append(cur)
                    cur, rows = [], 0
                cur.append(i)
                rows += B
            launches.append(cur)
        outs = [None] * len(calls)
        keep = []
        for idx in launches:
            group = [calls[i] for i in idx]
            for i, o in zip(idx, self._launch_group(group, keep)):
                outs[i] = o
        # graph replay bakes the input pointers: keep them alive until the stream has consumed them
        self._last_io = keep
        return outs

    def _launch_group(self, calls: list, keep: list) -> list:
        dev = self.device
        if len(calls) == 1:
            z, m32 = calls[0]["z"], calls[0]["mask"]
        else:
            z = torch.cat([c["z"] for c in calls])
            m32 = None
            if any(c["mask"] is not None for c in calls):
                # a call without a mask gets the default one materialised (predicted codebooks masked,
                # transformer.py:749-751): the launch takes one mask for all rows
                default = (torch.arange(self.n_codebooks, device=dev) >= self.n_conditioning_codebooks).to(torch.int32)
                m32 = torch.cat([c["mask"] if c["mask"] is not None else default[None, :, None].expand_as(c["z"])
                                 for c in calls]).contiguous()
        B, _, T = z.shape
        steps = calls[0]["steps"]
        arrays = []
        groups = (_lib.GenGroup * len(calls))()
        for g, c in zip(groups, calls):
            tef = (C.c_float * steps)(*c["temp_eff"])
            dos = (C.c_int32 * steps)(*c["do_sample"])
            arrays += [tef, dos]
            g.rows, g.temperature, g.temp_eff, g.do_sample = c["z"].shape[0], c["temperature"], tef, dos
            g.seed_lo, g.seed_hi, g.top_p = c["key"] & 0xFFFFFFFF, (c["key"] >> 32) & 0xFFFFFFFF, c["top_p"]
        gam = (C.c_float * steps)(*calls[0]["gamma"])
        out = torch.empty_like(z)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().vnb_generate_many(self._handle, _lib.ptr(z), _lib.ptr(m32), B, T, steps, gam, groups,
                                                    len(calls), 1 if self.use_cuda_graph else 0, _lib.ptr(out),
                                                    _lib.stream_ptr(dev)))
        keep.append((z, m32, out))
        return list(out.split([c["z"].shape[0] for c in calls]))

    @torch.no_grad()
    def decode(self, z, codec):
        """reference transformer.py:661-684: mask tokens -> 0, codes -> latents -> codec.quantizer.from_latents
        -> codec.decode.  The per-frame silence loop at :678-682 is dead after the masked_fill at :669 and
        costs T host syncs in the reference; it is not reproduced."""
        assert z.ndim == 3
        z = z.masked_fill(z == self.mask_token, 0)
        from ..audio import AudioSignal
        zq = codec.quantizer.from_latents(self.embedding.from_codes(z, codec))[0]
        return AudioSignal(codec.decode(zq)["audio"], codec.sample_rate)
