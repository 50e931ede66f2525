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


def rel_bias_table(weight: torch.Tensor):
    """The attention kernel's bias operand from the per-bucket weights (32, H): the Toeplitz table (2*sat+1, H) fp32
    over key - query in [-sat, sat], and sat, the distance beyond which the bucket no longer changes (91 for the
    reference's 32 buckets / max_distance 128), found from the bucket function itself."""
    probe = relative_position_bucket(torch.arange(-REL_SAT, REL_SAT + 1))
    sat = REL_SAT
    while sat > 1 and probe[REL_SAT + sat - 1] == probe[-1] and probe[REL_SAT - (sat - 1)] == probe[0]:
        sat -= 1
    buckets = relative_position_bucket(torch.arange(-sat, sat + 1)).to(weight.device)
    return weight.float()[buckets].contiguous(), sat


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


# the five LoRA'd projections of every layer (reference transformer.py:109-114, 70-84): what a fine-tune differs in
LORA_MODULES = ("self_attn.w_qs", "self_attn.w_vs", "self_attn.fc", "feed_forward.w_1", "feed_forward.w_2")


def pack_adapter(lora: dict, norm1: torch.Tensor, norm3: torch.Tensor, d: int, device) -> dict:
    """A' / B' of one adapter in the layout include/vampnet_b200.h: vnb_adapter_weights documents.
    lora[(layer, module)] = (lora_A (8, in), lora_B (out, 8)); norm1 / norm3 (L, d) the base model's RMSNorm weights.
    A' = lora_A with the norm folded into its columns (as wqkv / w1 get it), k-major; B' = lora_B * alpha / r with rows
    permuted like the packed weight rows (w1: 128 value rows then 128 gate rows per 256-row tile).  All fp32."""
    L = norm1.shape[0]
    s = LORA_ALPHA / LORA_R
    f = lambda t: t.to(device, torch.float32)
    out = {k: [] for k in ("a_qkv", "b_qkv", "a_wo", "b_wo", "a_w1", "b_w1", "a_w2", "b_w2")}
    nt = (2 * d) // 128
    for l in range(L):
        (aq, bq), (av, bv), (ao, bo), (a1, b1), (a2, b2) = [tuple(map(f, lora[(l, m)])) for m in LORA_MODULES]
        n1, n3 = f(norm1[l]), f(norm3[l])
        out["a_qkv"].append(torch.cat([(aq * n1[None, :]).t(), (av * n1[None, :]).t()], 1))   # (d, 16)
        out["b_qkv"].append(torch.cat([bq, bv], 0) * s)                                      # (2d, 8)
        out["a_wo"].append(ao.t())
        out["b_wo"].append(bo * s)
        out["a_w1"].append((a1 * n3[None, :]).t())
        b1s = b1 * s                                                                         # (4d, 8): [value 2d | gate 2d]
        out["b_w1"].append(torch.cat([b1s[:2 * d].view(nt, 128, LORA_R), b1s[2 * d:].view(nt, 128, LORA_R)], 1)
                           .reshape(4 * d, LORA_R))
        out["a_w2"].append(a2.t())
        out["b_w2"].append(b2 * s)
    return {k: torch.stack(v).contiguous() for k, v in out.items()}


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
        self._adapters = {}       # name -> packed A' / B' (pack_adapter), registered with every handle
        self._adapter_ids = {}    # name -> id in the live handle's adapter table
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
        self._adapter_ids = {}
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
        # registered adapters belong to the current base: a new base (or a folded fine-tune) drops them
        drop = bool(getattr(self, "_adapters", None)) and self._differing_base_tensor(state_dict) is not None
        if not live:
            self._invalidate()
            result = super().load_state_dict(state_dict, *a, **k)
        else:
            result = super().load_state_dict(state_dict, *a, **k)
            self.repack()
        if drop or (getattr(self, "_adapters", None) and self._is_folded()):
            self._drop_adapters()
        return result

    # ------------------------------------------------------------------ per-request adapters
    def _differing_base_tensor(self, state_dict):
        """Name of the first non-LoRA tensor of state_dict that differs from this model's (shape or value), or None."""
        params = dict(self.named_parameters())
        for name, t in state_dict.items():
            if ".lora_" in name or name not in params:
                continue
            p = params[name]
            if tuple(t.shape) != tuple(p.shape) or not torch.equal(t.detach().to(p.device, p.dtype), p.detach()):
                return name
        return None

    def _is_folded(self) -> bool:
        return any(bool((p != 0).any()) for n, p in self.named_parameters() if n.endswith("lora_B"))

    def _drop_adapters(self):
        lib = _lib.lib() if self._handle is not None else None
        for name, i in self._adapter_ids.items():
            _lib.check(lib.vnb_adapter_remove(self._handle, i))
        self._adapters, self._adapter_ids = {}, {}

    @torch.no_grad()
    def add_adapter(self, name: str, location_or_state_dict):
        """Register a fine-tune of this base model as a per-request adapter: generate(adapter=name) and
        forward_codes(adapter=name) then apply its LoRA (rank 8 on w_qs, w_vs, fc, w_1, w_2) to their rows only, on top
        of the shared base weights.  Takes a checkpoint in the layout load_finetuned reads (a path or a loaded dict with
        'state_dict' and 'metadata'), or a plain state dict.  Refuses another architecture, a checkpoint whose non-LoRA
        tensors differ from this model's, a rank other than 8, and a live model that is itself a folded fine-tune."""
        blob = location_or_state_dict
        if not isinstance(blob, dict):
            blob = torch.load(str(blob), map_location="cpu", weights_only=False)
        sd = blob.get("state_dict", blob) if isinstance(blob.get("state_dict", None), dict) else blob
        if "metadata" in blob:
            import inspect
            defaults = {k: v.default for k, v in inspect.signature(type(self).__init__).parameters.items()}
            want = dict(blob["metadata"].get("kwargs", {}))
            bad = [k for k, v in self.architecture().items() if want.get(k, defaults[k]) != v]
            if bad:
                raise ValueError(f"add_adapter({name!r}): the checkpoint's architecture differs ({bad[0]} = "
                                 f"{want.get(bad[0], defaults[bad[0]])}, this model has {self.architecture()[bad[0]]})")
        if self._is_folded():
            raise ValueError(f"add_adapter({name!r}): the live model carries a non-zero lora_B (a folded fine-tune); "
                             "adapters apply on top of a base model only")
        lora = {}
        for l in range(self.n_layers):
            for m in LORA_MODULES:
                key = f"transformer.layers.{l}.{m}"
                if key + ".lora_A" not in sd or key + ".lora_B" not in sd:
                    raise ValueError(f"add_adapter({name!r}): {key}.lora_A / lora_B missing: not a LoRA fine-tune of "
                                     "this architecture")
                a, b = sd[key + ".lora_A"], sd[key + ".lora_B"]
                prm = self.get_submodule(key).weight
                if a.shape[0] != LORA_R or b.shape[1] != LORA_R:
                    raise ValueError(f"add_adapter({name!r}): {key} has LoRA rank {a.shape[0]}; only rank {LORA_R} "
                                     "is supported")
                if tuple(a.shape) != (LORA_R, prm.shape[1]) or tuple(b.shape) != (prm.shape[0], LORA_R):
                    raise ValueError(f"add_adapter({name!r}): {key} LoRA shapes {tuple(a.shape)}, {tuple(b.shape)} do "
                                     "not fit this architecture")
                lora[(l, m)] = (a, b)
        diff = self._differing_base_tensor(sd)
        if diff is not None:
            raise ValueError(f"add_adapter({name!r}): {diff} differs from the live model's: the checkpoint is not a "
                             "fine-tune of this base")
        if name in self._adapters:
            self.remove_adapter(name)
        if len(self._adapters) >= _lib.MAX_ADAPTERS:
            raise ValueError(f"add_adapter({name!r}): {_lib.MAX_ADAPTERS} adapters are already registered")
        lay = self.transformer.layers
        norm1 = torch.stack([x.norm_1.weight.detach() for x in lay])
        norm3 = torch.stack([x.norm_3.weight.detach() for x in lay])
        with torch.inference_mode():
            self._adapters[name] = pack_adapter(lora, norm1, norm3, self.embedding_dim, self.device)
        if self._handle is not None:
            self._register_adapter(name)

    def remove_adapter(self, name: str):
        if name not in self._adapters:
            raise KeyError(f"adapter {name!r} is not registered")
        if name in self._adapter_ids:
            _lib.check(_lib.lib().vnb_adapter_remove(self._handle, self._adapter_ids.pop(name)))
        del self._adapters[name]

    def adapters(self) -> list:
        """Names of the registered adapters."""
        return sorted(self._adapters)

    def _register_adapter(self, name: str):
        p = self._adapters[name]
        if p["a_qkv"].device != self.device:
            with torch.inference_mode():
                p = self._adapters[name] = {k: v.to(self.device) for k, v in p.items()}
        w = _lib.AdapterWeights(**{k: v.data_ptr() for k, v in p.items()})
        i = C.c_int32()
        _lib.check(_lib.lib().vnb_adapter_add(self._handle, C.byref(w), C.byref(i)))
        self._adapter_ids[name] = i.value

    def _adapter_id(self, name) -> int:
        """-1 for the base model, else the live handle's id of a registered adapter (raises for an unknown name)."""
        if name is None:
            return -1
        if name not in self._adapters:
            raise KeyError(f"adapter {name!r} is not registered (add_adapter; a hot swap of the base drops adapters)")
        return self._adapter_ids[name]

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
        p["rel_bias"], self._rel_sat = rel_bias_table(lay[0].self_attn.relative_attention_bias.weight.to(dev))
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
        for name in self._adapters:
            self._register_adapter(name)

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
    def forward_codes(self, codes: torch.Tensor, codec, adapter: str = None) -> torch.Tensor:
        """embedding.from_codes + forward fused: codes (B, C, T) int64 (mask token allowed) -> (B, S, V) fp32.
        adapter: the name of a registered adapter (add_adapter) to apply, None for the base model."""
        if adapter is not None and adapter not in self._adapters:
            self._adapter_id(adapter)  # raises
        self._ensure_handle(codec)
        B, C_, T = codes.shape
        assert C_ == self.n_codebooks
        codes = codes.to(self.device, torch.int64).contiguous()
        logits = torch.empty(B, T * self.n_predict_codebooks, self.vocab_size, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            if adapter is None:
                _lib.check(_lib.lib().vnb_forward_codes(self._handle, _lib.ptr(codes), B, T, _lib.ptr(logits),
                                                        _lib.stream_ptr(self.device)))
            else:
                rows = (C.c_int32 * B)(*([self._adapter_id(adapter)] * B))
                _lib.check(_lib.lib().vnb_forward_codes_adapted(self._handle, _lib.ptr(codes), B, T, rows,
                                                                _lib.ptr(logits), _lib.stream_ptr(self.device)))
        return logits

    @torch.no_grad()
    def validate(self, codec, z: torch.Tensor, r=None, mask: torch.Tensor = None, rng=None, label_smoothing: float = 0.1,
                 adapter: str = None) -> dict:
        """One validation step of the reference's training script (scripts/exp/train.py val_loop, :327-371) from codes.

        z: (B, C', T) codes with C' >= n_codebooks; the first n_codebooks are used (train.py:334).  Pass exactly one of
        r, each item's mask ratio (a number or a (B,) tensor), and rng, a torch.quasirandom.SobolEngine that draws it
        as rng.draw(B)[:, 0] (train.py:339).  Without a mask the mask is pmask.random(z, r) with the conditioning
        codebooks unmasked (the reference's torch calls, so the same RNG state gives the same mask); a given (B,
        n_codebooks or C', T) binary mask is used as given.  The logits are forward_codes(apply_mask(z, mask)), with
        adapter applied.

        Returns the reference's dict: "loss", CrossEntropyLoss(label_smoothing, ignore_index=-100) over the masked
        tokens, and "accuracy-{0-0.5,0.5-1.0}/top{1,25}/{unmasked,masked}", each a 0-d fp32 tensor on the model's
        device.  Nothing from the forward to the returned dict synchronises."""
        from .. import mask as pmask
        from ..metrics import KEYS, xent_metrics
        if z.ndim != 3 or z.shape[1] < self.n_codebooks:
            raise ValueError(f"validate: z must be (B, C >= {self.n_codebooks}, T), got {tuple(z.shape)}")
        if (r is None) == (rng is None):
            raise ValueError("validate: pass exactly one of r and rng")
        ls = float(label_smoothing)
        if not 0.0 <= ls <= 1.0:
            raise ValueError(f"validate: label_smoothing must be in [0, 1], got {label_smoothing}")
        full_shape = tuple(z.shape)
        B, T = z.shape[0], z.shape[-1]
        dev = self.device
        z = z[:, :self.n_codebooks].to(dev, torch.int64)
        if rng is not None:
            r = rng.draw(B)[:, 0]
        elif not torch.is_tensor(r):
            r = pmask._scalar_to_batch(r, B)
        if tuple(r.shape) != (B,):
            raise ValueError(f"validate: r must be a number or a ({B},) tensor, got shape {tuple(r.shape)}")
        r = r.to(dev)
        if mask is None:
            mask = pmask.codebook_unmask(pmask.random(z, r), self.n_conditioning_codebooks)
        else:
            if tuple(mask.shape) not in (full_shape, (B, self.n_codebooks, T)):
                raise ValueError(f"validate: mask {tuple(mask.shape)} must be (B, n_codebooks, T) = "
                                 f"{(B, self.n_codebooks, T)} or z's shape {full_shape}")
            mask = mask[:, :self.n_codebooks].to(dev, torch.int64)
            if not bool(((mask == 0) | (mask == 1)).all()):
                raise ValueError("validate: mask must be binary")
        z_mask, mask = pmask.apply_mask(z, mask, self.mask_token, check=False)
        logits = self.forward_codes(z_mask, codec, adapter=adapter)
        out = xent_metrics(logits, z, mask, r, self.n_conditioning_codebooks, ls)
        return {k: out[i] for i, k in enumerate(KEYS)}

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
        adapter: str = None,
    ):
        """Iterative parallel decoding, reference transformer.py:686-946.

        Accepted-and-ignored exactly as the reference ignores them (SURVEY.md §A.6): typical_filtering /
        typical_mass / typical_min_tokens (its result is discarded at :989-993), causal_weight, cond,
        cfg_scale, debug.  cfg_guidance only computes an unused tensor in the reference (:845-847) but also
        doubles the batch; it is None on every call path of Interface and is rejected here.
        philox_key (not in the reference): a key already drawn with draw_philox_key(); the global RNGs are then left
        alone, and `seed` must be None.
        adapter (not in the reference): the name of a registered adapter (add_adapter) to generate with, None for the
        base model.
        """
        call = self._prepare_call(codec, time_steps, _sampling_steps, start_tokens, temperature, mask,
                                  mask_temperature, ctrls, ctrl_masks, top_p, seed, sample_cutoff, cfg_guidance,
                                  philox_key, adapter)
        out = self._launch_calls([call])[0]
        if return_signal:
            return self.decode(out, codec)
        return out

    @torch.inference_mode()
    def generate_many(self, codec, calls, mixed_lengths: bool = False, mixed_steps: bool = False,
                      mixed_top_p: bool = False):
        """Run many independent generate() calls, batched into as few launches as the shapes allow.

        `calls` is a list of dicts of generate() keyword arguments.  The result equals
        [self.generate(codec, **c) for c in calls] bit for bit, return_signal included, and the random, numpy and torch
        global RNG states afterwards are those the sequential calls leave: keys are drawn (draw_philox_key) in list
        order.  Calls with the same T, sampling steps and top-p on/off share one vnb_generate_many launch, in which
        each keeps its own N0, temperatures, schedules, top_p, key and adapter; a launch whose B*T would exceed
        MANY_MAX_ROWS is split.

        mixed_lengths=True: calls of different T share launches too (one vnb_generate_ragged per (steps, top-p on/off)
        bucket and MANY_MAX_ROWS).  Each call is padded to its launch's longest T with kept frames (code 0, mask 0)
        that attention does not read, and its result is cut back to its own T; the results are still bit-identical.

        mixed_steps=True: calls of different sampling-step counts share launches too (vnb_generate_steps; the bucket key
        drops the steps, the MANY_MAX_ROWS split is unchanged).  Each launch's calls are ordered by steps, longest first
        (stable); a launch runs as many iterations as its longest call, and a call of fewer steps is idle, and costs
        close to nothing, until its own steps fill the launch's last iterations.  The results are still bit-identical.

        mixed_top_p=True: nucleus (top-p) and plain-sampling calls share launches too (vnb_generate_mixed_top_p; the
        bucket key drops top-p on/off, the MANY_MAX_ROWS split and the orders above are unchanged).  Each row draws as
        its own call would; the results are still bit-identical."""
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
                                               a["cfg_guidance"], a["philox_key"], a["adapter"]))
            want_signal.append(bool(a["return_signal"]))
        outs = self._launch_calls(prepared, mixed_lengths, mixed_steps, mixed_top_p)
        return [self.decode(o, codec) if sig_ else o for o, sig_ in zip(outs, want_signal)]

    def _prepare_call(self, codec, time_steps, steps, start_tokens, temperature, mask, mask_temperature, ctrls,
                      ctrl_masks, top_p, seed, sample_cutoff, cfg_guidance, philox_key, adapter=None) -> dict:
        """Validate one generate() call, draw its key and stage its device inputs and per-step host schedules."""
        if adapter is not None and adapter not in self._adapters:
            self._adapter_id(adapter)  # raises before any RNG is touched
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
                    top_p=float(top_p) if (top_p is not None and top_p < 1.0) else 0.0, adapter=adapter)

    def _launch_calls(self, calls: list, mixed_lengths: bool = False, mixed_steps: bool = False,
                      mixed_top_p: bool = False) -> list:
        """Launch prepared calls, one vnb_generate_many per (T, steps, top-p on) bucket of at most MANY_MAX_ROWS rows
        (a single larger call runs alone); returns each call's (B, C, T) int64 tokens in list order.
        mixed_lengths: buckets drop T; a bucket's calls, longest first, fill launches while rows * (the launch's longest
        T) stays within MANY_MAX_ROWS.
        mixed_steps: buckets drop the steps; each launch's calls are then ordered by steps, longest first (stable), as
        vnb_generate_steps requires.
        mixed_top_p: buckets drop top-p on/off."""
        buckets = {}
        for i, c in enumerate(calls):
            top_p_on = None if mixed_top_p else 0.0 < c["top_p"] < 1.0
            T = None if mixed_lengths else c["z"].shape[-1]
            buckets.setdefault((T, None if mixed_steps else c["steps"], top_p_on), []).append(i)
        launches = []
        for idx in buckets.values():
            if mixed_lengths:  # stable: calls of equal T keep their list order
                idx = sorted(idx, key=lambda i: -calls[i]["z"].shape[-1])
            cur, rows, T = [], 0, 0
            for i in idx:
                B = calls[i]["z"].shape[0]
                if cur and (rows + B) * T > MANY_MAX_ROWS:
                    launches.append(cur)
                    cur, rows = [], 0
                if not cur:
                    T = calls[i]["z"].shape[-1]  # the launch's T: its first (longest) call's
                cur.append(i)
                rows += B
            launches.append(cur)
        if mixed_steps:  # stable: calls of equal steps keep their order
            launches = [sorted(idx, key=lambda i: -calls[i]["steps"]) for idx in launches]
        outs = [None] * len(calls)
        keep = []
        for idx in launches:
            group = [calls[i] for i in idx]
            launch = self._launch_ragged if mixed_lengths else self._launch_group
            for i, o in zip(idx, launch(group, keep)):
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
        out = self._launch(calls, keep, z, m32)
        return list(out.split([c["z"].shape[0] for c in calls]))

    def _launch_ragged(self, calls: list, keep: list) -> list:
        """One vnb_generate_ragged launch of calls whose T may differ: each call's z and mask are padded to the longest
        T with kept frames (code 0, mask 0), every call gets a materialised mask (the default one where it has none:
        predicted codebooks masked, transformer.py:749-751), and each result is cut back to the call's own T."""
        T = max(c["z"].shape[-1] for c in calls)
        default = (torch.arange(self.n_codebooks, device=self.device) >= self.n_conditioning_codebooks).to(torch.int32)
        zs, ms = [], []
        for c in calls:
            m = c["mask"] if c["mask"] is not None else default[None, :, None].expand_as(c["z"])
            pad = (0, T - c["z"].shape[-1])
            zs.append(torch.nn.functional.pad(c["z"], pad, value=0))
            ms.append(torch.nn.functional.pad(m, pad, value=0))
        out = self._launch(calls, keep, torch.cat(zs).contiguous(), torch.cat(ms).contiguous(),
                           frames=[c["z"].shape[-1] for c in calls])
        parts = out.split([c["z"].shape[0] for c in calls])
        return [o if c["z"].shape[-1] == T else o[..., :c["z"].shape[-1]].contiguous() for o, c in zip(parts, calls)]

    def _launch(self, calls: list, keep: list, z, m32, frames=None):
        """One launch of the prepared calls on their concatenated (B, C, T) z / mask; frames: each call's own length
        (vnb_generate_ragged), None when all have T.  Calls of different step counts (longest first) launch through
        vnb_generate_steps, nucleus (top-p) calls next to plain ones through vnb_generate_mixed_top_p."""
        dev = self.device
        B, _, T = z.shape
        steps = calls[0]["steps"]
        mixed_steps = any(c["steps"] != steps for c in calls)
        mixed_top_p = len({0.0 < c["top_p"] < 1.0 for c in calls}) > 1
        arrays = []
        groups = (_lib.GenGroup * len(calls))()
        for g, c in zip(groups, calls):
            tef = (C.c_float * c["steps"])(*c["temp_eff"])
            dos = (C.c_int32 * c["steps"])(*c["do_sample"])
            arrays += [tef, dos]
            g.rows, g.temperature, g.temp_eff, g.do_sample = c["z"].shape[0], c["temperature"], tef, dos
            g.seed_lo, g.seed_hi, g.top_p = c["key"] & 0xFFFFFFFF, (c["key"] >> 32) & 0xFFFFFFFF, c["top_p"]
        gam = (C.c_float * steps)(*calls[0]["gamma"])
        ids = [self._adapter_id(c.get("adapter")) for c in calls]
        ids = (C.c_int32 * len(calls))(*ids) if any(i >= 0 for i in ids) else None
        out = torch.empty_like(z)
        graph = 1 if self.use_cuda_graph else 0
        with torch.cuda.device(dev):
            if mixed_steps or mixed_top_p:
                gams = [(C.c_float * c["steps"])(*c["gamma"]) for c in calls]
                gptr = (C.POINTER(C.c_float) * len(calls))(*[C.cast(a, C.POINTER(C.c_float)) for a in gams])
                fr = None if frames is None else (C.c_int32 * len(calls))(*frames)
                fn = _lib.lib().vnb_generate_mixed_top_p if mixed_top_p else _lib.lib().vnb_generate_steps
                _lib.check(fn(self._handle, _lib.ptr(z), _lib.ptr(m32), B, T,
                              (C.c_int32 * len(calls))(*[c["steps"] for c in calls]), gptr, groups, len(calls), fr, ids,
                              graph, _lib.ptr(out), _lib.stream_ptr(dev)))
            elif frames is not None:
                _lib.check(_lib.lib().vnb_generate_ragged(self._handle, _lib.ptr(z), _lib.ptr(m32), B, T, steps, gam,
                                                          groups, len(calls), (C.c_int32 * len(calls))(*frames), ids,
                                                          graph, _lib.ptr(out), _lib.stream_ptr(dev)))
            elif ids is not None:
                _lib.check(_lib.lib().vnb_generate_many_adapted(self._handle, _lib.ptr(z), _lib.ptr(m32), B, T, steps,
                                                                gam, groups, len(calls), ids, graph, _lib.ptr(out),
                                                                _lib.stream_ptr(dev)))
            else:  # no call has an adapter: the plain kernels and graph
                _lib.check(_lib.lib().vnb_generate_many(self._handle, _lib.ptr(z), _lib.ptr(m32), B, T, steps, gam,
                                                        groups, len(calls), graph, _lib.ptr(out), _lib.stream_ptr(dev)))
        keep.append((z, m32, out))
        return out

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

    @torch.no_grad()
    def decode_many(self, z_list, codec):
        """[decode(z, codec) for z in z_list], bit for bit, with the codec's decoder run over the rows of all entries
        together (DAC.decode_many: clips of different lengths share launches).  Entries are (B_i, n_codebooks, T_i) codes
        with the same codebook count."""
        if len(z_list) == 0:
            raise ValueError("decode_many: an empty list")
        books = {z.shape[1] if z.ndim == 3 else None for z in z_list}
        if None in books:
            raise ValueError("decode_many: every entry is (B_i, n_codebooks, T_i)")
        if len(books) > 1:
            raise ValueError(f"decode_many: entries of different codebook counts {sorted(books)}")
        from ..audio import AudioSignal
        zq = [codec.quantizer.from_latents(self.embedding.from_codes(z.masked_fill(z == self.mask_token, 0), codec))[0]
              for z in z_list]
        return [AudioSignal(d["audio"], codec.sample_rate) for d in codec.decode_many(zq)]
