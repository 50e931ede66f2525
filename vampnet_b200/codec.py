"""DAC-family neural codec on the sm_90a kernels (SURVEY.md §8a rows D1-D3).

Provides what the reference takes from ``lac.model.lac.LAC`` (imported "as DAC", reference
vampnet/interface.py:16):  DAC.load, .preprocess, .encode(...)["codes"], .decode(z)["audio"],
.quantizer.from_latents, .quantizer.from_codes, .quantizer.quantizers[i].codebook.weight,
.sample_rate, .hop_length  (call sites: interface.py:70, 179, 189, 215, 223; transformer.py:671-675;
layers.py:145).  ``lac`` is an un-vendored, unpinned third-party fork of the Descript Audio Codec whose
source and checkpoints are not available here; the architecture below is the published DAC (encoder
dim 64, strides (2,4,8,12) -> hop 768, 14 x 1024 x 8 RVQ, decoder dim 1536) with hyper-parameters read
from the checkpoint's metadata when one is loaded.  Parameter names follow the HF DacModel layout
(encoder.block.{i}.res_unit{r}.conv1.weight ...); weight-norm pairs (weight_g / weight_v) are folded
on load.

All compute goes through the C ABI (vnb_codec_conv1d, vnb_codec_rvq); there is no torch fallback.
"""
from __future__ import annotations

import math
import re
from pathlib import Path
from typing import Dict

import torch
import torch.nn as nn

from . import _lib

# Rows x launch samples of one encode_many / decode_many launch: config [3]'s encode, 32 ten-second clips of 441 600
# samples, so that the peak memory of a mixed launch stays where that batch puts it.
CODEC_MANY_MAX_SAMPLES = 32 * 441_600


def plan_launches(lengths, budget: int = CODEC_MANY_MAX_SAMPLES):
    """Items (by index) -> launches: longest first (stable), each launch as many items as keep rows x its longest length
    within `budget` (an item longer than the budget alone still gets a launch of its own)."""
    order = sorted(range(len(lengths)), key=lambda k: -lengths[k])
    launches = []
    for k in order:
        if launches and (len(launches[-1]) + 1) * lengths[launches[-1][0]] <= budget:
            launches[-1].append(k)
        else:
            launches.append([k])
    return launches


def encoder_lengths(samples, rates):
    """Valid rows of each item at every rate of the encoder: row 0 audio samples (encoder.conv1 and block 0), row i + 1
    the output of block i's strided conv; the last row is frames (encoder.conv2 and the quantiser)."""
    table = [list(samples)]
    for s in rates:
        table.append([n // s for n in table[-1]])
    return table


def decoder_lengths(frames, rates):
    """Valid rows of each item at every rate of the decoder: row 0 frames (decoder.conv1), row i + 1 the output of block
    i's transposed conv, T * s - s % 2 (ConvTranspose1d(2s, stride s, pad ceil(s/2))); the last row is audio samples."""
    table = [list(frames)]
    for s in rates:
        table.append([t * s - s % 2 for t in table[-1]])
    return table


def upload_lengths(table, device):
    """(rates, items) int32 on `device`, in one asynchronous copy from pinned memory (no synchronisation)."""
    host = torch.tensor(table, dtype=torch.int32)
    if torch.device(device).type != "cuda":
        return host
    return host.pin_memory().to(device, non_blocking=True)


def zero_frames_past(zc, frames):
    """zc (B, T, D) channels-last with +0 in every frame t >= frames[b] (frames: int32 [B] on zc's device), one select:
    the decoder input of a clip coded alone has no such frames, and its first conv reads zeros there."""
    t = torch.arange(zc.shape[1], device=zc.device, dtype=torch.int32)
    return torch.where(t.view(1, -1, 1) < frames.view(-1, 1, 1), zc, torch.zeros((), dtype=zc.dtype, device=zc.device))


class _Params(nn.Module):
    """Nested parameter holder addressed by dotted names."""

    def add(self, dotted: str, tensor: torch.Tensor):
        head, _, rest = dotted.partition(".")
        if not rest:
            self.register_parameter(head, nn.Parameter(tensor, requires_grad=False))
            return
        if head not in self._modules:
            self.add_module(head, _Params())
        self._modules[head].add(rest, tensor)

    def get(self, dotted: str) -> torch.Tensor:
        obj = self
        for part in dotted.split("."):
            obj = obj._modules[part] if part in obj._modules else obj._parameters[part]
        return obj


def _layout(cfg) -> Dict[str, tuple]:
    """name -> shape of every tensor of the codec."""
    sh = {}
    d = cfg["encoder_dim"]

    def conv(n, co, ci, k):
        sh[n + ".weight"], sh[n + ".bias"] = (co, ci, k), (co,)

    def res(n, c):
        sh[n + ".snake1.alpha"] = (c,)
        conv(n + ".conv1", c, c, 7)
        sh[n + ".snake2.alpha"] = (c,)
        conv(n + ".conv2", c, c, 1)

    conv("encoder.conv1", d, 1, 7)
    for i, s in enumerate(cfg["encoder_rates"]):
        for r in range(3):
            res(f"encoder.block.{i}.res_unit{r + 1}", d)
        sh[f"encoder.block.{i}.snake1.alpha"] = (d,)
        conv(f"encoder.block.{i}.conv1", 2 * d, d, 2 * s)
        d *= 2
    sh["encoder.snake1.alpha"] = (d,)
    conv("encoder.conv2", cfg["latent_dim"], d, 3)
    for i in range(cfg["n_codebooks"]):
        conv(f"quantizer.quantizers.{i}.in_proj", cfg["codebook_dim"], cfg["latent_dim"], 1)
        conv(f"quantizer.quantizers.{i}.out_proj", cfg["latent_dim"], cfg["codebook_dim"], 1)
        sh[f"quantizer.quantizers.{i}.codebook.weight"] = (cfg["codebook_size"], cfg["codebook_dim"])
    c = cfg["decoder_dim"]
    conv("decoder.conv1", c, cfg["latent_dim"], 7)
    for i, s in enumerate(cfg["decoder_rates"]):
        sh[f"decoder.block.{i}.snake1.alpha"] = (c,)
        sh[f"decoder.block.{i}.conv_t1.weight"], sh[f"decoder.block.{i}.conv_t1.bias"] = (c, c // 2, 2 * s), (c // 2,)
        for r in range(3):
            res(f"decoder.block.{i}.res_unit{r + 1}", c // 2)
        c //= 2
    sh["decoder.snake1.alpha"] = (c,)
    conv("decoder.conv2", 1, c, 7)
    return sh


_WN_SUFFIXES = ((".parametrizations.weight.original0", ".weight_g"), (".parametrizations.weight.original1", ".weight_v"))


def remap_descript_keys(sd: Dict[str, torch.Tensor], n_blocks: int) -> Dict[str, torch.Tensor]:
    """descript-audio-codec / ``lac`` state_dict names -> the flat names of :func:`_layout`.

    The reference loads ``lac.model.lac.LAC`` (interface.py:16, 70), a fork of the Descript Audio Codec whose
    modules are ``nn.Sequential`` stacks, so its checkpoints address tensors by position:
    ``encoder.block.0`` is the input conv, ``encoder.block.{i+1}.block.{r}.block.{0..3}`` are (snake, conv7, snake,
    conv1) of residual unit r of block i, ``encoder.block.{i+1}.block.{3,4}`` the block's snake + strided conv,
    ``encoder.block.{n+1}/{n+2}`` the final snake + conv; the decoder is ``decoder.model.0``, then per block
    ``.block.0`` snake, ``.block.1`` transposed conv, ``.block.{2,3,4}`` residual units, then ``decoder.model.{n+1}``
    snake and ``.{n+2}`` output conv.  Weight-norm pairs arrive as ``weight_g``/``weight_v`` (or the newer
    ``parametrizations.weight.original0/1``) and Snake ``alpha`` as (1, C, 1); both are normalised by
    :meth:`DAC.load_flat`.  Keys already in the flat layout pass through unchanged.
    """
    n = n_blocks
    unit = {"0.alpha": "snake1.alpha", "1.": "conv1.", "2.alpha": "snake2.alpha", "3.": "conv2."}

    def res_unit(rest: str):
        for k, v in unit.items():
            if rest.startswith(k):
                return v + rest[len(k):] if k.endswith(".") else v
        raise KeyError(rest)

    out = {}
    for key, t in sd.items():
        for a, b in _WN_SUFFIXES:
            if key.endswith(a):
                key = key[: -len(a)] + b
        m = re.match(r"^(encoder\.block|decoder\.model)\.(\d+)\.(.*)$", key)
        if m is None or re.match(r"^encoder\.block\.\d+\.(res_unit\d|snake1|conv1)\.", key):
            out[key] = t
            continue
        side, idx, rest = m.group(1), int(m.group(2)), m.group(3)
        enc = side.startswith("encoder")
        root = "encoder" if enc else "decoder"
        if idx == 0:
            new = f"{root}.conv1.{rest}"
        elif idx == n + 1:
            new = f"{root}.snake1.{rest}"
        elif idx == n + 2:
            new = f"{root}.conv2.{rest}"
        elif 1 <= idx <= n:
            mm = re.match(r"^block\.(\d+)\.(.*)$", rest)
            if mm is None:
                raise KeyError(f"unrecognised codec key {key}")
            j, tail = int(mm.group(1)), mm.group(2)
            blk = f"{root}.block.{idx - 1}"
            if enc:
                if j < 3:
                    new = f"{blk}.res_unit{j + 1}." + res_unit(tail[len("block."):])
                elif j == 3:
                    new = f"{blk}.snake1.{tail}"
                else:
                    new = f"{blk}.conv1.{tail}"
            else:
                if j == 0:
                    new = f"{blk}.snake1.{tail}"
                elif j == 1:
                    new = f"{blk}.conv_t1.{tail}"
                else:
                    new = f"{blk}.res_unit{j - 1}." + res_unit(tail[len("block."):])
        else:
            raise KeyError(f"unrecognised codec key {key} (expected at most {n + 3} stages)")
        out[new] = t
    return out


class _Quantizer:
    """codec.quantizer: .quantizers[i].codebook.weight, from_latents, from_codes, forward (encode)."""

    def __init__(self, codec: "DAC"):
        self._codec = codec

    @property
    def quantizers(self):
        return list(self._codec.params._modules["quantizer"]._modules["quantizers"]._modules.values())

    def _rvq(self, mode, in_f=None, in_codes=None, channels_last=False, split=False):
        """channels_last: z / zq are (B, T, D) (tensor-core codec path); split: also return zq as hi/lo bf16."""
        c = self._codec
        pk = c._packed()
        src = in_f if in_f is not None else in_codes
        B = src.shape[0]
        T = src.shape[1] if (channels_last and mode == 0) else src.shape[-1]
        dev = src.device
        D, L, V = c.latent_dim, c.n_codebooks, c.codebook_size
        if mode == 1:
            L = in_f.shape[1] // c.codebook_dim
        elif mode == 2:
            L = in_codes.shape[1]
        zq = torch.empty((B, T, D) if channels_last else (B, D, T), device=dev, dtype=torch.float32)
        hi = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16) if split else None
        lo = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16) if split else None
        codes = torch.empty(B, L, T, device=dev, dtype=torch.int64) if mode == 0 else None
        lat = torch.empty(B, L * c.codebook_dim, T, device=dev, dtype=torch.float32) if mode == 0 else None
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().vnb_codec_rvq(mode, _lib.ptr(in_f), _lib.ptr(in_codes), _lib.ptr(pk["win"]),
                                                _lib.ptr(pk["bin"]), _lib.ptr(pk["wout"]), _lib.ptr(pk["bout"]),
                                                _lib.ptr(pk["cb"]), _lib.ptr(pk["cbn"]), _lib.ptr(codes), _lib.ptr(zq),
                                                _lib.ptr(lat), B, D, T, L, V, 1 if channels_last else 0, _lib.ptr(hi),
                                                _lib.ptr(lo), _lib.stream_ptr(dev)))
        if split:
            return zq, codes, lat, hi, lo
        return zq, codes, lat

    def __call__(self, z):
        zq, codes, lat = self._rvq(0, in_f=z.float().contiguous())
        return zq, codes, lat

    def from_latents(self, latents: torch.Tensor):
        """(B, 8*L, T) -> (z_q, quantised latents): re-quantise each 8-d chunk then out_proj and sum."""
        latents = latents.float().contiguous()
        zq, _, _ = self._rvq(1, in_f=latents)
        return zq, latents

    def from_codes(self, codes: torch.Tensor):
        codes = codes.to(torch.int64).contiguous()
        zq, _, _ = self._rvq(2, in_codes=codes)
        return zq, None, codes


class DAC(nn.Module):
    def __init__(self, encoder_dim: int = 64, encoder_rates=(2, 4, 8, 12), latent_dim: int = None,
                 decoder_dim: int = 1536, decoder_rates=None, n_codebooks: int = 14, codebook_size: int = 1024,
                 codebook_dim: int = 8, sample_rate: int = 44100, precision: str = "tc", **_ignored):
        super().__init__()
        self.encoder_dim = encoder_dim
        self.encoder_rates = tuple(encoder_rates)
        self.decoder_rates = tuple(decoder_rates) if decoder_rates is not None else tuple(reversed(self.encoder_rates))
        self.latent_dim = latent_dim if latent_dim is not None else encoder_dim * 2 ** len(self.encoder_rates)
        self.decoder_dim = decoder_dim
        self.n_codebooks = n_codebooks
        self.codebook_size = codebook_size
        self.codebook_dim = codebook_dim
        self.sample_rate = sample_rate
        # "tc": wgmma tensor-core convolutions with split-bf16 operands (fp32-grade); "fp32": CUDA-core kernels
        assert precision in ("tc", "fp32")
        widths = [encoder_dim * 2 ** i for i in range(len(self.encoder_rates) + 1)] + \
                 [decoder_dim // 2 ** i for i in range(len(self.decoder_rates) + 1)]
        if precision == "tc" and any(w % 32 for w in widths):
            raise ValueError(f"precision='tc' needs every channel width to be a multiple of 32, got {widths}; "
                             "use precision='fp32'")
        self.precision = precision
        self.hop_length = int(math.prod(self.encoder_rates))
        self._cfg = dict(encoder_dim=encoder_dim, encoder_rates=self.encoder_rates, latent_dim=self.latent_dim,
                         decoder_dim=decoder_dim, decoder_rates=self.decoder_rates, n_codebooks=n_codebooks,
                         codebook_size=codebook_size, codebook_dim=codebook_dim)
        self.params = _Params()
        g = torch.Generator().manual_seed(0)
        for name, shape in _layout(self._cfg).items():
            if name.endswith(".alpha"):
                t = torch.ones(shape, device="cpu")
            elif name.endswith(".bias"):
                t = torch.zeros(shape, device="cpu")
            else:
                fan = shape[1] * (shape[2] if len(shape) == 3 else 1)
                t = torch.randn(shape, generator=g, device="cpu") / math.sqrt(max(fan, 1))
            self.params.add(name, t)
        self.quantizer = _Quantizer(self)
        self._pack = None
        self.eval()

    # ---- state ---------------------------------------------------------------------------------
    def _invalidate(self):
        """Drop every tensor derived from the parameters (normalised codebooks, split-bf16 / transposed-conv packs);
        called by parallel.broadcast_module_weights after parameters were overwritten in place."""
        self._pack = None

    def _apply(self, fn, *a, **k):
        self._invalidate()
        return super()._apply(fn, *a, **k)

    def load_flat(self, weights: Dict[str, torch.Tensor]):
        """Load a flat {dotted name: tensor} dict, in the HF DacModel naming or in the descript-audio-codec / lac
        naming the reference's checkpoints use (see remap_descript_keys).  weight_g / weight_v pairs are folded."""
        weights = remap_descript_keys(dict(weights), len(self.encoder_rates))
        for k in [k for k in weights if k.endswith(".weight_v")]:
            base = k[: -len("_v")]
            v, gk = weights.pop(k), base + "_g"
            g = weights.pop(gk)
            weights[base] = v * (g / v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1))))
        own = _layout(self._cfg)
        missing = [k for k in own if k not in weights]
        if missing:
            raise KeyError(f"codec weights missing {len(missing)} tensors, e.g. {missing[:3]}")
        with torch.no_grad():
            for k, shape in own.items():
                t = weights[k].float().reshape(shape)
                self.params.get(k).data.copy_(t.to(self.params.get(k).device))
        self._pack = None
        return self

    @classmethod
    def load(cls, location, *_, **overrides):
        """audiotools BaseModel.load layout: {'state_dict': ..., 'metadata': {'kwargs': {...}}} (interface.py:70).
        Keyword arguments override the checkpoint's constructor arguments (e.g. precision="fp32")."""
        blob = torch.load(str(Path(location)), map_location="cpu", weights_only=False)
        kwargs = dict(blob.get("metadata", {}).get("kwargs", {}))
        kwargs.update(overrides)
        import inspect
        known = set(inspect.signature(cls.__init__).parameters) - {"self", "_ignored"}
        model = cls(**{k: v for k, v in kwargs.items() if k in known})  # e.g. quantizer_dropout is training-only
        sd = {k[len("params."):] if k.startswith("params.") else k: v for k, v in blob["state_dict"].items()}
        model.load_flat(sd)
        return model

    @property
    def device(self):
        return self.params.get("encoder.conv1.weight").device

    def _packed(self):
        if self._pack is not None:
            return self._pack
        if self.device.type != "cuda":
            raise RuntimeError("vampnet_b200.codec.DAC runs only on a CUDA (sm_90a) device; there is no CPU fallback")
        P = self.params.get
        L = self.n_codebooks
        q = "quantizer.quantizers."
        pk = {
            "win": torch.stack([P(f"{q}{i}.in_proj.weight").squeeze(-1) for i in range(L)]).contiguous(),
            "bin": torch.stack([P(f"{q}{i}.in_proj.bias") for i in range(L)]).contiguous(),
            "wout": torch.stack([P(f"{q}{i}.out_proj.weight").squeeze(-1) for i in range(L)]).contiguous(),
            "bout": torch.stack([P(f"{q}{i}.out_proj.bias") for i in range(L)]).contiguous(),
            "cb": torch.stack([P(f"{q}{i}.codebook.weight") for i in range(L)]).contiguous(),
        }
        pk["cbn"] = torch.nn.functional.normalize(pk["cb"], dim=-1).contiguous()
        # ConvTranspose1d(k=2s, stride s) as s two-tap convolutions: Wp[r][co][ci][j] = W[ci][co][r + j*s]
        for i, s in enumerate(self.decoder_rates):
            w = P(f"decoder.block.{i}.conv_t1.weight")  # (cin, cout, 2s)
            pk[f"convt{i}"] = torch.stack([w[:, :, r::s].permute(1, 0, 2) for r in range(s)]).contiguous()
        if self.precision == "tc":
            self._pack_tc(pk)
        self._pack = pk
        return pk

    # ---- tensor-core path: weights as (N, taps * cblocks * 64) split-bf16, tap-major -----------------------
    @staticmethod
    def _split(w: torch.Tensor):
        hi = w.to(torch.bfloat16)
        lo = (w - hi.float()).to(torch.bfloat16)
        return hi.contiguous(), lo.contiguous()

    def _pack_conv_tc(self, w: torch.Tensor):
        """(Cout, Cin, K) -> (Cout, K * cblocks * 64)."""
        co, ci, k = w.shape
        cb = (ci + 63) // 64
        t = torch.zeros(co, k, cb * 64, device=w.device, dtype=torch.float32)
        t[:, :, :ci] = w.permute(0, 2, 1)
        return self._split(t.reshape(co, k * cb * 64))

    def _pack_convt_tc(self, w: torch.Tensor, s: int):
        """ConvTranspose1d weight (Cin, Cout, 2s) -> (s*Cout, 2 * cblocks * 64): row r*Cout+co, tap j uses k = r + j*s."""
        ci, co, k = w.shape
        cb = (ci + 63) // 64
        t = torch.zeros(s, co, 2, cb * 64, device=w.device, dtype=torch.float32)
        for j in range(2):
            t[:, :, j, :ci] = w[:, :, j * s:(j + 1) * s].permute(2, 1, 0)  # (r, co, ci)
        return self._split(t.reshape(s * co, 2 * cb * 64))

    def _pack_tc(self, pk):
        P = self.params.get
        for name in _layout(self._cfg):
            if not name.endswith(".weight") or ".quantizer." in "." + name or name.endswith("codebook.weight"):
                continue
            base = name[:-len(".weight")]
            w = P(name).float()
            if base in ("encoder.conv1", "decoder.conv2"):
                continue  # Cin = 1 / Cout = 1 edge layers run on CUDA cores
            if ".conv_t1" in base:
                idx = int(base.split(".")[2])
                pk["tc:" + base] = self._pack_convt_tc(w, self.decoder_rates[idx])
            else:
                pk["tc:" + base] = self._pack_conv_tc(w)

    # ---- kernels -------------------------------------------------------------------------------
    def _conv(self, x, name, K, stride=1, dil=1, pad=0, alpha=None, resid=None, tanh=False, out=None):
        w, b = self.params.get(name + ".weight"), self.params.get(name + ".bias")
        B, Cin, Tin = x.shape
        Cout = w.shape[0]
        Tout = (Tin + 2 * pad - dil * (K - 1) - 1) // stride + 1
        y = out if out is not None else torch.empty(B, Cout, Tout, device=x.device, dtype=torch.float32)
        _lib.check(_lib.lib().vnb_codec_conv1d(_lib.ptr(x), _lib.ptr(w), _lib.ptr(b), _lib.ptr(alpha), _lib.ptr(resid),
                                               _lib.ptr(y), B, Cin, Tin, Cout, Tout, K, stride, dil, pad, 1, 0, Tout,
                                               1 if tanh else 0, _lib.stream_ptr(x.device)))
        return y

    def _convt(self, x, idx, s, alpha):
        B, Cin, Tin = x.shape
        wp = self._packed()[f"convt{idx}"]  # (s, cout, cin, 2)
        b = self.params.get(f"decoder.block.{idx}.conv_t1.bias")
        Cout = wp.shape[1]
        pad = math.ceil(s / 2)
        Tout = (Tin - 1) * s - 2 * pad + 2 * s
        y = torch.empty(B, Cout, Tout, device=x.device, dtype=torch.float32)
        for r in range(s):
            _lib.check(_lib.lib().vnb_codec_conv1d(_lib.ptr(x), _lib.ptr(wp[r]), _lib.ptr(b), _lib.ptr(alpha), None,
                                                   _lib.ptr(y), B, Cin, Tin, Cout, Tout, 2, 1, -1, 0, s, r - pad, Tin + 1,
                                                   0, _lib.stream_ptr(x.device)))
        return y

    def _res_unit(self, x, name, dil):
        P = self.params.get
        y = self._conv(x, name + ".conv1", 7, dil=dil, pad=3 * dil, alpha=P(name + ".snake1.alpha"))
        return self._conv(y, name + ".conv2", 1, alpha=P(name + ".snake2.alpha"), resid=x, out=x)  # in place: x += ...

    # ---- public surface ------------------------------------------------------------------------
    def preprocess(self, audio_data, sample_rate=None):
        """Right-pad to a multiple of hop_length; returns (padded, original_length) (interface.py:215)."""
        if sample_rate is not None:
            assert sample_rate == self.sample_rate, f"expected {self.sample_rate} Hz, got {sample_rate}"
        length = audio_data.shape[-1]
        right = math.ceil(length / self.hop_length) * self.hop_length - length
        return torch.nn.functional.pad(audio_data, (0, right)), length

    @torch.no_grad()
    def encode(self, audio_data: torch.Tensor, sample_rate: int = None, n_quantizers: int = None):
        """(B, 1, N) -> dict(z, codes (B, n_codebooks, N/hop) int64, latents)  (interface.py:223)."""
        self._packed()
        x = audio_data.to(self.device, torch.float32).contiguous()
        P = self.params.get
        if self.precision == "tc":
            return self._encode_tc(x)
        with torch.cuda.device(self.device):
            h = self._conv(x, "encoder.conv1", 7, pad=3)
            for i, s in enumerate(self.encoder_rates):
                p = f"encoder.block.{i}"
                for r, dil in enumerate((1, 3, 9)):
                    h = self._res_unit(h, f"{p}.res_unit{r + 1}", dil)
                h = self._conv(h, p + ".conv1", 2 * s, stride=s, pad=math.ceil(s / 2), alpha=P(p + ".snake1.alpha"))
            z = self._conv(h, "encoder.conv2", 3, pad=1, alpha=P("encoder.snake1.alpha"))
            zq, codes, lat = self.quantizer(z)
        return {"z": zq, "codes": codes, "latents": lat, "length": audio_data.shape[-1]}

    @torch.no_grad()
    def decode(self, z: torch.Tensor, length: int = None):
        """(B, latent_dim, T) -> dict(audio (B, 1, T*hop))  (transformer.py:671-675)."""
        self._packed()
        P = self.params.get
        z = z.to(self.device, torch.float32).contiguous()
        if self.precision == "tc":
            audio = self._decode_tc(z)
            return {"audio": audio if length is None else audio[..., :length]}
        with torch.cuda.device(self.device):
            h = self._conv(z, "decoder.conv1", 7, pad=3)
            for i, s in enumerate(self.decoder_rates):
                p = f"decoder.block.{i}"
                h = self._convt(h, i, s, P(p + ".snake1.alpha"))
                for r, dil in enumerate((1, 3, 9)):
                    h = self._res_unit(h, f"{p}.res_unit{r + 1}", dil)
            audio = self._conv(h, "decoder.conv2", 7, pad=3, alpha=P("decoder.snake1.alpha"), tanh=True)
        return {"audio": audio if length is None else audio[..., :length]}

    # ---- many clips of different lengths -----------------------------------------------------------------------
    @staticmethod
    def _refuse_empty(entries, what):
        if len(entries) == 0:
            raise ValueError(f"{what}: an empty list")
        for i, e in enumerate(entries):
            if e.dim() != 3 or e.shape[0] == 0 or e.shape[-1] == 0:
                raise ValueError(f"{what}: entry {i} has shape {tuple(e.shape)}; every entry is (B_i >= 1, C, N_i >= 1)")

    @torch.no_grad()
    def encode_many(self, audio_list, sample_rate=None, budget: int = CODEC_MANY_MAX_SAMPLES):
        """[encode(a) for a in audio_list], with the rows of all entries sharing launches.  Each entry is (B_i, 1, N_i),
        N_i a multiple of hop_length (as encode needs, see preprocess); sample_rate: None, one rate, or one per entry
        (all equal to the codec's).  Rows are sorted longest first and grouped so that rows x launch samples <= budget;
        a launch runs at its longest row, shorter rows zero-padded, and every row's codes, z and latents equal the
        row's own encode, bit for bit.  Nothing here synchronises the host."""
        self._refuse_empty(audio_list, "encode_many")
        rates = sample_rate if isinstance(sample_rate, (list, tuple)) else [sample_rate] * len(audio_list)
        if len(rates) != len(audio_list):
            raise ValueError("encode_many: one sample rate per entry")
        known = {r for r in rates if r is not None}
        if len(known) > 1:
            raise ValueError(f"encode_many: entries of different sample rates {sorted(known)}; resample them first")
        if known and known != {self.sample_rate}:
            raise ValueError(f"encode_many: expected {self.sample_rate} Hz, got {known.pop()}")
        for i, a in enumerate(audio_list):
            if a.shape[1] != 1 or a.shape[-1] % self.hop_length:
                raise ValueError(f"encode_many: entry {i} has shape {tuple(a.shape)}; each is (B_i, 1, N_i) with N_i a "
                                 f"multiple of {self.hop_length} (see preprocess)")
        if self.precision != "tc":
            return [self.encode(a) for a in audio_list]
        items = [(i, j) for i, a in enumerate(audio_list) for j in range(a.shape[0])]
        samples = [audio_list[i].shape[-1] for i, _ in items]
        rows = [None] * len(items)
        for launch in plan_launches(samples, budget):
            n = samples[launch[0]]
            x = torch.cat([torch.nn.functional.pad(audio_list[items[k][0]][items[k][1]:items[k][1] + 1]
                                                   .to(self.device, torch.float32), (0, n - samples[k]))
                           for k in launch])
            table = encoder_lengths([samples[k] for k in launch], self.encoder_rates)
            out = self._encode_launch(x.contiguous(), upload_lengths(table, self.device))
            for r, k in enumerate(launch):
                t = table[-1][r]
                rows[k] = (out["z"][r, :t], out["codes"][r, :, :t], out["latents"][r, :, :t])
        result, k = [], 0
        for a in audio_list:
            mine = rows[k:k + a.shape[0]]
            k += a.shape[0]
            zq, codes, lat = (torch.stack([m[f] for m in mine]) for f in range(3))
            result.append({"z": zq.permute(0, 2, 1), "codes": codes, "latents": lat, "length": a.shape[-1]})
        return result

    def _encode_launch(self, x, lens):
        """One ragged encoder launch: x (B, 1, N) -> channels-last z (B, T, D), codes (B, L, T), latents (B, 8L, T)."""
        self._packed()
        enc = self._encode_tc(x, lens=lens)
        return {"z": enc["z"].permute(0, 2, 1), "codes": enc["codes"], "latents": enc["latents"]}

    @torch.no_grad()
    def decode_many(self, z_list, budget: int = CODEC_MANY_MAX_SAMPLES):
        """[decode(z) for z in z_list], with the rows of all entries sharing launches.  Each entry is (B_i, D, T_i) with
        the same D.  Rows are sorted longest first and grouped so that rows x launch samples (frames x hop_length) <=
        budget; every row's audio equals the row's own decode, bit for bit.  Nothing here synchronises the host."""
        self._refuse_empty(z_list, "decode_many")
        dims = {z.shape[1] for z in z_list}
        if len(dims) > 1:
            raise ValueError(f"decode_many: entries of different latent counts {sorted(dims)}")
        if self.precision != "tc":
            return [self.decode(z) for z in z_list]
        items = [(i, j) for i, z in enumerate(z_list) for j in range(z.shape[0])]
        frames = [z_list[i].shape[-1] for i, _ in items]
        rows = [None] * len(items)
        D = z_list[0].shape[1]
        for launch in plan_launches([t * self.hop_length for t in frames], budget):
            T = frames[launch[0]]
            # frames past an item's own are left as they are here: the launch's select sets them to +0
            zc = torch.empty(len(launch), T, D, device=self.device, dtype=torch.float32)
            for r, k in enumerate(launch):
                i, j = items[k]
                zc[r, :frames[k]].copy_(z_list[i][j].transpose(0, 1))
            table = decoder_lengths([frames[k] for k in launch], self.decoder_rates)
            audio = self._decode_launch(zc, upload_lengths(table, self.device))
            for r, k in enumerate(launch):
                rows[k] = audio[r, :, :table[-1][r]]
        result, k = [], 0
        for z in z_list:
            result.append({"audio": torch.stack(rows[k:k + z.shape[0]])})
            k += z.shape[0]
        return result

    def _decode_launch(self, zc, lens):
        """One ragged decoder launch: zc (B, T, D) channels-last, any values past an item's frames -> audio (B, 1, N)."""
        self._packed()
        return self._decode_tc(zc.permute(0, 2, 1), lens=lens)

    # ---- tensor-core forward passes (activations channels-last, carried as fp32 stream + hi/lo bf16 operand) ----
    def _tc(self, act, base, N, taps, dil, pad, Tq, s=1, alpha=None, alpha_mod=1, resid=None, out_f32=False,
            out_split=True, bias_mod=None, out_rows=None, out_offset=0, lens=None, zeroed=False):
        """One tensor-core convolution.  act = (hi, lo) (B, Tin, Cin).  Returns (f32 | None, (hi, lo) | None).
        lens: DEVICE int32 [B] valid output rows of each item (a ragged launch: vnb_codec_conv_tc_ragged); zeroed: the
        fp32 output starts as zeros (rows past an item's halo are not written by a ragged launch)."""
        hi, lo = act
        B, Tin, Cin = hi.shape
        wh, wl = self._pack["tc:" + base]
        bias = self.params.get(base + ".bias")
        out_rows = Tq if out_rows is None else out_rows
        dev = hi.device
        # output tensor geometry: normal conv (B, Tq, N); transposed conv (B, T*s, Cout) written through the
        # (Tq, s*Cout) view shifted by out_offset
        cout = bias.shape[0]
        shape = (B, out_rows, cout)
        new = torch.zeros if zeroed else torch.empty
        f32 = resid if resid is not None else (new(shape, device=dev, dtype=torch.float32) if out_f32 else None)
        oh = torch.empty(shape, device=dev, dtype=torch.bfloat16) if out_split else None
        ol = torch.empty(shape, device=dev, dtype=torch.bfloat16) if out_split else None
        args = (_lib.ptr(hi), _lib.ptr(lo), B, Tin, Cin, s, _lib.ptr(wh), _lib.ptr(wl), N, taps, dil, pad, Tq,
                _lib.ptr(bias), cout if bias_mod is None else bias_mod, _lib.ptr(alpha), alpha_mod, _lib.ptr(resid),
                _lib.ptr(f32) if (out_f32 or resid is not None) else None, _lib.ptr(oh), _lib.ptr(ol),
                out_rows * cout, out_offset, out_rows * cout, 0)
        if lens is None:
            _lib.check(_lib.lib().vnb_codec_conv_tc(*args, _lib.stream_ptr(dev)))
        else:
            _lib.check(_lib.lib().vnb_codec_conv_tc_ragged(*args, _lib.ptr(lens), cout, _lib.stream_ptr(dev)))
        return f32, ((oh, ol) if out_split else None)

    def _res_unit_tc(self, skip, act, name, dil, next_alpha, lens=None):
        """skip: fp32 stream (updated in place); act = split(snake1(skip)); returns split(next_alpha(skip'))."""
        P = self.params.get
        C = skip.shape[-1]
        T = skip.shape[1]
        _, a2 = self._tc(act, name + ".conv1", C, 7, dil, 3 * dil, T, alpha=P(name + ".snake2.alpha"), alpha_mod=C,
                         lens=lens)
        _, nxt = self._tc(a2, name + ".conv2", C, 1, 1, 0, T, alpha=next_alpha, alpha_mod=C, resid=skip, lens=lens)
        return nxt

    def _encode_tc(self, x, lens=None):
        """x (B, 1, N).  lens: None, or the DEVICE (rates, B) table of encoder_lengths for a launch of items of
        different lengths (x zero-padded to the longest): each item's rows then equal its own launch, bit for bit,
        and the outputs past an item's frames are meaningless but finite."""
        P = self.params.get
        row = (lambda i: None) if lens is None else (lambda i: lens[i])
        B, _, N = x.shape
        lib = _lib.lib()
        with torch.cuda.device(self.device):
            d = self.encoder_dim
            skip = torch.empty(B, N, d, device=x.device, dtype=torch.float32)
            hi = torch.empty(B, N, d, device=x.device, dtype=torch.bfloat16)
            lo = torch.empty_like(hi)
            args = (_lib.ptr(x), _lib.ptr(P("encoder.conv1.weight")), _lib.ptr(P("encoder.conv1.bias")),
                    _lib.ptr(P("encoder.block.0.res_unit1.snake1.alpha")), _lib.ptr(skip), _lib.ptr(hi), _lib.ptr(lo), B,
                    N, d, 7, 3)
            if lens is None:
                _lib.check(lib.vnb_codec_conv_in(*args, _lib.stream_ptr(x.device)))
            else:
                _lib.check(lib.vnb_codec_conv_in_ragged(*args, _lib.ptr(row(0)), _lib.stream_ptr(x.device)))
            act = (hi, lo)
            T = N
            nb = len(self.encoder_rates)
            for i, s in enumerate(self.encoder_rates):
                p = f"encoder.block.{i}"
                for r, dil in enumerate((1, 3, 9)):
                    nxt = P(f"{p}.res_unit{r + 2}.snake1.alpha") if r < 2 else P(p + ".snake1.alpha")
                    act = self._res_unit_tc(skip, act, f"{p}.res_unit{r + 1}", dil, nxt, lens=row(i))
                # strided conv: input viewed as (B, T/s, s*C); output feeds the next block (or encoder.snake1)
                nxt = P(f"encoder.block.{i + 1}.res_unit1.snake1.alpha") if i + 1 < nb else P("encoder.snake1.alpha")
                skip, act = self._tc(act, p + ".conv1", 2 * d, 2 * s, 1, math.ceil(s / 2), T // s, s=s, alpha=nxt,
                                     alpha_mod=2 * d, out_f32=(i + 1 < nb), lens=row(i + 1))
                d *= 2
                T //= s
            # ragged: the quantiser reads every frame of the launch, so frames past an item's halo start as zeros
            z, _ = self._tc(act, "encoder.conv2", self.latent_dim, 3, 1, 1, T, out_f32=True, out_split=False,
                            lens=row(nb), zeroed=lens is not None)
            zq_cl, codes, lat = self.quantizer._rvq(0, in_f=z, channels_last=True)
        return {"z": zq_cl.permute(0, 2, 1), "codes": codes, "latents": lat, "length": N}

    def _decode_tc(self, z, lens=None):
        """z: (B, latent, T) fp32 (the reference's layout) -> audio (B, 1, T*hop), or shorter for odd decoder rates.
        lens: None, or the DEVICE (rates, B) table of decoder_lengths for a launch of items of different lengths: frames
        past an item's own are set to +0 first (one select), and each item's samples then equal its own launch."""
        P = self.params.get
        lib = _lib.lib()
        row = (lambda i: None) if lens is None else (lambda i: lens[i])
        with torch.cuda.device(self.device):
            zc = z.permute(0, 2, 1).contiguous()  # channels-last
            if lens is not None:
                zc = zero_frames_past(zc, lens[0])
            act = self._split(zc)
            B, T, _ = zc.shape
            c = self.decoder_dim
            _, act = self._tc(act, "decoder.conv1", c, 7, 1, 3, T, alpha=P("decoder.block.0.snake1.alpha"), alpha_mod=c,
                              lens=row(0))
            nb = len(self.decoder_rates)
            for i, s in enumerate(self.decoder_rates):
                p = f"decoder.block.{i}"
                co = c // 2
                pad = math.ceil(s / 2)
                # transposed conv as ONE GEMM with N = s*Cout phase-major columns and taps (x[q], x[q-1]); its output has
                # (T-1)*s - 2*pad + 2*s = T*s - s % 2 rows (ConvTranspose1d), so odd strides drop the last row
                rows = T * s - s % 2
                skip, act = self._tc(act, p + ".conv_t1", s * co, 2, -1, 0, T + 1, alpha=P(p + ".res_unit1.snake1.alpha"),
                                     alpha_mod=co, out_f32=True, bias_mod=co, out_rows=rows, out_offset=-pad * co,
                                     lens=row(i + 1))
                T = rows
                for r, dil in enumerate((1, 3, 9)):
                    if r < 2:
                        nxt = P(f"{p}.res_unit{r + 2}.snake1.alpha")
                    else:
                        nxt = P(f"decoder.block.{i + 1}.snake1.alpha") if i + 1 < nb else P("decoder.snake1.alpha")
                    act = self._res_unit_tc(skip, act, f"{p}.res_unit{r + 1}", dil, nxt, lens=row(i + 1))
                c = co
            audio = torch.empty(B, 1, T, device=z.device, dtype=torch.float32)
            args = (_lib.ptr(act[0]), _lib.ptr(act[1]), _lib.ptr(P("decoder.conv2.weight")),
                    _lib.ptr(P("decoder.conv2.bias")), _lib.ptr(audio), B, T, c, 7, 3)
            if lens is None:
                _lib.check(lib.vnb_codec_conv_out(*args, _lib.stream_ptr(z.device)))
            else:
                _lib.check(lib.vnb_codec_conv_out_ragged(*args, _lib.ptr(row(nb)), _lib.stream_ptr(z.device)))
        return audio

    def forward(self, audio_data, sample_rate=None):
        enc = self.encode(audio_data, sample_rate)
        return {**enc, **self.decode(enc["z"], audio_data.shape[-1])}
