"""Interface — drop-in for the reference's ``vampnet.interface.Interface`` surface
(reference vampnet/interface.py:54-562): checkpoint loading, encode, build_mask, chunked coarse_vamp,
coarse_to_fine, vamp, decode.  Same method names, arguments, defaults, return types and error behaviour;
the compute underneath is the sm_90a CUDA path (VampNet.generate, the codec kernels).

Chunk loops are kept (they define the reference's results: every chunk is an independent generate() call
with its own whole-batch N0), but each chunk's loop body is one CUDA-graph replay.
"""
from __future__ import annotations

import logging
import math
from pathlib import Path

import numpy as np
import torch

from . import mask as pmask
from .audio import AudioSignal
from .beats import BeatTracker, beat_mask
from .mask import *  # noqa: F401,F403  (reference does `from .mask import *`, interface.py:13)
from .modules.transformer import VampNet


def signal_concat(audio_signals: list):
    """interface.py:19-24."""
    audio_data = torch.cat([x.audio_data for x in audio_signals], dim=-1)
    return AudioSignal(audio_data, sample_rate=audio_signals[0].sample_rate)


def _load_model(ckpt: str, lora_ckpt: str = None, device: str = "cpu", chunk_size_s: int = 10):
    """interface.py:27-50.  A missing LoRA checkpoint raises instead of blocking on input()."""
    model = VampNet.load(location=Path(ckpt), map_location="cpu", strict=False)
    if lora_ckpt is not None:
        if not Path(lora_ckpt).exists():
            raise FileNotFoundError(f"lora checkpoint {lora_ckpt} does not exist")
        model.load_state_dict(torch.load(lora_ckpt, map_location="cpu"), strict=False)
    model.to(device)
    model.eval()
    model.chunk_size_s = chunk_size_s
    return model


class Interface(torch.nn.Module):
    def __init__(
        self,
        coarse_ckpt: str = None,
        coarse_lora_ckpt: str = None,
        coarse2fine_ckpt: str = None,
        coarse2fine_lora_ckpt: str = None,
        codec_ckpt: str = None,
        wavebeat_ckpt: str = "./models/vampnet/wavebeat.pth",
        device: str = "cpu",
        coarse_chunk_size_s: int = 10,
        coarse2fine_chunk_size_s: int = 3,
        compile=True,
    ):
        super().__init__()
        from .codec import DAC
        assert codec_ckpt is not None, "must provide a codec checkpoint"
        self.codec = DAC.load(Path(codec_ckpt))
        self.codec.eval()
        self.codec.to(device)
        self.codec_path = Path(codec_ckpt)

        assert coarse_ckpt is not None, "must provide a coarse checkpoint"
        self.coarse = _load_model(ckpt=coarse_ckpt, lora_ckpt=coarse_lora_ckpt, device=device,
                                  chunk_size_s=coarse_chunk_size_s)
        self.coarse_path = Path(coarse_ckpt)
        if coarse2fine_ckpt is not None:
            self.c2f_path = Path(coarse2fine_ckpt)
            self.c2f = _load_model(ckpt=coarse2fine_ckpt, lora_ckpt=coarse2fine_lora_ckpt, device=device,
                                   chunk_size_s=coarse2fine_chunk_size_s)
        else:
            self.c2f_path = None
            self.c2f = None
        # WaveBeat (interface.py:96-101) is a separate network whose package is not available; beat masks use the
        # librosa-style tracker of beats.py instead (any object with extract_beats can be assigned in its place)
        self.beat_tracker = BeatTracker(device)
        if wavebeat_ckpt is not None and Path(wavebeat_ckpt).exists():
            logging.debug("wavebeat checkpoint ignored: beat masks use the built-in librosa-style beat tracker")
        self.device = device
        self.loudness = -24.0
        # `compile` (torch.compile in the reference, interface.py:107-112) is accepted and ignored:
        # there is no tracing compiler on this path, the generate loop is a captured CUDA graph.

    @classmethod
    def from_models(cls, codec, coarse, c2f=None, device="cuda", coarse_chunk_size_s=10, coarse2fine_chunk_size_s=3):
        """Build an Interface around already-constructed modules (tests, benchmarks, synthetic weights)."""
        self = cls.__new__(cls)
        torch.nn.Module.__init__(self)
        self.codec, self.coarse, self.c2f = codec, coarse, c2f
        self.coarse.chunk_size_s = coarse_chunk_size_s
        if c2f is not None:
            self.c2f.chunk_size_s = coarse2fine_chunk_size_s
        self.codec_path = self.coarse_path = self.c2f_path = None
        self.beat_tracker = BeatTracker(device)
        self.device = device
        self.loudness = -24.0
        return self.to(device)

    # ------------------------------------------------------------------ checkpoints (interface.py:115-174)
    # The reference keeps a local cache under <repo>/models/vampnet ({codec,coarse,c2f}.pth, loras/<name>/{coarse,
    # c2f}.pth) and fills it from the HF hub on a miss (vampnet/__init__.py:19-76).  Here the cache is the only
    # source: $VAMPNET_MODELS_DIR or ./models/vampnet; a miss raises (no network access in this build).
    @staticmethod
    def models_dir() -> Path:
        import os
        return Path(os.environ.get("VAMPNET_MODELS_DIR", "./models/vampnet"))

    @classmethod
    def _cached(cls, *parts: str) -> Path:
        path = cls.models_dir().joinpath(*parts)
        if not path.exists():
            raise RuntimeError(f"{path} is not in the local model cache and this build cannot download it from the HF "
                               f"hub (vampnet/__init__.py:19-59); place the checkpoint there or set VAMPNET_MODELS_DIR")
        return path

    @classmethod
    def default(cls, **kwargs):
        """interface.py:115-126, from the local cache."""
        wavebeat = cls.models_dir() / "wavebeat.pth"
        return cls(coarse_ckpt=cls._cached("coarse.pth"), coarse2fine_ckpt=cls._cached("c2f.pth"),
                   codec_ckpt=cls._cached("codec.pth"), wavebeat_ckpt=str(wavebeat), **kwargs)

    @classmethod
    def available_models(cls):
        """interface.py:128-131: fine-tuned names (those with both coarse.pth and c2f.pth) + "default"."""
        loras = cls.models_dir() / "loras"
        names = sorted(d.name for d in loras.iterdir() if (d / "coarse.pth").exists() and (d / "c2f.pth").exists()) \
            if loras.is_dir() else []
        return names + ["default"]

    def load_finetuned(self, name: str):
        """interface.py:134-144."""
        assert name in self.available_models(), f"{name} is not a valid model name"
        where = () if name == "default" else ("loras", name)
        self.reload(coarse_ckpt=self._cached(*where, "coarse.pth"), c2f_ckpt=self._cached(*where, "c2f.pth"))

    def add_finetuned(self, name: str):
        """Register the fine-tune `name` (loras/<name>/{coarse,c2f}.pth, resolved as load_finetuned resolves them) as a
        per-request adapter of the live coarse and c2f models: vamp / vamp_many requests then take adapter=name, and
        requests for different fine-tunes share launches.  The live models stay as they are (see load_finetuned for
        swapping a fine-tune in)."""
        coarse, c2f = self._cached("loras", name, "coarse.pth"), self._cached("loras", name, "c2f.pth")
        self.coarse.add_adapter(name, coarse)
        if self.c2f is not None:
            self.c2f.add_adapter(name, c2f)

    def reload(self, coarse_ckpt: str = None, c2f_ckpt: str = None):
        """Swap checkpoints (interface.py:146-174); a checkpoint already loaded is skipped.  A checkpoint of the same
        architecture is hot-swapped into the live model (VampNet.swap_checkpoint: packed device buffers rewritten in
        place, workspaces / tensor maps / captured generate graphs kept); otherwise the model is rebuilt."""
        for attr, path_attr, ckpt in (("coarse", "coarse_path", coarse_ckpt), ("c2f", "c2f_path", c2f_ckpt)):
            if ckpt is None or getattr(self, path_attr) == Path(ckpt):
                continue
            model = getattr(self, attr)
            if model is None or not model.swap_checkpoint(ckpt):
                chunk_size_s = model.chunk_size_s if model is not None else (10 if attr == "coarse" else 3)
                setattr(self, attr, _load_model(ckpt=ckpt, device=self.device, chunk_size_s=chunk_size_s))
            setattr(self, path_attr, Path(ckpt))

    # ------------------------------------------------------------------ unit helpers (interface.py:176-201)
    def s2t(self, seconds: float):
        """seconds to tokens"""
        if isinstance(seconds, np.ndarray):
            return np.ceil(seconds * self.codec.sample_rate / self.codec.hop_length)
        return math.ceil(seconds * self.codec.sample_rate / self.codec.hop_length)

    def s2t2s(self, seconds: float):
        return self.t2s(self.s2t(seconds))

    def t2s(self, tokens: int):
        return tokens * self.codec.hop_length / self.codec.sample_rate

    def to(self, device):
        self.device = device
        self.coarse.to(device)
        self.codec.to(device)
        if self.c2f is not None:
            self.c2f.to(device)
        if isinstance(self.beat_tracker, BeatTracker):
            self.beat_tracker.device = device
        return self

    def set_chunk_size(self, chunk_size_s: float):
        self.coarse.chunk_size_s = chunk_size_s

    # ------------------------------------------------------------------ codec boundary (interface.py:203-224)
    def decode(self, z: torch.Tensor):
        return self.coarse.decode(z, self.codec)

    def _preprocess(self, signal: AudioSignal):
        signal = (signal.clone().resample(self.codec.sample_rate).to_mono().normalize(self.loudness)
                  .ensure_max_of_audio(1.0))
        signal.samples, length = self.codec.preprocess(signal.samples, signal.sample_rate)
        return signal

    @torch.inference_mode()
    def encode(self, signal: AudioSignal):
        signal = signal.to(self.device)
        signal = self._preprocess(signal)
        return self.codec.encode(signal.samples, signal.sample_rate)["codes"]

    def decode_many(self, z_list: list):
        """[decode(z) for z in z_list], bit for bit, with the codec's decoder run over all entries together (clips of
        different lengths share launches)."""
        return self.coarse.decode_many(z_list, self.codec)

    @torch.inference_mode()
    def encode_many(self, signals: list):
        """[encode(s) for s in signals], bit for bit: each signal is preprocessed as encode does (resample, mono,
        loudness, peak, hop padding), then the codec's encoder runs over all of them together (clips of different
        lengths share launches)."""
        if len(signals) == 0:
            raise ValueError("encode_many: an empty list")
        prepared = [self._preprocess(s.to(self.device)) for s in signals]
        enc = self.codec.encode_many([s.samples for s in prepared], [s.sample_rate for s in prepared])
        return [e["codes"] for e in enc]

    # ------------------------------------------------------------------ validation (scripts/exp/train.py:327-371)
    def validate(self, signal: AudioSignal, model: str = "coarse", **kwargs) -> dict:
        """The reference training script's validation metrics for `signal`: encode(signal), then the coarse or c2f
        model's VampNet.validate(codec, codes, **kwargs) (r / rng, mask, label_smoothing, adapter).  Returns the
        reference's dict of 9 0-d fp32 device tensors ("loss", "accuracy-..."); held-out clips score a checkpoint or a
        fine-tune registered with add_finetuned (adapter=name)."""
        if model not in ("coarse", "c2f"):
            raise ValueError(f"validate: model must be 'coarse' or 'c2f', got {model!r}")
        vn = self.coarse if model == "coarse" else self.c2f
        if vn is None:
            raise ValueError("validate: this Interface has no c2f model")
        return vn.validate(self.codec, self.encode(signal), **kwargs)

    # ------------------------------------------------------------------ beats (interface.py:226-322)
    def snap_to_beats(self, signal: AudioSignal):
        """The signal trimmed to start at the first beat and end at the last."""
        assert hasattr(self, "beat_tracker"), "No beat tracker loaded"
        beats, downbeats = self.beat_tracker.extract_beats(signal)
        samples_begin = int(beats[0] * signal.sample_rate)
        samples_end = int(beats[-1] * signal.sample_rate)
        return signal.clone().trim(samples_begin, signal.length - samples_end)

    def make_beat_mask(self, signal: AudioSignal = None, before_beat_s: float = 0.0, after_beat_s: float = 0.02,
                       mask_downbeats: bool = True, mask_upbeats: bool = True, downbeat_downsample_factor: int = None,
                       beat_downsample_factor: int = None, dropout: float = 0.0, invert: bool = True):
        """A mask that keeps (0 after the inversion) the codes at and around each beat: before_beat_s before it,
        after_beat_s after it.  The beat times come from self.beat_tracker (librosa-style by default: no downbeats,
        so beat_downsample_factor thins all beats); the mask is built from them as the reference builds it."""
        if torch.device(self.device).type != "cuda":
            raise RuntimeError(f"make_beat_mask: the beat tracker runs on a CUDA device; this Interface is on "
                               f"{self.device}")
        assert self.beat_tracker is not None, "No beat tracker loaded"
        if signal is None:
            raise TypeError("make_beat_mask: a signal is required")
        beats, downbeats = self.beat_tracker.extract_beats(signal)
        n_codebooks = self.c2f.n_codebooks if self.c2f is not None else self.coarse.n_codebooks
        return beat_mask(beats, downbeats, signal.duration, self.s2t, n_codebooks, self.device,
                         before_beat_s=before_beat_s, after_beat_s=after_beat_s, mask_downbeats=mask_downbeats,
                         mask_upbeats=mask_upbeats, downbeat_downsample_factor=downbeat_downsample_factor,
                         beat_downsample_factor=beat_downsample_factor, dropout=dropout, invert=invert)

    # ------------------------------------------------------------------ chunk helpers
    @staticmethod
    def _spans(total: int, span: int):
        """[lo, hi) frame ranges of consecutive chunks of `span` frames covering `total` frames."""
        return [(lo, min(lo + span, total)) for lo in range(0, total, span)]

    # ------------------------------------------------------------------ coarse -> fine (interface.py:327-380)
    def _c2f_plan(self, z: torch.Tensor, mask: torch.Tensor = None):
        """The chunks of coarse_to_fine: the generate() arguments of each chunk (time_steps, start_tokens, mask) and
        the state _c2f_stitch needs."""
        assert self.c2f is not None, "No coarse2fine model loaded"
        n_frames = z.shape[-1]
        span = self.s2t(self.c2f.chunk_size_s)
        tail = (-n_frames) % span
        if tail:
            z = torch.nn.functional.pad(z, (0, tail))
            if mask is not None:
                mask = torch.nn.functional.pad(mask, (0, tail), value=1)
        missing = self.c2f.n_codebooks - z.shape[1]
        if missing > 0:
            z = torch.cat([z, z.new_zeros(z.shape[0], missing, z.shape[-1])], dim=1)
        if mask is not None:
            mask = mask.clone()
            mask[:, :self.c2f.n_conditioning_codebooks, :] = 0
        chunks = [dict(time_steps=span, start_tokens=z[..., lo:hi], mask=None if mask is None else mask[..., lo:hi])
                  for lo, hi in self._spans(z.shape[-1], span)]
        return chunks, (n_frames, mask)

    def _c2f_stitch(self, parts: list, state, return_mask: bool):
        n_frames, mask = state
        fine = torch.cat(parts, dim=-1)
        result = fine[..., :n_frames].clone()
        if not return_mask:
            return result
        remasked, _ = pmask.apply_mask(fine, mask, self.c2f.mask_token)
        return result, remasked[..., :n_frames].clone()

    @torch.inference_mode()
    def coarse_to_fine(self, z: torch.Tensor, mask: torch.Tensor = None, return_mask: bool = False, **kwargs):
        """Fill the fine codebooks given the coarse ones, c2f.chunk_size_s seconds at a time.  The sequence is
        zero-padded to a whole number of chunks (padding frames masked), missing codebooks are appended as zeros and
        the conditioning codebooks are never masked; every chunk is an independent generate() call."""
        chunks, state = self._c2f_plan(z, mask)
        parts = [self.c2f.generate(codec=self.codec, **c, return_signal=False, cfg_guidance=None, **kwargs)
                 for c in chunks]
        return self._c2f_stitch(parts, state, return_mask)

    # ------------------------------------------------------------------ coarse (interface.py:382-452)
    def _coarse_plan(self, z, mask):
        """The chunks of coarse_vamp: the generate() arguments of each chunk (time_steps, start_tokens, mask)."""
        n_books = self.coarse.n_codebooks
        tokens, keep = z[:, :n_books, :].clone(), mask[:, :n_books, :]
        assert keep.dtype == torch.long, f"mask must be long dtype, but got {keep.dtype}"
        assert bool(((keep == 0) | (keep == 1)).all()), "mask must be binary"   # the one host sync of this call
        span = self.s2t(self.coarse.chunk_size_s)
        chunks = []
        for lo, hi in self._spans(tokens.shape[-1], span):
            # a chunk that keeps anything also keeps its first and last frame; decided on the device (no sync):
            # edge value = 0 where any(m == 0) else unchanged
            m = keep[..., lo:hi].clone()
            anchors = (m == 0).any()
            m[..., 0] = torch.where(anchors, torch.zeros_like(m[..., 0]), m[..., 0])
            m[..., -1] = torch.where(anchors, torch.zeros_like(m[..., -1]), m[..., -1])
            start, m = pmask.apply_mask(tokens[..., lo:hi], m, self.coarse.mask_token, check=False)
            chunks.append(dict(time_steps=span, start_tokens=start, mask=m))
        return chunks

    def _coarse_stitch(self, z, chunks: list, results: list, return_mask: bool):
        out = torch.cat([torch.cat(results, dim=-1), z[:, self.coarse.n_codebooks:, :]], dim=1)
        return (out, torch.cat([c["start_tokens"] for c in chunks], dim=-1)) if return_mask else out

    @torch.inference_mode()
    def coarse_vamp(self, z, mask, return_mask=False, gen_fn=None, **kwargs):
        """Regenerate the masked coarse tokens, coarse.chunk_size_s seconds at a time.  A chunk that keeps at least one
        frame also keeps its first and last frame as anchors so that stitched chunks do not jump
        (interface.py:407-413).  Fine codebooks ride along untouched."""
        chunks = self._coarse_plan(z, mask)
        run = gen_fn or self.coarse.generate
        results = [run(codec=self.codec, **c, return_signal=False, **kwargs) for c in chunks]
        return self._coarse_stitch(z, chunks, results, return_mask)

    # ------------------------------------------------------------------ masks (interface.py:454-489)
    def build_mask(self, z: torch.Tensor, sig: AudioSignal = None, rand_mask_intensity: float = 1.0,
                   prefix_s: float = 0.0, suffix_s: float = 0.0, periodic_prompt: int = 7,
                   periodic_prompt_width: int = 1, onset_mask_width: int = 0, _dropout: float = 0.0,
                   upper_codebook_mask: int = 3, ncc: int = 0):
        """1 = regenerate, 0 = keep.  Intersection (mask_and) of: Bernoulli(rand_mask_intensity), kept prefix/suffix,
        periodic prompt (random roll), optional onset prompt; then time dropout, `ncc` always-kept codebooks and every
        codebook >= upper_codebook_mask fully masked.  Order and RNG use follow the reference exactly."""
        layers = [
            pmask.linear_random(z, rand_mask_intensity),
            pmask.inpaint(z, self.s2t(prefix_s), self.s2t(suffix_s)),
            pmask.periodic_mask(z, periodic_prompt, periodic_prompt_width, random_roll=True),
        ]
        if onset_mask_width > 0:
            assert sig is not None, "must provide a signal to use onset mask"
            layers.append(pmask.onset_mask(sig, z, self, width=onset_mask_width))
        mask = layers[0]
        for other in layers[1:]:
            mask = pmask.mask_and(mask, other)
        mask = pmask.codebook_unmask(pmask.dropout(mask, _dropout), ncc)
        return pmask.codebook_mask(mask, int(upper_codebook_mask), None)

    # ------------------------------------------------------------------ vamp (interface.py:491-562)
    @staticmethod
    def _vamp_inputs(codes, mask, batch_size: int, time_stretch_factor: int):
        z = codes.expand(batch_size, -1, -1)
        mask = mask.expand(batch_size, -1, -1)
        k = int(time_stretch_factor)
        if k > 1:
            z = z.repeat_interleave(k, dim=-1)
            inserted = torch.ones_like(z)
            inserted[..., ::k] = 0
            mask = (mask.repeat_interleave(k, dim=-1).bool() | inserted.bool()).long()
        return z, mask

    def _vamp_result(self, z, zv, coarse_start, fine_start, return_mask: bool):
        if not return_mask:
            return zv
        n_coarse = self.coarse.n_codebooks
        return zv, torch.cat([coarse_start[:, :n_coarse, :], fine_start[:, n_coarse:, :]], dim=1).cpu()

    def _with_fine_books(self, z, zv):
        """The coarse stage's output with the input's fine codebooks re-attached when the coarse model lacks them."""
        return torch.cat([zv, z[:, self.coarse.n_codebooks:, :]], dim=1) if zv.shape[1] < z.shape[1] else zv

    # the fine stage's generate arguments, pinned by the reference (interface.py:545-551)
    _C2F_KWARGS = dict(typical_filtering=True, _sampling_steps=2)

    def vamp(self, codes: torch.Tensor, mask: torch.Tensor, batch_size: int = 1, feedback_steps: int = 1,
             time_stretch_factor: int = 1, return_mask: bool = False, adapter: str = None, **kwargs):
        """codes, mask (1|B, 14, T) -> (B, 14, T'): coarse stage (`feedback_steps` passes, kwargs forwarded to
        generate) then the fine stage, which the reference pins to 2 sampling steps with default temperature
        (interface.py:545-551).  time_stretch_factor k > 1 inserts k-1 always-masked frames after every frame.
        adapter: a fine-tune registered with add_finetuned, applied in both stages (None: the live models)."""
        z, mask = self._vamp_inputs(codes, mask, batch_size, time_stretch_factor)
        with_adapter = {} if adapter is None else dict(adapter=adapter)
        zv = z
        for i in range(feedback_steps):
            zv, coarse_start = self.coarse_vamp(zv, mask=mask, return_mask=True, **with_adapter, **kwargs)
            coarse_start = coarse_start.roll(shifts=(i + 1) % feedback_steps, dims=-1)
        zv, fine_start = self.coarse_to_fine(self._with_fine_books(z, zv), mask=mask, return_mask=True,
                                             **self._C2F_KWARGS, **with_adapter)
        return self._vamp_result(z, zv, coarse_start, fine_start, return_mask)

    @torch.inference_mode()
    def vamp_many(self, requests: list, mixed_lengths: bool = False, mixed_steps: bool = False,
                  mixed_top_p: bool = False):
        """Serve many vamp() calls together.  Each request is a dict of vamp() arguments (codes, mask, and optionally
        batch_size, feedback_steps, time_stretch_factor, return_mask and generate keyword arguments).  Returns the
        list the sequential vamp() calls return, bit for bit, and leaves the random, numpy and torch RNG states as
        they would: every chunk's key is drawn first, in the sequential calls' order.

        The requests advance stage by stage: feedback pass i runs the chunks of every request that has a pass i as
        one generate_many(), then the fine stage runs every request's chunks as one more.  Chunks of equal length,
        within a request or across requests, so share launches.

        mixed_lengths=True: chunks of different lengths share launches too (generate_many(mixed_lengths=True) in both
        stages), so a request's remainder chunk need not run in a launch of its own; the results are the same.

        mixed_steps=True: chunks of requests with different sampling-step counts share launches too
        (generate_many(mixed_steps=True) in both stages); the results are the same.

        mixed_top_p=True: chunks of nucleus (top-p) and plain-sampling requests share launches too
        (generate_many(mixed_top_p=True) in both stages); the results are the same."""
        many = dict(mixed_lengths=True) if mixed_lengths else {}
        if mixed_steps:
            many["mixed_steps"] = True
        if mixed_top_p:
            many["mixed_top_p"] = True
        reqs = []
        for r in requests:
            r = dict(r)
            codes, mask, batch_size = r.pop("codes"), r.pop("mask"), r.pop("batch_size", 1)
            feedback_steps, k = r.pop("feedback_steps", 1), r.pop("time_stretch_factor", 1)
            return_mask = r.pop("return_mask", False)
            z, mask = self._vamp_inputs(codes, mask, batch_size, k)
            seed, key = r.pop("seed", None), r.pop("philox_key", None)
            adapter = r.pop("adapter", None)
            with_adapter = {} if adapter is None else dict(adapter=adapter)
            q = self._vamp_request(z, mask, feedback_steps, dict(r, **with_adapter),
                                   fine=dict(self._C2F_KWARGS, **with_adapter), fine_mask=mask, seed=seed, key=key)
            q["return_mask"] = return_mask
            reqs.append(q)
        self._run_vamp_requests(reqs, many)
        return [self._vamp_result(q["z"], q["zv"], q.get("coarse_start"), q["fine_start"], q["return_mask"])
                for q in reqs]

    def _vamp_request(self, z, mask, feedback_steps: int, gen: dict, fine: dict = None, fine_mask=None, seed=None,
                      key=None) -> dict:
        """A request for _run_vamp_requests, with the Philox keys of all its generate calls drawn now, in the order the
        sequential calls draw them: `feedback_steps` coarse_vamp passes over codes z with `mask` and generate keyword
        arguments `gen` (0 passes: no coarse stage; seed / key as generate's seed / philox_key), then, unless fine is
        None, coarse_to_fine of the result with generate keyword arguments `fine` and mask fine_mask."""
        from .modules.transformer import draw_philox_key
        n_frames = z.shape[-1]
        n_coarse = len(self._spans(n_frames, self.s2t(self.coarse.chunk_size_s)))
        keys = [[key if key is not None else draw_philox_key(seed) for _ in range(n_coarse)]
                for _ in range(feedback_steps)]
        c2f_keys = [] if fine is None else [draw_philox_key(None)
                                            for _ in self._spans(n_frames, self.s2t(self.c2f.chunk_size_s))]
        return dict(z=z, mask=mask, zv=z, feedback_steps=feedback_steps, gen=gen, keys=keys, fine=fine,
                    fine_mask=fine_mask, c2f_keys=c2f_keys)

    def _run_vamp_requests(self, reqs: list, many: dict):
        """Run prepared requests (_vamp_request) stage by stage: coarse pass i of every request that has one as one
        coarse generate_many(**many), then the fine stage of every request that has one as one c2f generate_many.  Sets
        each request's "zv" (its result), "coarse_start" and "fine_start" (the masked inputs of its last coarse pass and
        of its fine stage, where it has them and a fine_mask)."""
        for i in range(max((q["feedback_steps"] for q in reqs), default=0)):
            stage = [q for q in reqs if q["feedback_steps"] > i]
            plans = [self._coarse_plan(q["zv"], q["mask"]) for q in stage]
            calls = [dict(**c, return_signal=False, philox_key=k, **q["gen"])
                     for q, plan in zip(stage, plans) for c, k in zip(plan, q["keys"][i])]
            results = iter(self.coarse.generate_many(self.codec, calls, **many))
            for q, plan in zip(stage, plans):
                q["zv"], start = self._coarse_stitch(q["zv"], plan, [next(results) for _ in plan], True)
                q["coarse_start"] = start.roll(shifts=(i + 1) % q["feedback_steps"], dims=-1)
        stage = [q for q in reqs if q["fine"] is not None]
        if not stage:
            return
        plans = [self._c2f_plan(self._with_fine_books(q["z"], q["zv"]), q["fine_mask"]) for q in stage]
        calls = [dict(**c, return_signal=False, cfg_guidance=None, philox_key=k, **q["fine"])
                 for q, (chunks, _) in zip(stage, plans) for c, k in zip(chunks, q["c2f_keys"])]
        results = iter(self.c2f.generate_many(self.codec, calls, **many))
        for q, (chunks, state) in zip(stage, plans):
            out = self._c2f_stitch([next(results) for _ in chunks], state, q["fine_mask"] is not None)
            q["zv"], q["fine_start"] = out if q["fine_mask"] is not None else (out, None)
