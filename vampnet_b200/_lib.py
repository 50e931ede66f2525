"""ctypes binding of the C ABI declared in include/vampnet_b200.h.

The library is built in-tree by ``python -m vampnet_b200.build`` (nvcc, sm_90a).  There is no
CPU fallback: if the shared object is missing or cannot be loaded, every entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvampnet_b200.so")

EPI_BF16, EPI_QKV, EPI_RESID, EPI_GEGLU, EPI_BIAS_F32 = range(5)
FAMILIES = ("embed", "rmsnorm", "gemm_qkv", "attention", "gemm_attn_out", "gemm_ffn_up", "gemm_ffn_down",
            "gemm_classifier", "sample_remask", "state")
LORA_DOWN_FAMILY = 10  # profile family of the LoRA down-projections (adapted launches only); VNB_NUM_FAMILIES = 11
MAX_ADAPTERS = 16      # VNB_MAX_ADAPTERS


class Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "n_heads", "n_layers", "n_codebooks", "n_conditioning_codebooks", "latent_dim", "d_model", "vocab_size")]


class Weights(C.Structure):
    _fields_ = [
        ("emb_table", C.c_void_p), ("emb_w3", C.c_void_p), ("emb_b", C.c_void_p), ("norm1", C.c_void_p),
        ("wqkv", C.c_void_p), ("wo", C.c_void_p), ("norm3", C.c_void_p), ("w1", C.c_void_p), ("w2", C.c_void_p),
        ("norm_f", C.c_void_p), ("wcls", C.c_void_p), ("bcls", C.c_void_p), ("rel_bias", C.c_void_p),
        ("rel_sat", C.c_int32),
    ]


class AdapterWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("a_qkv", "b_qkv", "a_wo", "b_wo", "a_w1", "b_w1", "a_w2", "b_w2")]


class GenParams(C.Structure):
    _fields_ = [
        ("sampling_steps", C.c_int32), ("temperature", C.c_float), ("gamma", C.POINTER(C.c_float)),
        ("temp_eff", C.POINTER(C.c_float)), ("do_sample", C.POINTER(C.c_int32)), ("seed_lo", C.c_uint32),
        ("seed_hi", C.c_uint32), ("use_graph", C.c_int32), ("top_p", C.c_float),
    ]


class GenGroup(C.Structure):
    _fields_ = [
        ("rows", C.c_int32), ("temperature", C.c_float), ("temp_eff", C.POINTER(C.c_float)),
        ("do_sample", C.POINTER(C.c_int32)), ("seed_lo", C.c_uint32), ("seed_hi", C.c_uint32), ("top_p", C.c_float),
    ]


class SampleGroup(C.Structure):
    _fields_ = [
        ("rows", C.c_int32), ("temperature", C.c_float), ("gamma", C.c_float), ("temp_eff", C.c_float),
        ("do_sample", C.c_int32), ("is_last", C.c_int32), ("step", C.c_int32), ("seed_lo", C.c_uint32),
        ("seed_hi", C.c_uint32), ("top_p", C.c_float),
    ]


class MelScale(C.Structure):
    _fields_ = [("n_fft", C.c_int32), ("hop", C.c_int32), ("n_mels", C.c_int32), ("fmin", C.c_double),
                ("fmax", C.c_double)]


_SIGS = {
    "vnb_abi_version": (C.c_int32, []),
    "vnb_last_error": (C.c_char_p, []),
    "vnb_model_create": (C.c_int32, [C.POINTER(Config), C.POINTER(Weights), C.POINTER(C.c_void_p)]),
    "vnb_model_destroy": (None, [C.c_void_p]),
    "vnb_forward_codes": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "vnb_forward_latents": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "vnb_forward_latents_acts": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                             C.c_void_p]),
    "vnb_get_hidden": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "vnb_generate": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(GenParams),
                                 C.c_void_p, C.c_void_p]),
    "vnb_generate_many": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                      C.POINTER(C.c_float), C.POINTER(GenGroup), C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_void_p]),
    "vnb_generate_many_adapted": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                              C.POINTER(C.c_float), C.POINTER(GenGroup), C.c_int32,
                                              C.POINTER(C.c_int32), C.c_int32, C.c_void_p, C.c_void_p]),
    "vnb_generate_ragged": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                        C.POINTER(C.c_float), C.POINTER(GenGroup), C.c_int32, C.POINTER(C.c_int32),
                                        C.POINTER(C.c_int32), C.c_int32, C.c_void_p, C.c_void_p]),
    "vnb_generate_steps": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32),
                                       C.POINTER(C.POINTER(C.c_float)), C.POINTER(GenGroup), C.c_int32,
                                       C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int32, C.c_void_p, C.c_void_p]),
    "vnb_generate_mixed_top_p": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                             C.POINTER(C.c_int32), C.POINTER(C.POINTER(C.c_float)), C.POINTER(GenGroup),
                                             C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int32,
                                             C.c_void_p, C.c_void_p]),
    "vnb_adapter_add": (C.c_int32, [C.c_void_p, C.POINTER(AdapterWeights), C.POINTER(C.c_int32)]),
    "vnb_adapter_remove": (C.c_int32, [C.c_void_p, C.c_int32]),
    "vnb_forward_codes_adapted": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32),
                                              C.c_void_p, C.c_void_p]),
    "vnb_launch_count": (C.c_uint64, []),
    "vnb_graph_capture_count": (C.c_uint64, []),
    "vnb_set_option": (C.c_int32, [C.c_char_p, C.c_int32]),
    "vnb_get_option": (C.c_int32, [C.c_char_p, C.POINTER(C.c_int32)]),
    "vnb_profile_begin": (C.c_int32, [C.c_void_p]),
    "vnb_profile_end": (C.c_int32, [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_int32), C.c_int32]),
    "vnb_sample_step": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                    C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float,
                                    C.c_float, C.c_uint32, C.c_uint32, C.c_void_p]),
    "vnb_op_gemm": (C.c_int32, [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "vnb_op_attention": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                     C.c_int32, C.c_int32, C.c_void_p]),
    "vnb_dbg_attention_ragged": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                             C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "vnb_codec_conv1d": (C.c_int32, [C.c_void_p] * 6 + [C.c_int32] * 13 + [C.c_void_p]),
    "vnb_codec_rvq": (C.c_int32, [C.c_int32] + [C.c_void_p] * 11 + [C.c_int32] * 6 + [C.c_void_p] * 3),
    "vnb_codec_conv_tc": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_void_p]),
    "vnb_codec_conv_in": (C.c_int32, [C.c_void_p] * 7 + [C.c_int32] * 5 + [C.c_void_p]),
    "vnb_codec_conv_out": (C.c_int32, [C.c_void_p] * 5 + [C.c_int32] * 5 + [C.c_void_p]),
    "vnb_codec_conv_tc_ragged": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                             C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                             C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                             C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "vnb_codec_conv_in_ragged": (C.c_int32, [C.c_void_p] * 7 + [C.c_int32] * 5 + [C.c_void_p, C.c_void_p]),
    "vnb_codec_conv_out_ragged": (C.c_int32, [C.c_void_p] * 5 + [C.c_int32] * 5 + [C.c_void_p, C.c_void_p]),
    "vnb_set_error_cuda": (C.c_int32, [C.c_char_p, C.c_int32]),
    "vnb_dbg_set_live": (C.c_int32, [C.c_void_p]),
    "vnb_dbg_gemm_ref": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "vnb_dbg_gemm_fused": (C.c_int32, [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_float,
                                       C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vnb_dbg_gemm_adapted": (C.c_int32, [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                         C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_float,
                                         C.c_float, C.c_void_p, C.c_void_p, C.POINTER(AdapterWeights), C.c_int32,
                                         C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vnb_dbg_gemm_qkv_frames": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                            C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_float, C.c_float,
                                            C.c_void_p, C.POINTER(AdapterWeights), C.c_int32, C.c_int32, C.c_void_p,
                                            C.c_void_p, C.c_void_p]),
    "vnb_dbg_gemm_sample": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                        C.c_int32, C.c_float, C.c_float, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_uint32, C.c_uint32,
                                        C.c_void_p, C.c_void_p]),
    "vnb_onset_workspace_bytes": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    "vnb_onset_detect": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                     C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vnb_onset_mask": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                   C.c_int32, C.c_int32, C.c_void_p]),
    "vnb_beat_workspace_bytes": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    "vnb_beat_track": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_double,
                                   C.c_int32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p]),
    "vnb_dbg_beat_from_envelope": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double,
                                               C.c_double, C.c_int32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p]),
    "vnb_pitch_workspace_bytes": (C.c_int32, [C.c_int32] * 6 + [C.c_double, C.POINTER(C.c_uint64)]),
    "vnb_pitch_shift": (C.c_int32, [C.c_void_p] + [C.c_int32] * 6 + [C.c_double, C.c_void_p, C.c_uint64, C.c_void_p,
                                                                      C.c_void_p]),
    "vnb_dbg_pitch_layout": (C.c_int32, [C.c_int32] * 6 + [C.c_double, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "vnb_dbg_pitch_time_steps": (C.c_int32, [C.c_double, C.c_int32, C.c_void_p, C.c_void_p]),
    "vnb_xent_metrics_workspace_bytes": (C.c_int32, [C.c_int32, C.c_int64, C.POINTER(C.c_uint64)]),
    "vnb_xent_metrics": (C.c_int32, [C.c_void_p] * 4 + [C.c_int32] * 5 + [C.c_double, C.c_void_p, C.c_uint64, C.c_void_p,
                                                                          C.c_void_p, C.c_void_p]),
    "vnb_dbg_xent_rows": (C.c_int32, [C.c_void_p] * 2 + [C.c_int32] * 5 + [C.c_void_p, C.c_void_p]),
    "vnb_mel_spectrogram": (C.c_int32, [C.c_void_p] + [C.c_int32] * 3 + [C.POINTER(MelScale), C.c_void_p, C.c_void_p]),
    "vnb_mel_workspace_bytes": (C.c_int32, [C.c_int32] * 4 + [C.POINTER(MelScale), C.c_int32, C.POINTER(C.c_uint64)]),
    "vnb_mel_loss": (C.c_int32, [C.c_void_p] * 2 + [C.c_int32] * 4 + [C.POINTER(MelScale), C.c_int32] + [C.c_double] * 4
                     + [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vnb_dbg_sample": (C.c_int32, [C.c_int32] + [C.c_void_p] * 7 + [C.c_int32] * 6 + [C.POINTER(SampleGroup),
                                                                                        C.c_int32, C.c_void_p]),
    "vnb_dbg_sample_split": (C.c_int32, [C.c_void_p] * 7 + [C.c_int32] * 6 + [C.POINTER(SampleGroup), C.c_int32,
                                                                             C.c_void_p]),
    "vnb_dbg_gemm_sample_split": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                              C.c_void_p, C.c_int32, C.c_float, C.c_float, C.c_void_p, C.c_int32,
                                              C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(SampleGroup),
                                              C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
}

_lib = None


def exported_symbols():
    return sorted(_SIGS)


def lib():
    """Load (once) and return the shared library.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        # not a fallback: the only way to get the kernels is to compile them (nvcc cross-compiles sm_90a anywhere)
        try:
            from . import build as _build
            _build.build()
        except Exception as e:
            raise RuntimeError(
                f"{LIB_PATH} not found and building it failed ({e}); build it with `python -m vampnet_b200.build` "
                "(nvcc, sm_90a). vampnet_b200 has no CPU or PyTorch fallback.") from e
    L = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGS.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    if L.vnb_abi_version() != 2:
        raise RuntimeError("ABI version mismatch between _lib.py and libvampnet_b200.so")
    _lib = L
    return L


def check(rc: int):
    if rc != 0:
        raise RuntimeError("vampnet_b200: " + lib().vnb_last_error().decode(errors="replace"))


def ptr(t):
    """Raw device/host address of a torch tensor (or None)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr(device=None):
    import torch
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def workspace(device, query, *args):
    """(workspace, size): a uint8 tensor on ``device`` of the size in bytes that ``query``, one of the
    ``vnb_*_workspace_bytes`` entry points, reports for ``args``."""
    import torch
    n = C.c_uint64(0)
    check(query(*args, C.byref(n)))
    return torch.empty(n.value, dtype=torch.uint8, device=device), n.value
