"""Bit-level record of the audio kernels (vnb_pitch_shift and its float64 intermediates, vnb_beat_track,
vnb_onset_detect, vnb_mel_spectrogram, vnb_mel_loss) on seeded inputs:

    python tools/audio_bits.py --write tests/golden/audio_bits.npz

Every case builds its input on the CPU from a fixed seed, runs the library on cuda:0 and stores the SHA-256 of all of
its outputs (bit patterns, in a fixed order) plus a fixed seeded sample of its first output's values (for diagnosing a
mismatch).  tests/test_gpu_audio_bits.py requires a build to reproduce every hash, so a rewrite of an audio kernel
that alters any float operation or its order is caught bit for bit, even where the change stays inside the float64
tolerances of tests/test_gpu_pitch_ops.py.

The pitch cases store the fp32 output and the four intermediates that vnb_dbg_pitch_layout locates in the workspace
(spectrum, stretched spectrum, inverse-DFT frames, overlap-added signal); they cover odd and even n_fft, the three
stages isolated (rate 1 with new_freq = sr, the vocoder alone, the resampler alone) and the full composition.  The
beat cases store the envelope, tempo and beat frames at three tempo-window sizes W, the onset cases the envelope and
onset frames at three (sr, hop).  The mel spectrogram cases store the spectrogram at every window length from 32 to
4096, with empty Slaney bands at 48 kHz and one clip of the shortest accepted length; the mel loss cases store the
loss and the per-item losses of the default two scales and of seven scales at 48 kHz (empty bands at 32 and 64).  The
library wrappers here are shared with tests/test_gpu_pitch_ops.py,
tests/test_gpu_beat_ops.py and tests/test_gpu_onset_ops.py.
"""
from __future__ import annotations

import argparse
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import beat_oracle as bo  # noqa: E402
from oracle import gen_pitch_golden as gg  # noqa: E402
from oracle import mel_oracle as mo  # noqa: E402
from oracle import onset_oracle as oo  # noqa: E402
from oracle import pitch_oracle as po  # noqa: E402
from tools.gemm_bits import digest, lib, sample_index  # noqa: E402


# ---------------------------------------------------------------------------------------------------- wrappers
def pitch_signal(rows, N, sr, seed):
    """(rows, N) float32: gg.signal's partials, vibrato and noise floor, one seed per row."""
    return np.stack([gg.signal(sr, (N + 1) / sr, seed + 101 * r)[:N] for r in range(rows)])


def pitch_plan(rows, N, sr, new_freq, n_fft, hop, rate):
    """(workspace bytes, offsets[4], dims[4]) from vnb_pitch_workspace_bytes and vnb_dbg_pitch_layout, or None when
    either refuses (both must agree).  Needs only the library, not a device."""
    L = lib().lib()
    args = (rows, N, sr, new_freq, n_fft, hop, float(rate))
    need = ctypes.c_uint64(0)
    offs, dims = (ctypes.c_int64 * 4)(), (ctypes.c_int64 * 4)()
    rc_ws = L.vnb_pitch_workspace_bytes(*args, ctypes.byref(need))
    rc_layout = L.vnb_dbg_pitch_layout(*args, offs, dims)
    assert (rc_ws == 0) == (rc_layout == 0), (args, rc_ws, rc_layout)
    if rc_ws:
        return None
    return need.value, list(offs), list(dims)


def pitch_run(x, sr, new_freq, n_fft, hop, rate):
    """vnb_pitch_shift on x (rows, N) float32, then its intermediates read from the workspace through
    vnb_dbg_pitch_layout.  Returns CPU tensors: out (rows, N) fp32; spec (rows, F, nb, 2) float64 (re, im) when
    rate == 1, (|X|, angle X) otherwise; stretched (rows, F2, nb, 2) (re, im) or None; frames (rows, F2, n_fft);
    y (rows, L); and dims (F, F2, L, target)."""
    L = lib()
    x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()
    rows, N = x.shape
    plan = pitch_plan(rows, N, sr, new_freq, n_fft, hop, rate)
    assert plan is not None, "refused"
    need, offs, dims = plan
    F, F2, Ly, _ = dims
    nb = n_fft // 2 + 1
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.empty(rows, N, dtype=torch.float32, device="cuda")
    L.check(L.lib().vnb_pitch_shift(L.ptr(x), rows, N, sr, new_freq, n_fft, hop, float(rate), L.ptr(ws), need,
                                    L.ptr(out), L.stream_ptr()))
    w = ws.cpu()

    def region(i, shape):
        n = int(np.prod(shape))
        return w[offs[i]:offs[i] + 8 * n].view(torch.float64).reshape(shape).clone()

    return dict(out=out.cpu(), spec=region(0, (rows, F, nb, 2)),
                stretched=region(1, (rows, F2, nb, 2)) if offs[1] >= 0 else None,
                frames=region(2, (rows, F2, n_fft)), y=region(3, (rows, Ly)), dims=tuple(dims))


def beat_from_envelope(env, sr, hop, start_bpm=120.0, tightness=100.0, trim=True):
    """vnb_dbg_beat_from_envelope on a (B, F) float32 envelope: (tempo (B,), [beat frames per row])."""
    L = lib()
    env = torch.as_tensor(np.ascontiguousarray(env, dtype=np.float32)).reshape(-1, np.shape(env)[-1]).cuda()
    B, F = env.shape
    need = ctypes.c_uint64(0)
    L.check(L.lib().vnb_beat_workspace_bytes(B, (F - 1) * hop + 1, hop, ctypes.byref(need)))
    ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    tempo = torch.empty(B, dtype=torch.float64, device="cuda")
    beats = torch.empty(B, F, dtype=torch.int32, device="cuda")
    counts = torch.empty(B, dtype=torch.int32, device="cuda")
    L.check(L.lib().vnb_dbg_beat_from_envelope(L.ptr(env), B, F, sr, hop, float(start_bpm), float(tightness),
                                               int(trim), L.ptr(ws), need.value, L.ptr(tempo), L.ptr(beats),
                                               L.ptr(counts), L.stream_ptr()))
    counts = counts.cpu()
    return tempo.cpu().numpy(), [beats[b, :int(counts[b])].cpu().numpy() for b in range(B)]


def beat_track(y, sr, hop):
    """vampnet_b200.beats.beat_track on a (B, N) float32 signal: (envelope, tempo, [beat frames per row])."""
    from vampnet_b200.beats import beat_track as track
    r = track(torch.from_numpy(np.ascontiguousarray(y, dtype=np.float32)).cuda(), sr, hop)
    counts = r.counts.cpu()
    return r.envelope.cpu(), r.tempo.cpu(), [r.frames[b, :int(counts[b])].cpu() for b in range(counts.numel())]


def onset_detect(y, sr, hop, backtrack=True):
    """vampnet_b200.onset.onset_detect on a (B, N) float32 signal: (envelope, [onset frames per row])."""
    from vampnet_b200.onset import onset_detect as detect
    r = detect(torch.from_numpy(np.ascontiguousarray(y, dtype=np.float32)).cuda(), sr, hop, backtrack=backtrack)
    counts = r.counts.cpu()
    return r.envelope.cpu(), [r.frames[b, :int(counts[b])].cpu() for b in range(counts.numel())]


def mel_spectrogram(x, sr, n_fft, hop, n_mels):
    """vnb_mel_spectrogram on x (rows, N) float32, fmin 0 and fmax sr / 2: (rows, n_mels, F) fp32 on the CPU."""
    L = lib()
    xd = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()
    rows, N = xd.shape
    sc = L.MelScale(n_fft, hop, n_mels, 0.0, sr / 2)
    out = torch.empty(rows, n_mels, 1 + N // hop, dtype=torch.float32, device="cuda")
    L.check(L.lib().vnb_mel_spectrogram(L.ptr(xd), rows, N, sr, ctypes.byref(sc), L.ptr(out), L.stream_ptr()))
    return out.cpu()


def mel_loss(x, y, sr, scales):
    """MelSpectrogramLoss over (n_mels, fmin, fmax, window) scales on (B, C, N) float32 pairs: (loss (1,), items (B,))."""
    from vampnet_b200.audio import AudioSignal
    from vampnet_b200.metrics import MelSpectrogramLoss
    m, lo, hi, w = zip(*scales)
    fn = MelSpectrogramLoss(n_mels=list(m), window_lengths=list(w), mel_fmin=list(lo), mel_fmax=list(hi))
    xs, ys = (AudioSignal(torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda(), sr) for a in (x, y))
    return fn(xs, ys).reshape(1).cpu(), fn.per_item(xs, ys).cpu()


# ---------------------------------------------------------------------------------------------------- record
PITCH_CASES = {  # name: rows, N, sr, new_freq, rate, n_fft, hop
    "pitch_n16_h1": (1, 200, 44100, 44100, 1.0, 16, 1),
    "pitch_n65_h16_vocoder": (2, 3000, 44100, 44100, 2.0 ** (-1 / 12), 65, 16),
    "pitch_n128_h32_r2": (1, 4000, 44100, 44100, 2.0, 128, 32),
    "pitch_n689_h21_default_p5": (1, 6000, 44100, *po.shift_params(5, 44100)[2:], 689, 21),
    "pitch_n750_h23_default_m7": (1, 6000, 48000, *po.shift_params(-7, 48000)[2:], 750, 23),
    "pitch_n1024_h256_resample": (1, 5000, 44100, 41625, 1.0, 1024, 256),
    "pitch_n2047_h511_r05": (1, 8000, 44100, 44100, 0.5, 2047, 511),
    "pitch_n4096_h1024_full": (1, 12000, 16000, 15999, 2.0 ** (1 / 12), 4096, 1024),
}
BEAT_CASES = {  # name: sr, hop, signal   (W = int(8 sr) // hop)
    "beat_w459": (44100, 768, "bursts_4"),
    "beat_w1024": (16000, 125, "bursts_4"),
    "beat_w4096": (2048, 4, "clicks120"),
}
ONSET_CASES = {  # name: sr, hop, signal
    "onset_44100_h32": (44100, 32, "clicks"),
    "onset_22050_h1324": (22050, 1324, "bursts"),
    "onset_96000_h4096": (96000, 4096, "bursts"),
}
MEL_SPEC_CASES = {  # name: n_fft, hop, n_mels, sr, N; rows: mo.test_pair's two signals
    "melspec_w32_sr48000": (32, 8, 5, 48000, 2000),  # band 0 is empty
    "melspec_w64_sr48000": (64, 16, 10, 48000, 3000),  # an empty band
    "melspec_w128": (128, 32, 20, 16000, 3000),
    "melspec_w256": (256, 64, 40, 22050, 5000),
    "melspec_w512_Nmin": (512, 128, 80, 44100, 257),  # N = n_fft / 2 + 1: the reflection reaches the far end
    "melspec_w1024": (1024, 256, 160, 48000, 9000),
    "melspec_w2048": (2048, 512, 150, 44100, 20000),
    "melspec_w4096": (4096, 1000, 128, 44100, 30000),  # a hop that does not divide N
}
MEL_LOSS_CASES = {  # name: sr, N, B, C, scales; item b is mo.test_pair at seed b
    "mel_loss_default": (44100, 22050, 3, 1, mo.DEFAULT_SCALES),
    "mel_loss_seven_sr48000": (48000, 12000, 2, 2, mo.SEVEN_SCALES),
}
CASES = list(PITCH_CASES) + list(BEAT_CASES) + list(ONSET_CASES) + list(MEL_SPEC_CASES) + list(MEL_LOSS_CASES)


def run_named(name):
    """All outputs of the record case `name`, as CPU tensors in a fixed order."""
    if name in PITCH_CASES:
        rows, N, sr, new_freq, rate, n_fft, hop = PITCH_CASES[name]
        r = pitch_run(pitch_signal(rows, N, sr, 7), sr, new_freq, n_fft, hop, rate)
        return [r[k] for k in ("out", "spec", "stretched", "frames", "y") if r[k] is not None]
    if name in BEAT_CASES:
        sr, hop, sig = BEAT_CASES[name]
        env, tempo, beats = beat_track(bo.test_signal(sig, sr)[None], sr, hop)
        return [env, tempo, beats[0]]
    if name in ONSET_CASES:
        sr, hop, sig = ONSET_CASES[name]
        env, onsets = onset_detect(oo.test_signal(sig, sr)[None], sr, hop)
        return [env, onsets[0]]
    if name in MEL_SPEC_CASES:
        n_fft, hop, n_mels, sr, N = MEL_SPEC_CASES[name]
        return [mel_spectrogram(np.concatenate(mo.test_pair(N, sr, seed=11)), sr, n_fft, hop, n_mels)]
    if name in MEL_LOSS_CASES:
        sr, N, B, C, scales = MEL_LOSS_CASES[name]
        pairs = [mo.test_pair(N, sr, seed=b, channels=C) for b in range(B)]
        return list(mel_loss(np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs]), sr, scales))
    raise KeyError(name)


def sample_values(outs, name):
    flat = outs[0].double().reshape(-1).numpy()
    return flat[sample_index(flat.size, name)]


def record():
    rec = {}
    for name in CASES:
        outs = run_named(name)
        rec["sha256_" + name] = np.array(digest(outs))
        rec["sample_" + name] = sample_values(outs, name)
        print(f"{name}: {rec['sha256_' + name]}", flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--write", metavar="NPZ", help="where to store the hashes and samples (default: only print them)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    rec = record()
    dev = torch.cuda.get_device_properties(0)
    rec["device"] = np.array(dev.name)
    if args.write:
        os.makedirs(os.path.dirname(os.path.abspath(args.write)), exist_ok=True)
        np.savez_compressed(args.write, **rec)
        print(f"wrote {len(CASES)} cases to {args.write}")


if __name__ == "__main__":
    main()
