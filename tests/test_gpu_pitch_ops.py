"""GPU: the pitch-shift kernels (csrc/pitch.cu) stage by stage against float64, across the n_fft, hop, N, rate and
rate pairs that vnb_pitch_shift accepts, and end to end through vampnet_b200.pitch.pitch_shift at sample rates and
arguments other than the app's.

vnb_dbg_pitch_layout locates the float64 intermediates in the workspace, and the C ABI takes new_freq and rate
separately, so setting one of them to identity isolates the other.  Each stage is compared against the oracle's
(oracle/pitch_oracle.py) statement of that stage applied to the device's own previous stage, within a bound from the
analysis of the stage's float64 arithmetic (u = 2^-53):

  forward DFT   per frame, |X - rfft(frame)| <= C_DFT n_fft u sum|frame|: every basis value is cos or sin of an argument
                reduced exactly and rounded a few times (error < 22 u), and the K = n_fft products are summed in some
                order (error < K u sum|terms|); numpy's FFT adds O(log n_fft) u.  Magnitudes are held to the same bound
                where the vocoder reads them as (|X|, angle X).
  vocoder       |Y - ref| <= C_VOC u |Y| (F2 P + 1), P the largest running sum of |phase increment|: the increments are
                the oracle's expressions on the device's own (|X|, angle), so only the running sum's order (chunk sums,
                then offsets) and sincos differ.
  inverse DFT   per frame, |frame - irfft(Y)| <= C_DFT nb u (2 / n_fft) sum_k(|Re Y_k| + |Im Y_k|), the same analysis
                with K = 2 nb and the 2 / n_fft folded into the basis.
  overlap-add   |y - ola(frames)| <= 4 u ola(|frames|): the same sums in the same frame order.
  resampler     |out - float32(resample(y))| <= one fp32 ulp of the reference (taken at no less than 2^-24, where the
                float64 sum's own rounding would exceed it).

The bounds are analytic; the worst ratio of error to bound per stage is printed by the last test of this file.  End to
end, the outputs are held to test_gpu_pitch.py's ATOL on signals whose conditioning figure exceeds COND_MIN."""
import math

import numpy as np
import pytest
import torch

from oracle import pitch_oracle as po
from tools import audio_bits as AB

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
C_DFT = 4
C_VOC = 4
ATOL = 1e-6
COND_MIN = 1e-8
R12 = 2.0 ** (1 / 12)
_worst = {}

# name: rows, N, sr, new_freq, rate, n_fft, hop.  F = 1 + (N + 2 (n_fft // 2) - n_fft) // hop, F2 = ceil(F / rate);
# tests/test_audio_params_cpu.py checks the shapes noted here.
CASES = [
    # forward DFT, inverse DFT and overlap-add (rate 1, new_freq = sr)
    ("n16_h1_Nmin", 3, 9, 44100, 44100, 1.0, 16, 1),               # N = n_fft // 2 + 1: reflects at both ends
    ("n17_h2_Nmin", 1, 9, 44100, 44100, 1.0, 17, 2),
    ("n63_h15_F64", 1, 946, 44100, 44100, 1.0, 63, 15),            # F = 0 (mod 64), F2 = 0 (mod 32)
    ("n64_h32_F65", 1, 2048, 44100, 44100, 1.0, 64, 32),           # F = 1 (mod 64), F2 = 1 (mod 32)
    ("n65_h64_F63", 3, 3969, 44100, 44100, 1.0, 65, 64),           # F = 63 (mod 64), F2 = 31 (mod 32)
    ("n127_h127_Nmin", 1, 64, 44100, 44100, 1.0, 127, 127),        # one frame, L = 1
    ("n128_h1_Nmin", 1, 65, 44100, 44100, 1.0, 128, 1),
    ("n129_h2", 1, 300, 44100, 44100, 1.0, 129, 2),
    ("n2047_h2046", 1, 30000, 44100, 44100, 1.0, 2047, 2046),
    ("n2048_h512_Nmin", 1, 1025, 44100, 44100, 1.0, 2048, 512),
    ("n4096_h2048", 1, 20000, 44100, 44100, 1.0, 4096, 2048),
    # + the vocoder (rate != 1, new_freq = sr)
    ("v_n16_h1_r05", 1, 40, 44100, 44100, 0.5, 16, 1),             # F2 = 2 F
    ("v_n17_h4_r_near1", 1, 100, 44100, 44100, 1 - 2.0 ** -20, 17, 4),  # steps just below whole frames; F2 = F + 1
    ("v_n64_h16_r05_F2_0", 3, 752, 44100, 44100, 0.5, 64, 16),     # F2 = 96 = 0 (mod 32)
    ("v_n128_h32_up_F2_31", 1, 2080, 44100, 44100, R12, 128, 32),  # F2 = 63 = 31 (mod 32)
    ("v_n689_h21_down_F63", 1, 4000, 44100, 44100, 1 / R12, 689, 21),
    ("v_n750_h375_down_F2_0", 1, 10875, 44100, 44100, 1 / R12, 750, 375),
    ("v_n1024_h256_r2_F2_1", 1, 16384, 44100, 44100, 2.0, 1024, 256),  # F2 = 33 = 1 (mod 32)
    ("v_n2047_h511_r2", 3, 12000, 44100, 44100, 2.0, 2047, 511),
    ("v_n2048_h2048_Nmin_r05", 1, 1025, 44100, 44100, 0.5, 2048, 2048),  # one frame, stretched to two
    ("v_n4095_h4094_r05", 1, 30000, 44100, 44100, 0.5, 4095, 4094),
    ("v_n4096_h1024_up", 1, 20000, 44100, 44100, R12, 4096, 1024),
    # + the resampler (rate 1, new_freq != sr)
    ("s_44100_41625_n689", 1, 4000, 44100, 41625, 1.0, 689, 21),   # gcd 225; target < N: zero padded
    ("s_44100_44101_n750", 1, 3000, 44100, 44101, 1.0, 750, 187),  # coprime
    ("s_48000_96000_n1024", 3, 5000, 48000, 96000, 1.0, 1024, 256),  # target > N: cut
    ("s_16000_15999_n4095", 1, 9000, 16000, 15999, 1.0, 4095, 4095),
    ("s_8000_16001_n129", 1, 3000, 8000, 16001, 1.0, 129, 64),
]
BATCHED = [c[0] for c in CASES if c[1] > 1]

# end to end through pitch_shift: (sample rate, shift, n_fft, hop_length), 0 for the default n_fft and hop
END_TO_END = [
    (8000, 1, 0, 0), (8000, -12, 0, 0),
    (16000, -1, 0, 0), (16000, 7, 0, 0),
    (22050, -7, 0, 0), (22050, 12, 0, 0),
    (32000, "fast", 0, 0), (32000, -12, 0, 0),
    (96000, 12, 0, 0), (96000, -1, 0, 0),
    (44100, 5, 1024, 256), (16000, -3, 129, 64), (48000, "fast", 2048, 2047), (22050, 2, 500, 500),
]
E2E_SECONDS = 0.5


def signal(name, rows, N, sr):
    return AB.pitch_signal(rows, N, sr, 1000 + [c[0] for c in CASES].index(name))


def e2e_case(i):
    """(signal (1, 1, N), shift, sample rate, n_fft, hop) of END_TO_END[i]; "fast" is one of get_fast_shifts' ratios."""
    sr, shift, n_fft, hop = END_TO_END[i]
    if shift == "fast":
        from vampnet_b200.pitch import get_fast_shifts
        fast = get_fast_shifts(sr)
        shift = fast[len(fast) // 3]
    return AB.pitch_signal(1, int(E2E_SECONDS * sr), sr, 2000 + i)[None], shift, sr, n_fft, hop


@pytest.fixture(scope="module", params=CASES, ids=[c[0] for c in CASES])
def run(request):
    name, rows, N, sr, new_freq, rate, n_fft, hop = request.param
    x = signal(name, rows, N, sr)
    return dict(name=name, x=x, sr=sr, new_freq=new_freq, rate=rate, n_fft=n_fft, hop=hop,
                dev={k: (v.numpy() if torch.is_tensor(v) else v) for k, v in
                     AB.pitch_run(x, sr, new_freq, n_fft, hop, rate).items()})


def _ratio(stage, name, err, bound):
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    worst = float(np.max(r)) if r.size else 0.0
    if worst >= _worst.get(stage, (-1.0, ""))[0]:
        _worst[stage] = (worst, name)
    return worst


def _complex(a):
    return a[..., 0] + 1j * a[..., 1]


def ola(frames, n_fft, hop):
    """oracle.pitch_oracle.istft's overlap-add on given frames (rows, F2, n_fft): the same loop, without the irfft."""
    rows, F2, _ = frames.shape
    total = n_fft + hop * (F2 - 1)
    y = np.zeros((rows, total))
    cnt = np.zeros(total)
    for f in range(F2):
        y[:, f * hop:f * hop + n_fft] += frames[:, f]
        cnt[f * hop:f * hop + n_fft] += 1
    s = n_fft // 2
    return y[:, s:total - s] / cnt[s:total - s]


def vocoder_from_polar(mag, ang, rate, hop):
    """oracle.pitch_oracle.phase_vocoder's steps on a given (|X|, angle X): (re, im, |Y|, running sum of |increment|)."""
    rows, F, nb = mag.shape
    ts = po.time_steps(F, rate)
    alphas = (ts % np.float32(1.0)).astype(np.float64)[None, :, None]
    i0 = np.floor(ts).astype(np.int64)
    zeros = np.zeros((rows, 2, nb))
    pm, pa = np.concatenate([mag, zeros], axis=1), np.concatenate([ang, zeros], axis=1)
    adv = po.phase_advance(nb, hop)[None, None, :]
    ph = pa[:, i0 + 1] - pa[:, i0] - adv
    ph = ph - 2 * math.pi * np.round(ph / (2 * math.pi))
    ph = ph + adv
    ph = np.concatenate([ang[:, :1], ph[:, :-1]], axis=1)
    acc = np.cumsum(ph, axis=1)
    m = alphas * pm[:, i0 + 1] + (1 - alphas) * pm[:, i0]
    return m * np.cos(acc), m * np.sin(acc), m, np.cumsum(np.abs(ph), axis=1)


def plan_dims(N, sr, new_freq, rate, n_fft, hop):
    """(F, F2, L, target) as the oracle's stages produce them."""
    F = po.stft(np.zeros((1, N)), n_fft, hop).shape[1]
    F2 = len(po.time_steps(F, rate)) if rate != 1.0 else F
    L = n_fft - 2 * (n_fft // 2) + hop * (F2 - 1)
    return F, F2, L, po.resample(np.zeros((1, L)), sr, new_freq).shape[1]


def test_dims_match_oracle(run):
    N = run["x"].shape[1]
    assert run["dev"]["dims"] == plan_dims(N, run["sr"], run["new_freq"], run["rate"], run["n_fft"], run["hop"])


def test_forward_dft(run):
    d, n_fft, hop = run["dev"], run["n_fft"], run["hop"]
    x = run["x"].astype(np.float64)
    want = po.stft(x, n_fft, hop)
    pad = n_fft // 2
    xp = np.pad(x, ((0, 0), (pad, pad)), mode="reflect")
    idx = np.arange(want.shape[1])[:, None] * hop + np.arange(n_fft)[None, :]
    bound = (C_DFT * n_fft * U * np.abs(xp[:, idx]).sum(-1))[..., None]  # (rows, F, 1)
    spec = d["spec"]
    if run["rate"] == 1.0:
        got = _complex(spec)
        err = np.maximum(np.abs(got.real - want.real), np.abs(got.imag - want.imag))
    else:  # (|X|, angle X): the magnitudes on their own, and the spectrum they describe
        err_mag = np.abs(spec[..., 0] - np.abs(want))
        assert _ratio("forward DFT |X|", run["name"], err_mag, bound) <= 1.0, "magnitudes"
        got = spec[..., 0] * np.exp(1j * spec[..., 1])
        err = np.maximum(np.abs(got.real - want.real), np.abs(got.imag - want.imag))
    assert _ratio("forward DFT", run["name"], err, bound) <= 1.0


def test_vocoder(run):
    d = run["dev"]
    if run["rate"] == 1.0:
        assert d["stretched"] is None
        return
    re, im, mag, run_sum = vocoder_from_polar(d["spec"][..., 0], d["spec"][..., 1], run["rate"], run["hop"])
    F2 = re.shape[1]
    assert d["stretched"].shape[:3] == re.shape
    bound = C_VOC * U * mag * (F2 * run_sum.max() + 1)
    err = np.maximum(np.abs(d["stretched"][..., 0] - re), np.abs(d["stretched"][..., 1] - im))
    assert _ratio("vocoder", run["name"], err, bound) <= 1.0


def test_inverse_dft(run):
    d, n_fft = run["dev"], run["n_fft"]
    Y = d["stretched"] if d["stretched"] is not None else d["spec"]
    want = np.fft.irfft(_complex(Y), n=n_fft, axis=-1)
    nb = n_fft // 2 + 1
    bound = (C_DFT * nb * U * (2.0 / n_fft) * np.abs(Y).sum(axis=(-1, -2)))[..., None]
    err = np.abs(d["frames"] - want)
    assert _ratio("inverse DFT", run["name"], err, bound) <= 1.0


def test_overlap_add(run):
    d = run["dev"]
    want = ola(d["frames"], run["n_fft"], run["hop"])
    bound = 4 * U * ola(np.abs(d["frames"]), run["n_fft"], run["hop"])
    assert d["y"].shape == want.shape
    err = np.abs(d["y"] - want)
    assert _ratio("overlap-add", run["name"], err, bound) <= 1.0


def test_resampler_and_output(run):
    d = run["dev"]
    rows, N = run["x"].shape
    y = po.resample(d["y"], run["sr"], run["new_freq"])
    want = np.zeros((rows, N), dtype=np.float32)
    n = min(N, y.shape[1])
    want[:, :n] = y[:, :n].astype(np.float32)
    got = d["out"]
    bound = np.spacing(np.maximum(np.abs(want), np.float32(2.0 ** -24))).astype(np.float64)
    err = np.abs(got.astype(np.float64) - want.astype(np.float64))
    assert _ratio("resampler", run["name"], err, bound) <= 1.0
    assert not got[:, n:].any(), "the zero padding past the resampled length"


@pytest.mark.parametrize("name", BATCHED)
def test_batched_rows_equal_rows_alone(name):
    _, rows, N, sr, new_freq, rate, n_fft, hop = next(c for c in CASES if c[0] == name)
    x = signal(name, rows, N, sr)
    many = AB.pitch_run(x, sr, new_freq, n_fft, hop, rate)
    for r in range(rows):
        one = AB.pitch_run(x[r:r + 1], sr, new_freq, n_fft, hop, rate)
        for k in ("out", "spec", "stretched", "frames", "y"):
            if one[k] is not None:
                assert torch.equal(many[k][r], one[k][0]), (name, r, k)


@pytest.mark.parametrize("i", range(len(END_TO_END)), ids=[f"{sr}_{s}_{n}_{h}" for sr, s, n, h in END_TO_END])
def test_end_to_end(i):
    from vampnet_b200.pitch import pitch_shift
    x, shift, sr, n_fft, hop = e2e_case(i)
    want, cond = po.pitch_shift(x, shift, sr, n_fft=n_fft, hop_length=hop)
    assert cond > COND_MIN, f"conditioning {cond:.2e}"
    kw = dict(n_fft=n_fft, hop_length=hop) if n_fft else {}
    got = pitch_shift(torch.from_numpy(x).cuda(), shift, sr, **kw).cpu().numpy().astype(np.float64)
    err = float(np.abs(got - want).max())
    key = f"end to end {sr} Hz"
    if err >= _worst.get(key, (-1.0, ""))[0]:
        _worst[key] = (err, f"shift {shift}, n_fft {n_fft or 'default'}")
    assert err <= ATOL, f"max |device - oracle| = {err:.3e}"


def test_report_worst_ratio():
    """Runs last in this file: the worst error-to-bound ratio per stage, and the worst end-to-end error per sample
    rate."""
    for stage, (v, name) in sorted(_worst.items()):
        kind = "max |device - oracle|" if stage.startswith("end to end") else "worst error / bound"
        print(f"\npitch ops: {stage}: {kind} {v:.3e} ({name})", end="")
    print()
