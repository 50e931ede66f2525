"""TEST INFRASTRUCTURE — independent CPU restatement of the audio preprocessing either side of the hot path
(reference interface.py:206-217: resample -> mono -> normalize(-24 LUFS) -> ensure_max_of_audio; app.py:175-178, 247-248).

The reference delegates this to ``descript-audiotools`` (third-party, unpinned, absent from the original project's checkout and from the
image: PARITY UNPINNED against it).  What can be pinned is the published standard the library implements:

  * loudness: ITU-R BS.1770-4 integrated loudness — the two K-weighting biquads with the coefficients TABULATED IN THE
    STANDARD for 48 kHz, applied in the time domain (scipy.signal.lfilter), 400 ms blocks with 75 % overlap, absolute
    gate -70 LUFS, relative gate -10 LU, plain Python loops.  The product (vampnet_b200/audio.py) filters in the
    frequency domain with coefficients re-derived for any sample rate and gates with batched tensor ops; agreement of
    the two at 48 kHz pins both the derivation and the vectorised gating.
  * resampling: scipy.signal.resample_poly (another polyphase Kaiser design) — agreement inside the pass band.
Only tests/ may import this file."""
import numpy as np
from scipy import signal

# BS.1770-4, table 1 and 2 (48 kHz)
PRE_B = [1.53512485958697, -2.69169618940638, 1.19839281085285]
PRE_A = [1.0, -1.69065929318241, 0.73248077421585]
RLB_B = [1.0, -2.0, 1.0]
RLB_A = [1.0, -1.99004745483398, 0.99007225036621]


def integrated_loudness_48k(x: np.ndarray) -> float:
    """x: (channels, samples) at 48 kHz -> LUFS (channels weighted 1.0; surround weights not needed for mono/stereo)."""
    assert x.ndim == 2
    sr, blk, hop = 48000, int(0.4 * 48000), int(0.1 * 48000)
    y = signal.lfilter(RLB_B, RLB_A, signal.lfilter(PRE_B, PRE_A, x.astype(np.float64), axis=-1), axis=-1)
    n_blocks = (y.shape[-1] - blk) // hop + 1
    z = np.array([[np.mean(y[c, j * hop:j * hop + blk] ** 2) for j in range(n_blocks)] for c in range(y.shape[0])])
    zsum = z.sum(0)
    lj = -0.691 + 10 * np.log10(np.maximum(zsum, 1e-12))
    keep = lj > -70.0
    if not keep.any():
        return -70.0
    rel = -0.691 + 10 * np.log10(zsum[keep].mean()) - 10.0
    keep2 = keep & (lj > rel)
    if not keep2.any():
        return -70.0
    return max(-70.0, float(-0.691 + 10 * np.log10(zsum[keep2].mean())))


def resample_poly(x: np.ndarray, sr_in: int, sr_out: int) -> np.ndarray:
    g = np.gcd(sr_in, sr_out)
    return signal.resample_poly(x.astype(np.float64), sr_out // g, sr_in // g, axis=-1)
