"""Cases and a restatement of the loudness meter (csrc/loudness.cu, zeggs_loudness_gain, audio.LoudnessMeter).

* The reference for every comparison is oracle/loudness_oracle.py: pyloudnorm 0.1.0 restated in float64, rounding to float32
  where the package does (after each biquad, into the float32 channel buffer).
* `meter`: a numpy/scipy restatement of the kernel's own scheme: the segment geometry built as the host builds it, each segment
  filtered from a zero state `warm` samples early (float64 biquads, float32 rounding after each stage), segment energies summed
  into block energies, the absolute and the relative gate.  Its output is rounded to float32 like the kernel's.  It sets the
  bounds (tests/test_loudness_f64_cpu.py), and with `fault` it models kernel mistakes the bounds must reject.
* Signals: the speech-like synth.make_waveforms, white noise, a 38 Hz tone on a DC offset of 0.5 (the high pass's largest
  start-up transient: the worst case for the warm-up), a 1.5 kHz tone (the shelf), a full-scale clipped square, a loud burst in
  near-silence (the relative gate drops most blocks), alternating sections at -62 and -71 LUFS (the relative threshold falls
  below -70 LUFS, so the `l > -70` term of the second pass decides which blocks count), an all-zero clip and a clip wholly
  below the absolute gate.
* The kernel returns LUFS in float32: at |L| near 64 half an ulp is 3.8e-6 LU, so the cases keep finite loudness above -64 LUFS
  and the 1e-5 LU bound measures the meter, not the output format.
"""
import numpy as np
from scipy import signal

from oracle import loudness_oracle as lo

T_G, STEP = 0.4, 0.25

# bounds (tests/test_loudness_f64_cpu.py prints the restatement's and each fault's ratio to each)
LUFS_TOL = 1e-5                  # |L - L_ref| in LU, where L_ref is finite
GAIN_RTOL = 2e-6                 # |g - g_ref| / g_ref: 1e-5 LU is 1.15e-6 in gain; the rest covers rounding g to float32

FAULTS = {
    "warm0": "each segment filtered from a zero state at its own start (warm = 0)",
    "seg_off_by_one": "every interior segment bound one sample early",
    "no_clamp": "the last block not clamped to the clip (it reads on into the next clip)",
    "clamped_len": "a block energy divided by its clamped length instead of 0.4 s * rate",
    "no_abs_in_rel": "the l > -70 term dropped from the relative pass",
    "i16_32767": "int16 PCM decoded as x / 32767",
}


# ---------------------------------------------------------------------------------------------- geometry
def n_blocks(n, rate):
    return int(np.round(((n / rate - T_G) / (T_G * STEP))) + 1)


def samples_for_blocks(nb, rate=16000):
    """The clip length that gives exactly nb gating blocks (a whole number of hops past the first block)."""
    return int(T_G * rate) + int(T_G * STEP * rate) * (nb - 1)


def block_samples(n, rate, clamp=True):
    """(lo, hi) sample bounds of every block, as the host computes them (pyloudnorm's float64 expressions, hi clamped to n)."""
    nb = n_blocks(n, rate)
    lo_ = [int(T_G * (j * STEP) * rate) for j in range(nb)]
    hi_ = [int(T_G * (j * STEP + 1) * rate) for j in range(nb)]
    if clamp:
        hi_ = [min(h, n) for h in hi_]
    return np.array(lo_, dtype=np.int64), np.array(hi_, dtype=np.int64)


def geometry(n, rate, fault=None):
    """-> (segment bounds [n_seg + 1], block -> first segment [nb], block -> one past its last segment [nb]): the tables
    LoudnessMeter._geometry hands to the kernel."""
    lo_, hi_ = block_samples(n, rate, clamp=fault != "no_clamp")
    bounds = np.array(sorted(set(lo_.tolist()) | set(hi_.tolist())), dtype=np.int64)
    index = {int(b): i for i, b in enumerate(bounds)}
    blo = np.array([index[int(x)] for x in lo_], dtype=np.int64)
    bhi = np.array([index[int(x)] for x in hi_], dtype=np.int64)
    if fault == "seg_off_by_one":
        bounds = bounds.copy()
        bounds[1:-1] -= 1
    return bounds, blo, bhi


# ---------------------------------------------------------------------------------------------- the kernel's scheme
def decode(x, fault=None):
    """The samples as the kernel loads them: float32, or int16 PCM * (1 / 32768) in float32."""
    x = np.asarray(x)
    if x.dtype == np.int16:
        return x.astype(np.float32) * np.float32(1.0 / (32767.0 if fault == "i16_32767" else 32768.0))
    return x.astype(np.float32)


def segment_energies(x, rate, bounds, warm):
    """float64 energy of every segment of the K-weighted float32 signal x [n'] (n' may run past the last bound's clip when a
    fault reads on): each segment filtered from a zero state at max(0, s0 - warm).  Segments of equal filtered length go through
    scipy's lfilter together."""
    (b1, a1), (b2, a2) = lo.k_weighting(rate)
    s0, s1 = bounds[:-1], bounds[1:]
    start = np.maximum(s0 - warm, 0)
    e = np.zeros(len(s0))
    xd = x.astype(np.float64)
    length = s1 - start
    for L in np.unique(length):
        same = np.nonzero(length == L)[0]
        for idx in np.array_split(same, -(-len(same) // 256)):          # 256 rows at a time: bounded memory on long clips
            rows = xd[start[idx, None] + np.arange(L)[None, :]]
            ya = signal.lfilter(b1, a1, rows, axis=1).astype(np.float32).astype(np.float64)
            yb = signal.lfilter(b2, a2, ya, axis=1).astype(np.float32).astype(np.float64)
            keep = np.arange(L)[None, :] >= (s0[idx] - start[idx])[:, None]
            e[idx] = np.sum(np.where(keep, yb * yb, 0.0), axis=1)
    return e


def meter(x, rate, fault=None, next_clip=None):
    """-> (LUFS, gain to -20 LUFS), both float32, of one clip x [n] (float32 or int16) through the kernel's scheme.
    next_clip: what lies after x in the batch (the no_clamp fault reads it; zeros when absent)."""
    xf = decode(x, fault)
    n = len(xf)
    if n < T_G * rate:
        raise ValueError("Audio must have length greater than the block size.")
    bounds, blo, bhi = geometry(n, rate, fault)
    if bounds[-1] > n:
        tail = np.zeros(bounds[-1] - n, dtype=np.float32)
        if next_clip is not None:
            nx = decode(next_clip, fault)[:len(tail)]
            tail[:len(nx)] = nx
        xf = np.concatenate([xf, tail])
    warm = 0 if fault == "warm0" else int(0.3 * rate)
    se = segment_energies(xf, rate, bounds, warm)
    if fault == "clamped_len":
        lo_, hi_ = block_samples(n, rate)
        inv = 1.0 / (hi_ - lo_).astype(np.float64)
    else:
        inv = np.full(len(blo), 1.0 / (T_G * rate))
    z = np.array([np.sum(se[a:b]) for a, b in zip(blo, bhi)]) * inv
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        l = -0.691 + 10.0 * np.log10(z)
        za = np.mean(z[l >= -70.0]) if np.any(l >= -70.0) else np.nan
        gamma_r = -0.691 + 10.0 * np.log10(za) - 10.0
        sel = (l > gamma_r) if fault == "no_abs_in_rel" else ((l > gamma_r) & (l > -70.0))
        zr = np.mean(z[sel]) if np.any(sel) else 0.0
        lufs = -0.691 + 10.0 * np.log10(zr)
        gain = np.power(10.0, (-20.0 - lufs) / 20.0)
    return np.float32(lufs), np.float32(gain)


def oracle(x, rate):
    """-> (LUFS, gain) of oracle/loudness_oracle.py on the samples the kernel decodes from x (float64 results)."""
    xf = decode(x)
    L = lo.integrated_loudness(xf, rate)
    with np.errstate(over="ignore"):
        return L, float(np.power(10.0, (-20.0 - L) / 20.0))


def ratio(lufs, gain, L_ref, g_ref):
    """Worst ratio of (lufs, gain) to the bounds against (L_ref, g_ref).  Where the reference is -inf (nothing passes the
    absolute gate) the answer must be L = -inf and g = +inf exactly: 0 if so, inf if not."""
    lufs, gain = float(lufs), float(gain)
    if not np.isfinite(L_ref):
        return 0.0 if (lufs == L_ref and gain == np.inf) else np.inf
    if not (np.isfinite(lufs) and np.isfinite(gain)):
        return np.inf
    return max(abs(lufs - L_ref) / LUFS_TOL, abs(gain - g_ref) / (GAIN_RTOL * g_ref))


# ---------------------------------------------------------------------------------------------- signals
def _scaled_to(x, rate, target):
    """x scaled so that its oracle loudness is `target` LUFS."""
    L = lo.integrated_loudness(x.astype(np.float32), rate)
    return (x * 10.0 ** ((target - L) / 20.0)).astype(np.float32)


def white(n, seed, scale=0.1):
    return (scale * np.random.RandomState(seed).randn(n)).astype(np.float32)


def tone(n, rate, f, amp=0.3, offset=0.0, phase=0.4):
    return (offset + amp * np.sin(2.0 * np.pi * f * np.arange(n) / rate + phase)).astype(np.float32)


def square(n, rate, f=220.0):
    """Full scale: +-1 with 30 % of the samples driven past it and clipped."""
    return np.clip(1.3 * np.sign(np.sin(2.0 * np.pi * f * np.arange(n) / rate + 0.1)), -1.0, 1.0).astype(np.float32)


def burst(n, rate, seed):
    """Near-silence at about -65 LUFS with one 0.9 s burst at about -10 LUFS starting on a segment bound (0.1 s * rate)."""
    x = white(n, seed, 4e-4)
    a = int(T_G * STEP * rate) * max(1, (n // int(T_G * STEP * rate)) // 3)
    b = min(n, a + int(0.9 * rate))
    x[a:b] = white(b - a, seed + 1, 0.3)
    return x


def gate_sections(n, rate, seed, loud=-62.0, quiet=-71.0, sec=1.0):
    """Alternating sections of noise at `loud` and `quiet` LUFS.  The absolutely gated mean sits near -62 LUFS, so the relative
    threshold is near -72 LUFS: below -70, and the quiet blocks pass it but not the absolute term of the second pass."""
    m = int(sec * rate)
    base = white(2 * m, seed, 1.0)
    a, b = _scaled_to(base[:m], rate, loud), _scaled_to(base[m:], rate, quiet)
    reps = -(-n // (2 * m))
    return np.tile(np.concatenate([a, b]), reps)[:n].copy()


def below_gate(n, rate, seed):
    """Noise at about -80 LUFS: not zero, but no block reaches the absolute gate."""
    return white(n, seed, 3e-5)


def speech(n, rate, seed):
    from zeggs_b200 import synth
    return synth.make_waveforms(1, n, seed=seed)[0]


CONTENTS = ["speech", "white", "tone38_dc", "tone1500", "square", "burst", "gate_sections", "zeros", "below_gate", "const1e-5"]


def content(kind, n, rate, seed=0):
    if kind == "speech":
        return speech(n, rate, seed)
    if kind == "white":
        return white(n, seed)
    if kind == "tone38_dc":
        return tone(n, rate, 38.0, 0.3, 0.5)
    if kind == "tone1500":
        return tone(n, rate, 1500.0, 0.2)
    if kind == "square":
        return square(n, rate)
    if kind == "burst":
        return burst(n, rate, seed)
    if kind == "gate_sections":
        return gate_sections(n, rate, seed)
    if kind == "zeros":
        return np.zeros(n, dtype=np.float32)
    if kind == "below_gate":
        return below_gate(n, rate, seed)
    if kind == "const1e-5":
        return np.full(n, 1e-5, dtype=np.float32)
    raise ValueError(kind)


def batch(n_clips, n, rate, seed=0):
    """[n_clips, n] float32 cycling through CONTENTS, each clip scaled by its own factor (1 / 8 .. 1) so no two are alike."""
    out = np.empty((n_clips, n), dtype=np.float32)
    for i in range(n_clips):
        k = CONTENTS[i % len(CONTENTS)]
        s = 1.0 if k in ("gate_sections", "below_gate", "const1e-5", "zeros") else 2.0 ** (-(i % 4))
        out[i] = content(k, n, rate, seed + i) * np.float32(s)
    return out


def to_pcm16(x):
    return np.clip(np.round(np.asarray(x, dtype=np.float64) * 32768.0), -32768, 32767).astype(np.int16)


# ---------------------------------------------------------------------------------------------- lengths and rates
def clamped_length(rate, nb=28):
    """A length whose block count rounds up, so the last block ends 0.4375 of a hop past the clip and is clamped to it."""
    return int(T_G * rate) + int(T_G * STEP * rate) * (nb - 2) + int(0.5625 * T_G * STEP * rate)


TOO_SHORT = 6399                                                # one sample short of a block at 16 kHz: refused
LEN_16K = [6400, 6401, 7999, 8000, 8001, 48123, clamped_length(16000), 160000, 960000]   # (T - 0.4) / 0.1 rounds up at 7999
BLOCK_COUNTS = [5952, 5953, 6000, 6001]                         # around 48 KB of doubles per block and the former 6000 cap
MIN_20 = 20 * 60 * 16000
# 11025 Hz has 1102.5 samples per hop: int() truncation makes the segments alternate between 1102 and 1103 samples
OTHER_RATES = [8000, 11025, 22050, 44100, 48000]


def rate_lengths(rate):
    """One block exactly, one block plus one sample, a clamped ragged length and 10 s."""
    return [int(T_G * rate), int(T_G * rate) + 1, clamped_length(rate), 10 * rate]
