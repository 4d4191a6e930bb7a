"""float64 oracle of the rate conversion generate_gesture applies to a WAV that is not 16 kHz (zeggs_resample, csrc/resample.cu).

It restates what the reference gets back from SoX (audio_files.py:52-78, 115-146: `rate -h 16000`, `channels 1`, 32-bit output):
decode as SoX does, average the channels, filter with the given prototype h (gain L, centre tap (len(h) - 1) / 2, zero delay)
as a direct sum over the input samples, n_out = floor(n_in * L / M + 1/2), clamp to [-1, 1].  The 2^-31 output quantisation is
not reproduced.
"""
import numpy as np


def decode(pcm):
    """[n] or [n, C] PCM as scipy.io.wavfile.read returns it -> float64 mono [n]."""
    x = np.asarray(pcm)
    if x.dtype == np.float64:
        x = x.astype(np.float32)                    # the host casts float64 files to float32 before the upload
    if x.dtype == np.int16:
        y = x / 32768.0
    elif x.dtype == np.int32:
        y = x / 2147483648.0
    elif x.dtype == np.uint8:
        y = (x.astype(np.float64) - 128.0) / 128.0  # SoX's unsigned 8-bit conversion
    elif x.dtype == np.float32:
        y = np.clip(x.astype(np.float64), -1.0, 1.0)   # SoX clips float input when it converts it to integer samples
    else:
        raise TypeError(f"unsupported PCM dtype {x.dtype}")
    return y.mean(axis=1) if y.ndim == 2 else y


def n_out(n_in, L, M):
    return (2 * int(n_in) * L + M) // (2 * M)


def resample(pcm, h, L, M, chunk=1 << 16):
    """y[j] = sum_i x[i] h[j M + D - i L], D = (len(h) - 1) / 2, over 0 <= i < n_in; clamped to [-1, 1]."""
    x = decode(pcm)
    n_in, N = len(x), len(h)
    D = (N - 1) // 2
    K = -(-N // L)
    hp = np.zeros(K * L)                             # taps past the end of h are zero
    hp[:N] = h
    xp = np.concatenate([np.zeros(K), x, np.zeros(D // L + 2)])   # input outside [0, n_in) is zero
    y = np.zeros(n_out(n_in, L, M))
    for j0 in range(0, len(y), chunk):
        t = np.arange(j0, min(j0 + chunk, len(y)), dtype=np.int64) * M + D
        top, p = t // L + K, t % L
        acc = np.zeros(len(t))
        for q in range(K):
            acc += hp[p + q * L] * xp[top - q]
        y[j0:j0 + len(t)] = acc
    return np.clip(y, -1.0, 1.0)
