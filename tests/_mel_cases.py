"""Cases and oracles for the mel front end (csrc/mel.cu, csrc/mel_fft.cuh) at every shape it accepts.

* Signals: white noise, pure tones exactly on FFT bins and between them, a DC offset, a chirp (consecutive frames differ, so the
  two frames of a pair cannot be swapped unseen), silence (every band at the minimum amplitude) and full-scale int16 PCM.
* `front_end`: a vectorised restatement of the whole front end -- frames gathered through the kernel's own index map (zero
  extension of short clips, reflect padding), a symmetric Hann window, rfft, any sparse filterbank given as the kernel's
  (start, len, off, w) tables, clip -> dB -> [0,1], ln(10^(s/20)), the energy channel and the 60 fps lerp, with per-clip gains
  and the int16 decode (x / 32768).  In float64 it equals oracle/mel_oracle to 1e-12 and is fast enough for long takes; with
  f32=True every step runs in float32 (scipy.fft.rfft on float32 frames, float32 dB arithmetic) and only sets the bounds.
* FAULTS: kernel mistakes, each modelled in the restatement, that the bounds must reject (tests/test_mel_f64_cpu.py).
"""
import numpy as np
import scipy.fft

from oracle import mel_oracle

N_FFT = 800
NB = N_FFT // 2 + 1
LN10_20 = 0.11512925464970229          # ln(10) / 20: m = s * ln(10) / 20 = ln(10^(s/20))
MIN_AMP = 1e-5 / N_FFT                  # the shipped min_clipping / n_fft

# bounds (tests/test_mel_f64_cpu.py prints the float32 restatement's and each fault's ratio to each)
MEL_TOL = 1e-4                          # |s - s_ref|, s in [0, 1]  (the project's mel bound)
FEAT_TOL = 2e-4                         # |feat - feat_ref| on the ln-domain mel + energy features
BIN_MIN_AMP = 1e-15                     # single-bin tables: nothing of interest clips at this minimum amplitude
BIN_TAU = 1e-5                          # per frame: max_k |a - a_ref| <= BIN_TAU * (frame pair's ||w x||_2) / 800 + BIN_RHO * a_ref
BIN_RHO = 4e-5

FAULTS = {
    "pair_swap": "the two frames of a pair swapped",
    "lane0_partner": "lane 0 (bins 25 k) separates with the conjugate partner one 25-bin row off",
    "twiddle_sign": "the twiddle exp(-2 pi i m / 800) not negated for m > 400",
    "symmetric_pad": "symmetric padding instead of reflect",
    "periodic_hann": "a periodic Hann window instead of the symmetric one",
    "no_zero_extend": "short clips reflected at their own end, without zero extension to n_fft first",
    "lerp_tile": "the lerp takes frame i0 + 1 from the start of the tile when i0 is a tile's last frame",
    "energy_from_s": "the energy channel computed from s instead of exp(m)",
    "gain0": "gain[0] applied to every clip",
}

# ---------------------------------------------------------------------------------------------- signals


def white(n, seed, scale=0.3):
    return (scale * np.random.RandomState(seed).randn(n)).astype(np.float32)


def tone(n, k, amp=0.5, phase=0.3):
    """cos at k * fs / 800: exactly on FFT bin k when k is an integer."""
    return (amp * np.cos(2.0 * np.pi * k * np.arange(n) / N_FFT + phase)).astype(np.float32)


def dc(n, seed, offset=0.25):
    return (offset + white(n, seed, 0.05)).astype(np.float32)


def chirp(n, seed, f0=0.003, f1=0.49):
    """Linear chirp from f0 to f1 cycles per sample over the clip, plus a little noise (so no band sinks to float32 noise)."""
    t = np.arange(n, dtype=np.float64)
    ph = 2.0 * np.pi * (f0 * t + 0.5 * (f1 - f0) * t * t / max(n - 1, 1))
    return (0.4 * np.cos(ph) + white(n, seed, 0.1)).astype(np.float32)


def pcm16(n, seed):
    """Full-scale int16 PCM, both extremes included."""
    x = np.random.RandomState(seed).randint(-32768, 32768, size=n).astype(np.int16)
    x[: min(n, 2)] = [-32768, 32767][: min(n, 2)]
    return x


def signal(kind, n, seed):
    if kind == "white":
        return white(n, seed)
    if kind == "chirp":
        return chirp(n, seed)
    if kind == "dc":
        return dc(n, seed)
    if kind == "silence":
        return np.zeros(n, np.float32)
    if kind == "pcm16":
        return pcm16(n, seed)
    if kind == "pcm16_silence":
        return np.zeros(n, np.int16)
    raise ValueError(kind)


BIN_TONES = [1, 24, 25, 26, 199, 200, 375, 380, 399, 400]
OFF_BIN_TONES = [3.5, 123.37, 399.7]


def bin_signals(n):
    """[16, n] f32: the signals of the bin-by-bin test, one per clip."""
    xs = [tone(n, k) for k in BIN_TONES] + [tone(n, k, phase=1.1) for k in OFF_BIN_TONES]
    xs += [white(n, 1), dc(n, 2), chirp(n, 3)]
    return np.stack(xs)


# ---------------------------------------------------------------------------------------------- filterbank tables


def sparse_tables(fb):
    """Dense [n_mels, 401] filterbank -> the kernel's (start, len, off, w) tables, as zeggs_b200.audio.MelFrontEnd builds them."""
    start, length, off, ws = [], [], [], []
    for row in fb:
        nz = np.nonzero(row)[0]
        s, e = (int(nz[0]), int(nz[-1]) + 1) if len(nz) else (0, 0)
        start.append(s); length.append(e - s); off.append(len(ws)); ws.extend(row[s:e].tolist())
    return (np.array(start, np.int32), np.array(length, np.int32), np.array(off, np.int32),
            np.array(ws if ws else [0.0], np.float64))


def slaney_tables(fs, n_mels, fmin, fmax, normalize=True):
    return sparse_tables(mel_oracle.mel_filterbank(N_FFT, fs, n_mels, fmin, fmax, normalize))


def single_bin_tables(bins):
    """Band i = FFT bin bins[i] with weight 1."""
    n = len(bins)
    return (np.asarray(bins, np.int32), np.ones(n, np.int32), np.arange(n, dtype=np.int32), np.ones(n, np.float64))


def wide_tables(n_mels=64, width=80, seed=0):
    """Overlapping random-weight bands of `width` bins: n_mels * width weights (> 4096: the kernel reads them from global memory)."""
    rs = np.random.RandomState(seed)
    start = np.linspace(0, NB - width, n_mels).astype(np.int32)
    return (start, np.full(n_mels, width, np.int32), (np.arange(n_mels) * width).astype(np.int32),
            rs.uniform(0.001, 0.02, n_mels * width))


def dense(tables, dtype=np.float64):
    start, length, off, w = tables
    W = np.zeros((len(start), NB), dtype=np.float64)
    for i, (s, n, o) in enumerate(zip(start, length, off)):
        W[i, s:s + n] += w[o:o + n]
    return W.astype(dtype)


# ---------------------------------------------------------------------------------------------- restatement


def num_frames(n_samples, hop):
    return mel_oracle.num_frames(n_samples, N_FFT, hop)


def max_anim_length(n_samples, hop, fs, anim_fs):
    """The largest anim_length whose last 60 fps row needs no frame past L - 1 (data_pipeline.py:473 asserts no NaNs)."""
    L, fpa = num_frames(n_samples, hop), (fs / hop) / anim_fs
    n = int(np.floor((L - 1) / fpa + 1e-9)) + 1
    while (n - 1) * fpa > (L - 1) + 1e-9:
        n -= 1
    while n * fpa <= (L - 1) + 1e-9:
        n += 1
    return n


def hann(periodic=False):
    k = np.arange(N_FFT, dtype=np.float64)
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * k / (N_FFT if periodic else N_FFT - 1))


def sample_index(n_samples, hop, fault=None, n_frames=None):
    """[n_frames (default L), 800] source sample of every frame tap in the kernel's staging map; -1 reads zero.  Short clips are
    zero-extended to n_fft, then reflect-padded by n_fft / 2 (spectrograms.py:233-239)."""
    L = num_frames(n_samples, hop) if n_frames is None else n_frames
    o = np.arange(L, dtype=np.int64)[:, None] * hop + np.arange(N_FFT)[None, :] - N_FFT // 2
    Ts = n_samples
    Te = Ts if fault == "no_zero_extend" else max(Ts, N_FFT)
    if fault == "symmetric_pad":
        o = np.where(o < 0, -o - 1, o)
        o = np.where(o >= Te, 2 * Te - 1 - o, o)
    else:
        o = np.where(o < 0, -o, o)
        o = np.where(o >= Te, 2 * (Te - 1) - o, o)
    return np.where((o >= 0) & (o < Ts), o, -1)


def decode(x, gain, f32):
    """Samples as the kernel stages them: int16 -> x / 32768, then the per-clip gain."""
    dt = np.float32 if f32 else np.float64
    x = np.asarray(x)
    v = x.astype(dt) * dt(1.0 / 32768.0) if x.dtype == np.int16 else x.astype(dt)
    return v * dt(gain) if gain is not None else v


def frames(x, hop, f32=False, fault=None, gain=None):
    """Windowed frames of one clip, L rounded up to even (the kernel transforms frames in pairs; an odd L's last frame shares its
    transform with frame L, staged by the same map), and each frame's ||w x||_2 / 800 (float64)."""
    v = decode(x, gain, f32)
    L = num_frames(len(v), hop)
    idx = sample_index(len(v), hop, fault, L + L % 2)
    fr = np.concatenate([v, np.zeros(1, v.dtype)])[idx]
    w = hann(fault == "periodic_hann")
    wf = fr * (w.astype(np.float32) if f32 else w)
    return wf, np.linalg.norm(fr.astype(np.float64) * w, axis=1) / N_FFT


def split_fft(z, fault=None):
    """The kernel's 800-point transform, 32 x 25: sample n1 + 32 n2 -> DFT25 over n2, twiddle exp(-2 pi i n1 k2 / 800), DFT32 over
    n1; bin k2 + 25 k1.  twiddle_sign: the table value for m = n1 k2 > 400 is used without its sign flip."""
    A = np.fft.fft(z.reshape(-1, 25, 32), axis=1)                                  # [.., k2, n1]
    m = np.arange(25)[:, None] * np.arange(32)[None, :]
    tw = np.exp(-2j * np.pi * m / N_FFT)
    if fault == "twiddle_sign":
        tw = np.where(m > N_FFT // 2, -tw, tw)
    B = np.fft.fft(A * tw, axis=2)                                                 # [.., k2, k1]
    return B.transpose(0, 2, 1).reshape(-1, N_FFT)


def _paired_amp(wf, f32, fault):
    """Two real frames per complex transform, separated as the kernel does: X_A[k] = (Z[k] + conj Z[p(k)]) / 2, X_B likewise.
    In float32 the transform is scipy's complex64 FFT, so each frame carries the rounding of its pair."""
    if f32:
        Z = scipy.fft.fft((wf[0::2] + np.complex64(1j) * wf[1::2]).astype(np.complex64), axis=1)
    else:
        Z = split_fft(wf[0::2] + 1j * wf[1::2], fault)
    k = np.arange(NB)
    p = (N_FFT - k) % N_FFT
    if fault == "lane0_partner":
        p = np.where(k % 25 == 0, (N_FFT - 25 - k) % N_FFT, p)
    P, Q = Z[:, k], np.conj(Z[:, p])
    half = np.float32(0.5) if f32 else 0.5
    a, b = half * (P + Q), half * (P - Q)                     # X_B = (P - Q) / 2i: the same magnitude
    amp = np.empty((2 * len(Z), NB), dtype=np.float32 if f32 else np.float64)
    amp[0::2], amp[1::2] = np.abs(a), np.abs(b)
    return amp * (np.float32(1.0 / N_FFT) if f32 else 1.0 / N_FFT)


def spectra(x, hop, f32=False, fault=None, gain=None):
    """|rfft(w x)| / 800 per frame [L, 401] of one clip, and the norm of the frame pair each frame shares a transform with,
    sqrt(||w x_2p||^2 + ||w x_2p+1||^2) / 800 [L] (the scale of the transform's rounding error)."""
    wf, nrm = frames(x, hop, f32, fault, gain)
    L = num_frames(len(x), hop)
    if f32 or fault in ("twiddle_sign", "lane0_partner"):
        amp = _paired_amp(wf, f32, fault)[:L]
    else:
        amp = np.abs(np.fft.rfft(wf[:L], axis=1)) / N_FFT
    if fault == "pair_swap":
        n = amp.shape[0] // 2 * 2
        amp[0:n:2], amp[1:n:2] = amp[1:n:2].copy(), amp[0:n:2].copy()
    pair = np.repeat(np.sqrt(nrm[0::2] ** 2 + nrm[1::2] ** 2), 2)[:L]
    return amp, pair


def lerp(y, fpa, anim_length, f32=False, fault=None):
    """Rows of y [L, C] at positions k * fpa (data_pipeline.py:65-80), i0 clamped to [0, L - 2] as the kernel does."""
    L = y.shape[0]
    pos = fpa * np.arange(anim_length)
    i0 = np.clip(np.floor(pos).astype(np.int64), 0, max(L - 2, 0))
    i1 = np.minimum(i0 + 1, L - 1)
    if fault == "lerp_tile":
        i1 = np.where(i0 % 30 == 29, i1 - 30, i1)
    w = (pos - i0)[:, None]
    if f32:
        w = w.astype(np.float32)
    return y[i0] + (y[i1] - y[i0]) * w


def front_end(x, hop, tables, min_amp=MIN_AMP, gain=None, fpa=None, anim_length=None, f32=False, fault=None):
    """x [N, n] f32 or int16 -> (mel [N, n_mels, L], feat [N, anim_length, n_mels + 1] or None), float64 (float32 if f32)."""
    dt = np.float32 if f32 else np.float64
    x = np.asarray(x)
    if x.ndim == 1:
        x = x[None]
    W = dense(tables, dt)
    R = dt(-20.0) * np.log10(dt(min_amp))
    mels, feats = [], []
    for c in range(x.shape[0]):
        g = None if gain is None else gain[0 if fault == "gain0" else c]
        amp, _ = spectra(x[c], hop, f32, fault, g)
        acc = amp.astype(dt) @ W.T                                                  # [L, n_mels]
        v = np.maximum(np.abs(acc), dt(min_amp))
        s = (dt(20.0) * np.log10(v) + R) / R
        mels.append(s.T)
        if fpa is not None:
            m = s * dt(LN10_20)
            e = np.sqrt((s * s if fault == "energy_from_s" else np.exp(m) ** 2).sum(axis=1))
            feats.append(lerp(np.concatenate([m, e[:, None]], axis=1), fpa, anim_length, f32, fault))
    return np.stack(mels), (np.stack(feats) if feats else None)


def _s_of(v, min_amp):
    R = -20.0 * np.log10(min_amp)
    return (20.0 * np.log10(np.maximum(v, min_amp)) + R) / R


def mel_tolerance(x, hop, tables, min_amp=MIN_AMP, gain=None):
    """[N, n_mels, L] bound on |s - s_ref|: MEL_TOL, plus the spread of s over band values within the float32 transform's error
    (per bin BIN_TAU times the pair norm plus BIN_RHO of the bin, summed with the band's weights) of the float64 band value.  The
    spread matters only for a band far below its frame pair's level, such as the last frame of a short clip, which reads little
    but padding under the window's near-zero taps and shares its transform with a full frame."""
    x = np.asarray(x)
    if x.ndim == 1:
        x = x[None]
    W = dense(tables)
    out = []
    for c in range(x.shape[0]):
        amp, pair = spectra(x[c], hop, gain=None if gain is None else gain[c])
        acc = np.abs(amp @ W.T)
        E = BIN_TAU * pair[:, None] * np.abs(W).sum(axis=1)[None, :] + BIN_RHO * (amp @ np.abs(W).T)
        s0 = _s_of(acc, min_amp)
        out.append((MEL_TOL + np.maximum(_s_of(acc + E, min_amp) - s0, s0 - _s_of(acc - E, min_amp))).T)
    return np.stack(out)


def feat_tolerance(mel_ref, mel_tol, fpa, anim_length):
    """[N, anim_length, n_mels + 1] bound on the features: FEAT_TOL plus mel_tolerance's spread carried through m = s ln(10) / 20
    (the larger of the two frames a row interpolates) and, for the energy e = ||exp(m)||_2, through |de| <= e max_b |dm_b|."""
    ex = (mel_tol - MEL_TOL) * LN10_20                                               # [N, n_mels, L]
    e = np.sqrt(np.exp(2.0 * LN10_20 * mel_ref).sum(axis=1))                         # [N, L]
    y = np.concatenate([ex.transpose(0, 2, 1), (e * ex.max(axis=1))[..., None]], axis=2)
    L = y.shape[1]
    i0 = np.clip(np.floor(fpa * np.arange(anim_length)).astype(np.int64), 0, max(L - 2, 0))
    return FEAT_TOL + np.maximum(y[:, i0], y[:, np.minimum(i0 + 1, L - 1)])


# ---------------------------------------------------------------------------------------------- bin-by-bin bound


def amp_from_mel(s, min_amp):
    """Invert s = (20 log10 a + R) / R, R = -20 log10(min_amp): a = 10^((s - 1) R / 20)."""
    R = -20.0 * np.log10(np.float64(np.float32(min_amp)))
    return 10.0 ** ((np.asarray(s, np.float64) - 1.0) * R / 20.0)


def bin_ratio(a, a_ref, nrm):
    """Per frame: max_k |a - a_ref| / (BIN_TAU * nrm + BIN_RHO * a_ref); a, a_ref [L, K], nrm [L] the frame pair's norm."""
    return (np.abs(a - a_ref) / (BIN_TAU * nrm[:, None] + BIN_RHO * a_ref)).max(axis=1)


BIN_HALVES = (list(range(0, 201)), list(range(201, NB)))      # two calls of at most 256 bands cover bins 0..400


def bin_config_lengths(hop):
    """(even-L, odd-L) clip lengths near 6000 samples at this hop."""
    out = {}
    n = 6000
    while len(out) < 2:
        out.setdefault(num_frames(n, hop) % 2, n)
        n += 1
    return out[0], out[1]


BIN_HOPS = [200, 199, 160, 800]

# ---------------------------------------------------------------------------------------------- the shape grid

HOPS = [1, 7, 80, 160, 199, 200, 256, 400, 401, 799, 800]
N_MELS = [1, 31, 32, 33, 80, 128, 256]
CONFS = [(16000, 20, 7600), (16000, 0, 8000), (22050, 20, None), (8000, 20, 4000)]
N_SAMPLES = [401, 402, 799, 800, 801, 12345]
LONG_SAMPLES = 2_400_000
ANIM_FS = [60, 30, 25, 24]
N_CLIPS = [1, 3, 65]
_KINDS = ["white", "chirp", "dc", "silence"]
_MAX_FRAMES = 60000                     # clips x frames per grid case: keeps the float64 restatement to about a second


class Case:
    def __init__(self, cid, hop, n_mels, conf, normalize, n_samples, anim_fs, n_clips, pcm, tables=None):
        self.cid, self.hop, self.n_mels, self.normalize = cid, hop, n_mels, normalize
        self.fs, self.fmin, self.fmax = conf
        self.n_samples, self.anim_fs, self.n_clips, self.pcm = n_samples, anim_fs, n_clips, pcm
        self.L = num_frames(n_samples, hop)
        self.fpa = (self.fs / hop) / anim_fs
        self.anim_length = max_anim_length(n_samples, hop, self.fs, anim_fs)
        self.tables = tables if tables is not None else slaney_tables(self.fs, n_mels, self.fmin, self.fmax, normalize)
        seed = sum(map(ord, cid))
        kinds = ["pcm16", "pcm16_silence"] if pcm else _KINDS
        self.x = np.stack([signal(kinds[i % len(kinds)] if n_clips > 1 else kinds[0], n_samples, seed + i) for i in range(n_clips)])
        self.gain = (np.float32(0.35) + np.float32(0.23) * np.arange(n_clips, dtype=np.float32)) if n_clips > 1 or pcm else None

    def oracle(self, f32=False, fault=None):
        return front_end(self.x, self.hop, self.tables, MIN_AMP, self.gain, self.fpa, self.anim_length, f32, fault)

    def tolerances(self, mel_ref):
        """(mel, feature) bounds of this case, elementwise."""
        tol = mel_tolerance(self.x, self.hop, self.tables, MIN_AMP, self.gain)
        return tol, feat_tolerance(mel_ref, tol, self.fpa, self.anim_length)

    def default_conf(self):
        return (self.fs, self.fmin, self.fmax, self.normalize) == (16000, 20, 7600, True)


def grid():
    """Stratified grid: case i takes the i-th value of each list modulo its length (the periods 11, 7, 8, 6, 4, 3 cover every
    value of each list and many pairs), then the extra cases the grid cannot reach."""
    cases = []
    for i in range(33):
        hop, nm = HOPS[i % 11], N_MELS[i % 7]
        conf, normalize = CONFS[i % 4], (i // 4) % 2 == 0
        ns, afs, N = N_SAMPLES[i % 6], ANIM_FS[(i // 3) % 4], N_CLIPS[i % 3]
        while N > 1 and N * num_frames(ns, hop) > _MAX_FRAMES:
            N = N_CLIPS[N_CLIPS.index(N) - 1]
        cid = f"g{i:02d}_hop{hop}_m{nm}_fs{conf[0]}_{conf[1]}_{conf[2]}{'' if normalize else '_nonorm'}_n{ns}_a{afs}_N{N}"
        cases.append(Case(cid, hop, nm, conf, normalize, ns, afs, N, pcm=(i % 5 == 4)))
    cases += [
        Case("long_2.4M_hop200_m80", 200, 80, CONFS[0], True, LONG_SAMPLES, 60, 1, False),
        Case("L1_hop800_n600_m80", 800, 80, CONFS[0], True, 600, 60, 3, False),
        Case("hop800_m256_fmax8000", 800, 256, CONFS[1], True, 12345, 24, 3, False),
        Case("wide_fb_5120_hop200", 200, 64, CONFS[0], True, 12345, 60, 3, False, tables=wide_tables()),
        Case("n65_hop200_m80_pcm", 200, 80, CONFS[0], True, 4000, 30, 65, True),
    ]
    return cases
