"""Mel front end on the GPU -- host-side mirror of the reference's audio feature API.

Mirrors (same names / argument meaning):
  ZEGGS/audio/spectrograms.py:8-54   extract_mel_spectrogram_for_tts
  ZEGGS/data_pipeline.py:33-84       preprocess_audio
The arithmetic runs in `zeggs_mel_forward` (csrc/mel.cu); this file only builds the small
constant tables (Hann window, FFT twiddles, sparse Slaney filterbank) in float64 on the host
and moves buffers.  No CPU fallback.
"""
import math

import numpy as np
import torch

from . import _lib


def _hz_to_mel(f):  # spectrograms.py:446-473
    f = np.asarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz, min_log_mel, log_step = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-300) / min_log_hz) / log_step, f / f_sp)


def _mel_to_hz(m):  # spectrograms.py:476-503
    m = np.asarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz, min_log_mel, log_step = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(log_step * (m - min_log_mel)), f_sp * m)


def mel_filterbank(n_fft, fs, n_mels, fmin, fmax, normalize=True):
    """Slaney filterbank [n_mels, n_fft//2+1] (spectrograms.py:386-443)."""
    if fmax is None:
        fmax = fs / 2.0
    nb = 1 + n_fft // 2
    fft_freqs = np.linspace(0, fs / 2.0, nb)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fft_freqs[None, :]
    w = np.zeros((n_mels, nb))
    for i in range(n_mels):
        w[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    if normalize:
        w *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return w


class MelFrontEnd:
    """Device-resident tables + launcher for one audio configuration (data_pipeline_conf.audio_conf)."""

    def __init__(self, device, sampling_rate=16000, filter_length=800, hop_length=200, n_mel_channels=80,
                 mel_fmin=20, mel_fmax=7600, min_clipping=1e-5, real_amplitude=True, normalize_mel_bins=True):
        self.device = torch.device(device)
        self.fs, self.n_fft, self.hop, self.n_mels = sampling_rate, filter_length, hop_length, n_mel_channels
        self.min_amp = float(min_clipping / (filter_length if real_amplitude else 1))   # spectrograms.py:86-88
        n = filter_length
        k = np.arange(n, dtype=np.float64)
        window = 0.5 - 0.5 * np.cos(2.0 * np.pi * k / (n - 1))                           # sps.hann(n), :230
        n2 = n // 2
        a1 = -2.0 * np.pi * np.arange(n2) / n2
        a2 = -2.0 * np.pi * np.arange(n2 + 1) / n
        tw = np.concatenate([np.stack([np.cos(a1), np.sin(a1)], 1), np.stack([np.cos(a2), np.sin(a2)], 1)], 0)
        fb = mel_filterbank(n, sampling_rate, n_mel_channels, mel_fmin, mel_fmax, normalize_mel_bins)
        start, length, off, ws = [], [], [], []
        for i in range(n_mel_channels):
            nz = np.nonzero(fb[i])[0]
            s, e = (int(nz[0]), int(nz[-1]) + 1) if len(nz) else (0, 0)
            start.append(s); length.append(e - s); off.append(len(ws)); ws.extend(fb[i, s:e].tolist())
        dev = self.device
        self.window = torch.tensor(window, dtype=torch.float32, device=dev)
        self.twiddle = torch.tensor(tw, dtype=torch.float32, device=dev).contiguous()
        self.fb_start = torch.tensor(start, dtype=torch.int32, device=dev)
        self.fb_len = torch.tensor(length, dtype=torch.int32, device=dev)
        self.fb_off = torch.tensor(off, dtype=torch.int32, device=dev)
        self.fb_w = torch.tensor(ws if ws else [0.0], dtype=torch.float32, device=dev)

    def num_frames(self, n_samples):
        return _lib.lib().zeggs_mel_num_frames(int(n_samples), self.n_fft, self.hop)

    def forward(self, wav, anim_fs=None, anim_length=None, want_mel=False, want_feat=True, gain=None):
        """wav [N, n_samples] f32 (or int16 PCM) CUDA -> (mel [N, n_mels, L] or None, feat [N, anim_length, n_mels+1] or None).
        gain: optional [N] f32 per-clip factor applied to the samples at load (LoudnessMeter.gain)."""
        if wav.dim() == 1:
            wav = wav[None]
        pcm16 = wav.dtype == torch.int16
        wav = wav.contiguous() if pcm16 else wav.contiguous().float()
        N, ns = wav.shape
        L = self.num_frames(ns)
        mel = torch.empty((N, self.n_mels, L), dtype=torch.float32, device=wav.device) if want_mel else None
        feat = None
        fpa = 0.0
        if want_feat:
            fpa = (self.fs / self.hop) / anim_fs                                           # data_pipeline.py:68
            feat = torch.empty((N, anim_length, self.n_mels + 1), dtype=torch.float32, device=wav.device)
        a = _lib.MelArgs(n_clips=N, n_samples=ns, n_fft=self.n_fft, hop=self.hop, n_mels=self.n_mels,
                         anim_length=int(anim_length or 0), min_amp=self.min_amp, frames_per_anim=float(fpa),
                         wav=None if pcm16 else _lib.ptr(wav), wav_i16=_lib.ptr(wav) if pcm16 else None,
                         gain=None if gain is None else _lib.ptr(gain.contiguous().float()),
                         window=_lib.ptr(self.window), twiddle=_lib.ptr(self.twiddle),
                         fb_start=_lib.ptr(self.fb_start), fb_len=_lib.ptr(self.fb_len), fb_off=_lib.ptr(self.fb_off),
                         fb_w=_lib.ptr(self.fb_w), mel_out=_lib.ptr(mel), feat_out=_lib.ptr(feat), fb_total=int(self.fb_w.numel()))
        _lib.check(_lib.lib().zeggs_mel_forward(a, _lib.stream_ptr()), "zeggs_mel_forward")
        return mel, feat


class LoudnessMeter:
    """BS.1770 integrated loudness and the gain to `target` LUFS per clip, on the device (zeggs_loudness_gain) -- what
    data_pipeline.py:34-39 does with pyloudnorm.  Filter coefficients and gating-block geometry are built here on the host
    in float64 with the package's own expressions (pyloudnorm 0.1.0 IIRfilter.generate_coefficients / integrated_loudness)."""
    T_G, OVERLAP = 0.4, 0.75

    def __init__(self, device, rate=16000, target=-20.0):
        self.device, self.rate, self.target = torch.device(device), int(rate), float(target)
        self.coef = self._k_weighting(self.rate)
        self._geom = {}

    @staticmethod
    def _biquad(G, Q, fc, rate, kind):
        A = 10 ** (G / 40.0)
        w0 = 2.0 * np.pi * (fc / rate)
        alpha = np.sin(w0) / (2.0 * Q)
        c = np.cos(w0)
        if kind == "high_shelf":
            b = [A * ((A + 1) + (A - 1) * c + 2 * np.sqrt(A) * alpha), -2 * A * ((A - 1) + (A + 1) * c),
                 A * ((A + 1) + (A - 1) * c - 2 * np.sqrt(A) * alpha)]
            a = [(A + 1) - (A - 1) * c + 2 * np.sqrt(A) * alpha, 2 * ((A - 1) - (A + 1) * c), (A + 1) - (A - 1) * c - 2 * np.sqrt(A) * alpha]
        else:
            b = [(1 + c) / 2, -(1 + c), (1 + c) / 2]
            a = [1 + alpha, -2 * c, 1 - alpha]
        return [b[0] / a[0], b[1] / a[0], b[2] / a[0], a[1] / a[0], a[2] / a[0]]

    @classmethod
    def _k_weighting(cls, rate):
        return cls._biquad(4.0, 1.0 / np.sqrt(2.0), 1500.0, rate, "high_shelf") + cls._biquad(0.0, 0.5, 38.0, rate, "high_pass")

    def _geometry(self, n_samples):
        g = self._geom.get(n_samples)
        if g is None:
            if n_samples < self.T_G * self.rate:
                raise _lib.ZeggsError("Audio must have length greater than the block size.")          # pyloudnorm util.valid_audio
            step = 1.0 - self.OVERLAP
            T = n_samples / self.rate
            nb = int(np.round(((T - self.T_G) / (self.T_G * step))) + 1)
            lo = [int(self.T_G * (j * step) * self.rate) for j in range(nb)]
            hi = [min(int(self.T_G * (j * step + 1) * self.rate), n_samples) for j in range(nb)]     # numpy slicing clamps at the end
            bounds = sorted(set(lo) | set(hi))
            index = {b: i for i, b in enumerate(bounds)}
            mk = lambda v: torch.tensor(v, dtype=torch.int32, device=self.device)
            g = dict(n_seg=len(bounds) - 1, n_blocks=nb, bounds=mk(bounds), lo=mk([index[x] for x in lo]), hi=mk([index[x] for x in hi]))
            self._geom[n_samples] = g
        return g

    def gain(self, wav, want_lufs=False):
        """wav [N, n_samples] f32 / int16 CUDA -> gain [N] f32 (and the integrated loudness in LUFS)."""
        if wav.dim() == 1:
            wav = wav[None]
        pcm16 = wav.dtype == torch.int16
        wav = wav.contiguous() if pcm16 else wav.contiguous().float()
        N, ns = wav.shape
        g = self._geometry(ns)
        l = _lib.lib()
        wsb = l.zeggs_loudness_workspace_bytes(N, g["n_seg"])
        ws = torch.empty(wsb, dtype=torch.uint8, device=wav.device)
        gain = torch.empty(N, dtype=torch.float32, device=wav.device)
        lufs = torch.empty(N, dtype=torch.float32, device=wav.device)
        a = _lib.LoudnessArgs(n_clips=N, n_samples=ns, n_seg=g["n_seg"], n_blocks=g["n_blocks"], warm=int(0.3 * self.rate),
                              inv_block_len=1.0 / (self.T_G * self.rate), target_lufs=self.target,
                              wav=None if pcm16 else wav.data_ptr(), wav_i16=wav.data_ptr() if pcm16 else None,
                              seg_bounds=g["bounds"].data_ptr(), blk_seg_lo=g["lo"].data_ptr(), blk_seg_hi=g["hi"].data_ptr(),
                              gain_out=gain.data_ptr(), lufs_out=lufs.data_ptr(), workspace=ws.data_ptr(), workspace_bytes=wsb)
        for i, c in enumerate(self.coef):
            a.coef[i] = float(c)
        _lib.check(l.zeggs_loudness_gain(a, _lib.stream_ptr()), "zeggs_loudness_gain")
        return (gain, lufs) if want_lufs else gain


RESAMPLE_ATTEN_DB = 125.5        # Kaiser design attenuation: the measured stopband then stays below -124 dB in fp32 at every rate
RESAMPLE_MAX_L = 1024
PCM_DTYPES = {np.dtype(np.int16): 0, np.dtype(np.int32): 1, np.dtype(np.uint8): 2, np.dtype(np.float32): 3}   # zeggs_resample_args.dtype


def resample_ratio(fs_in, fs_out=16000):
    """(L, M) with L / M = fs_out / fs_in in lowest terms; a ZeggsError names the rate when L > RESAMPLE_MAX_L."""
    fs_in, fs_out = int(fs_in), int(fs_out)
    if fs_in <= 0 or fs_out <= 0:
        raise _lib.ZeggsError(f"cannot resample {fs_in} Hz audio to {fs_out} Hz")
    g = math.gcd(fs_in, fs_out)
    L, M = fs_out // g, fs_in // g
    if L > RESAMPLE_MAX_L:
        raise _lib.ZeggsError(f"cannot resample {fs_in} Hz audio to {fs_out} Hz: the rate ratio reduces to {L}/{M} and the "
                              f"polyphase filter supports at most {RESAMPLE_MAX_L} phases")
    return L, M


def resampled_length(n_in, fs_in, fs_out=16000):
    """floor(n_in * fs_out / fs_in + 0.5) in exact integers: the length SoX's rate effect flushes (samples_in / factor + .5)."""
    return (2 * int(n_in) * int(fs_out) + int(fs_in)) // (2 * int(fs_in))


def design_resampler(fs_in, fs_out=16000, atten_db=RESAMPLE_ATTEN_DB):
    """Linear-phase Kaiser-windowed sinc prototype at rate L * fs_in, float64, gain L (SoX `rate -h` parameters: passband to
    0.95 f_N, stopband from f_N = min(fs_in, fs_out) / 2, ~125 dB rejection).  Length from the Kaiser formula, rounded up to a
    multiple of L and made odd, so the filter is symmetric about its centre tap (n - 1) / 2.  Returns (h, L, M)."""
    L, M = resample_ratio(fs_in, fs_out)
    F = float(L * int(fs_in))
    f_n = min(int(fs_in), int(fs_out)) / 2.0
    f_pass, f_stop = 0.95 * f_n, f_n
    fc = 0.5 * (f_pass + f_stop)
    dw = 2.0 * np.pi * (f_stop - f_pass) / F
    n = int(math.ceil((atten_db - 7.95) / (2.285 * dw))) + 1
    n = -(-n // L) * L
    n += 1 - n % 2
    beta = 0.1102 * (atten_db - 8.7)
    k = np.arange(n, dtype=np.float64) - (n - 1) / 2.0
    h = L * (2.0 * fc / F) * np.sinc((2.0 * fc / F) * k) * np.kaiser(n, beta)
    return h, L, M


def polyphase_table(h, L):
    """Prototype h -> fp32 table [L, K4] with table[p, q] = h[p + q L] (zero past the end), K4 = ceil(len(h) / L) rounded up to 4."""
    K = -(-len(h) // L)
    K4 = -(-K // 4) * 4
    hp = np.zeros(L * K4, dtype=np.float64)
    hp[:len(h)] = h
    return np.ascontiguousarray(hp.reshape(K4, L).T.astype(np.float32)), K


class Resampler:
    """Rate conversion of raw WAV PCM to fs_out (zeggs_resample): decode as SoX does, average the channels, polyphase FIR with
    the design_resampler prototype, clamp to [-1, 1].  The polyphase table is built on the host in float64 and kept on the device."""

    def __init__(self, device, fs_in, fs_out=16000):
        self.device = torch.device(device)
        self.fs_in, self.fs_out = int(fs_in), int(fs_out)
        self.h, self.L, self.M = design_resampler(fs_in, fs_out)
        self.delay = (len(self.h) - 1) // 2
        table, self.K = polyphase_table(self.h, self.L)
        self.table = torch.from_numpy(table).to(self.device)

    def __call__(self, pcm):
        """pcm [n] or [n, C] (numpy or torch; int16, int32, uint8, float32 or float64) -> float32 [n_out] on the device."""
        if isinstance(pcm, np.ndarray):
            x = pcm.astype(np.float32) if pcm.dtype == np.float64 else pcm
            if x.dtype not in PCM_DTYPES:
                raise _lib.ZeggsError(f"unsupported PCM sample type {x.dtype}")
            x = torch.from_numpy(np.ascontiguousarray(x))
        else:
            x = pcm.float() if pcm.dtype == torch.float64 else pcm
        code = {torch.int16: 0, torch.int32: 1, torch.uint8: 2, torch.float32: 3}.get(x.dtype)
        if code is None:
            raise _lib.ZeggsError(f"unsupported PCM sample type {x.dtype}")
        if x.dim() == 1:
            x = x[:, None]
        if x.dim() != 2 or x.shape[1] < 1:
            raise _lib.ZeggsError(f"PCM must be [n_samples] or [n_samples, channels], got {tuple(x.shape)}")
        if not x.is_cuda:
            x = x.contiguous().pin_memory().to(self.device, non_blocking=True)
        x = x.contiguous()
        n_in, C = x.shape
        n_out = resampled_length(n_in, self.fs_in, self.fs_out)
        out = torch.empty(n_out, dtype=torch.float32, device=x.device)
        a = _lib.ResampleArgs(n_in=n_in, n_out=n_out, channels=C, dtype=code, L=self.L, M=self.M, K4=int(self.table.shape[1]),
                              delay=self.delay, pcm=_lib.ptr(x), taps=_lib.ptr(self.table), out=_lib.ptr(out))
        _lib.check(_lib.lib().zeggs_resample(a, _lib.stream_ptr()), "zeggs_resample")
        return out


_cache = {}
_meters = {}
_resamplers = {}


def resample(pcm, fs_in, fs_out=16000, device="cuda"):
    """Raw WAV PCM at fs_in ([n] or [n, C], as scipy.io.wavfile.read returns it) -> float32 [n_out] CUDA tensor at fs_out: what
    the reference's read_wavfile(..., desired_fs=16000) gets back from SoX (audio_files.py:52-78, 115-146)."""
    key = (str(torch.device(device)), int(fs_in), int(fs_out))
    if key not in _resamplers:
        _resamplers[key] = Resampler(device, fs_in, fs_out)
    return _resamplers[key](pcm)


def _meter(device, rate):
    key = (str(device), int(rate))
    if key not in _meters:
        _meters[key] = LoudnessMeter(device, rate)
    return _meters[key]


def _front_end(device, **kw):
    key = (str(device),) + tuple(sorted(kw.items()))
    if key not in _cache:
        _cache[key] = MelFrontEnd(device, **kw)
    return _cache[key]


def _conf_kwargs(params):
    g = (lambda k: params[k]) if isinstance(params, dict) else (lambda k: getattr(params, k))
    if g("pre_emphasis"):
        raise _lib.ZeggsError("pre_emphasis=True is not on the accelerated path (shipped confs use False)")
    if not (g("centered") and g("normalize_range") and g("resample_method") == "linear"):
        raise _lib.ZeggsError("only centered / normalize_range / linear resampling (the shipped audio_conf) is supported")
    return dict(sampling_rate=g("sampling_rate"), filter_length=g("filter_length"), hop_length=g("hop_length"),
                n_mel_channels=g("n_mel_channels"), mel_fmin=g("mel_fmin"), mel_fmax=g("mel_fmax"),
                min_clipping=g("min_clipping"), real_amplitude=g("real_amplitude"),
                normalize_mel_bins=g("normalize_mel_bins"))


def preprocess_audio(audio_data, anim_fs, anim_length, params, feature_type, device="cuda"):
    """Drop-in for data_pipeline.preprocess_audio (data_pipeline.py:33-84): numpy/torch [T] (or [N,T]) in,
    float32 [anim_length, 81] (numpy for numpy input, CUDA tensor for tensor input) out.  int16 PCM input is decoded on the
    device (x / 32768).  params.normalize_loudness (:34-39): BS.1770 integrated loudness -> gain to -20 LUFS, measured by
    zeggs_loudness_gain and folded into the mel kernel's sample load."""
    nl = params["normalize_loudness"] if isinstance(params, dict) else getattr(params, "normalize_loudness", False)
    if list(feature_type) != ["mel_spec", "energy"]:
        raise _lib.ZeggsError("feature_type must be ['mel_spec', 'energy'] (the shipped audio_feature_type)")
    as_numpy = isinstance(audio_data, np.ndarray)
    wav = torch.as_tensor(audio_data)
    if wav.dtype != torch.int16:
        wav = wav.to(torch.float32)
    if not wav.is_cuda:
        wav = wav.pin_memory().to(device, non_blocking=True) if (as_numpy and torch.cuda.is_available()) else wav.to(device)
    kw = _conf_kwargs(params)
    fe = _front_end(wav.device, **kw)
    gain = _meter(wav.device, kw["sampling_rate"]).gain(wav) if nl else None
    _, feat = fe.forward(wav, anim_fs, anim_length, want_mel=False, want_feat=True, gain=gain)
    if wav.dim() == 1 or (as_numpy and np.ndim(audio_data) == 1):
        feat = feat[0]
    return feat.cpu().numpy() if as_numpy else feat


def extract_mel_spectrogram_for_tts(wav_signal, fs, n_fft, step_size, n_mels, mel_fmin, mel_fmax, min_amplitude,
                                    pre_emphasis=True, pre_emph_coeff=0.97, dynamic_range=None, real_amplitude=True,
                                    centered=True, normalize_mel_bins=True, normalize_range=True, logger=None,
                                    device="cuda"):
    """Drop-in for spectrograms.extract_mel_spectrogram_for_tts (spectrograms.py:8-54) -> (mel[n_mels, L], wav)."""
    if pre_emphasis or dynamic_range or not (centered and normalize_range and min_amplitude):
        raise _lib.ZeggsError("unsupported option combination (accelerated path = the shipped audio_conf)")
    as_numpy = isinstance(wav_signal, np.ndarray)
    wav = torch.as_tensor(wav_signal, dtype=torch.float32).to(device)
    fe = _front_end(wav.device, sampling_rate=fs, filter_length=n_fft, hop_length=step_size, n_mel_channels=n_mels,
                    mel_fmin=mel_fmin, mel_fmax=mel_fmax, min_clipping=min_amplitude, real_amplitude=real_amplitude,
                    normalize_mel_bins=normalize_mel_bins)
    mel, _ = fe.forward(wav, want_mel=True, want_feat=False)
    mel = mel[0]
    return (mel.cpu().numpy() if as_numpy else mel), wav_signal
