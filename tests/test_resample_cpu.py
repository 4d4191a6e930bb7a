"""Rate conversion to 16 kHz (zeggs_b200.audio.design_resampler / zeggs_resample), host side: the filter meets SoX's `rate -h`
specification when measured, the rate rules, and the float64 oracle against scipy.signal.upfirdn on the same taps."""
import numpy as np
import pytest

from oracle import resample_oracle as ro
from zeggs_b200 import _lib, audio

RATES = [8000, 11025, 22050, 24000, 32000, 44100, 48000, 96000]


def _response_db(h, L, fs_in):
    """|H(f)| / L of a prototype at rate L * fs_in on a long FFT grid -> (passband deviation to 0.95 f_N, stopband peak from f_N, dB)."""
    f_n = min(fs_in, 16000) / 2.0
    nfft = 1 << int(np.ceil(np.log2(len(h) * 16)))
    H = np.abs(np.fft.rfft(h, nfft)) / L
    f = np.arange(len(H)) * (L * fs_in) / nfft
    return float(np.abs(H[f <= 0.95 * f_n] - 1.0).max()), float(20.0 * np.log10(H[f >= f_n].max()))


@pytest.mark.parametrize("fs_in", RATES)
def test_prototype_meets_the_rate_h_specification(fs_in):
    h, L, M = audio.design_resampler(fs_in)
    assert len(h) % 2 == 1 and np.array_equal(h, h[::-1])
    dev, stop = _response_db(h, L, fs_in)
    print(f"  {fs_in} Hz: L/M {L}/{M}, {len(h)} taps, passband deviation {dev:.2e}, stopband {stop:.2f} dB")
    assert dev <= 1e-6 and stop <= -124.0
    table, K = audio.polyphase_table(h, L)
    assert table.dtype == np.float32 and table.shape[0] == L and table.shape[1] % 4 == 0 and K == -(-len(h) // L)
    h32 = table.T.reshape(-1)[:len(h)].astype(np.float64)              # the taps the kernel multiplies by
    assert np.array_equal(h32, h.astype(np.float32).astype(np.float64)) and not table.T.reshape(-1)[len(h):].any()
    _, stop32 = _response_db(h32, L, fs_in)
    print(f"    fp32 table stopband {stop32:.2f} dB")
    assert stop32 <= -124.0


def test_rate_rules():
    assert audio.resample_ratio(48000) == (1, 3)
    assert audio.resample_ratio(44100) == (160, 441)
    assert audio.resample_ratio(11025) == (640, 441)
    assert audio.resample_ratio(8000) == (2, 1)
    assert audio.resample_ratio(192000) == (1, 12)
    assert audio.resample_ratio(176400) == (40, 441)
    for fs in (16001, 15999, 44101, 7):
        with pytest.raises(_lib.ZeggsError, match=str(fs)):
            audio.resample_ratio(fs)
    # n_out = floor(n_in * 16000 / fs_in + 0.5) in exact integers
    for n_in, fs, want in ((48000, 48000, 16000), (1, 48000, 0), (2, 48000, 1), (7, 48000, 2), (44100, 44100, 16000),
                           (1, 44100, 0), (1, 8000, 2), (441, 44100, 160)):
        assert audio.resampled_length(n_in, fs) == want, (n_in, fs)
    # exactly half-way rounds up: 0.5, 1.5 and 2.5 output samples
    assert audio.resampled_length(1, 32000) == 1 and audio.resampled_length(3, 96000) == 1
    assert audio.resampled_length(9, 96000) == 2 and audio.resampled_length(15, 96000) == 3
    rs = np.random.RandomState(0)
    for fs in RATES:
        for n in rs.randint(0, 10 ** 7, size=50):
            assert audio.resampled_length(int(n), fs) == int(np.floor(int(n) * 16000 / fs + 0.5))
            assert audio.resampled_length(int(n), fs) == ro.n_out(int(n), *audio.resample_ratio(fs))


def test_decode_rules():
    assert np.array_equal(ro.decode(np.array([-32768, 0, 16384], np.int16)), [-1.0, 0.0, 0.5])
    assert np.array_equal(ro.decode(np.array([-2 ** 31, 2 ** 30], np.int32)), [-1.0, 0.5])
    assert np.array_equal(ro.decode(np.array([0, 128, 255], np.uint8)), [-1.0, 0.0, 127 / 128])
    assert np.array_equal(ro.decode(np.array([-3.0, 0.25, 1.5], np.float32)), [-1.0, 0.25, 1.0])
    assert np.array_equal(ro.decode(np.array([[0.5, -0.25], [1.0, 1.0]], np.float64)), [0.125, 1.0])
    assert np.array_equal(ro.decode(np.array([[100, 300, -400]], np.int16)), [0.0])


def _upfirdn_reference(x, h, L, M, n_out):
    """scipy.signal.upfirdn on the same taps, shifted by the filter delay D and cut to n_out: y[j] = (h * up_L(x))[j M + D]."""
    from scipy.signal import upfirdn
    D = (len(h) - 1) // 2
    s = (-D) % M                                                        # front zeros so that the delay is a whole number of outputs
    y = upfirdn(np.concatenate([np.zeros(s), h]), np.concatenate([x, np.zeros(len(h) // L + 2)]), L, M)
    return y[(D + s) // M:(D + s) // M + n_out]


@pytest.mark.parametrize("fs_in", RATES)
def test_oracle_matches_upfirdn(fs_in):
    h, L, M = audio.design_resampler(fs_in)
    rs = np.random.RandomState(fs_in % 1000)
    for n_in, C, dtype in ((1, 1, np.int16), (7, 2, np.float32), (len(h) // L // 3, 2, np.int32), (4000, 1, np.uint8), (3001, 6, np.int16)):
        if dtype == np.float32:
            pcm = (rs.randn(n_in, C) * 0.8).astype(np.float32)
        elif dtype == np.uint8:
            pcm = rs.randint(0, 256, size=(n_in, C)).astype(np.uint8)
        else:
            info = np.iinfo(dtype)
            pcm = rs.randint(info.min, info.max, size=(n_in, C), dtype=np.int64).astype(dtype)
        pcm = pcm[:, 0] if C == 1 else pcm
        got = ro.resample(pcm, h, L, M)
        n_out = audio.resampled_length(n_in, fs_in)
        ref = np.clip(_upfirdn_reference(ro.decode(pcm), h, L, M, n_out), -1.0, 1.0)
        assert got.shape == ref.shape == (n_out,)
        if n_out:
            err = float(np.abs(got - ref).max())
            print(f"  {fs_in} Hz n_in={n_in} C={C} {np.dtype(dtype).name}: max |oracle - upfirdn| {err:.2e}")
            assert err <= 1e-12
