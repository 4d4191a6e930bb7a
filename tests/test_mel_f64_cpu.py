"""CPU (no GPU): the mel front end's float64 restatement (tests/_mel_cases.py) equals oracle/mel_oracle, the float32 restatement
meets every bound tests/test_mel_f64_gpu.py holds the kernel to with headroom, and every modelled kernel fault breaks one.
Also the host-side refusal of more clips than one grid can hold, through the C ABI with placeholder pointers."""
import numpy as np
import pytest

from oracle import mel_oracle
from tests import _mel_cases as mc
from tests._util import ensure_built

F32_HEADROOM = 4.0        # the float32 restatement stays below 1 / F32_HEADROOM of every bound


def _ratio_line(tag, r):
    print(f"  [{tag}] {r:.3g} of its bound")
    return r


# ---------------------------------------------------------------------------------------------- restatement == oracle
ORACLE_CONFS = [dict(hop=200), dict(hop=160), dict(hop=199), dict(hop=800), dict(hop=7),
                dict(hop=200, fs=16000, n_mels=256, fmin=0, fmax=8000), dict(hop=256, fs=22050, n_mels=33, fmin=20, fmax=None),
                dict(hop=80, fs=8000, n_mels=128, fmin=20, fmax=4000), dict(hop=401, fs=16000, n_mels=1, fmin=20, fmax=7600)]


@pytest.mark.parametrize("n", [401, 799, 800, 12345])
@pytest.mark.parametrize("conf", ORACLE_CONFS, ids=lambda c: "_".join(f"{k}{v}" for k, v in c.items()))
def test_restatement_equals_mel_oracle(conf, n):
    kw = dict(fs=16000, n_mels=80, fmin=20, fmax=7600) | conf
    hop, fs = kw["hop"], kw["fs"]
    x = mc.chirp(n, 5)
    tables = mc.slaney_tables(fs, kw["n_mels"], kw["fmin"], kw["fmax"])
    n60 = mc.max_anim_length(n, hop, fs, 60)
    s, f = mc.front_end(x, hop, tables, mc.MIN_AMP, None, (fs / hop) / 60, n60)
    s_ref = mel_oracle.mel_spectrogram(x, **kw)
    assert s.shape[1:] == s_ref.shape
    assert np.abs(s[0] - s_ref).max() <= 1e-12
    if fs == 16000 and kw["fmin"] == 20 and kw["fmax"] == 7600:
        f_ref = mel_oracle.preprocess_audio(x, 60, n60, hop=hop, n_mels=kw["n_mels"])      # rounded to float32 by the oracle
        assert np.all(np.abs(f[0] - f_ref) <= 1e-12 + np.abs(f_ref) * 2.0 ** -24)
    # the non-normalised bank, and a non-default minimum amplitude
    s, _ = mc.front_end(x, hop, mc.slaney_tables(fs, kw["n_mels"], kw["fmin"], kw["fmax"], False), 1e-4 / 800)
    s_ref = mel_oracle.mel_spectrogram(x, min_clipping=1e-4, normalize_mel_bins=False, **kw)
    assert np.abs(s[0] - s_ref).max() <= 1e-12


def test_restatement_covers_gain_pcm16_and_single_frame():
    """int16 is decoded as x / 32768 before the gain; a call with L = 1 has one 60 fps row, equal to that frame."""
    x16 = mc.pcm16(700, 3)
    g = np.float32(0.61)
    x = (x16.astype(np.float64) / 32768.0) * np.float64(g)
    s, f = mc.front_end(x16[None], 800, mc.slaney_tables(16000, 80, 20, 7600), mc.MIN_AMP, np.array([g]), 80 / 60 * 0.25, 1)
    assert mc.num_frames(700, 800) == 1
    assert np.abs(s[0] - mel_oracle.mel_spectrogram(x, hop=800)).max() <= 1e-12
    f_ref = mel_oracle.preprocess_audio(x, 60, 1, hop=800)                            # rounded to float32 by the oracle
    assert np.all(np.abs(f[0] - f_ref) <= 1e-12 + np.abs(f_ref) * 2.0 ** -24)


def test_host_tables_match_the_restatement():
    """MelFrontEnd builds its tables on the host (no device needed on a CPU device): the same sparse tables as the restatement's."""
    from zeggs_b200 import audio
    for fs, nm, fmin, fmax, norm in [(16000, 80, 20, 7600, True), (22050, 256, 20, None, False), (8000, 33, 0, 4000, True)]:
        fe = audio.MelFrontEnd("cpu", sampling_rate=fs, n_mel_channels=nm, mel_fmin=fmin, mel_fmax=fmax, normalize_mel_bins=norm)
        st, ln, off, w = mc.slaney_tables(fs, nm, fmin, fmax, norm)
        assert np.array_equal(fe.fb_start.numpy(), st) and np.array_equal(fe.fb_len.numpy(), ln)
        assert np.array_equal(fe.fb_off.numpy(), off) and np.array_equal(fe.fb_w.numpy(), w.astype(np.float32))
        assert np.array_equal(fe.window.numpy(), mc.hann().astype(np.float32))


def test_grid_covers_every_listed_value():
    cases = mc.grid()
    for attr, values in [("hop", mc.HOPS), ("n_mels", mc.N_MELS), ("anim_fs", mc.ANIM_FS), ("n_clips", mc.N_CLIPS),
                         ("n_samples", mc.N_SAMPLES + [mc.LONG_SAMPLES])]:
        assert set(values) <= {getattr(c, attr) for c in cases}, attr
    assert {(c.fs, c.fmin, c.fmax, c.normalize) for c in cases} >= {conf + (nz,) for conf in mc.CONFS for nz in (True, False)}
    assert any(c.L == 1 for c in cases) and any(c.pcm for c in cases)
    assert any(int(c.tables[3].size) > 4096 for c in cases)
    assert any(c.hop == 800 and c.n_mels == 256 for c in cases)


# ---------------------------------------------------------------------------------------------- float32 meets the bounds
def test_float32_meets_the_grid_bounds_with_headroom():
    worst = []
    for c in mc.grid():
        m, f = c.oracle()
        m32, f32 = c.oracle(f32=True)
        mt, ft = c.tolerances(m)
        worst.append(((np.abs(m32 - m) / mt).max(), f"{c.cid} mel"))
        worst.append(((np.abs(f32 - f) / ft).max(), f"{c.cid} feat"))
    worst.sort(reverse=True)
    for r, tag in worst[:4]:
        _ratio_line(f"float32 {tag}", r)
    assert worst[0][0] * F32_HEADROOM <= 1.0


def _bin_case(hop, n, f32=False, fault=None):
    """-> per-frame bin ratios [clips, L] of `fault` (or float32) against float64, amplitudes through the dB encoding as the kernel
    returns them from single-bin tables."""
    x = mc.bin_signals(n)
    out = []
    for c in range(x.shape[0]):
        a_ref, nrm = mc.spectra(x[c], hop)
        a, _ = mc.spectra(x[c], hop, f32, fault)
        if f32:
            s, _ = mc.front_end(x[c], hop, mc.single_bin_tables(range(mc.NB)), mc.BIN_MIN_AMP, f32=True)
            a = mc.amp_from_mel(s[0].T, mc.BIN_MIN_AMP)
        out.append(mc.bin_ratio(a, a_ref, nrm))
    return np.stack(out)


def test_float32_meets_the_bin_bound_with_headroom():
    worst = 0.0
    for hop in mc.BIN_HOPS:
        for n in mc.bin_config_lengths(hop):
            r = _bin_case(hop, n, f32=True).max()
            _ratio_line(f"float32 bin hop{hop} n{n}", r)
            worst = max(worst, r)
    assert worst * F32_HEADROOM <= 1.0


# ---------------------------------------------------------------------------------------------- faults break a bound
def _grid_case(cid):
    return next(c for c in mc.grid() if c.cid == cid)


def _grid_ratio(cid, fault):
    c = _grid_case(cid)
    m, f = c.oracle()
    mf, ff = c.oracle(fault=fault)
    if mf.shape != m.shape:
        return np.inf
    mt, ft = c.tolerances(m)
    return max((np.abs(mf - m) / mt).max(), (np.abs(ff - f) / ft).max())


FAULT_CASES = {
    "pair_swap": ("bin", 200),
    "lane0_partner": ("bin", 160),
    "twiddle_sign": ("bin", 199),
    "symmetric_pad": ("bin", 800),
    "periodic_hann": ("bin", 200),
    "no_zero_extend": ("grid", "g01_hop7_m31_fs16000_0_8000_n402_a60_N3"),
    "lerp_tile": ("grid", "g05_hop200_m128_fs16000_0_8000_nonorm_n12345_a30_N65"),
    "energy_from_s": ("grid", "g17_hop256_m33_fs16000_0_8000_n12345_a30_N65"),
    "gain0": ("grid", "n65_hop200_m80_pcm"),
}


def test_every_fault_has_a_case():
    assert set(FAULT_CASES) == set(mc.FAULTS)


@pytest.mark.parametrize("fault", list(mc.FAULTS))
def test_fault_breaks_a_bound(fault):
    kind, arg = FAULT_CASES[fault]
    if kind == "bin":
        r = _bin_case(arg, mc.bin_config_lengths(arg)[1], fault=fault).max()
    else:
        r = _grid_ratio(arg, fault)
    _ratio_line(f"fault {fault} ({mc.FAULTS[fault]}) on {kind} {arg}", r)
    assert r > 1.0


def test_lane0_fault_is_seen_by_the_tones_on_its_bins():
    """The tones on bins 25, 200, 375 and 400 (lane 0's bins) each break the bin bound under the lane-0 fault on their own."""
    n = mc.bin_config_lengths(200)[0]
    r = _bin_case(200, n, fault="lane0_partner").max(axis=1)
    for k in (25, 200, 375, 400):
        assert r[mc.BIN_TONES.index(k)] > 1.0, k


# ---------------------------------------------------------------------------------------------- host refusals
def test_more_clips_than_one_grid_holds_are_refused():
    """One grid row per clip: 65535 clips at most.  Refused with a message that names the limit, before any CUDA call (this runs
    without a GPU: the pointers are placeholders that nothing reads)."""
    import ctypes
    ensure_built()
    from zeggs_b200 import _lib
    l = _lib.lib()
    dummy = ctypes.create_string_buffer(64)
    p = ctypes.addressof(dummy)
    a = _lib.MelArgs(n_clips=65536, n_samples=16000, n_fft=800, hop=200, n_mels=80, anim_length=60, min_amp=mc.MIN_AMP,
                     frames_per_anim=4 / 3, wav=p, window=p, twiddle=p, fb_start=p, fb_len=p, fb_off=p, fb_w=p, mel_out=p,
                     feat_out=p, fb_total=742)
    launches = l.zeggs_launch_count()
    assert l.zeggs_mel_forward(ctypes.byref(a), None) == -1          # ZEGGS_ERR_ARG
    msg = l.zeggs_last_error().decode()
    print(f"  [n_clips 65536] {msg}")
    assert "65535" in msg
    assert l.zeggs_launch_count() == launches
