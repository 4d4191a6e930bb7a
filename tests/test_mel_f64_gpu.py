"""GPU: the mel front end (csrc/mel.cu, zeggs_mel_forward) against the float64 restatement of tests/_mel_cases.py, bin by bin,
at every shape it accepts, and bitwise invariances between its staging paths and call forms.

* Bin by bin: single-bin filterbank tables (band i = FFT bin k_i, weight 1; two calls cover bins 0..400) and a minimum amplitude
  of 1e-15 turn mel_out into |X_k| / 800.  Per frame: max_k |a - a_ref| <= BIN_TAU * ||w x||_2 / 800 + BIN_RHO * a_ref, on tones
  on bins 1, 24, 25, 26, 199, 200, 375, 380, 399, 400, off-bin tones, white noise, a DC offset and a chirp, at hops 200, 199, 160
  and 800, with an even and an odd frame count.
* Every accepted shape: a stratified grid over hop, n_mels, (fs, fmin, fmax) with and without normalised bands, clip length
  (401 .. 12345 and 2.4 M samples), anim_fs, 1 / 3 / 65 clips with distinct gains, int16 PCM, L = 1, a 5120-weight table (read
  from global memory) and hop 800 with 256 bands and mel_out (past the shared-memory limit with staged weights).  mel_out
  |s - s_ref| <= 1e-4, features <= 2e-4; anim_length at its limit, and one more is refused.  The drop-in
  extract_mel_spectrogram_for_tts at each configuration.
* Bitwise: int16 PCM equals float32 x / 32768 (with and without gain, on both 16-byte staging paths and the general one); mel
  only, features only and both agree; each clip of a batch equals the clip alone; appending 1..7 samples leaves every frame
  that reads no padded sample unchanged; an unaligned view equals its aligned copy.
tests/test_mel_f64_cpu.py shows the float32 restatement meets these bounds with >= 4x headroom and that each modelled fault
breaks one.
"""
import numpy as np
import pytest
import torch

from tests import _mel_cases as mc
from tests._util import ensure_built

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


def _front_end(dev, hop, fs=16000, n_mels=80, fmin=20, fmax=7600, normalize=True, tables=None, min_amp=None):
    from zeggs_b200 import audio
    fe = audio.MelFrontEnd(dev, sampling_rate=fs, hop_length=hop, n_mel_channels=n_mels, mel_fmin=fmin, mel_fmax=fmax,
                           normalize_mel_bins=normalize)
    if tables is not None:
        _set_tables(fe, tables)
    if min_amp is not None:
        fe.min_amp = float(min_amp)
    return fe


def _set_tables(fe, tables):
    start, length, off, w = tables
    it = lambda v: torch.tensor(np.asarray(v), dtype=torch.int32, device=fe.device)
    fe.fb_start, fe.fb_len, fe.fb_off = it(start), it(length), it(off)
    fe.fb_w = torch.tensor(np.asarray(w), dtype=torch.float32, device=fe.device)
    fe.n_mels = len(start)


def _report(tag, ratios):
    for name, r in ratios:
        print(f"  [{tag}] {name}: {r:.3g} of its bound")
    bad = [x for x in ratios if not x[1] <= 1.0]
    assert not bad, bad


# ---------------------------------------------------------------------------------------------- 1. bin by bin
@pytest.mark.parametrize("parity", ["even_L", "odd_L"])
@pytest.mark.parametrize("hop", mc.BIN_HOPS)
def test_every_fft_bin_against_float64(dev, hop, parity):
    n = mc.bin_config_lengths(hop)[parity == "odd_L"]
    x = mc.bin_signals(n)
    fe = _front_end(dev, hop, min_amp=mc.BIN_MIN_AMP)
    a = []
    for bins in mc.BIN_HALVES:
        _set_tables(fe, mc.single_bin_tables(bins))
        mel, _ = fe.forward(torch.from_numpy(x).to(dev), want_mel=True, want_feat=False)
        a.append(mc.amp_from_mel(mel.cpu().numpy(), mc.BIN_MIN_AMP))
    a = np.concatenate(a, axis=1)                                                   # [clips, 401, L]
    names = [f"tone{k}" for k in mc.BIN_TONES + mc.OFF_BIN_TONES] + ["white", "dc", "chirp"]
    ratios = []
    for c in range(x.shape[0]):
        a_ref, nrm = mc.spectra(x[c], hop)
        r = mc.bin_ratio(a[c].T, a_ref, nrm)
        ratios.append((f"{names[c]} worst frame {int(r.argmax())}/{len(r)} bin {int(np.abs(a[c].T - a_ref)[r.argmax()].argmax())}",
                       float(r.max())))
    print(f"  [bins hop{hop} n{n} L{mc.num_frames(n, hop)}] WORST {max(r for _, r in ratios):.3g}")
    _report(f"bins hop{hop} n{n}", ratios)


# ---------------------------------------------------------------------------------------------- 2. every accepted shape
_grid = {}


def _case(cid):
    if not _grid:
        _grid.update((c.cid, c) for c in mc.grid())
    return _grid[cid]


def _grid_ids():
    return [c.cid for c in mc.grid()]


def _run(dev, fe, x, gain, anim_fs, anim_length, want_mel=True, want_feat=True):
    g = None if gain is None else torch.from_numpy(np.asarray(gain, np.float32)).to(dev)
    return fe.forward(torch.from_numpy(np.ascontiguousarray(x)).to(dev), anim_fs, anim_length, want_mel=want_mel,
                      want_feat=want_feat, gain=g)


@pytest.mark.parametrize("cid", _grid_ids())
def test_every_accepted_shape_against_float64(dev, cid):
    from zeggs_b200 import _lib
    c = _case(cid)
    fe = _front_end(dev, c.hop, c.fs, c.n_mels, c.fmin, c.fmax, c.normalize, tables=c.tables)
    mel, feat = _run(dev, fe, c.x, c.gain, c.anim_fs, c.anim_length)
    m_ref, f_ref = c.oracle()
    assert mel.shape == m_ref.shape and feat.shape == f_ref.shape
    mt, ft = c.tolerances(m_ref)
    em = float((np.abs(mel.cpu().numpy() - m_ref) / mt).max())
    ef = float((np.abs(feat.cpu().numpy() - f_ref) / ft).max())
    print(f"  [{cid}] L={c.L} anim_length={c.anim_length} fb_total={c.tables[3].size}")
    _report(cid, [("mel_out", em), ("feat", ef)])
    # one 60 fps row more than the frames reach is refused before any launch
    torch.cuda.synchronize()
    launches = _lib.lib().zeggs_launch_count()
    with pytest.raises(_lib.ZeggsError, match="anim_length"):
        _run(dev, fe, c.x, c.gain, c.anim_fs, c.anim_length + 1)
    assert _lib.lib().zeggs_launch_count() == launches


DROPIN_CONFS = [(fs, fmin, fmax, nz) for fs, fmin, fmax in mc.CONFS for nz in (True, False)]


@pytest.mark.parametrize("conf", DROPIN_CONFS, ids=lambda c: f"fs{c[0]}_{c[1]}_{c[2]}{'' if c[3] else '_nonorm'}")
def test_dropin_extract_mel_spectrogram_at_each_configuration(dev, conf):
    from zeggs_b200 import audio
    fs, fmin, fmax, normalize = conf
    x = mc.chirp(9001, 7)
    for hop, n_mels in [(160, 80), (199, 256)]:
        mel, wav = audio.extract_mel_spectrogram_for_tts(x, fs, 800, hop, n_mels, fmin, fmax, 1e-5, pre_emphasis=False,
                                                         normalize_mel_bins=normalize, device=dev)
        assert wav is x and isinstance(mel, np.ndarray)
        tables = mc.slaney_tables(fs, n_mels, fmin, fmax, normalize)
        ref, _ = mc.front_end(x, hop, tables)
        assert mel.shape == ref[0].shape
        _report(f"drop-in fs{fs} hop{hop} m{n_mels}", [("mel", float((np.abs(mel - ref[0]) / mc.mel_tolerance(x, hop, tables)[0]).max()))])


# ---------------------------------------------------------------------------------------------- 3. bitwise invariances
def _pcm_pair(n, seed=11):
    x16 = np.stack([mc.pcm16(n, seed + i) for i in range(3)])
    return x16, (x16.astype(np.float32) / np.float32(32768.0))            # exact: x * 2^-15 rounds once either way


@pytest.mark.parametrize("gain", [None, "gains"])
@pytest.mark.parametrize("hop,n", [(200, 16000), (200, 16004), (199, 16000), (160, 12808)],
                         ids=["interior_f4_i16", "f4_and_general", "general", "hop160"])
def test_int16_equals_float_x_over_32768_bitwise(dev, hop, n, gain):
    """(200, 16000): float4 and 8-sample int16 paths on interior tiles; (200, 16004): float4 for float, general for int16;
    hop 199: the general path everywhere."""
    x16, xf = _pcm_pair(n)
    g = None if gain is None else np.array([0.37, 1.0, 2.53], np.float32)
    fe = _front_end(dev, hop)
    n60 = mc.max_anim_length(n, hop, 16000, 60)
    m16, f16 = _run(dev, fe, x16, g, 60, n60)
    mf, ff = _run(dev, fe, xf, g, 60, n60)
    assert torch.equal(m16, mf) and torch.equal(f16, ff)


def test_output_selection_does_not_change_values(dev):
    x = np.stack([mc.chirp(20000, 1), mc.white(20000, 2)])
    fe = _front_end(dev, 200, n_mels=128)
    n30 = mc.max_anim_length(20000, 200, 16000, 30)
    both = _run(dev, fe, x, [0.5, 1.5], 30, n30)
    mel_only = _run(dev, fe, x, [0.5, 1.5], 30, n30, want_feat=False)[0]
    feat_only = _run(dev, fe, x, [0.5, 1.5], 30, n30, want_mel=False)[1]
    assert torch.equal(both[0], mel_only) and torch.equal(both[1], feat_only)


@pytest.mark.parametrize("pcm", [False, True])
def test_each_clip_of_a_batch_equals_the_clip_alone(dev, pcm):
    n, N = 7777, 5
    x = np.stack([mc.pcm16(n, i) if pcm else mc.signal(["white", "chirp", "dc", "silence"][i % 4], n, i) for i in range(N)])
    g = np.linspace(0.3, 2.0, N).astype(np.float32)
    fe = _front_end(dev, 160, n_mels=33)
    n60 = mc.max_anim_length(n, 160, 16000, 25)
    mel, feat = _run(dev, fe, x, g, 25, n60)
    for i in range(N):
        mi, fi = _run(dev, fe, x[i:i + 1], g[i:i + 1], 25, n60)
        assert torch.equal(mel[i:i + 1], mi) and torch.equal(feat[i:i + 1], fi), i


@pytest.mark.parametrize("pcm", [False, True])
@pytest.mark.parametrize("hop", [200, 160, 400])
def test_appended_samples_leave_unpadded_frames_unchanged(dev, hop, pcm):
    """n = 16000 stages interior tiles on a 16-byte path; 1..7 more samples move them to the general path.  A frame pair that
    reads no padded sample (i hop - 400 >= 0 and i hop + 399 < n for both frames) sees the same samples either way.  The pair,
    not the frame: both frames share one complex transform, so each one's rounding depends on the other."""
    n = 16000
    base = mc.pcm16(n + 7, 3) if pcm else mc.white(n + 7, 3)
    fe = _front_end(dev, hop)
    m0, _ = _run(dev, fe, base[None, :n], None, None, None, want_feat=False)
    i = np.arange(m0.shape[2])
    lo, hi = i & ~1, i | 1
    inner = torch.from_numpy(np.nonzero((lo * hop - 400 >= 0) & (hi * hop + 399 < n))[0]).to(dev)
    assert len(inner) > 30
    for j in range(1, 8):
        mj, _ = _run(dev, fe, base[None, :n + j], None, None, None, want_feat=False)
        assert torch.equal(m0.index_select(2, inner), mj.index_select(2, inner)), j


@pytest.mark.parametrize("dtype", [torch.float32, torch.int16])
def test_unaligned_view_equals_aligned_copy(dev, dtype):
    """A 1-D view with a storage offset is contiguous, so forward() passes it as it is: its base is not 16-byte aligned, and the
    kernel must stage it on the general path (the same values as the 16-byte paths)."""
    n = 16000
    buf = torch.from_numpy(mc.pcm16(n + 1, 5) if dtype == torch.int16 else mc.white(n + 1, 5)).to(dev)
    view = buf[1:]
    assert view.is_contiguous() and view.data_ptr() % 16 != 0
    fe = _front_end(dev, 200)
    n60 = mc.max_anim_length(n, 200, 16000, 60)
    got = fe.forward(view, 60, n60, want_mel=True, want_feat=True)
    want = fe.forward(view.clone(), 60, n60, want_mel=True, want_feat=True)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
