"""zeggs_resample (csrc/resample.cu) on the device: against the float64 oracle (oracle/resample_oracle.py), analytic checks that
do not use the oracle's filter, the audio features of its output, and generate_gesture on audio that is not 16 kHz."""
import json
import shutil

import numpy as np
import pytest
import torch

from oracle import resample_oracle as ro
from tests._util import ensure_built

pytestmark = pytest.mark.gpu

RATES = [8000, 11025, 22050, 24000, 32000, 44100, 48000, 96000]
KERNEL_TOL = 2e-6        # fp32 accumulation in four partial sums; measured on an H100 at most 7.3e-7 over these cases


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


def _pcm(rs, n, C, dtype):
    if dtype == np.float32:
        x = (rs.randn(n, C) * 0.7).astype(np.float32)          # about 15 % of the samples lie outside [-1, 1]
    elif dtype == np.uint8:
        x = rs.randint(0, 256, size=(n, C)).astype(np.uint8)
    else:
        info = np.iinfo(dtype)
        x = (np.clip(rs.randn(n, C) * 0.3, -1, 1) * info.max).astype(dtype)
    return x[:, 0] if C == 1 else x


def _check(dev, pcm, fs_in, tag):
    from zeggs_b200 import audio
    r = audio.Resampler(dev, fs_in)
    got = r(pcm)
    ref = ro.resample(pcm, r.h, r.L, r.M)
    assert tuple(got.shape) == ref.shape == (audio.resampled_length(len(pcm), fs_in),)
    err = float(np.abs(got.cpu().numpy().astype(np.float64) - ref).max()) if len(ref) else 0.0
    print(f"  [{tag}] n_out {len(ref)}: max-abs err {err:.3e}")
    assert err <= KERNEL_TOL
    return err


@pytest.mark.parametrize("fs_in", RATES)
def test_kernel_matches_float64_oracle(dev, fs_in):
    """Every dtype and 1 / 2 channels at every rate; lengths 1, 7, shorter than the filter, 2 s and 10 s."""
    from zeggs_b200 import audio
    h, L, _ = audio.design_resampler(fs_in)
    short = max(2, (len(h) // L) // 2)                  # fewer input samples than taps per output
    rs = np.random.RandomState(fs_in % 977)
    cases = [(1, 1, np.int16), (7, 2, np.uint8), (short, 2, np.float32), (short, 1, np.int32),
             (2 * fs_in, 1, np.uint8), (2 * fs_in, 2, np.int32), (2 * fs_in, 1, np.float32), (10 * fs_in, 2, np.int16)]
    worst = max(_check(dev, _pcm(rs, n, C, dt), fs_in, f"{fs_in} Hz n={n} C={C} {np.dtype(dt).name}") for n, C, dt in cases)
    print(f"  {fs_in} Hz worst {worst:.3e}")


def test_kernel_six_channels_and_a_long_take(dev):
    rs = np.random.RandomState(5)
    _check(dev, _pcm(rs, 3 * 44100, 6, np.int16), 44100, "44.1 kHz 6 channels int16")
    _check(dev, _pcm(rs, 3 * 48000, 6, np.float32), 48000, "48 kHz 6 channels float32")
    _check(dev, _pcm(rs, 150 * 48000, 2, np.int16), 48000, "150 s 48 kHz stereo int16")


def _interior(h, L, fs_in, n):
    """Output samples further than half a filter length from either end."""
    e = int(np.ceil(len(h) / (2.0 * L * fs_in) * 16000)) + 1
    return slice(e, n - e)


@pytest.mark.parametrize("fs_in", RATES)
def test_analytic_tones_silence_and_full_scale(dev, fs_in):
    """Independent of the oracle: tones below 7.5 kHz (and below 0.9 f_N) synthesised at fs_in and directly at 16 kHz agree to
    1e-5; tones at 9 and 11 kHz leave an interior RMS <= 1e-6 of their amplitude; silence gives exact zeros; a full-scale square
    wave stays inside [-1, 1]."""
    from zeggs_b200 import audio
    r = audio.Resampler(dev, fs_in)
    rs = np.random.RandomState(fs_in % 1013)
    n_in = 2 * fs_in
    t_in = np.arange(n_in) / fs_in
    fmax = min(7500.0, 0.9 * min(fs_in, 16000) / 2)
    freq, phase = rs.uniform(40.0, fmax, 10), rs.uniform(0, 2 * np.pi, 10)
    sig = lambda t: sum(0.09 * np.sin(2 * np.pi * f * t + p) for f, p in zip(freq, phase))
    y = r(sig(t_in).astype(np.float32)).cpu().numpy().astype(np.float64)
    z = sig(np.arange(len(y)) / 16000.0)
    s = _interior(r.h, r.L, fs_in, len(y))
    err = float(np.abs(y[s] - z[s]).max())
    print(f"  {fs_in} Hz passband tones: interior max-abs err {err:.3e}")
    assert err <= 1e-5
    if fs_in >= 24000:
        amp = 0.45
        x = amp * np.sin(2 * np.pi * 9000 * t_in + 0.4) + amp * np.sin(2 * np.pi * 11000 * t_in + 2.0)
        y = r(x.astype(np.float32)).cpu().numpy().astype(np.float64)
        rms = float(np.sqrt(np.mean(y[_interior(r.h, r.L, fs_in, len(y))] ** 2)))
        print(f"  {fs_in} Hz 9 + 11 kHz tones: interior RMS / amplitude {rms / amp:.3e}")
        assert rms <= 1e-6 * amp
    for dt, zero in ((np.int16, 0), (np.int32, 0), (np.uint8, 128), (np.float32, 0)):
        y = r(np.full((n_in // 4, 2), zero, dtype=dt))
        assert int(torch.count_nonzero(y)) == 0
    sq = np.where(np.sin(2 * np.pi * 997.0 * t_in) >= 0, 32767, -32768).astype(np.int16)
    y = r(sq)
    assert float(y.abs().max()) <= 1.0
    print(f"  {fs_in} Hz square wave: output range [{float(y.min()):.6f}, {float(y.max()):.6f}]")


@pytest.mark.parametrize("loud", [0, 1])
def test_features_of_kernel_output_match_oracle_output(dev, loud):
    """preprocess_audio on the kernel's 16 kHz signal vs on the oracle's, abs <= 3e-4 (the audio-feature tolerance)."""
    from oracle.make_golden import audio_params
    from zeggs_b200 import audio, synth
    p = audio_params(200)
    p.normalize_loudness = bool(loud)
    for fs_in, C in ((48000, 2), (44100, 2), (22050, 1)):
        x = synth.make_waveforms(C, 3 * fs_in, seed=fs_in % 100).T
        pcm = np.round(x * 20000.0).astype(np.int16)
        pcm = pcm[:, 0] if C == 1 else np.ascontiguousarray(pcm)
        r = audio.Resampler(dev, fs_in)
        y = r(pcm)
        ref = ro.resample(pcm, r.h, r.L, r.M).astype(np.float32)
        n60 = int(round(60.0 * len(ref) / 16000))
        got = audio.preprocess_audio(y, 60, n60, p, ["mel_spec", "energy"]).cpu().numpy()
        want = audio.preprocess_audio(ref, 60, n60, p, ["mel_spec", "energy"])
        err = float(np.abs(got - want).max())
        print(f"  {fs_in} Hz C={C} loud={loud}: features max-abs err {err:.3e}")
        assert err <= 3e-4


def _generate_setup(tmp_path):
    """Synthetic networks, stats and style BVH as tests/test_gpu_parity.py's generate_gesture end-to-end test builds them."""
    import os
    from tests import _fixtures as fx
    from zeggs_b200 import modules, synth
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "generate_e2e.npz"))
    H = int(g["H"])
    P = synth.make_params(H=H, seed=int(g["param_seed"]))

    def load(mod, prefix):
        mod.load_state_dict({k[len(prefix):]: torch.from_numpy(v) for k, v in P.items() if k.startswith(prefix)})
        return mod

    net = tmp_path / "net"; net.mkdir()
    torch.save(load(modules.SpeechEncoder(81, 64, 64), "speech_encoder."), net / "speech_encoder.pt")
    torch.save(load(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), "style_encoder."), net / "style_encoder.pt")
    torch.save(load(modules.Decoder(1134, 1131, 64, 64, H, 2), "decoder."), net / "decoder.pt")
    data = tmp_path / "data"; data.mkdir()
    stats = synth.load_stats()
    np.savez(data / "stats.npz", **{k: stats[k] for k in ("audio_input_mean", "audio_input_std", "anim_input_mean", "anim_input_std",
                                                         "anim_output_mean", "anim_output_std")})
    shutil.copy(os.path.join(fx.DATA, "data_definition_v1.json"), data / "data_definition.json")
    conf = json.load(open(os.path.join(fx.DATA, "data_pipeline_conf_v1.json")))
    conf["audio_conf"]["normalize_loudness"] = True
    json.dump(conf, open(data / "data_pipeline_conf.json", "w"))
    bvh = fx.make_synthetic_bvh(str(tmp_path / "style.bvh"))
    return net, data, bvh


def _generate(path, net, data, bvh, res):
    from zeggs_b200 import generate
    enc = generate.generate_gesture(path, [(bvh, (10, 300))], net, data, res, style_encoding_type="example", file_name="out",
                                    temperature=1e6, seed=1234, use_gpu=True)
    return enc, (res / "out.bvh").read_bytes()


def test_generate_gesture_48k_stereo_equals_16k_path_fed_the_kernel_output(dev, tmp_path):
    """A 48 kHz stereo int16 WAV through generate_gesture gives the same style encoding and the same BVH bytes as the 16 kHz path
    fed the kernel's output (written as a float32 WAV); out.wav is a byte copy of the 48 kHz file; the frame count follows n_out."""
    from scipy.io import wavfile
    from zeggs_b200 import animation, audio, synth
    net, data, bvh = _generate_setup(tmp_path)
    x = synth.make_waveforms(2, int(4.3 * 48000) + 7, seed=44).T
    pcm = np.ascontiguousarray(np.round(x * 20000.0).astype(np.int16))
    wav48 = tmp_path / "speech48.wav"
    wavfile.write(str(wav48), 48000, pcm)
    y = audio.resample(pcm, 48000, device=dev).cpu().numpy()
    wav16 = tmp_path / "speech16.wav"
    wavfile.write(str(wav16), 16000, y)
    enc48, bvh48 = _generate(wav48, net, data, bvh, tmp_path / "res48")
    enc16, bvh16 = _generate(wav16, net, data, bvh, tmp_path / "res16")
    assert torch.equal(enc48, enc16)
    assert bvh48 == bvh16
    assert (tmp_path / "res48" / "out.wav").read_bytes() == wav48.read_bytes()
    n_out = audio.resampled_length(len(pcm), 48000)
    assert len(y) == n_out
    frames = animation.load_bvh(str(tmp_path / "res48" / "out.bvh"))["positions"].shape[0]
    assert frames == int(round(60.0 * n_out / 16000))
    print(f"  {len(pcm)} samples at 48 kHz -> {n_out} at 16 kHz -> {frames} frames")


def test_16k_files_never_reach_the_resampler(dev, tmp_path, monkeypatch):
    """16 kHz files take the existing path: with audio.Resampler replaced by a stub that raises, a mono int16 file and a stereo file
    both generate, and the stereo one uses channel 0."""
    from scipy.io import wavfile
    from zeggs_b200 import audio, synth

    class Refuse:
        def __init__(self, *a, **k):
            raise AssertionError("a 16 kHz file reached the resampler")

    monkeypatch.setattr(audio, "Resampler", Refuse)
    monkeypatch.setattr(audio, "_resamplers", {})
    net, data, bvh = _generate_setup(tmp_path)
    x = np.round(synth.make_waveforms(2, 3 * 16000, seed=45).T * 20000.0).astype(np.int16)
    mono, stereo = tmp_path / "mono.wav", tmp_path / "stereo.wav"
    wavfile.write(str(mono), 16000, np.ascontiguousarray(x[:, 0]))
    wavfile.write(str(stereo), 16000, np.ascontiguousarray(x))
    enc_m, bvh_m = _generate(mono, net, data, bvh, tmp_path / "res_mono")
    enc_s, bvh_s = _generate(stereo, net, data, bvh, tmp_path / "res_stereo")
    assert torch.equal(enc_m, enc_s) and bvh_m == bvh_s
