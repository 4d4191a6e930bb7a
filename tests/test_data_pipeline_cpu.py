"""CPU checks of the training-set pipeline: the chunked spline restated in numpy (oracle/dataset_oracle.py) against scipy's griddata,
the sign-scan unroll against the reference semantics, and the host bookkeeping (timecodes, silence mask, trims, stretched lengths,
ranges, labels) against the reference's outputs stored in tests/golden/data_pipeline.npz."""
import hashlib
import os

import numpy as np
import pytest
from scipy.interpolate import griddata

from oracle import dataset_oracle as do
from tests import _pipeline_inputs as pin


def _griddata(x, m):
    n = x.shape[0]
    return griddata(np.linspace(0, n - 1, n), x, np.linspace(0, n - 1, m), method="cubic")


@pytest.mark.parametrize("n", [4, 5, 6, 7, 8, 255, 256, 257, 303, 304, 305, 511, 512, 513, 560, 1031])
def test_chunked_spline_matches_scipy(n):
    rs = np.random.RandomState(n)
    x = rs.randn(n, 3).astype(np.float32) * np.array([1.0, 50.0, 1e-3], dtype=np.float32)
    for m in sorted({int(0.9 * n), n, 2 * n - 1, 1, 2}):
        ref = _griddata(x, m)
        got = do.spline_resample(x, m)
        assert np.abs(got - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), (n, m)


def test_chunked_spline_matches_scipy_on_a_take_length_signal():
    n = 2_400_000
    x = (np.random.RandomState(1).randn(n) * 0.3).astype(np.float32)
    m = int(0.9 * n)
    ref = _griddata(x, m)
    got = do.spline_resample(x, m)
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())


def test_scan_unroll_equals_reference_semantics():
    from zeggs_b200 import animation
    rs = np.random.RandomState(0)
    e = np.cumsum(rs.randn(400, 6, 3) * 20.0, axis=0)
    e[rs.rand(400, 6) < 0.2] += 360.0                       # a full turn of one channel negates the quaternion: many flips
    q = animation.q_from_euler_deg(e, "zyx")
    q[50, 2] = 0.0                                           # exact zero dots against both neighbours
    q[50, 2, 0] = 1.0
    q[51, 2] = np.array([0.0, 1.0, 0.0, 0.0])
    ref = animation.q_unroll(q)
    assert np.array_equal(do.unroll_by_scan(q), ref)
    assert (np.sum(q[1:] * q[:-1], -1) < 0).sum() > 100


def _bookkeeping(g, base):
    """The pipeline's host steps on the golden's inputs -> (ranges, labels by name, trimmed wav lengths / hashes)."""
    from zeggs_b200 import animation
    from zeggs_b200 import data_pipeline as dp
    conf = pin.conf_for(base)
    info = dp.read_csv_rows(os.path.join(base, "info.csv"))
    ranges = {"train": [], "valid": []}
    labels = {"train": [], "valid": []}
    wavs = {}
    cur = 0
    for row in info:
        anim = animation.load_bvh(os.path.join(base, "original", row["anim_bvh"]))
        wav_path = os.path.join(base, "original", row["audio_filename"])
        wav = dp._read_take_audio(wav_path, 16000)
        mask = dp.silence_mask(dp.read_csv_rows(wav_path[:-4] + ".csv"), len(wav), 16000)
        a0, a1, m0, m1 = dp.trim_bounds(row, 16000, 60)
        wav = (wav * mask).astype(wav.dtype)[a0:a1]
        n = len(anim["rotations"][m0:m1])
        folder = "valid" if dp._truthy(row["validation"]) else "train"
        for r in conf["len_ratios"]:
            nf = n if r == 1.0 else dp.stretched_length(r, n)
            stem = row["anim_bvh"].split(".")[0] + "_x_" + str(r).replace(".", "_")
            wavs[f"{folder}/{stem}.wav"] = (len(wav) if r == 1.0 else dp.stretched_length(r, len(wav)),
                                           hashlib.sha256(wav.tobytes()).hexdigest() if r == 1.0 else None)
            ranges[folder].append([cur, cur + nf])
            labels[folder].append(row["style"])
            cur += nf
    return ranges, labels, wavs


def test_host_bookkeeping_reproduces_the_reference(tmp_path):
    g = pin.load_golden()
    base = pin.write_inputs(g, str(tmp_path))
    ranges, labels, wavs = _bookkeeping(g, base)
    names = pin.data_definition(g)["label_names"]
    for split in ("train", "valid"):
        assert np.array_equal(np.array(ranges[split], dtype=np.int32).reshape(-1, 2), g[f"out:ranges_{split}"]), split
        assert [names[i] for i in g[f"out:ranges_{split}_labels"]] == labels[split], split
    for k, (n, sha) in wavs.items():
        assert int(g["trimlen:" + k]) == n, k
        if sha is not None:                                   # ratio 1.0: the masked, trimmed samples themselves
            assert str(g["trimsha:" + k]) == sha, k


def test_label_order_is_first_appearance_or_explicit():
    from zeggs_b200 import _lib
    from zeggs_b200 import data_pipeline as dp
    rows = [{"style": s} for s in ("Sad", "Happy", "Sad", "Old")]
    assert dp.label_order(rows) == ["Sad", "Happy", "Old"]
    assert dp.label_order(rows, ["Old", "Happy", "Sad", "Extra"]) == ["Old", "Happy", "Sad", "Extra"]
    with pytest.raises(_lib.ZeggsError):
        dp.label_order(rows, ["Sad", "Happy"])


def test_unsupported_inputs_raise_naming_the_file_or_key(tmp_path):
    from scipy.io import wavfile
    from zeggs_b200 import _lib
    from zeggs_b200 import data_pipeline as dp
    p = str(tmp_path / "stereo.wav")
    wavfile.write(p, 16000, np.zeros((100, 2), np.int16))
    with pytest.raises(_lib.ZeggsError, match="stereo.wav"):
        dp._read_take_audio(p, 16000)
    wavfile.write(p, 22050, np.zeros(100, np.int16))
    with pytest.raises(_lib.ZeggsError, match="stereo.wav"):
        dp._read_take_audio(p, 16000)
    with pytest.raises(_lib.ZeggsError, match="save_normalized_animations"):
        dp._check_conf({"save_normalized_animations": True})


def test_deterministic_npz_writer_round_trips(tmp_path):
    from zeggs_b200 import data_pipeline as dp
    arrays = dict(a=np.arange(5, dtype=np.int32), b=np.float64(2.5), c=np.ones((2, 3), np.float32))
    dp.savez_deterministic(tmp_path / "x.npz", arrays)
    b1 = (tmp_path / "x.npz").read_bytes()
    dp.savez_deterministic(tmp_path / "x.npz", arrays)
    assert (tmp_path / "x.npz").read_bytes() == b1
    with np.load(tmp_path / "x.npz") as d:
        for k, v in arrays.items():
            assert d[k].dtype == np.asarray(v).dtype and np.array_equal(d[k], v)
