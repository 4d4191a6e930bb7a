"""The training-set pipeline on the GPU: data_pipeline() end to end against the reference's outputs (tests/golden/data_pipeline.npz),
its kernels against scipy / the host feature code / numpy float64, run-to-run byte identity, and train() on a dataset it built."""
import json
import os
import random

import numpy as np
import pytest
import torch
from scipy.interpolate import griddata

from tests import _pipeline_inputs as pin
from tests._util import ensure_built

pytestmark = pytest.mark.gpu

POSE = ["Y_root_pos", "Y_root_rot", "Y_root_vel", "Y_root_vrt", "Y_lpos", "Y_ltxy", "Y_lvel", "Y_lvrt", "Y_gaze_pos"]
STAT_DTYPES = dict(audio_input_mean=np.float32, audio_input_std=np.float64, anim_input_mean=np.float32, anim_input_std=np.float64,
                   anim_output_mean=np.float32, anim_output_std=np.float32)


@pytest.fixture(scope="module", autouse=True)
def built():
    ensure_built()


def _run(g, base, processed="processed"):
    from zeggs_b200.data_pipeline import data_pipeline
    pin.write_inputs(g, base)
    return data_pipeline(pin.conf_for(base, processed), label_names=pin.data_definition(g)["label_names"])


def test_pipeline_matches_reference_golden(tmp_path):
    g = pin.load_golden()
    base = str(tmp_path)
    processed, ddef = _run(g, base)
    out = os.path.join(base, "processed")
    with np.load(os.path.join(out, "processed_data.npz")) as d:
        got = {k: d[k] for k in d.files}
    ref = {k[4:]: v for k, v in g.items() if k.startswith("out:")}
    assert set(got) == set(ref)
    with np.load(os.path.join(out, "stats.npz")) as d:
        assert sorted(d.files) == sorted(g["stats_keys"].tolist())
    for k in ("ranges_train", "ranges_valid", "ranges_train_labels", "ranges_valid_labels"):
        assert got[k].dtype == np.int32 and np.array_equal(got[k], ref[k]), k
    # per array, relative to max(1, max |ref|) as the other pose-feature checks: the reference runs ratio 1.0 in float32 (float32 BVH
    # channels), so a root velocity carries ~1e-5 / dt of rounding from positions of magnitude ~100
    for k in POSE:
        assert got[k].shape == ref[k].shape and got[k].dtype == np.float32, k
        err = np.abs(got[k].astype(np.float64) - ref[k]).max() / max(1.0, float(np.abs(ref[k]).max()))
        assert err <= 1e-4, (k, err)
    a = np.abs(got["X_audio_features"].astype(np.float64) - ref["X_audio_features"]).max()
    assert got["X_audio_features"].shape == ref["X_audio_features"].shape and a <= 3e-4, a
    # 1e-5 relative.  The reference accumulates its means in float32 row by row, which is exact to ~1e-7 of the data's spread rather
    # than of the mean: a mean is scaled by |mean| + its group's pooled std, a per-channel std by max(|std|, 1e-2 x that pooled std)
    pooled = ref["anim_input_std"].astype(np.float64)
    n_out = len(ref["anim_output_mean"])
    spread = dict(anim_input_mean=pooled, anim_output_mean=pooled[:n_out], anim_output_std=1e-2 * pooled[:n_out],
                  audio_input_mean=float(ref["audio_input_std"]), anim_input_std=0.0, audio_input_std=0.0)
    for k, dt in STAT_DTYPES.items():
        assert got[k].dtype == dt and got[k].shape == ref[k].shape, k
        r = ref[k].astype(np.float64)
        scale = np.abs(r) + spread[k] if k.endswith("mean") else np.maximum(np.abs(r), spread[k])
        bad = np.abs(got[k] - r) > 1e-5 * scale
        assert not bad.any(), (k, np.flatnonzero(bad)[:5], np.atleast_1d(got[k])[bad][:5], np.atleast_1d(r)[bad][:5])
    z = ref["anim_output_std"] == 0
    # exactly 0 wherever the reference's is (a constant channel); a float32 reference can leave rounding noise where the float64
    # two-pass std is exactly 0, which the relative check above accepts
    assert z.any() and np.all(got["anim_output_std"][z] == 0.0), np.flatnonzero(got["anim_output_std"][z] != 0)
    assert ddef == pin.data_definition(g)
    with open(os.path.join(out, "data_definition.json")) as f:
        assert json.load(f) == pin.data_definition(g)
    # trimmed takes: the same files, BVH values within print precision of the centring (fp32 in the reference, fp64 here)
    from zeggs_b200 import animation
    for k, v in g.items():
        if k.startswith("trim:"):
            p = os.path.join(out, "trimmed", k[5:])
            rp = os.path.join(base, "ref.bvh")
            with open(rp, "wb") as f:
                f.write(v.tobytes())
            a, b = animation.load_bvh(p), animation.load_bvh(rp)
            assert a["names"] == b["names"] and np.array_equal(a["offsets"], b["offsets"]), k
            assert np.abs(a["positions"] - b["positions"]).max() <= 1e-3, k
            assert np.abs(a["rotations"] - b["rotations"]).max() <= 1e-2, k
        elif k.startswith("trimlen:"):
            from scipy.io import wavfile
            assert len(wavfile.read(os.path.join(out, "trimmed", k[8:]))[1]) == int(v), k


def test_two_runs_write_identical_files(tmp_path):
    g = pin.load_golden()
    _run(g, str(tmp_path), "a")
    _run(g, str(tmp_path), "b")
    for d, _, fns in os.walk(tmp_path / "a"):
        for fn in fns:
            pa = os.path.join(d, fn)
            pb = os.path.join(str(tmp_path / "b"), os.path.relpath(pa, str(tmp_path / "a")))
            if fn == "data_pipeline_conf.json":
                continue                                        # names its own output directory
            assert open(pa, "rb").read() == open(pb, "rb").read(), fn


@pytest.mark.parametrize("n,C,in_dtype", [(n, 3, np.float32) for n in range(4, 9)] + [(n, 2, np.float64) for n in range(4, 9)] +
                         [(2_400_000, 1, np.float32), (9000, 525, np.float64)])
def test_spline_resample_matches_scipy(n, C, in_dtype):
    from zeggs_b200 import ops
    rs = np.random.RandomState(n)
    x = (rs.randn(n, C) * (0.3 if C == 1 else 20.0)).astype(in_dtype)
    if C == 1:
        x = x[:, 0]
    for m in sorted({int(0.9 * n), 1, 2 * n}):
        if n > 10000 and m != int(0.9 * n):
            continue
        ref = griddata(np.linspace(0, n - 1, n), x, np.linspace(0, n - 1, m), method="cubic")
        got = ops.spline_resample(torch.from_numpy(x).cuda(), m).cpu().numpy()
        assert got.shape == ref.shape and got.dtype == np.float64
        assert np.all(np.abs(got - ref) <= 1e-10 * np.maximum(1.0, np.abs(ref))), (n, m, np.abs(got - ref).max())


def _flip_take(T=9000, seed=5):
    from tests import _fixtures as fx
    from zeggs_b200 import synth
    d = fx.skeleton()
    J = len(d["parents"])
    rs = np.random.RandomState(seed)
    offsets = synth.load_stats()["anim_input_mean"][6:6 + 3 * J].reshape(J, 3).astype(np.float64)
    rot = np.cumsum(rs.randn(T, J, 3) * 0.5, axis=0) + 15.0 * np.sin(np.arange(T)[:, None, None] / 50.0 + rs.rand(1, J, 3) * 6.28)
    rot[rs.rand(T, J) < 0.05] += 360.0                        # a full turn negates the quaternion: thousands of hemisphere flips
    rot[:, 0] = np.cumsum(rs.randn(T, 3) * 0.2, axis=0) + np.array([0.0, 25.0, 0.0])
    pos = np.repeat(offsets[None], T, axis=0)
    pos[:, 0] = np.array([0.0, 92.0, 0.0]) + np.cumsum(rs.randn(T, 3) * 0.3, axis=0) * np.array([1.0, 0.05, 1.0])
    return dict(rotations=rot.astype(np.float32), positions=pos.astype(np.float32), parents=np.asarray(d["parents"], np.int32),
                names=d["bone_names"], order="zyx", frametime=d["dt"])


@pytest.mark.parametrize("T", [9000, 9001])
def test_anim_features_match_host_preprocess_animation(T):
    from zeggs_b200 import animation, ops
    anim = _flip_take(T)
    ref = animation.preprocess_animation(anim)
    names = anim["names"]
    got = ops.anim_features(anim["rotations"], anim["positions"], anim["parents"], "zyx", anim["frametime"], names.index("Spine2"),
                            names.index("Hips"), names.index("Head"))
    for k, v in got.items():
        v = v.cpu().numpy().astype(np.float64)
        r = ref[k].astype(np.float64)
        assert v.shape == r.shape, k
        assert np.all(np.abs(v - r) <= 1e-5 * np.maximum(1.0, np.abs(r))), (k, np.abs(v - r).max())
    q = animation.q_from_euler_deg(anim["rotations"].astype(np.float64), "zyx")
    assert (np.sum(q[1:] * q[:-1], -1) < 0).sum() > 1000
    uq = ops.unrolled_quaternions(anim["rotations"], anim["parents"], "zyx").cpu().numpy()
    ref_q = animation.q_unroll(q)
    assert np.array_equal(np.sign(uq[..., 0]) * np.sign(ref_q[..., 0]), np.ones(uq.shape[:2]))   # the same sign on every frame
    assert np.abs(uq - ref_q).max() <= 1e-12


def test_anim_features_reject_short_takes():
    from zeggs_b200 import _lib, ops
    anim = _flip_take(3)
    with pytest.raises(_lib.ZeggsError):
        ops.anim_features(anim["rotations"], anim["positions"], anim["parents"], "zyx", 1 / 60, 3, 0, 5)


def test_masked_moments_match_float64():
    from zeggs_b200 import ops
    rs = np.random.RandomState(3)
    N = 20000
    groups = [rs.randn(N, 3).astype(np.float32) * 5 + 2, rs.randn(N, 75, 3).astype(np.float32), rs.randn(N, 81).astype(np.float32) - 4]
    groups[1][:, 10:20] = rs.randn(1, 10, 3).astype(np.float32)             # constant channels
    rows = np.sort(rs.choice(N, 15000, replace=False)).astype(np.int32)
    mean, std, gstd = ops.masked_moments([torch.from_numpy(g).cuda() for g in groups], torch.from_numpy(rows).cuda())
    mean, std, gstd = mean.cpu().numpy(), std.cpu().numpy(), gstd.cpu().numpy()
    flat = [g.reshape(N, -1)[rows].astype(np.float64) for g in groups]
    rm = np.concatenate([f.mean(0) for f in flat])
    rsd = np.concatenate([f.std(0) for f in flat])
    rg = np.array([f.std() for f in flat])
    assert np.all(np.abs(mean - rm) <= 1e-12 * np.maximum(np.abs(rm), 1e-300) + 1e-15)
    nz = rsd > 0
    assert np.all(np.abs(std[nz] - rsd[nz]) <= 1e-12 * rsd[nz])
    assert np.all(np.abs(gstd - rg) <= 1e-12 * rg)
    const = np.zeros(groups[1].shape[1:], bool)
    const[10:20] = True
    assert np.all(std[3:3 + 225][const.ravel()] == 0.0)
    assert np.count_nonzero(std == 0.0) == 30


def test_train_runs_on_a_pipeline_built_75_joint_dataset(tmp_path):
    """Four 75-joint takes (the shipped skeleton) through the pipeline, then WindowDataset / DeviceWindowDataset and 2 train() iterations."""
    from scipy.io import wavfile
    from tests import _fixtures as fx
    from zeggs_b200 import bvhio, data, synth
    from zeggs_b200.data_pipeline import data_pipeline
    base = tmp_path / "set"
    (base / "original").mkdir(parents=True)
    rows = []
    for k, style in enumerate(["Neutral", "Happy", "Neutral", "Happy"]):
        anim = _flip_take(420, seed=40 + k)
        bvhio.save_bvh(base / "original" / f"t{k}.bvh", anim["positions"], anim["rotations"], anim["parents"], anim["names"], "zyx", 1 / 60)
        x = synth.make_waveforms(1, 16000 * 7, seed=50 + k)[0]
        wavfile.write(base / "original" / f"t{k}.wav", 16000, np.round(x * 20000).astype(np.int16))
        (base / "original" / f"t{k}.csv").write_text("#,Name,Start,End\nR1,S,0:00.000,0:06.900\n")
        rows.append(f"t{k}.wav,10:00:00:00,,,,t{k}.fbx,10:00:00:00,,,,{style},1,10:00:00:10,10:00:06:50,t{k}.bvh,{'TRUE' if k == 3 else 'FALSE'}")
    cols = "audio_filename,audio_start_time,audio_end_time,audio_duration,audio_clap_time,anim_fbx_file,anim_start_time,anim_end_time," \
           "anim_duration,anim_clap_time,style,capture_session,acting_start_time,acting_end_time,anim_bvh,validation"
    (base / "info.csv").write_text(cols + "\n" + "\n".join(rows) + "\n")
    data_pipeline(pin.conf_for(str(base)))
    dproc, ddef = str(base / "processed" / "processed_data.npz"), str(base / "processed" / "data_definition.json")
    ds = data.WindowDataset(ddef, dproc, 64, "example", 64)
    dds = data.DeviceWindowDataset(ddef, dproc, 64, "example", 64)
    assert len(ds.starts) > 0 and len(dds.starts) == len(ds.starts)
    from zeggs_b200.train import train
    to = dict(seed=21, use_gpu=True, resume=False, learning_rate=1e-3, learning_rate_decay=0.999, eps=1e-5, niterations=2 / 1000.0,
              batchsize=4, window=64, style_encoding_type="example", generate_samples_step=1, use_tensorboard=False,
              decoder_engine="fp32", cuda_graph=True, device_dataset=True)
    no = dict(speech_encoder=dict(nhidden=64, speech_encoding_size=64),
              style_encoder=dict(nhidden=512, style_encoding_size=64, example_length=64, type="attn", use_vae=True),
              decoder=dict(nhidden=64))
    state = random.getstate()
    random.seed(0)
    try:
        train(str(tmp_path / "models"), str(tmp_path / "logs"), dproc, ddef, to, no)
    finally:
        random.setstate(state)
    recs = [json.loads(ln) for ln in open(tmp_path / "logs" / "valid_loss.jsonl").read().strip().split("\n")]
    assert recs and all(np.isfinite(r["train_loss"]) for r in recs)
    written = [os.path.join(d, f) for d, _, fs in os.walk(tmp_path / "models") for f in fs]
    assert any(f.endswith(".pt") for f in written), written
