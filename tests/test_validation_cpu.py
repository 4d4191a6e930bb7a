"""The held-out split of the window supplier (zeggs_b200.data) against the reference dataset (ZEGGS/dataset.py), on a synthetic
processed_data.npz whose validation ranges are disjoint from the training ranges:

  * validation tiles: non-overlapping windows at s, s+W, ... inside every validation range, each of them a window the reference's
    own enumeration (dataset.py:82-93) produces for a dataset built on the validation ranges; a range shorter than W + 1 gives none;
  * the style example of every tile: the rows of the reference's get_example (dataset.py:176-204) over the validation range;
  * the sample clips of train.py:520-729: get_sample(split, 30) (dataset.py:206-233) and get_example([s,e], [s,e], L).

What the reference returns is stored as row indices in tests/golden/validation_windows.npz (scripts/make_validation_golden.py);
where the reference tree is importable the test also recomputes it live."""
import json
import os

import numpy as np
import pytest
import torch

from zeggs_b200.data import KEYS, WindowDataset, validation_windows

N_FRAMES = 3000
RANGES_TRAIN = [[0, 300], [300, 420], [420, 2400]]                    # the last one is longer than 30 s: get_sample cuts it
RANGES_VALID = [[2400, 2750], [2750, 2810], [2810, 2875], [2875, 3000]]  # 60 rows (< W+1 at W=64), exactly W+1 = 65 rows, the tail
LABELS_TRAIN, LABELS_VALID = [0, 2, 1], [1, 0, 2, 2]
CASES = [(64, 128), (100, 200), (64, 256)]                             # (window, configured example length)
SAMPLE_LENGTHS = (128, 200)                                            # example lengths of the sample clips


def make_files(d, with_valid=True):
    """processed_data.npz + data_definition.json with the reference's schema (data_pipeline.py:650-684) in directory d."""
    from zeggs_b200 import synth
    st = synth.load_stats()
    rs = np.random.RandomState(13)
    data = {"X_audio_features": rs.randn(N_FRAMES, 81).astype(np.float32)}
    win = synth.make_pose_windows(1, N_FRAMES, seed=14)
    for k in KEYS:
        data["Y_" + k] = win[k][0]
    data.update(ranges_train=np.array(RANGES_TRAIN, np.int64), ranges_train_labels=np.array(LABELS_TRAIN))
    if with_valid:
        data.update(ranges_valid=np.array(RANGES_VALID, np.int64), ranges_valid_labels=np.array(LABELS_VALID))
    for k in ("audio_input_mean", "audio_input_std", "anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std"):
        data[k] = st[k]
    os.makedirs(d, exist_ok=True)
    np.savez(os.path.join(d, "processed_data.npz"), **data)
    details = dict(bone_names=[f"b{i}" for i in range(75)], label_names=["Neutral", "Happy", "Sad"],
                   parents=[int(p) for p in st["parents"]], dt=float(st["dt"]))
    with open(os.path.join(d, "data_definition.json"), "w") as f:
        json.dump(details, f)
    return os.path.join(d, "data_definition.json"), os.path.join(d, "processed_data.npz")


def _rows_of(ex, root_vel):
    """Row indices of the data whose root_vel the example rows carry (the synthetic rows are all distinct)."""
    lut = {tuple(r): i for i, r in enumerate(np.asarray(root_vel).reshape(len(root_vel), -1).tolist())}
    return np.array([lut[tuple(r)] for r in np.asarray(ex)[:, :3].tolist()], dtype=np.int64)


def reference_values(d):
    """What the reference's SGDataset returns on the fixture in directory d -> {name: int array}."""
    from oracle import ref_shim
    ref_shim.install()
    from dataset import SGDataset        # ZEGGS/dataset.py
    ddef, dproc = make_files(d)
    raw = dict(np.load(dproc))
    vd = os.path.join(d, "valid_as_train")
    os.makedirs(vd, exist_ok=True)
    np.savez(os.path.join(vd, "processed_data.npz"), **dict(raw, ranges_train=raw["ranges_valid"],
                                                          ranges_train_labels=raw["ranges_valid_labels"]))
    out = {}
    for W, L in CASES:
        ref = SGDataset(ddef, os.path.join(vd, "processed_data.npz"), W, "example", L)
        out[f"w{W}_enum"] = ref.R[:, 0].numpy().astype(np.int64)
        out[f"w{W}_enum_range"] = ref.S.numpy().astype(np.int64)
        starts, ri = validation_windows(raw["ranges_valid"], W)
        for j, (s, r) in enumerate(zip(starts, ri)):
            ex = ref.get_example(torch.arange(s, s + W), ref.ranges_train[r], L)
            out[f"w{W}_L{L}_ex{j}"] = _rows_of(ex, raw["Y_root_vel"])
    ref = SGDataset(ddef, dproc, 64, "example", 128)
    for split, ranges in (("train", RANGES_TRAIN), ("valid", RANGES_VALID)):
        for i in range(len(ranges)):
            sample = ref.get_sample(split, 30, range_index=i)
            out[f"sample_{split}{i}_se"] = np.array(sample[11], np.int64)
            out[f"sample_{split}{i}_label"] = np.array([int(sample[10])], np.int64)
            assert torch.equal(sample[0][0], torch.from_numpy(raw["X_audio_features"][sample[11][0]:sample[11][1]]))
            for L in SAMPLE_LENGTHS:
                out[f"sample_{split}{i}_L{L}_ex"] = _rows_of(ref.get_example(sample[11], sample[11], L), raw["Y_root_vel"])
    return out


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    return make_files(str(tmp_path_factory.mktemp("valid_ds")))


@pytest.fixture(scope="module", params=["golden", "live"])
def ref(request, golden_dir, tmp_path_factory):
    if request.param == "golden":
        return dict(np.load(os.path.join(golden_dir, "validation_windows.npz")))
    from oracle import ref_shim
    if not ref_shim.available():
        pytest.skip("the reference tree is not importable here; the golden case covers the same values")
    return reference_values(str(tmp_path_factory.mktemp("valid_ref")))


def _example_from_rows(raw, rows):
    n = len(rows)
    parts = [raw["Y_" + k][rows].reshape(n, -1) for k in ("root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt")]
    return torch.from_numpy(np.concatenate(parts + [np.zeros((n, 3), np.float32)], axis=1))


@pytest.mark.parametrize("W,L", CASES)
def test_validation_tiles_match_reference_enumeration(files, ref, W, L):
    ddef, dproc = files
    ds = WindowDataset(ddef, dproc, W, "example", L, seed=0)
    enum = set(zip(ref[f"w{W}_enum"].tolist(), ref[f"w{W}_enum_range"].tolist()))
    assert len(ds.valid_starts) > 0
    for s, r in zip(ds.valid_starts.tolist(), ds.valid_rng_idx.tolist()):
        assert (s, r) in enum, (s, r)                           # a window the reference would also draw, from the same range
    for r, (s0, e0) in enumerate(RANGES_VALID):
        st = np.sort(ds.valid_starts[ds.valid_rng_idx == r])
        assert np.all(st >= s0) and np.all(st + W <= e0)        # inside the range
        assert np.all(np.diff(st) >= W)                         # no overlap
        if e0 - s0 < W + 1:
            assert len(st) == 0, (s0, e0)
    # every tile s0 + kW <= e0 - W - 1 is kept unless the reference's example rule cannot fill L rows for it
    tiles, _ = validation_windows(np.array(RANGES_VALID), W)
    assert len(tiles) == sum((e0 - s0 - 1) // W if e0 - s0 >= W + 1 else 0 for s0, e0 in RANGES_VALID)
    full = [len(ref[f"w{W}_L{L}_ex{j}"]) == L for j in range(len(tiles))]
    assert ds.valid_starts.tolist() == [s for s, f in zip(tiles.tolist(), full) if f]


@pytest.mark.parametrize("W,L", CASES)
def test_validation_examples_match_reference(files, ref, W, L):
    ddef, dproc = files
    raw = dict(np.load(dproc))
    ds = WindowDataset(ddef, dproc, W, "example", L, seed=0)
    ds.example_window_length = 2 * (L // 3)                     # the per-iteration random length must not leak into validation
    b = ds.valid_host_batch(np.arange(len(ds.valid_starts)))
    assert b["style"].shape == (len(ds.valid_starts), L, 1134)
    tiles = validation_windows(np.array(RANGES_VALID), W)[0].tolist()
    for j, s in enumerate(ds.valid_starts.tolist()):
        assert torch.equal(b["style"][j], _example_from_rows(raw, ref[f"w{W}_L{L}_ex{tiles.index(s)}"])), j
        assert torch.equal(b["audio"][j], torch.from_numpy(raw["X_audio_features"][s:s + W]))
        for k in KEYS:
            assert torch.equal(b[k][j], torch.from_numpy(raw["Y_" + k][s:s + W])), k


def test_validation_label_batch(files):
    ddef, dproc = files
    ds = WindowDataset(ddef, dproc, 64, "label", 128, seed=0)
    b = ds.valid_host_batch(np.arange(len(ds.valid_starts)))
    want = torch.zeros(len(ds.valid_starts), 3)
    want[torch.arange(len(ds.valid_starts)), torch.as_tensor(np.array(LABELS_VALID)[ds.valid_rng_idx])] = 1.0
    assert torch.equal(b["style"], want)


def test_validation_draws_nothing_from_the_training_generator(files):
    ddef, dproc = files
    a = WindowDataset(ddef, dproc, 64, "example", 128, seed=4)
    b = WindowDataset(ddef, dproc, 64, "example", 128, seed=4)
    a.valid_host_batch(np.arange(len(a.valid_starts)))
    ha, hb = a.sample_host_batch(5), b.sample_host_batch(5)
    for k in ha:
        assert torch.equal(ha[k], hb[k]), k


@pytest.mark.parametrize("split", ["train", "valid"])
def test_sample_clips_match_reference(files, ref, split):
    ddef, dproc = files
    raw = dict(np.load(dproc))
    ds = WindowDataset(ddef, dproc, 64, "example", 128, seed=0)
    for i in range(len(RANGES_TRAIN if split == "train" else RANGES_VALID)):
        clip, label, se, ri = ds.get_sample(split, 30, range_index=i)
        assert ri == i and se == ref[f"sample_{split}{i}_se"].tolist() and label == int(ref[f"sample_{split}{i}_label"][0])
        s, e = se
        assert torch.equal(clip["audio"][0], torch.from_numpy(raw["X_audio_features"][s:e]))
        for k in KEYS:
            assert clip[k].shape[:2] == (1, e - s) and torch.equal(clip[k][0], torch.from_numpy(raw["Y_" + k][s:e])), k
        for L in SAMPLE_LENGTHS:
            assert torch.equal(ds.get_example(se, se, L), _example_from_rows(raw, ref[f"sample_{split}{i}_L{L}_ex"])), (i, L)
    assert ref["sample_train2_se"].tolist() == [420, 420 + 30 * 60]     # the 30 s cut is exercised


def test_sample_range_picks_follow_the_given_generator(files):
    ddef, dproc = files
    ds = WindowDataset(ddef, dproc, 64, "example", 128, seed=0)
    picks = [ds.get_sample("valid", 30, rs=np.random.RandomState(7))[3] for _ in range(2)]
    assert picks[0] == picks[1] == int(np.random.RandomState(7).randint(len(RANGES_VALID)))


def test_no_validation_split(tmp_path):
    ddef, dproc = make_files(str(tmp_path), with_valid=False)
    ds = WindowDataset(ddef, dproc, 64, "example", 128, seed=0)
    assert len(ds.valid_starts) == 0 and len(ds.ranges_valid) == 0
    d = dict(np.load(dproc))
    np.savez(dproc, **dict(d, ranges_valid=np.zeros((0, 2), np.int64), ranges_valid_labels=np.zeros(0, np.int64)))
    ds = WindowDataset(ddef, dproc, 64, "example", 128, seed=0)
    assert len(ds.valid_starts) == 0
