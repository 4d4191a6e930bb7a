"""Training-set construction with the reference's call surface (ZEGGS/data_pipeline.py:234-736): recorded takes (BVH + 16 kHz WAV,
info.csv, per-WAV speaker-timing CSVs) in, processed_data.npz / stats.npz / data_definition.json out, as train() reads them.

Host side (this file): manifest and timing CSVs (stdlib csv), silence mask, timecode sync and trim, ranges / labels bookkeeping,
file writing.  Device side: the time-stretch (ops.spline_resample), Euler / quaternion conversions and the per-frame animation
features (ops.anim_features), loudness and mel features (audio.preprocess_audio) and the dataset statistics (ops.masked_moments).
Takes are processed one at a time; the concatenated arrays stay in device memory until the statistics are taken.

    python -m zeggs_b200.data_pipeline -c data_pipeline_conf.json [--label-names Neutral,Happy,...]
"""
import argparse
import csv
import io
import json
import zipfile
from pathlib import Path

import numpy as np
import torch

from . import _lib, animation, audio, bvhio, ops
from .generate import read_wav

ANIM_KEYS = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt", "gaze_pos", "gaze_dir"]
IN_GROUPS = ["root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt", "gaze_dir"]        # anim_input_* order (:581-591)


# ---------------------------------------------------------------------------------------------- host bookkeeping
def read_csv_rows(path):
    with open(path, newline="") as f:
        return list(csv.DictReader(f))


def _truthy(v):
    return str(v).strip().lower() in ("true", "1", "yes")


def silence_mask(rows, n_samples, fs):
    """:307-329: 1 over the speaker-timing rows whose `#` contains R; times M:SS.mmm (only the first three fields are used)."""
    mask = np.zeros(n_samples, dtype=bool)
    for row in rows:
        if "R" in row["#"]:
            t = []
            for key in ("Start", "End"):
                f = [int(num) for num in row[key].replace(".", ":").rsplit(":")]
                t.append(f[0] * 60 * fs + f[1] * fs + int(f[2] * (fs / 1000)))
            mask[t[0]:t[1]] = True
    return mask


def _thirds(tc, audio):
    f = [int(num) for num in tc.rsplit(":")]
    return f[0] * 216000 + f[1] * 3600 + f[2] * 60 + f[3] * (2 if audio else 1)


def trim_bounds(row, audio_sr, anim_fps):
    """:334-400 -> (audio start, audio end, anim start, anim end): audio timecodes at 30 fps, animation and acting at 60 fps."""
    a0 = _thirds(row["audio_start_time"], True)
    m0 = _thirds(row["anim_start_time"], False)
    s = _thirds(row["acting_start_time"], False)
    e = _thirds(row["acting_end_time"], False)
    b = (int(np.round((s - a0) * (audio_sr / 60))), int(np.round((e - a0) * (audio_sr / 60))),
         int(np.round((s - m0) * (anim_fps / 60))), int(np.round((e - m0) * (anim_fps / 60))))
    if min(b) < 0:
        raise ValueError("The timings are incorrect!")
    return b


def stretched_length(len_ratio, n):
    return int(len_ratio * n)


def label_order(info_rows, label_names=None):
    """Default: first appearance in info.csv (the reference's list(set(...)) order depends on PYTHONHASHSEED)."""
    styles = [r["style"] for r in info_rows]
    if label_names is None:
        return list(dict.fromkeys(styles))
    label_names = list(label_names)
    missing = sorted(set(styles) - set(label_names))
    if missing:
        raise _lib.ZeggsError(f"label_names lacks the styles {missing} of info.csv")
    return label_names


def train_rows(ranges_train):
    """Training rows with 2 frames cut from each end of every range (:564-566), in row order."""
    rows = [np.arange(s + 2, e - 2) for s, e in ranges_train if e - 2 > s + 2]
    if not rows:
        raise _lib.ZeggsError("no training rows: every training range is shorter than 5 frames")
    return np.unique(np.concatenate(rows)).astype(np.int32)


def savez_deterministic(path, arrays):
    """np.savez with a fixed member timestamp, so the same arrays give the same bytes (np.load reads it like any .npz)."""
    with zipfile.ZipFile(path, mode="w", compression=zipfile.ZIP_STORED, allowZip64=True) as z:
        for k, v in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(v), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue())


def _q_to_euler(q, order):
    x0, x1, x2, x3 = q[..., 0:1], q[..., 1:2], q[..., 2:3], q[..., 3:4]
    if order == "zyx":
        return np.concatenate([np.arctan2(2.0 * (x0 * x3 + x1 * x2), 1.0 - 2.0 * (x2 * x2 + x3 * x3)),
                               np.arcsin(np.clip(2.0 * (x0 * x2 - x3 * x1), -1.0, 1.0)),
                               np.arctan2(2.0 * (x0 * x1 + x2 * x3), 1.0 - 2.0 * (x1 * x1 + x2 * x2))], axis=-1)
    return np.concatenate([np.arctan2(2.0 * (x1 * x0 - x2 * x3), -x1 * x1 + x2 * x2 - x3 * x3 + x0 * x0),
                           np.arctan2(2.0 * (x2 * x0 - x1 * x3), x1 * x1 - x2 * x2 - x3 * x3 + x0 * x0),
                           np.arcsin(np.clip(2.0 * (x1 * x2 + x3 * x0), -1.0, 1.0))], axis=-1)


def centre_root_in_place(positions, rotations, order):
    """:449-459, joint 0 only.  The reference's `output = anim_data.copy()` is a shallow copy, so these writes land in the take
    itself: the saved BVH and the features computed after it both see the centred root.  offset_rot keeps the first frame's w and y
    components without renormalising, exactly as written there."""
    lrot0 = animation.q_from_euler_deg(rotations[:, 0].astype(np.float64), order)
    off_pos = positions[0:1, 0].astype(np.float64) * np.array([1.0, 0.0, 1.0])
    off_rot = lrot0[0:1] * np.array([1.0, 0.0, 1.0, 0.0])
    inv = animation.q_inv(off_rot)
    positions[:, 0] = animation.q_rot(inv, positions[:, 0] - off_pos)
    rotations[:, 0] = np.degrees(_q_to_euler(animation.q_mul(inv, lrot0), order))


# ---------------------------------------------------------------------------------------------- the pipeline
def _get(conf, key, default=None):
    return conf[key] if key in conf else default


def _check_conf(conf):
    for key in ("save_normalized_animations", "visualize_spectrogram", "visualize_gaze"):
        if _get(conf, key, False):
            raise _lib.ZeggsError(f"conf key {key!r} is set: it needs matplotlib / writes normalised BVHs and has no device path; set it false")


def _read_take_audio(path, fs):
    from scipy.io import wavfile
    file_fs, x = wavfile.read(str(path))
    if x.ndim > 1 or file_fs != fs:
        raise _lib.ZeggsError(f"{path}: {file_fs} Hz, {1 if x.ndim == 1 else x.shape[1]} channel(s); expected {fs} Hz mono "
                              "(the reference converts other formats with SoX: convert the file first)")
    return read_wav(path)             # int16 as is (decoded x / 32768 on the device), other formats rescaled to float32


def data_pipeline(conf, label_names=None, device="cuda"):
    """ZEGGS/data_pipeline.py:234 -> (processed_data, data_definition), writing the same files under base_path/processed_data_path.
    label_names: explicit label order (default: the conf's "label_names", else first appearance in info.csv)."""
    dev = torch.device(device)
    _check_conf(conf)
    len_ratios = conf["len_ratios"]
    base_path = Path(conf["base_path"])
    out_dir = base_path / conf["processed_data_path"]
    out_dir.mkdir(parents=True, exist_ok=True)
    original = base_path / "original"
    with open(out_dir / "data_pipeline_conf.json", "w") as f:
        json.dump(conf, f, indent=4)
    aconf = conf["audio_conf"]
    fs = int(aconf["sampling_rate"])
    feature_type = conf["audio_feature_type"]
    info = read_csv_rows(base_path / conf["info_filename"])
    label_names = label_order(info, label_names if label_names is not None else _get(conf, "label_names"))

    X, Y = [], {k: [] for k in ANIM_KEYS}
    ranges = {"train": [], "valid": []}
    labels = {"train": [], "valid": []}
    cur = 0
    anim = None
    for row in info:
        anim = animation.load_bvh(str(original / row["anim_bvh"]))
        anim_fps = int(np.ceil(1 / anim["frametime"]))
        if anim_fps != 60:
            raise _lib.ZeggsError(f"{row['anim_bvh']}: {anim_fps} fps, the pipeline expects 60")
        names = anim["names"]
        joints = [names.index(n) for n in ("Spine2", "Hips", "Head")]
        wav_path = original / row["audio_filename"]
        wav = _read_take_audio(wav_path, fs)
        mask = silence_mask(read_csv_rows(wav_path.with_suffix(".csv")), len(wav), fs)
        wav = (wav * mask).astype(wav.dtype)
        a0, a1, m0, m1 = trim_bounds(row, fs, anim_fps)
        wav = wav[a0:a1]
        rot0, pos0 = anim["rotations"][m0:m1], anim["positions"][m0:m1]
        folder = "valid" if _truthy(row["validation"]) else "train"
        for len_ratio in len_ratios:
            # every ratio starts from the trimmed take (the reference's ratio 1.0 modifies it in place: DESIGN.md §7)
            rot, pos = rot0.copy(), pos0.copy()
            wav_dev = torch.from_numpy(np.ascontiguousarray(wav)).to(dev)
            if len_ratio != 1.0:
                n, J = pos.shape[0], pos.shape[1]
                m = stretched_length(len_ratio, n)
                pos_dev = ops.spline_resample(torch.from_numpy(pos.reshape(n, -1)).to(dev), m).reshape(m, J, 3)
                q = ops.unrolled_quaternions(rot, anim["parents"], anim["order"], device=dev)
                q = ops.spline_resample(q.reshape(n, -1), m).reshape(m, J, 4)
                rot_dev = ops.quat_to_euler_deg(q, anim["order"])
                if wav_dev.dtype == torch.int16:
                    wav_dev = wav_dev.to(torch.float32) / 32768.0
                wav_dev = ops.spline_resample(wav_dev, stretched_length(len_ratio, len(wav)))
                pos, rot = pos_dev.cpu().numpy(), rot_dev.cpu().numpy()
            stem = row["anim_bvh"].split(".")[0] + "_x_" + str(len_ratio).replace(".", "_")
            if conf["save_trimmed_audio"]:
                (out_dir / "trimmed" / folder).mkdir(parents=True, exist_ok=True)
                _write_trimmed_wav(out_dir / "trimmed" / folder / (stem + ".wav"), wav_dev, fs)
            if conf["save_trimmed_animation"]:
                (out_dir / "trimmed" / folder).mkdir(parents=True, exist_ok=True)
                centre_root_in_place(pos, rot, anim["order"])
                bvhio.save_bvh(out_dir / "trimmed" / folder / (stem + ".bvh"), pos, rot, anim["parents"], names, anim["order"],
                               anim["frametime"], offsets=anim["offsets"])
            nframes = len(rot)
            wav_in = wav_dev if wav_dev.dtype == torch.int16 else wav_dev.to(torch.float32)
            feats = audio.preprocess_audio(wav_in, anim_fps, nframes, aconf, feature_type, device=dev)
            f = ops.anim_features(rot, pos, anim["parents"], anim["order"], anim["frametime"], *joints, device=dev)
            X.append(feats)
            for k in ANIM_KEYS:
                Y[k].append(f[k])
            ranges[folder].append([cur, cur + nframes])
            labels[folder].append(row["style"])
            cur += nframes

    X = torch.cat(X)
    Y = {k: torch.cat(v) for k, v in Y.items()}
    if not bool(torch.isfinite(X).all()):
        raise _lib.ZeggsError("non-finite audio features")
    ranges_train = np.array(ranges["train"], dtype=np.int32).reshape(-1, 2)
    ranges_valid = np.array(ranges["valid"], dtype=np.int32).reshape(-1, 2)
    lab_train = np.array([label_names.index(s) for s in labels["train"]], dtype=np.int32)
    lab_valid = np.array([label_names.index(s) for s in labels["valid"]], dtype=np.int32)

    # statistics (:562-648): per-channel means / stds and pooled stds of every group over the cut training rows
    groups = IN_GROUPS + ["audio"]
    mean, std, gstd = ops.masked_moments([Y[k] for k in IN_GROUPS] + [X], train_rows(ranges_train))
    mean, std, gstd = mean.cpu().numpy(), std.cpu().numpy(), gstd.cpu().numpy()
    widths = [int(Y[k][0].numel()) for k in IN_GROUPS] + [int(X.shape[1])]
    off = np.concatenate([[0], np.cumsum(widths)])
    sl = {g: slice(off[i], off[i + 1]) for i, g in enumerate(groups)}
    in_mean = np.concatenate([mean[sl[g]] for g in IN_GROUPS]).astype(np.float32)
    in_std = np.concatenate([np.repeat(gstd[i] + 1e-10, widths[i]) for i in range(len(IN_GROUPS))]).astype(np.float64)
    out_groups = IN_GROUPS[:-1]
    stats = dict(ranges_train=ranges_train, ranges_valid=ranges_valid, ranges_train_labels=lab_train, ranges_valid_labels=lab_valid,
                 audio_input_mean=mean[sl["audio"]].astype(np.float32), audio_input_std=np.float64(gstd[-1] + 1e-10),
                 anim_input_mean=in_mean, anim_input_std=in_std,
                 anim_output_mean=np.concatenate([mean[sl[g]] for g in out_groups]).astype(np.float32),
                 anim_output_std=np.concatenate([std[sl[g]] for g in out_groups]).astype(np.float32))
    processed = dict(X_audio_features=X.cpu().numpy())
    for k in ANIM_KEYS:
        if k != "gaze_dir":
            processed["Y_" + k] = Y[k].cpu().numpy()
    processed.update(stats)
    data_definition = dict(dt=anim["frametime"], label_names=label_names, parents=[int(p) for p in anim["parents"]],
                           bone_names=list(anim["names"]))
    if conf["save_final_data"]:
        savez_deterministic(out_dir / "processed_data.npz", processed)
        savez_deterministic(out_dir / "stats.npz", stats)
        with open(out_dir / "data_definition.json", "w") as f:
            json.dump(data_definition, f, indent=4)
    print(summary_table(label_names, ranges_train, lab_train, ranges_valid, lab_valid))
    return processed, data_definition


def _write_trimmed_wav(path, wav_dev, fs):
    """audio_files.write_wavefile: float samples * 2^15 cast to int16; int16 samples as they are."""
    from scipy.io import wavfile
    x = wav_dev.cpu().numpy()
    if x.dtype != np.int16:
        x = (x * 2 ** 15).astype(np.int16)
    wavfile.write(str(path), fs, x)


def summary_table(label_names, ranges_train, lab_train, ranges_valid, lab_valid):
    """The per-style table of :702-731 as plain text (frame counts halved as there)."""
    cols, total = [], 0.0
    for i, name in enumerate(label_names):
        tr = np.sum(ranges_train[lab_train == i, 1] - ranges_train[lab_train == i, 0]) / 2 if len(ranges_train) else 0.0
        va = np.sum(ranges_valid[lab_valid == i, 1] - ranges_valid[lab_valid == i, 0]) / 2 if len(ranges_valid) else 0.0
        cols.append((name, [f"{tr} frames - {tr / 60:.1f} secs", f"{va} frames - {va / 60:.1f} secs",
                            f"{tr + va} frames - {(tr + va) / 60:.1f} secs"]))
        total += tr + va
    lines = ["Data Info", " | ".join(["Dataset"] + [c[0] for c in cols])]
    for r, name in enumerate(("Train", "Validation", "Total")):
        lines.append(" | ".join([name] + [c[1][r] for c in cols]))
    lines.append(f"Total length of dataset is {total} frames - {total / 60:.1f} seconds")
    return "\n".join(lines)


def main(argv=None):
    p = argparse.ArgumentParser(description="Build processed_data.npz / stats.npz / data_definition.json from recorded takes.")
    p.add_argument("-c", "--config", required=True, help="data_pipeline_conf.json")
    p.add_argument("--label-names", default=None, help="comma-separated label order (default: first appearance in info.csv)")
    args = p.parse_args(argv)
    with open(args.config) as f:
        conf = json.load(f)
    data_pipeline(conf, label_names=args.label_names.split(",") if args.label_names else None)


if __name__ == "__main__":
    main()
