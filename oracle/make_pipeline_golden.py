"""Generate tests/golden/data_pipeline.npz: a synthetic mini-dataset run through the UNMODIFIED reference data_pipeline
(ZEGGS/data_pipeline.py:234, imported via oracle/ref_shim.py), len_ratios [0.9, 1.0], loudness normalisation on (the
oracle-backed pyloudnorm stub of make_golden.py), PYTHONHASHSEED fixed.

The mini-dataset: a 10-joint BVH skeleton (Hips with 6 channels, Spine2, Head, ...), 3 training takes and 1 validation take in 2
styles, 16 kHz int16 WAVs of 2.2 s, speaker-timing CSVs mixing R and non-R rows (some running past the end of the audio), and an info.csv in the real manifest's
column layout whose timecodes make np.round differ from truncation.  The golden keeps the input files' bytes, so the inputs can be
rebuilt without the reference, every output array, the trimmed BVH text of the first take (both ratios) and the length and
sample hash of every trimmed WAV.  Acting regions of 80-90 frames keep the file small.

    python -m oracle.make_pipeline_golden
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "data_pipeline.npz")
HASHSEED = "7"

NAMES = ["Hips", "Spine", "Spine1", "Spine2", "Neck", "Head", "LeftShoulder", "LeftArm", "RightShoulder", "RightArm"]
PARENTS = [-1, 0, 1, 2, 3, 4, 3, 6, 3, 8]
OFFSETS = np.array([[0, 92, 0], [0, 8, 0.5], [0, 9, 0], [0, 9, -0.5], [0, 12, 1], [0, 8, 1.5], [3, 7, 0], [12, 0, 0], [-3, 7, 0],
                    [-12, 0, 0]], dtype=np.float64)
FS = 16000
# (audio, style, validation, audio_start, anim_start, acting_start, acting_end, speaker rows (#, start, end))
TAKES = [
    ("001_Happy_0", "Happy", "FALSE", "10:00:00:05", "10:00:00:07", "10:00:00:33", "10:00:02:03",
     [("R1", "0:00.250", "0:01.100"), ("O1", "0:01.100", "0:01.400"), ("R2", "0:01.400", "0:02.450")]),
    ("002_Sad_0", "Sad", "FALSE", "11:30:10:11", "11:30:10:30", "11:30:10:59", "11:30:12:21",
     [("R1", "0:00.100", "0:02.500")]),
    ("003_Happy_1", "Happy", "FALSE", "12:01:00:00", "12:01:00:09", "12:01:00:35", "12:01:01:53",
     [("R1", "0:00.300", "0:00.900"), ("S1", "0:00.900", "0:01.300"), ("R2", "0:01.300", "0:01.950"), ("O2", "0:01.950", "0:02.600")]),
    ("004_Sad_1", "Sad", "TRUE", "09:15:20:13", "09:15:20:28", "09:15:20:55", "09:15:22:16",
     [("O1", "0:00.000", "0:00.500"), ("R1", "0:00.500", "0:02.400")]),
]
INFO_COLS = ["audio_filename", "audio_start_time", "audio_end_time", "audio_duration", "audio_clap_time", "anim_fbx_file", "anim_start_time",
             "anim_end_time", "anim_duration", "anim_clap_time", "style", "capture_session", "acting_start_time", "acting_end_time",
             "anim_bvh", "validation"]


def conf_for(base):
    with open(os.path.join(ROOT, "ubisoft-laforge-zeroeggs_b200", "data", "data_pipeline_conf_v1.json")) as f:
        conf = json.load(f)
    conf.update(base_path=str(base), processed_data_path="processed", info_filename="info.csv")
    return conf


def write_inputs(base):
    """The mini-dataset's files under base/ (info.csv) and base/original/ -> {relative path: bytes}."""
    from scipy.io import wavfile
    from zeggs_b200 import bvhio, synth
    orig = os.path.join(base, "original")
    os.makedirs(orig, exist_ok=True)
    rows = []
    for k, (name, style, valid, a0, m0, s, e, spk) in enumerate(TAKES):
        rs = np.random.RandomState(100 + k)
        T = 130
        rot = np.cumsum(rs.randn(T, len(NAMES), 3) * 0.8, axis=0) + 10.0 * np.sin(np.arange(T)[:, None, None] / 11.0 + rs.rand(1, len(NAMES), 3) * 6)
        rot[:, 0] = np.cumsum(rs.randn(T, 3) * 0.5, axis=0) + np.array([20.0 * k, 15.0, 0.0])
        pos = np.repeat(OFFSETS[None], T, axis=0)
        pos[:, 0] = OFFSETS[0] + np.cumsum(rs.randn(T, 3) * 0.4, axis=0) * np.array([1.0, 0.05, 1.0]) + np.array([5.0 * k, 0.0, -3.0])
        bvhio.save_bvh(os.path.join(orig, name + ".bvh"), pos, rot, PARENTS, NAMES, "zyx", 1.0 / 60.0, offsets=OFFSETS)
        x = synth.make_waveforms(1, int(FS * 2.2), seed=200 + k)[0]
        wavfile.write(os.path.join(orig, name + ".wav"), FS, np.round(x * 20000.0).astype(np.int16))
        with open(os.path.join(orig, name + ".csv"), "w") as f:
            f.write("#,Name,Start,End\n")
            for tag, t0, t1 in spk:
                f.write(f"{tag},Speaker,{t0},{t1}\n")
        rows.append({"audio_filename": name + ".wav", "audio_start_time": a0, "audio_end_time": "", "audio_duration": "",
                     "audio_clap_time": "", "anim_fbx_file": name + ".fbx", "anim_start_time": m0, "anim_end_time": "",
                     "anim_duration": "", "anim_clap_time": "", "style": style, "capture_session": "1", "acting_start_time": s,
                     "acting_end_time": e, "anim_bvh": name + ".bvh", "validation": valid})
    with open(os.path.join(base, "info.csv"), "w") as f:
        f.write(",".join(INFO_COLS) + "\n")
        for r in rows:
            f.write(",".join(r[c] for c in INFO_COLS) + "\n")
    files = {}
    for d, _, fns in os.walk(base):
        for fn in fns:
            p = os.path.join(d, fn)
            files[os.path.relpath(p, base)] = open(p, "rb").read()
    return files


def _run_reference(base):
    """Child process (fixed PYTHONHASHSEED): the reference pipeline on the files under base."""
    sys.path.insert(0, ROOT)
    from oracle import ref_shim
    from oracle.make_golden import _pyloudnorm_stub
    ref_shim.install()
    _pyloudnorm_stub()
    import data_pipeline as ref_dp                     # ZEGGS/data_pipeline.py
    ref_dp.data_pipeline(conf_for(base))


def main():
    with tempfile.TemporaryDirectory() as base:
        files = write_inputs(base)
        env = dict(os.environ, PYTHONHASHSEED=HASHSEED, PYTHONPATH=ROOT)
        subprocess.run([sys.executable, "-m", "oracle.make_pipeline_golden", "--reference", base], check=True, env=env, cwd=ROOT)
        out_dir = os.path.join(base, "processed")
        g = {"file:" + k: np.frombuffer(v, dtype=np.uint8) for k, v in files.items()}
        with np.load(os.path.join(out_dir, "processed_data.npz")) as d:
            g.update({"out:" + k: d[k] for k in d.files})
        with np.load(os.path.join(out_dir, "stats.npz")) as d:
            g["stats_keys"] = np.array(sorted(d.files))
        g["data_definition"] = np.frombuffer(open(os.path.join(out_dir, "data_definition.json"), "rb").read(), dtype=np.uint8)
        for folder in ("train", "valid"):
            d = os.path.join(out_dir, "trimmed", folder)
            for fn in sorted(os.listdir(d)):
                p = os.path.join(d, fn)
                if fn.endswith(".bvh"):
                    if fn.startswith(TAKES[0][0]):
                        g[f"trim:{folder}/{fn}"] = np.frombuffer(open(p, "rb").read(), dtype=np.uint8)
                else:
                    from scipy.io import wavfile
                    x = wavfile.read(p)[1]
                    g[f"trimlen:{folder}/{fn}"] = np.array(len(x))
                    g[f"trimsha:{folder}/{fn}"] = np.array(hashlib.sha256(x.tobytes()).hexdigest())
    np.savez_compressed(GOLD, **g)
    print("data_pipeline golden:", os.path.getsize(GOLD), "bytes")


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--reference":
        _run_reference(sys.argv[2])
    else:
        main()
