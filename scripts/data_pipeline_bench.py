"""Time the device training-set pipeline against the host path on a synthetic ZeroEGGS-sized set (default: 67 takes of 150 s,
75 joints, len_ratios [0.9, 1.0]), built from a seed in a temporary directory.

  device: data_pipeline() end to end (host clock after a synchronise), and per stage on the same takes: BVH parse, stretch
          (ops.spline_resample of positions, unrolled quaternions and audio + quat_to_euler_deg), animation features
          (ops.anim_features), audio features (loudness + mel), statistics (ops.masked_moments), writing (processed_data.npz).
          Device stages are timed with CUDA events.
  host:   animation.preprocess_animation + scipy griddata for the stretch on the same takes.

    python scripts/data_pipeline_bench.py [--takes 67] [--seconds 150] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def make_set(base, takes, seconds, seed):
    from scipy.io import wavfile
    from tests import _fixtures as fx
    from zeggs_b200 import bvhio, synth
    d = fx.skeleton()
    J = len(d["parents"])
    offsets = synth.load_stats()["anim_input_mean"][6:6 + 3 * J].reshape(J, 3).astype(np.float64)
    os.makedirs(os.path.join(base, "original"), exist_ok=True)
    rows = []
    T = int(60 * seconds)
    for k in range(takes):
        rs = np.random.RandomState(seed + k)
        rot = np.cumsum(rs.randn(T, J, 3) * 0.35, axis=0) + 12.0 * np.sin(np.arange(T)[:, None, None] / 37.0 + rs.rand(1, J, 3) * 6.28)
        pos = np.repeat(offsets[None], T, axis=0)
        pos[:, 0] = np.array([0.0, 92.0, 0.0]) + np.cumsum(rs.randn(T, 3) * 0.3, axis=0) * np.array([1.0, 0.05, 1.0])
        bvhio.save_bvh(os.path.join(base, "original", f"{k:03d}.bvh"), pos, rot, d["parents"], d["bone_names"], "zyx", d["dt"])
        x = synth.make_waveforms(1, int(16000 * seconds), seed=seed + 1000 + k)[0]
        wavfile.write(os.path.join(base, "original", f"{k:03d}.wav"), 16000, np.round(x * 20000).astype(np.int16))
        with open(os.path.join(base, "original", f"{k:03d}.csv"), "w") as f:
            f.write(f"#,Name,Start,End\nR1,S,0:00.000,{int(seconds) // 60}:{int(seconds) % 60:02d}.000\n")
        end = int(60 * seconds) - 30
        rows.append(f"{k:03d}.wav,10:00:00:00,,,,{k:03d}.fbx,10:00:00:00,,,,{'Style%d' % (k % 19)},1,10:00:00:10,"
                    f"10:{end // 3600:02d}:{(end // 60) % 60:02d}:{end % 60:02d},{k:03d}.bvh,{'TRUE' if k % 10 == 9 else 'FALSE'}")
    cols = ("audio_filename,audio_start_time,audio_end_time,audio_duration,audio_clap_time,anim_fbx_file,anim_start_time,anim_end_time,"
            "anim_duration,anim_clap_time,style,capture_session,acting_start_time,acting_end_time,anim_bvh,validation")
    with open(os.path.join(base, "info.csv"), "w") as f:
        f.write(cols + "\n" + "\n".join(rows) + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--takes", type=int, default=67)
    ap.add_argument("--seconds", type=float, default=150.0)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--host-takes", type=int, default=None, help="takes timed on the host path (default: all)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("data_pipeline_bench needs a CUDA device")
    import __graft_entry__ as g
    g.build()
    from scipy.interpolate import griddata
    from zeggs_b200 import animation, audio, ops
    from zeggs_b200 import data_pipeline as dp
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip()
    print("card:", card)
    res = dict(card=card, takes=args.takes, seconds_per_take=args.seconds, len_ratios=[0.9, 1.0])
    with tempfile.TemporaryDirectory() as base:
        t0 = time.time()
        make_set(base, args.takes, args.seconds, args.seed)
        print(f"synthetic set written in {time.time() - t0:.1f} s")
        with open(os.path.join(ROOT, "ubisoft-laforge-zeroeggs_b200", "data", "data_pipeline_conf_v1.json")) as f:
            conf = json.load(f)
        conf.update(base_path=base, processed_data_path="processed", info_filename="info.csv", save_trimmed_audio=False,
                    save_trimmed_animation=False)
        t0 = time.time()
        dp.data_pipeline(conf)
        torch.cuda.synchronize()
        res["device_end_to_end_s"] = time.time() - t0

        # per stage on the same takes
        info = dp.read_csv_rows(os.path.join(base, "info.csv"))
        ev = lambda: torch.cuda.Event(enable_timing=True)
        st = dict(parse_s=0.0, stretch_ms=0.0, features_ms=0.0, audio_ms=0.0)
        host = dict(preprocess_animation_s=0.0, griddata_s=0.0)
        n_host = len(info) if args.host_takes is None else min(args.host_takes, len(info))
        Xs, Ys = [], []
        for i, row in enumerate(info):
            t0 = time.time()
            anim = animation.load_bvh(os.path.join(base, "original", row["anim_bvh"]))
            st["parse_s"] += time.time() - t0
            wav = dp._read_take_audio(os.path.join(base, "original", row["audio_filename"]), 16000)
            names = anim["names"]
            jn = [names.index(n) for n in ("Spine2", "Hips", "Head")]
            for r in (0.9, 1.0):
                rot, pos = anim["rotations"], anim["positions"]
                wav_dev = torch.from_numpy(wav).cuda()
                if r != 1.0:
                    e0, e1 = ev(), ev()
                    e0.record()
                    n, J = pos.shape[:2]
                    m = int(r * n)
                    p = ops.spline_resample(torch.from_numpy(pos.reshape(n, -1)).cuda(), m).reshape(m, J, 3)
                    qq = ops.spline_resample(ops.unrolled_quaternions(rot, anim["parents"], "zyx").reshape(n, -1), m).reshape(m, J, 4)
                    e = ops.quat_to_euler_deg(qq, "zyx")
                    wav_dev = ops.spline_resample(wav_dev.float() / 32768.0, int(r * len(wav))).float()
                    e1.record(); torch.cuda.synchronize()
                    st["stretch_ms"] += e0.elapsed_time(e1)
                    rot, pos = e, p
                e0, e1, e2 = ev(), ev(), ev()
                e0.record()
                f = ops.anim_features(rot, pos, anim["parents"], "zyx", anim["frametime"], *jn)
                e1.record()
                x = audio.preprocess_audio(wav_dev, 60, f["lpos"].shape[0], conf["audio_conf"], conf["audio_feature_type"])
                e2.record(); torch.cuda.synchronize()
                st["features_ms"] += e0.elapsed_time(e1)
                st["audio_ms"] += e1.elapsed_time(e2)
                Xs.append(x); Ys.append(f)
            if i < n_host:
                t0 = time.time()
                n = len(anim["rotations"])
                m = int(0.9 * n)
                ot, sp = np.linspace(0, n - 1, n), np.linspace(0, n - 1, m)
                ps = griddata(ot, anim["positions"].reshape(n, -1), sp, method="cubic")
                qs = griddata(ot, animation.q_unroll(animation.q_from_euler_deg(anim["rotations"].astype(np.float64), "zyx")).reshape(n, -1),
                              sp, method="cubic")
                na = len(wav)
                griddata(np.linspace(0, na - 1, na), wav.astype(np.float32) / 32768.0, np.linspace(0, na - 1, int(0.9 * na)), method="cubic")
                host["griddata_s"] += time.time() - t0
                qs = qs.reshape(m, -1, 4)
                qs /= np.linalg.norm(qs, axis=-1, keepdims=True)
                e = np.degrees(dp._q_to_euler(qs, "zyx"))
                t0 = time.time()
                animation.preprocess_animation(dict(anim, rotations=e, positions=ps.reshape(m, -1, 3)))
                animation.preprocess_animation(anim)
                host["preprocess_animation_s"] += time.time() - t0
        groups = [torch.cat([y[k] for y in Ys]) for k in dp.IN_GROUPS] + [torch.cat(Xs)]
        rows = torch.arange(2, groups[0].shape[0] - 2, dtype=torch.int32, device="cuda")
        e0, e1 = ev(), ev()
        e0.record()
        ops.masked_moments(groups, rows)
        e1.record(); torch.cuda.synchronize()
        st["statistics_ms"] = e0.elapsed_time(e1)
        t0 = time.time()
        dp.savez_deterministic(os.path.join(base, "bench_write.npz"), {f"a{i}": g.cpu().numpy() for i, g in enumerate(groups)})
        st["writing_s"] = time.time() - t0
        res["device_stages"] = st
        res["host_takes_timed"] = n_host
        res["host"] = host
        scale = len(info) / max(1, n_host)
        res["host_anim_stretch_features_s_all_takes"] = (host["griddata_s"] + host["preprocess_animation_s"]) * scale
        res["device_anim_stretch_features_s"] = (st["stretch_ms"] + st["features_ms"]) / 1000.0
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=2)


if __name__ == "__main__":
    main()
