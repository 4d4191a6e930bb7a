"""Time the device BVH MOTION text paths (csrc/bvh_text.cu) against the host code, on one GPU, in one process.

  parse:   animation.load_bvh of a synthetic 150 s, 75-joint take: device path and host path (host clock, the call ends with the copy of
           the parsed values to the host), the parse kernels alone (CUDA events around zeggs_bvh_parse_motion), and np.fromstring(block,
           sep=" ") over the same MOTION block as the cheapest vectorised host parse.
  format:  bvhio.save_bvh of the same take from CUDA tensors and from numpy arrays (host clock), the format kernels alone (CUDA events).
  callers: generate_gesture wall time for a 10 s and a 60 s clip and data_pipeline() end to end on --takes takes of 150 s, each with the
           device text paths and with them patched out, alternating.

    python scripts/bvh_text_bench.py [--reps 3] [--takes 4] [--out results.json]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


class HostOnly:
    """Patch the device text entry points out, as the GPU tests do to get the host path."""
    def __enter__(self):
        from zeggs_b200 import animation, bvhio
        self.saved = animation._device_parse_available, bvhio._format_motion_device
        animation._device_parse_available = lambda: False
        bvhio._format_motion_device = lambda *a, **k: None

    def __exit__(self, *exc):
        from zeggs_b200 import animation, bvhio
        animation._device_parse_available, bvhio._format_motion_device = self.saved


def timed_kernels(l, name, store):
    """Wrap the library entry point `name` with CUDA events on the current stream; store gets the milliseconds of every call."""
    import torch
    fn = getattr(l, name)

    def wrapped(*a):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = fn(*a)
        e1.record()
        e1.synchronize()
        store.append(e0.elapsed_time(e1))
        return rc
    setattr(l, name, wrapped)


def clock(fn, reps):
    import torch
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return min(out), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--takes", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bvh_text_bench needs a CUDA device")
    import __graft_entry__ as g
    g.build()
    from tests import _fixtures as fx
    from zeggs_b200 import _lib, animation, bvhio
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = dict(card=q.stdout.strip())
    print("card:", res["card"])
    l = _lib.lib()
    parse_ms, format_ms = [], []
    timed_kernels(l, "zeggs_bvh_parse_motion", parse_ms)
    timed_kernels(l, "zeggs_bvh_format_motion", format_ms)
    with tempfile.TemporaryDirectory() as base:
        path = fx.make_synthetic_bvh(os.path.join(base, "take.bvh"), frames=9000, seed=3)
        raw = open(path, "rb").read()
        block = raw.split(b"Frame Time:", 1)[1].split(b"\n", 1)[1]
        nvals = 9000 * 228
        res["take"] = dict(frames=9000, joints=75, file_bytes=len(raw), motion_bytes=len(block), values=nvals)
        animation.load_bvh(path)                                                    # warm-up
        parse_ms.clear()
        dev_s, _ = clock(lambda: animation.load_bvh(path), args.reps)
        kern_ms = min(parse_ms)
        with HostOnly():
            host_s, _ = clock(lambda: animation.load_bvh(path), args.reps)
        text = block.decode("ascii")
        np_s, _ = clock(lambda: np.fromstring(text, sep=" "), args.reps)
        mb = len(block) / 1e6
        res["parse"] = dict(device_call_s=dev_s, device_kernels_ms=kern_ms, host_call_s=host_s, numpy_fromstring_s=np_s,
                            device_call_MB_s=mb / dev_s, device_kernels_MB_s=mb / (kern_ms / 1e3), host_call_MB_s=mb / host_s,
                            numpy_fromstring_MB_s=mb / np_s, device_kernels_values_s=nvals / (kern_ms / 1e3),
                            host_call_values_s=nvals / host_s)
        print("parse", json.dumps(res["parse"]))

        a = animation.load_bvh(path)
        d = fx.skeleton()
        pos_d, rot_d = torch.from_numpy(a["positions"]).cuda(), torch.from_numpy(a["rotations"]).cuda()
        out = os.path.join(base, "w.bvh")
        bvhio.save_bvh(out, pos_d, rot_d, d["parents"], d["bone_names"], "zyx", d["dt"])      # warm-up
        format_ms.clear()
        fdev_s, _ = clock(lambda: bvhio.save_bvh(out, pos_d, rot_d, d["parents"], d["bone_names"], "zyx", d["dt"]), args.reps)
        fk_ms = min(format_ms)
        dev_bytes = open(out, "rb").read()
        fhost_s, _ = clock(lambda: bvhio.save_bvh(out, a["positions"], a["rotations"], d["parents"], d["bone_names"], "zyx", d["dt"]),
                           args.reps)
        assert open(out, "rb").read() == dev_bytes
        mb = len(block) / 1e6
        res["format"] = dict(device_call_s=fdev_s, device_kernels_ms=fk_ms, host_call_s=fhost_s, device_kernels_MB_s=mb / (fk_ms / 1e3),
                             device_kernels_values_s=nvals / (fk_ms / 1e3), host_call_values_s=nvals / fhost_s)
        print("format", json.dumps(res["format"]))

        # generate_gesture, 10 s and 60 s clips, device text paths on and off, alternating
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from tests.test_bvh_text_gpu import _generate_setup
        from zeggs_b200 import generate
        net, data = _generate_setup(Path(base))
        style = Path(fx.make_synthetic_bvh(os.path.join(base, "style.bvh"), frames=9000, seed=4))
        res["generate_gesture"] = {}
        for secs in (10, 60):
            wav = Path(fx.make_wav(os.path.join(base, f"speech{secs}.wav"), seconds=float(secs)))
            call = lambda r: generate.generate_gesture(wav, [(style, None)], net, data, Path(base) / r, style_encoding_type="example",
                                                       file_name="out", first_pose=style, temperature=1e6, seed=1234, use_gpu=True)
            call("warm")
            times = dict(device=[], host=[])
            for _ in range(args.reps):
                times["device"].append(clock(lambda: call("dev"), 1)[0])
                with HostOnly():
                    times["host"].append(clock(lambda: call("host"), 1)[0])
            assert (Path(base) / "dev" / "out.bvh").read_bytes() == (Path(base) / "host" / "out.bvh").read_bytes()
            res["generate_gesture"][f"{secs}s"] = dict(device_s=min(times["device"]), host_s=min(times["host"]), all=times)
            print("generate_gesture", secs, json.dumps(res["generate_gesture"][f"{secs}s"]))

        # data_pipeline() end to end
        from data_pipeline_bench import make_set
        from zeggs_b200 import data_pipeline as dp
        dpb = os.path.join(base, "dp")
        make_set(dpb, args.takes, 150.0, 0)
        with open(os.path.join(ROOT, "ubisoft-laforge-zeroeggs_b200", "data", "data_pipeline_conf_v1.json")) as f:
            conf = json.load(f)
        conf.update(base_path=dpb, info_filename="info.csv", save_trimmed_audio=False, save_trimmed_animation=True)
        times = dict(device=[], host=[])
        for i in range(args.reps):
            for mode in ("device", "host"):
                c = dict(conf, processed_data_path=f"p_{mode}")
                if mode == "host":
                    with HostOnly():
                        times[mode].append(clock(lambda: dp.data_pipeline(c), 1)[0])
                else:
                    times[mode].append(clock(lambda: dp.data_pipeline(c), 1)[0])
                shutil.rmtree(os.path.join(dpb, f"p_{mode}"))
        res["data_pipeline"] = dict(takes=args.takes, seconds_per_take=150, save_trimmed_animation=True, device_s=min(times["device"]),
                                    host_s=min(times["host"]), all=times)
        print("data_pipeline", json.dumps(res["data_pipeline"]))
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
