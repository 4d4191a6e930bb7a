"""Cost of the training monitor at the reference configuration (B=32, T=256, H=1024, T_ex=384, tensor-core decoder engine) on a
synthetic processed_data.npz with a ~13 minute validation split: one validate() sweep (device gather + forward-only step per
batch) and one round of sample animations (6 clips of up to 30 s: encoders, decoder, pose -> BVH channels, BVH text), each
timed with the device synchronised, and both amortised over generate_samples_step = 5000 training iterations.

    python scripts/validation_bench.py [--repeats 3] [--valid-minutes 13]

Prints one JSON line.  Writes nothing into the tree (the synthetic data goes to a temporary directory)."""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def make_data(d, valid_minutes, train_minutes=3, range_s=60):
    from zeggs_b200 import synth
    from zeggs_b200.data import KEYS
    st = synth.load_stats()
    n_tr, n_va = int(train_minutes * 3600), int(valid_minutes * 3600)
    N = n_tr + n_va
    rs = np.random.RandomState(0)
    data = {"X_audio_features": (st["audio_input_mean"] + st["audio_input_std"] * rs.randn(N, 81)).astype(np.float32)}
    win = synth.make_pose_windows(1, N, seed=1)
    for k in KEYS:
        data["Y_" + k] = win[k][0]
    cut = lambda a, b: np.array([[s, min(s + range_s * 60, b)] for s in range(a, b, range_s * 60)], np.int64)
    tr, va = cut(0, n_tr), cut(n_tr, N)
    data.update(ranges_train=tr, ranges_train_labels=np.arange(len(tr)) % 3, ranges_valid=va, ranges_valid_labels=np.arange(len(va)) % 3)
    for k in ("audio_input_mean", "audio_input_std", "anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std"):
        data[k] = st[k]
    np.savez(os.path.join(d, "processed_data.npz"), **data)
    with open(os.path.join(d, "data_definition.json"), "w") as f:
        json.dump(dict(bone_names=[f"b{i}" for i in range(75)], label_names=["Neutral", "Happy", "Sad"],
                       parents=[int(p) for p in st["parents"]], dt=float(st["dt"])), f)
    return os.path.join(d, "data_definition.json"), os.path.join(d, "processed_data.npz")


def timed(fn, dev):
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize(dev)
    return (time.perf_counter() - t0) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--valid-minutes", type=float, default=13.0)
    ap.add_argument("--gss", type=int, default=5000)
    args = ap.parse_args()
    from zeggs_b200 import ops
    from zeggs_b200.data import DeviceWindowDataset
    from zeggs_b200.train import TrainStep, build_networks, validate, write_samples
    dev = torch.device("cuda:0")
    ops.set_decoder_engine("tc")
    B, T, H, T_ex = 32, 256, 1024, 384
    with tempfile.TemporaryDirectory() as d:
        ddef, dproc = make_data(d, args.valid_minutes)
        details = json.load(open(ddef))
        ds = DeviceWindowDataset(ddef, dproc, T, "example", T_ex, seed=0, device=dev)
        torch.manual_seed(0)
        se, de, st = build_networks(dict(speech_encoder=dict(nhidden=64, speech_encoding_size=64),
                                         style_encoder=dict(nhidden=512, style_encoding_size=64, type="attn", use_vae=True),
                                         decoder=dict(nhidden=H)), ds.get_shapes(), "example", 3, dev)
        step = TrainStep(se, de, st, ds.stats, details["parents"], details["dt"])
        n_win = len(ds.valid_starts)
        validate(step, ds, B)                                            # warm-up: weight packs, workspaces
        sweep = [timed(lambda: validate(step, ds, B), dev)[0] for _ in range(args.repeats)]
        # the sweep split into its stages: the device gathers alone, then the forward-only steps on pre-gathered batches
        idx = [np.arange(i, min(i + B, n_win)) for i in range(0, n_win, B)]
        gather = [timed(lambda: [ds.valid_batch(ix) for ix in idx], dev)[0] for _ in range(args.repeats)]
        batches = [ds.valid_batch(ix) for ix in idx]
        evals = [timed(lambda: [step.evaluate(b, index=k) for k, b in enumerate(batches)], dev)[0] for _ in range(args.repeats)]
        samples_dir = os.path.join(d, "samples")
        os.makedirs(samples_dir)
        run_samples = lambda rs: write_samples(samples_dir, 0, ds, se, de, st, ds.stats, details, "example", rs, dev)
        run_samples(np.random.RandomState(0))                            # warm-up
        rounds = [timed(lambda: run_samples(np.random.RandomState(1 + r)), dev)[0] for r in range(args.repeats)]
        # the host-side part of a round: the BVH text of its 12 files at the 30 s cap
        from zeggs_b200 import bvhio
        pos, eul = np.zeros((1800, 75, 3), np.float32), np.zeros((1800, 75, 3), np.float32)
        t0 = time.perf_counter()
        for i in range(12):
            bvhio.save_bvh(os.path.join(samples_dir, f"text_{i}.bvh"), pos, eul, details["parents"], details["bone_names"], "zyx", 1 / 60)
        bvh_text_ms = (time.perf_counter() - t0) * 1e3
    med = lambda v: float(sorted(v)[len(v) // 2])
    res = dict(gpu=torch.cuda.get_device_name(dev), B=B, T=T, H=H, T_ex=T_ex, engine="tc", valid_minutes=args.valid_minutes,
               windows=n_win, sweep_ms=round(med(sweep), 2), ms_per_window=round(med(sweep) / n_win, 4),
               gather_ms=round(med(gather), 2), evaluate_ms=round(med(evals), 2), sample_round_ms=round(med(rounds), 1), bvh_text_ms_12_files=round(bvh_text_ms, 1),
               generate_samples_step=args.gss, amortised_ms_per_iteration=round((med(sweep) + med(rounds)) / args.gss, 4),
               sweep_ms_all=[round(x, 2) for x in sweep], sample_round_ms_all=[round(x, 1) for x in rounds])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
