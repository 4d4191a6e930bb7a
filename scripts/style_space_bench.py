"""Time zeggs_b200.style_space.build() on a synthetic processed set of ZeroEGGS size (default: about 570 k rows of 75 joints in
ranges of 20..90 s over 19 labels, the size of the training set of DESIGN.md 7a) with the v1 style encoder's sizes (attention,
hidden 512, Z = 64, VAE, example length 256), written from a seed to a temporary directory.

  build_s       wall time of build() (load, gather, encode, moments, eigendecomposition) to a device synchronise
  encoder_ms    the style encoder over the same number of 256-window batches, CUDA events
  moments_ms    ops.embedding_moments over the space's embeddings, CUDA events, mean of --reps calls
  device, power_limit   read in the same run

    python scripts/style_space_bench.py [--rows 570000] [--reps 20] [--out results.json]
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

L, Z, HIDDEN, BATCH, LABELS = 256, 64, 512, 256, 19


def make_set(d, rows, seed):
    """processed_data.npz / stats.npz / data_definition.json with the pipeline's schema; values are seeded noise."""
    from tests import _fixtures as fx
    from zeggs_b200 import synth
    from zeggs_b200.data import KEYS
    from zeggs_b200.data_pipeline import savez_deterministic
    rs = np.random.default_rng(seed)
    shapes = dict(root_pos=(3,), root_rot=(4,), root_vel=(3,), root_vrt=(3,), lpos=(75, 3), ltxy=(75, 2, 3), lvel=(75, 3),
                  lvrt=(75, 3), gaze_pos=(3,))
    arrays = {"X_audio_features": rs.standard_normal((rows, 81), dtype=np.float32)}
    for k in KEYS:
        arrays["Y_" + k] = rs.standard_normal((rows,) + shapes[k], dtype=np.float32)
    lens = rs.integers(20 * 60, 90 * 60, size=rows // (20 * 60) + 1)
    ends = np.minimum(np.cumsum(lens), rows)
    starts = np.concatenate([[0], ends[:-1]])
    keep = ends - starts > L + 1
    ranges = np.stack([starts[keep], ends[keep]], 1).astype(np.int64)
    st = synth.load_stats()
    stats = dict(ranges_train=ranges, ranges_train_labels=(np.arange(len(ranges)) % LABELS).astype(np.int64),
                 ranges_valid=np.zeros((0, 2), np.int64), ranges_valid_labels=np.zeros(0, np.int64),
                 audio_input_mean=np.zeros(81, np.float32), audio_input_std=np.float64(1.0),
                 anim_input_mean=np.zeros(1134, np.float32), anim_input_std=np.ones(1134, np.float32),
                 anim_output_mean=st["anim_output_mean"], anim_output_std=st["anim_output_std"])
    arrays.update(stats)
    savez_deterministic(os.path.join(d, "processed_data.npz"), arrays)
    savez_deterministic(os.path.join(d, "stats.npz"), stats)
    sk = fx.skeleton()
    with open(os.path.join(d, "data_definition.json"), "w") as f:
        json.dump(dict(dt=sk["dt"], label_names=[f"style{i}" for i in range(LABELS)], parents=sk["parents"], bone_names=sk["bone_names"]), f)
    return len(ranges)


def make_nets(d, seed):
    import torch
    from zeggs_b200 import modules
    torch.manual_seed(seed)
    torch.save(modules.SpeechEncoder(81, 64, 64), os.path.join(d, "speech_encoder.pt"))
    torch.save(modules.Decoder(1134, 1131, 64, Z, 64, 2), os.path.join(d, "decoder.pt"))
    torch.save(modules.StyleEncoder(1134, HIDDEN, Z, type="attn", use_vae=True), os.path.join(d, "style_encoder.pt"))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (r.stdout.strip().split("\n")[0].split(", ") + ["?"])[:2] if r.returncode == 0 else ("?", "?")
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=570_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("style_space_bench needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from zeggs_b200 import generate, ops, style_space
    dev = torch.device("cuda:0")
    with tempfile.TemporaryDirectory() as tmp:
        n_ranges = make_set(tmp, args.rows, 1)
        make_nets(tmp, 2)
        style_space.build(tmp, tmp, example_length=L, device=dev)          # warm-up: module loads, workspaces, positional table
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        space = style_space.build(tmp, tmp, example_length=L, device=dev)
        torch.cuda.synchronize()
        build_s = time.perf_counter() - t0
        N = len(space.labels)
        enc = generate.load_networks(tmp, dev)["style_encoder"]
    x = torch.randn((BATCH, L, 1134), device=dev)
    xr = x[:N % BATCH] if N % BATCH else None
    eps, eps_r = torch.zeros((BATCH, Z), device=dev), torch.zeros((N % BATCH, Z), device=dev)
    with torch.no_grad():
        enc(x, 1.0, eps=eps)
        if xr is not None:
            enc(xr, 1.0, eps=eps_r)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(N // BATCH):
            enc(x, 1.0, eps=eps)
        if xr is not None:
            enc(xr, 1.0, eps=eps_r)
        e1.record()
        torch.cuda.synchronize()
        encoder_ms = e0.elapsed_time(e1)
        E = torch.from_numpy(space.embeddings).to(dev)
        g = torch.from_numpy(space.labels.astype(np.int32)).to(dev)
        ops.embedding_moments(E, g, LABELS)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.reps):
            ops.embedding_moments(E, g, LABELS)
        e1.record()
        torch.cuda.synchronize()
        moments_ms = e0.elapsed_time(e1) / args.reps
    name, power = card()
    res = dict(rows=args.rows, ranges=n_ranges, windows=N, Z=Z, example_length=L, style_hidden=HIDDEN, build_s=round(build_s, 3),
               encoder_ms=round(encoder_ms, 2), moments_ms=round(moments_ms, 4), device=name, power_limit=power)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
