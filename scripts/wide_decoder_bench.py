"""Train-step and generation time of the fp32 decoder engine at H = 1024, 1536 and 2048 (1536 and 2048 run at 16 units per CTA).

  * train step: B=32, T=256, attention style encoder with the VAE, style example T_ex=384, the whole step captured as a CUDA graph and
    replayed, timed with CUDA events (best of --rounds);
  * generation: the decoder window of a one-minute clip, T=3600 frames at B=1 (speech and style encodings given), forward only.

One TrainStep at a time: a captured step keeps the addresses of the library's grow-only workspaces (ops.WS).  Also reported: the fp32
weights one recurrence step streams (the slices of layer0 / GRU0 / GRU1 / layer2 every CTA reads each step) and the card's name and
power limit.  Prints a table and one JSON line.

    python scripts/wide_decoder_bench.py [--steps 10] [--warmup 3] [--rounds 3] [--gen-rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from film_bench import make_batch, make_step  # noqa: E402

NAMES = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt"]


def step_weight_bytes(H):
    """fp32 bytes of the packed slices one forward step reads: P1 (1136 x 4H), P2 and P3 (H x 6H each), P4 (padded layer-2 rows)."""
    U = 4 if H // 4 <= 132 else (8 if H // 8 <= 132 else 16)
    G = H // U
    n4t = -(-(-(-1131 // G)) // 16)
    return 4 * (1136 * 4 * H + 12 * H * H + G * n4t * 16 * H)


def time_train(H, dev, batch, args):
    from zeggs_b200 import ops
    s = make_step("normal", dev, H=H)
    for _ in range(args.warmup):
        s.step(batch)
    torch.cuda.synchronize()
    rounds = []
    for _ in range(args.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            s.step(batch)
        e1.record()
        torch.cuda.synchronize()
        rounds.append(e0.elapsed_time(e1) / args.steps)
    del s
    ops.WS.bufs.clear()
    return rounds


def time_generate(H, dev, args, T=3600):
    from zeggs_b200 import modules, ops, synth
    P = synth.make_params(H=H, seed=2, with_style=False)
    dec = modules.Decoder(1134, 1131, 64, 64, H, 2)
    dec.load_state_dict({k[len("decoder."):]: torch.from_numpy(v) for k, v in P.items() if k.startswith("decoder.")})
    dec = dec.to(dev).eval()
    st = synth.load_stats()
    f = lambda k: torch.as_tensor(st[k], dtype=torch.float32, device=dev)
    win = {k: torch.from_numpy(v).to(dev) for k, v in synth.make_pose_windows(1, T, seed=5).items()}
    rs = np.random.RandomState(0)
    speech = torch.from_numpy(rs.randn(1, T, 64).astype(np.float32) * 0.5).to(dev)
    style = torch.from_numpy(rs.randn(1, 1, 64).astype(np.float32)).to(dev).repeat(1, T, 1)
    args_ = [win[n][:, 0] for n in NAMES] + [win["gaze_pos"], speech, style, torch.as_tensor(st["parents"]), f("anim_input_mean"),
                                             f("anim_input_std"), f("anim_output_mean"), f("anim_output_std"), float(st["dt"])]
    rounds = []
    with torch.no_grad():
        dec(*args_)
        torch.cuda.synchronize()
        for _ in range(args.gen_rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = dec(*args_)
            e1.record()
            torch.cuda.synchronize()
            rounds.append(e0.elapsed_time(e1))
    assert all(torch.isfinite(o).all() for o in out)
    del dec
    ops.WS.bufs.clear()
    return rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--gen-rounds", type=int, default=3)
    ap.add_argument("--H", type=int, nargs="+", default=[1024, 1536, 2048])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wide_decoder_bench needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from zeggs_b200 import ops
    ops.set_decoder_engine("fp32")
    dev = torch.device("cuda:0")
    batch = make_batch(dev)
    rows = []
    for H in args.H:
        tr = time_train(H, dev, batch, args)
        gen = time_generate(H, dev, args)
        w = step_weight_bytes(H)
        rows.append({"H": H, "train_step_ms": min(tr), "train_rounds_ms": tr, "generate_T3600_ms": min(gen), "generate_rounds_ms": gen,
                     "generate_us_per_frame": 1e3 * min(gen) / 3599, "fwd_step_weight_MB": w / 1e6})
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"{'H':>6} {'train step ms':>14} {'generate T=3600 ms':>19} {'us / frame':>11} {'fwd weights / step MB':>22}")
    for r in rows:
        print(f"{r['H']:>6} {r['train_step_ms']:>14.2f} {r['generate_T3600_ms']:>19.1f} {r['generate_us_per_frame']:>11.2f} "
              f"{r['fwd_step_weight_MB']:>22.1f}")
    print(json.dumps({"metric": "wide_decoder", "engine": "fp32", "B": 32, "T": 256, "T_ex": 384, "rows": rows,
                      "gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q.stdout.strip()}))


if __name__ == "__main__":
    main()
