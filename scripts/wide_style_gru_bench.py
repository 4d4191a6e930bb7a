"""Train-step and long-example times of the GRU style encoder at style hidden 512, 1056, 1536 and 2112 (1536 and 2112 run at 16 units per
CTA, reading W_hh from L2 / HBM every step).

  * train step: B=32, T=256, decoder H=1024 (tensor-core engine), GRU style encoder with the VAE, style example T_ex=384, the whole step
    captured as a CUDA graph and replayed, timed with CUDA events (best of --rounds);
  * generation: the style encoder's forward on one T_ex=3600 example (B=1, no eps), as generate_gesture runs it.

Also reported per width: W_hh's fp32 bytes (what one forward step reads across the grid), and those bytes times the 3599 steps after the
first over the whole generation forward: a lower bound on the recurrence's read rate, to set against the card's L2 and HBM bandwidth.
One TrainStep at a time (a captured step keeps the addresses of ops.WS).  Prints a table and one JSON line with the card's name and
power limit.

    python scripts/wide_style_gru_bench.py [--steps 10] [--warmup 3] [--rounds 3] [--gen-rounds 3] [--Hs 512 1056 1536 2112]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from film_bench import make_batch  # noqa: E402


def _load(mod, P, prefix, dev):
    mod.load_state_dict({k[len(prefix):]: torch.from_numpy(v) for k, v in P.items() if k.startswith(prefix)})
    return mod.to(dev)


def time_train(Hs, dev, batch, args):
    from zeggs_b200 import modules, ops, synth
    from zeggs_b200.train import TrainStep
    P = synth.make_params(H=1024, seed=1, style_hidden=Hs, style_type="gru")
    se = _load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", dev)
    st = _load(modules.StyleEncoder(1134, Hs, 64, type="gru", use_vae=True), P, "style_encoder.", dev)
    de = _load(modules.Decoder(1134, 1131, 64, 64, 1024, 2), P, "decoder.", dev)
    stats = synth.load_stats()
    s = TrainStep(se, de, st, stats, stats["parents"], float(stats["dt"]), use_graph=True)
    for _ in range(args.warmup):
        s.step(batch)
    torch.cuda.synchronize()
    rounds = []
    for _ in range(args.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            loss = s.step(batch)
        e1.record()
        torch.cuda.synchronize()
        rounds.append(e0.elapsed_time(e1) / args.steps)
    assert torch.isfinite(loss).all()
    del s
    ops.WS.bufs.clear()
    return rounds


def time_generate(Hs, dev, args, T=3600):
    from zeggs_b200 import modules, ops, synth
    P = synth.make_params(H=64, seed=2, style_hidden=Hs, style_type="gru")
    st = _load(modules.StyleEncoder(1134, Hs, 64, type="gru", use_vae=True), P, "style_encoder.", dev).eval()
    x = torch.from_numpy(synth.make_style_example(1, T, seed=4)).to(dev)
    rounds = []
    with torch.no_grad():
        ops.style_encoder_fwd(st, x, None, None, 1.0)
        torch.cuda.synchronize()
        for _ in range(args.gen_rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            outs = ops.style_encoder_fwd(st, x, None, None, 1.0)[0]
            e1.record()
            torch.cuda.synchronize()
            rounds.append(e0.elapsed_time(e1))
    assert all(torch.isfinite(o).all() for o in outs if o is not None)
    del st
    ops.WS.bufs.clear()
    return rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--gen-rounds", type=int, default=3)
    ap.add_argument("--Hs", type=int, nargs="+", default=[512, 1056, 1536, 2112])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wide_style_gru_bench needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from zeggs_b200 import ops
    ops.set_decoder_engine("auto")
    dev = torch.device("cuda:0")
    batch = make_batch(dev)
    rows = []
    for Hs in args.Hs:
        tr = time_train(Hs, dev, batch, args)
        gen = time_generate(Hs, dev, args)
        whh = 4 * 3 * Hs * Hs
        rows.append({"style_hidden": Hs, "train_step_ms": min(tr), "train_rounds_ms": tr, "generate_T3600_ms": min(gen),
                     "generate_rounds_ms": gen, "whh_MB": whh / 1e6, "whh_read_GBps_lower_bound": whh * 3599 / (min(gen) * 1e-3) / 1e9})
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"{'style H':>8} {'train step ms':>14} {'style fwd T=3600 ms':>20} {'W_hh MB':>8} {'W_hh read GB/s >=':>18}")
    for r in rows:
        print(f"{r['style_hidden']:>8} {r['train_step_ms']:>14.2f} {r['generate_T3600_ms']:>20.1f} {r['whh_MB']:>8.1f} "
              f"{r['whh_read_GBps_lower_bound']:>18.0f}")
    print(json.dumps({"metric": "wide_style_gru", "decoder_H": 1024, "B": 32, "T": 256, "T_ex": 384, "rows": rows,
                      "gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q.stdout.strip()}))


if __name__ == "__main__":
    main()
