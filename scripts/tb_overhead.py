"""What the TensorBoard logs of train() cost per step, at the bench geometry (B=32, T=256, H=1024, T_ex=384, tc engine, the step replayed
from a CUDA graph, batches resident in HBM).  Three variants alternate in one process on one TrainStep, `--repeats` times each, in
rotating order:
  none       the step alone;
  collector  what train() does with use_tensorboard: LossLog.push after every step, TensorBoardLog.write of each returned block;
  naive      the reference's way: the step's terms read back with .cpu() after every step, then written.
A repeat times `--steps` steps (a multiple of the 100-step block) with the host clock, up to a device synchronise after the last one,
so the host's writing counts where it holds the GPU up.  The collector starts a block ahead, so a timed repeat writes as many blocks
as it closes: its steady state.  Prints one JSON line: ms/step per variant (median, min, max over the repeats) with the card's name
and power limit.

    python scripts/tb_overhead.py [--steps 300] [--repeats 5] [--warmup 10]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tb_overhead needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from bench import build_stepper, synth_batch
    from zeggs_b200 import ops
    from zeggs_b200.train import LossLog, TensorBoardLog
    ops.set_decoder_engine("tc")
    dev = torch.device("cuda:0")
    torch.manual_seed(1000)
    stepper, _, _ = build_stepper(1024, dev, 1, use_graph=True)
    batch = synth_batch(32, 256, 384, seed=100, device=dev)
    for _ in range(args.warmup):
        stepper.step(batch)
    torch.cuda.synchronize()
    assert stepper.use_graph and len(stepper._graphs) == 1, "the CUDA-graph path did not run"
    K = args.steps
    times = {"none": [], "collector": [], "naive": []}
    with tempfile.TemporaryDirectory() as tmp:
        tb = TensorBoardLog(os.path.join(tmp, "tb"), {"decoder": {"nhidden": 1024}}, {"batchsize": 32, "use_tensorboard": True})

        def none():
            for _ in range(K):
                stepper.step(batch)

        def collector():
            log = LossLog(dev)
            for _ in range(log.hist.shape[0]):             # untimed: the first block, so every timed close writes one
                stepper.step(batch)
                log.push(stepper)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(K):
                stepper.step(batch)
                tb.write("losses", *log.push(stepper))
            torch.cuda.synchronize()
            t = time.perf_counter() - t0
            tb.write("losses", *log.drain())
            return t

        def naive():
            for _ in range(K):
                stepper.step(batch)
                tb.write("losses", [stepper.iteration - 1], stepper.terms.cpu().numpy()[None])

        def timed(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            t = fn()
            torch.cuda.synchronize()
            return (t if t is not None else time.perf_counter() - t0) * 1e3 / K

        order = list(times)
        for r in range(args.repeats):
            for name in order[r % 3:] + order[:r % 3]:
                times[name].append(timed({"none": none, "collector": collector, "naive": naive}[name]))
        tb.close()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"metric": "train_step_ms", "B": 32, "T": 256, "H": 1024, "T_ex": 384, "engine": "tc", "cuda_graph": True, "steps": K,
           "repeats": args.repeats, "gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q.stdout.strip()}
    for name, ts in times.items():
        out[name] = {"median_ms": round(statistics.median(ts), 3), "min_ms": round(min(ts), 3), "max_ms": round(max(ts), 3),
                     "ms": [round(t, 3) for t in ts]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
