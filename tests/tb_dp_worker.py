"""Worker of tests/test_tensorboard_gpu.py::test_data_parallel_rows_are_rank_means (launched by torch.distributed.run, one rank per
GPU): LossLog under data parallelism against the mean of the ranks' own per-step terms, and the gradient all-reduces per step."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rank, world, lrank = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", lrank)
    torch.cuda.set_device(dev)
    torch.distributed.init_process_group("nccl", device_id=dev)
    import __graft_entry__ as ge
    if rank == 0:
        ge.build()
    torch.distributed.barrier()
    from zeggs_b200 import ops
    from zeggs_b200.train import LossLog
    from bench import build_stepper, synth_batch
    ops.set_decoder_engine("fp32")
    torch.manual_seed(50 + rank)
    step, _, _ = build_stepper(64, dev, world, use_graph=True)
    step.ar_events = []
    log = LossLog(dev, block=4)
    mine, steps, rows = [], [], []
    for i in range(10):
        step.step(synth_batch(4, 16, 24, seed=100 + 10 * i + rank, device=dev))
        mine.append(step.terms.clone())
        s, r = log.push(step)
        steps += s.tolist(); rows.append(r)
    s, r = log.drain()
    steps += s.tolist(); rows.append(r)
    torch.cuda.synchronize()
    mine = torch.stack(mine)
    every = [torch.empty_like(mine) for _ in range(world)]
    torch.distributed.all_gather(every, mine)
    want = every[0]
    for t in every[1:]:
        want = want + t
    want = (want * (1.0 / world)).cpu().numpy()
    rows = np.concatenate(rows)
    if rank == 0:
        print("TBDPRESULT " + json.dumps(dict(world=world, steps=steps, rows_equal_rank_mean=bool(rows.tobytes() == want.tobytes()),
                                              ranks_differ=bool(not torch.equal(every[0], every[1])), allreduces=len(step.ar_events),
                                              graphed=bool(step.use_graph and len(step._graphs) == 1))))
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
