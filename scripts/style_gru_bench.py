#!/usr/bin/env python
"""Train-step time with each style encoder at the train_v1 sizes (B=32, T=256, decoder hidden 1024, T_ex=384, style hidden 512, VAE):

    python scripts/style_gru_bench.py [--steps K] [--warmup W] [--types attn,gru]

CUDA-graph replay, lanes on, tensor-core decoder engine, as bench.py's headline.  Prints one JSON line: per style encoder type the
ms per step and the library's encoders_fwd / encoders_bwd spans (CUDA events recorded inside the replayed graph, mean of K
synchronised replays).  The spans cover both encoders (speech and style)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch

from bench import read_spans, synth_batch


def measure(style_type, K, W, device):
    from zeggs_b200 import _lib, modules, synth
    from zeggs_b200.train import TrainStep
    lib = _lib.lib()
    torch.manual_seed(1000)
    P = synth.make_params(H=1024, seed=1234, style_type=style_type)
    ld = lambda m, pre: (m.load_state_dict({k[len(pre):]: torch.from_numpy(v) for k, v in P.items() if k.startswith(pre)}), m.to(device))[1]
    se = ld(modules.SpeechEncoder(81, 64, 64), "speech_encoder.")
    st = ld(modules.StyleEncoder(1134, 512, 64, type=style_type, use_vae=True), "style_encoder.")
    de = ld(modules.Decoder(1134, 1131, 64, 64, 1024, 2), "decoder.")
    stats = synth.load_stats()
    step = TrainStep(se, de, st, stats, stats["parents"], float(stats["dt"]), use_graph=True)
    batch = synth_batch(32, 256, 384, seed=100, device=device)
    step.step(batch)                                   # eager: first sight of the geometry
    lib.zeggs_timing_reset(); lib.zeggs_timing_enable(1)
    step.step(batch)                                   # captured: span events become nodes of the graph
    lib.zeggs_timing_enable(0)
    assert step.use_graph and step._graphs, "the CUDA-graph path did not run"
    for _ in range(W):
        step.step(batch)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(K):
        loss = step.step(batch)
    e1.record()
    torch.cuda.synchronize()
    acc = {"encoders_fwd": 0.0, "encoders_bwd": 0.0}
    for _ in range(K):
        step.step(batch)
        torch.cuda.synchronize()
        sp = read_spans(lib)
        for n in acc:
            acc[n] += sp[n][0]
    out = dict(ms_per_step=round(e0.elapsed_time(e1) / K, 3), loss=float(loss.item()),
               **{n + "_ms": round(v / K, 3) for n, v in acc.items()})
    del step
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--types", default="attn,gru")
    a = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    from zeggs_b200 import ops
    ops.set_decoder_engine("tc")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    res = {t: measure(t, a.steps, a.warmup, device) for t in a.types.split(",")}
    print(json.dumps(dict(config="B=32, T=256, decoder hidden 1024, T_ex=384, style hidden 512, VAE, CUDA graph, lanes, tc engine",
                          gpu=torch.cuda.get_device_name(device), steps=a.steps, results=res)))


if __name__ == "__main__":
    main()
