"""Train-step time of the FiLM-conditioned decoder (rnn_cond "film") beside the normal one, in the same process, at the v1 training
sizes (B=32, T=256, H=1024, attention style encoder with the VAE, style example T_ex=384): the whole step (encoders, decoder window
and BPTT, loss, RAdam) captured as a CUDA graph and replayed, timed with CUDA events.  One TrainStep at a time: a captured step keeps
the addresses of the library's grow-only workspaces (ops.WS), which a second decoder with larger workspaces would reallocate under
it.  Prints one JSON line with the card's name and power limit.

    python scripts/film_bench.py [--steps 20] [--warmup 3] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def make_step(rnn_cond, dev, H=1024):
    from zeggs_b200 import modules, synth
    from zeggs_b200.train import TrainStep
    P = synth.make_params(H=H, seed=1, rnn_cond=rnn_cond)

    def ld(m, prefix):
        m.load_state_dict({k[len(prefix):]: torch.from_numpy(v) for k, v in P.items() if k.startswith(prefix)})
        return m.to(dev)
    se = ld(modules.SpeechEncoder(81, 64, 64), "speech_encoder.")
    st = ld(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), "style_encoder.")
    de = ld(modules.Decoder(1134, 1131, 64, 64, H, 2, rnn_cond=rnn_cond), "decoder.")
    stats = synth.load_stats()
    return TrainStep(se, de, st, stats, stats["parents"], float(stats["dt"]), use_graph=True)


def make_batch(dev, B=32, T=256, T_ex=384, seed=3):
    from zeggs_b200 import synth
    b = {k: torch.from_numpy(v).to(dev) for k, v in synth.make_pose_windows(B, T, seed=seed).items()}
    b["audio"] = torch.from_numpy(synth.make_audio_features(B, T, seed=seed)).to(dev)
    b["style"] = torch.from_numpy(synth.make_style_example(B, T_ex, seed=seed)).to(dev)
    return b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("film_bench needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from zeggs_b200 import ops
    ops.set_decoder_engine("fp32")          # the FiLM decoder runs on the fp32 engine: time both decoders on it
    dev = torch.device("cuda:0")
    batch = make_batch(dev)
    times = {}
    for c in ("normal", "film"):
        s = make_step(c, dev)
        for _ in range(args.warmup):
            s.step(batch)
        torch.cuda.synchronize()
        times[c] = []
        for _ in range(args.rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                s.step(batch)
            e1.record()
            torch.cuda.synchronize()
            times[c].append(e0.elapsed_time(e1) / args.steps)
        del s
        ops.WS.bufs.clear()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"metric": "train_step_ms", "B": 32, "T": 256, "H": 1024, "T_ex": 384, "engine": "fp32",
           "normal_ms": min(times["normal"]), "film_ms": min(times["film"]), "rounds_ms": times,
           "gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q.stdout.strip()}
    out["film_over_normal"] = out["film_ms"] / out["normal_ms"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
