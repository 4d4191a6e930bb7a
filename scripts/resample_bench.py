"""Device time of zeggs_resample on 60 s clips (48 kHz stereo int16, 44.1 kHz stereo int16, 22.05 kHz mono int16) -> 16 kHz,
CUDA events around 200 back-to-back launches after warm-up, with the PCM already on the device.  Reports us per clip, output
samples/s, multiply-adds/s (n_out x taps per output) as a share of the H100 SXM data-sheet FP32 rate, and, labelled as such,
the host time of scipy.signal.upfirdn on the same taps.  The card's name and power limit are read in the same run.  Dev tool."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import __graft_entry__ as g

g.build()
from zeggs_b200 import _lib, audio, synth

FP32_FMA_PER_S = 67e12 / 2          # H100 SXM data sheet: 67 TFLOP/s FP32, one multiply-add = 2 FLOP
SECONDS, LAUNCHES = 60, 200


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else f"unknown ({torch.cuda.get_device_name(0)})"


def main():
    from scipy.signal import upfirdn
    dev = torch.device("cuda:0")
    res = {"card": card(), "clip_seconds": SECONDS, "launches": LAUNCHES}
    for fs, C in ((48000, 2), (44100, 2), (22050, 1)):
        x = synth.make_waveforms(C, SECONDS * fs, seed=fs % 97).T
        pcm = np.ascontiguousarray(np.round(x * 20000.0).astype(np.int16))
        r = audio.Resampler(dev, fs)
        pcm_d = torch.from_numpy(pcm).to(dev).reshape(len(pcm), C)
        n_out = audio.resampled_length(len(pcm), fs)
        out = torch.empty(n_out, dtype=torch.float32, device=dev)
        a = _lib.ResampleArgs(n_in=len(pcm), n_out=n_out, channels=C, dtype=0, L=r.L, M=r.M, K4=int(r.table.shape[1]),
                              delay=r.delay, pcm=pcm_d.data_ptr(), taps=r.table.data_ptr(), out=out.data_ptr())
        lib, s = _lib.lib(), _lib.stream_ptr()
        for _ in range(10):
            _lib.check(lib.zeggs_resample(a, s), "zeggs_resample")
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(LAUNCHES):
            lib.zeggs_resample(a, s)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / LAUNCHES
        assert torch.equal(out, r(pcm_d))
        macs = n_out * r.K
        mono = pcm.astype(np.float64).reshape(len(pcm), C).mean(axis=1) / 32768.0
        t0 = time.perf_counter()
        upfirdn(r.h, mono, r.L, r.M)
        host_s = time.perf_counter() - t0
        res[f"{fs}Hz_{C}ch"] = dict(L=r.L, M=r.M, taps_per_output=r.K, n_out=n_out, us_per_clip=round(us, 2),
                                    output_samples_per_s=round(n_out / us * 1e6), gmac_per_clip=round(macs / 1e9, 4),
                                    tmac_per_s=round(macs / us * 1e-6, 3), share_of_fp32_datasheet=round(macs / (us * 1e-6) / FP32_FMA_PER_S, 4),
                                    host_scipy_upfirdn_s=round(host_s, 3))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
