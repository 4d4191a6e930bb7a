"""One process driving two GPUs: the library sets kernel attributes and checks co-residency per device, so the same work on cuda:0 and
then on cuda:1 must run on both and give bitwise-equal results.  Covered: a tensor-core decoder window forward and backward, an fp32
decoder window forward and backward, a split-bf16 gemm_f32 product and the training loss."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests._util import NAMES, ensure_built, loss_case, make_decoder, stats_tensors, tt

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def devs():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    ensure_built()
    return torch.device("cuda:0"), torch.device("cuda:1")


def _decoder_window(dev, engine, H, B, T, seed):
    """Forward and backward of one decoder window on `dev` -> the 8 outputs and every gradient, on the CPU."""
    from zeggs_b200 import ops, synth
    prev = ops.DECODER_ENGINE
    ops.set_decoder_engine(engine)
    try:
        P = synth.make_params(H=H, seed=seed, with_style=False)
        win = tt(synth.make_pose_windows(B, T, seed=seed))
        rs = np.random.RandomState(seed)
        speech = torch.from_numpy((rs.randn(B, T, 64) * 0.5).astype(np.float32)).to(dev).requires_grad_(True)
        style = torch.from_numpy(rs.randn(B, T, 64).astype(np.float32)).to(dev).requires_grad_(True)
        cot = [torch.from_numpy(rs.randn(*win[n].shape).astype(np.float32)).to(dev) for n in NAMES]
        st = stats_tensors(dev)
        dec = make_decoder(P, H, device=dev).train()
        out = dec(*[win[n][:, 0].to(dev) for n in NAMES], win["gaze_pos"].to(dev), speech, style, st["parents"],
                  *[st[k] for k in ("anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")], st["dt"])
        params = [p for _, p in sorted(dec.named_parameters())]
        g = torch.autograd.grad(sum((o * c).sum() for o, c in zip(out, cot)), params + [speech, style])
        torch.cuda.synchronize(dev)
        return [o.detach().cpu() for o in out] + [x.cpu() for x in g]
    finally:
        ops.set_decoder_engine(prev)


def _gemm(dev):
    """C = A B^T + bias through the split-bf16 tensor-core front end (gemm mode 1, the device's own scratch)."""
    from zeggs_b200 import _lib, ops
    rs = np.random.RandomState(3)
    M, N, K = 256, 384, 520
    A = torch.from_numpy(rs.randn(M, K).astype(np.float32)).to(dev)
    B = torch.from_numpy(rs.randn(N, K).astype(np.float32)).to(dev)
    bias = torch.from_numpy(rs.randn(N).astype(np.float32)).to(dev)
    out = torch.empty(M, N, device=dev)
    _lib.check(_lib.lib().zeggs_gemm_f32_ctx(ops.ctx_ptr(dev), 0, M, N, K, A.data_ptr(), K, B.data_ptr(), K, bias.data_ptr(),
                                             out.data_ptr(), N, 0, 0, _lib.stream_ptr()), "zeggs_gemm_f32_ctx")
    torch.cuda.synchronize(dev)
    return [out.cpu()]


def _loss(dev):
    from zeggs_b200 import ops, synth
    from zeggs_b200.train import kl_weight, pack_pose
    O, W, gaze, mu, lv = loss_case(4, 17, seed=21)
    Og, Wg = [o.to(dev) for o in O], [w.to(dev) for w in W]
    par = torch.as_tensor(synth.load_stats()["parents"], dtype=torch.int32, device=dev)
    terms = torch.zeros(19, device=dev)
    _, grads = ops.loss_fwd_bwd(pack_pose(*Og[2:]), Og[0], Og[1], pack_pose(*Wg[2:]), Wg[0], Wg[1], gaze.to(dev), par,
                                float(synth.load_stats()["dt"]), mu.to(dev), lv.to(dev), kl_weight(7000), terms)
    torch.cuda.synchronize(dev)
    return [terms.cpu()] + [g.cpu() for g in grads]


@pytest.mark.parametrize("what", ["tc_window", "fp32_window", "gemm", "loss"])
def test_same_results_on_two_devices(devs, what):
    run = {"tc_window": lambda d: _decoder_window(d, "tc", 512, 5, 9, seed=41),
           "fp32_window": lambda d: _decoder_window(d, "fp32", 64, 33, 9, seed=42),
           "gemm": _gemm, "loss": _loss}[what]
    results = []
    for dev in devs:
        with torch.cuda.device(dev):
            results.append(run(dev))
    assert len(results[0]) == len(results[1])
    for i, (a, b) in enumerate(zip(*results)):
        assert torch.equal(a, b), f"{what}: result {i} differs between {devs[0]} and {devs[1]}"
