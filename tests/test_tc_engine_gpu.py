"""The tensor-core decoder kernels (engine 1) against their own precision contract: oracle/tc_oracle.decoder_forward_tc(bf16=True), the
float64 restatement that rounds every MMA operand to bf16 where the kernels do.  Forward: per pose-channel group max-abs error
<= TC_FWD_TOL * max(1, max|ref|); backward: relative L2 error <= TC_GRAD_TOL for every decoder parameter gradient, dSpeech and dStyle.
Every eligible hidden size runs (U = 4: H = 384, 512; U = 8: H = 640 ... 1024), with the batch / window edges B = 1, B = 33 (two batch
tiles), T = 2 (one recurrent step) and T = 1 (no recurrence).  Each case also prints its error against the fp32 oracle (model_oracle),
the reference semantics the long-horizon tests in test_gpu_parity.py bound.  Windows stay short: bf16 rounding-boundary flips of h
compound once the recurrence runs free."""
import numpy as np
import pytest
import torch

from oracle import model_oracle as mo
from oracle import tc_oracle as tco
from tests._util import NAMES, ensure_built, make_decoder, run_with_grads, stats_tensors, tt

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


@pytest.fixture
def engine():
    from zeggs_b200 import ops
    prev = ops.DECODER_ENGINE
    yield ops.set_decoder_engine
    ops.set_decoder_engine(prev)


def _case(H, B, T, Z, seed):
    from zeggs_b200 import synth
    P = synth.make_params(H=H, Z=Z, seed=seed, with_style=False)
    win = tt(synth.make_pose_windows(B, T, seed=seed))
    rs = np.random.RandomState(seed)
    speech = torch.from_numpy((rs.randn(B, T, 64) * 0.5).astype(np.float32))
    style = torch.from_numpy(rs.randn(B, T, Z).astype(np.float32))
    cot = [torch.from_numpy(rs.randn(*win[n].shape).astype(np.float32)) for n in NAMES]
    return P, win, speech, style, cot


def _run_gpu(dev, P, win, speech, style, cot, H, Z, grads):
    """The decoder module on the GPU -> (8 outputs, {name: gradient} or None) for the loss sum(out * cot)."""
    st = stats_tensors(dev)
    dec = make_decoder(P, H, Z=Z, device=dev)
    args = [win[n][:, 0].to(dev) for n in NAMES] + [win["gaze_pos"].to(dev)]
    stats = [st[k] for k in ("anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")]
    if not grads:
        with torch.no_grad():
            out = dec(*args, speech.to(dev), style.to(dev), st["parents"], *stats, st["dt"])
        torch.cuda.synchronize()
        return [o.cpu() for o in out], None
    dec.train()
    sp, sy = speech.to(dev).requires_grad_(True), style.to(dev).requires_grad_(True)
    out = dec(*args, sp, sy, st["parents"], *stats, st["dt"])
    named = dict(dec.named_parameters())
    keys = sorted("decoder." + k for k in named)
    g = torch.autograd.grad(sum((o * c.to(dev)).sum() for o, c in zip(out, cot)), [named[k[len("decoder."):]] for k in keys] + [sp, sy])
    torch.cuda.synchronize()
    return [o.detach().cpu() for o in out], {k: v.cpu() for k, v in zip(keys + ["speech", "style"], g)}


FWD_CASES = [(H, B, T, 64) for H in (384, 512, 640, 768, 896, 1024) for B, T in ((1, 2), (7, 9), (32, 33))] + \
            [(768, 33, 9, 64), (512, 4, 1, 64), (512, 5, 9, 9)]


@pytest.mark.parametrize("H,B,T,Z", FWD_CASES)
def test_tc_forward_vs_matched_oracle(dev, engine, H, B, T, Z):
    engine("tc")
    case = _case(H, B, T, Z, seed=900 + H + B + T + Z)
    got, _ = _run_gpu(dev, *case, H, Z, grads=False)
    P, win, speech, style, _ = case
    st = stats_tensors()
    ref_args = ([win[n][:, 0].double() for n in NAMES] + [win["gaze_pos"].double(), speech.double(), style.double()] +
                [st[k].double() for k in ("anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")] + [st["dt"]])
    Pd = {k: torch.from_numpy(v).double() for k, v in P.items()}
    with torch.no_grad():
        ref_tc = tco.decoder_forward_tc(Pd, *ref_args, bf16=True)
        ref_32 = mo.decoder_forward(Pd, *ref_args)
    e_tc, e_32 = tco.forward_errors(got, ref_tc), tco.forward_errors(got, ref_32)
    for n, o in zip(NAMES, got):
        assert torch.isfinite(o).all(), n
        print(f"  [tc fwd H{H} B{B} T{T} Z{Z}] {n:9s} vs matched {e_tc[n]:.3e}  vs fp32 oracle {e_32[n]:.3e}  "
              f"ratio {e_32[n] / max(e_tc[n], 1e-30):.1f}")
    bad = {n: e for n, e in e_tc.items() if not e <= tco.TC_FWD_TOL}
    assert not bad, bad


BWD_CASES = [(H, B, T) for H in (384, 640, 896, 1024) for B, T in ((1, 5), (16, 12), (32, 17))] + [(640, 33, 5)]


@pytest.mark.parametrize("H,B,T", BWD_CASES)
def test_tc_backward_vs_matched_oracle(dev, engine, H, B, T):
    """Every decoder parameter gradient, dSpeech and dStyle of the tc forward + BPTT kernels against autograd through the matched
    oracle with the same cotangents (B = 33 runs the two batch tiles through autograd one after the other)."""
    engine("tc")
    case = _case(H, B, T, 64, seed=1300 + H + B + T)
    _, g_got = _run_gpu(dev, *case, H, 64, grads=True)
    _, g_tc = run_with_grads(tco.decoder_forward_tc, *case, bf16=True)
    _, g_32 = run_with_grads(mo.decoder_forward, *case)
    bad = []
    for k in g_tc:
        e_tc, e_32 = tco.rel_l2(g_got[k], g_tc[k]), tco.rel_l2(g_got[k], g_32[k])
        print(f"  [tc bwd H{H} B{B} T{T}] {k:48s} relL2 vs matched {e_tc:.3e}  vs fp32 oracle {e_32:.3e}  ratio {e_32 / max(e_tc, 1e-30):.1f}")
        if not e_tc <= tco.TC_GRAD_TOL:
            bad.append((k, e_tc))
    assert not bad, bad


@pytest.mark.parametrize("name", ["fp32", "tc"])
def test_one_frame_window(dev, engine, name):
    """T = 1: the window is the given first pose (frame 0 bit-identical), and since no weight and no conditioning input reaches it,
    every parameter gradient, dSpeech and dStyle is exactly zero -- what the reference's autograd gives (model_oracle, checked on the
    CPU by tests/test_tc_oracle_cpu.py).  Both engines."""
    engine(name)
    H = 512
    case = _case(H, 3, 1, 64, seed=77)
    got, g = _run_gpu(dev, *case, H, 64, grads=True)
    win = case[1]
    for n, o in zip(NAMES, got):
        assert o.shape[1] == 1 and torch.equal(o[:, 0], win[n][:, 0]), n
    nonzero = [k for k, v in g.items() if bool((v != 0).any())]
    assert not nonzero, nonzero
