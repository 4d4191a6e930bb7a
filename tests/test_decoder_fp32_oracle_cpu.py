"""CPU checks of oracle/fp32_oracle.py, the restatement of the fp32 decoder engine (normal and FiLM), and of the bounds
tests/test_decoder_fp32_f64_gpu.py asserts against the float64 oracle:
(1) in float64 without a fault the restatement IS the reference decoder: outputs and every gradient equal model_oracle's / film_oracle's
    autograd to 1e-12;
(2) a float32 evaluation (GEMM mode 0: plain; GEMM mode 1: split-bf16 front-end and weight-gradient products) meets every bound with at
    least 4x headroom, at the hidden sizes, batch tiles and window lengths the GPU tests run, the training shape included;
(3) every modelled kernel fault exceeds a bound; the printout shows which of them the older, looser bounds would have missed.
No GPU involved."""
import numpy as np
import pytest
import torch

from oracle import film_oracle as fo
from oracle import fp32_oracle as f3
from oracle import model_oracle as mo
from tests._util import NAMES, run_with_grads, stats_tensors, tt
from zeggs_b200 import synth


def _case(H, B, T, Z, seed, film=False, S=64):
    P = synth.make_params(H=H, S=S, Z=Z, seed=seed, with_style=False, rnn_cond="film" if film else "normal")
    win = tt(synth.make_pose_windows(B, T, seed=seed))
    rs = np.random.RandomState(seed)
    speech = torch.from_numpy((rs.randn(B, T, S) * 0.5).astype(np.float32))
    style = torch.from_numpy(rs.randn(B, T, Z).astype(np.float32))
    cot = [torch.from_numpy(rs.randn(*win[n].shape).astype(np.float32)) for n in NAMES]
    return P, win, speech, style, cot


@pytest.fixture(scope="module")
def stats():
    st = stats_tensors()
    return tuple(st[k] for k in ("anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")) + (st["dt"],)


def _worst(d):
    return max(d.items(), key=lambda kv: kv[1])


@pytest.mark.parametrize("film", [False, True])
@pytest.mark.parametrize("H,B,T,Z", [(16, 3, 5, 9), (64, 33, 4, 64), (544, 2, 3, 64), (128, 2, 1, 64)])
def test_restatement_is_the_reference_decoder(stats, film, H, B, T, Z):
    case = _case(H, B, T, Z, seed=10 + H + B + T, film=film)
    out_r, g_r = run_with_grads(fo.decoder_forward_film if film else mo.decoder_forward, *case)
    out_t, g_t = f3.run(*case, stats, film=film)
    for n, a, b in zip(NAMES, out_t, out_r):
        assert a.shape == b.shape, n
        assert float((a - b).abs().max()) <= 1e-12 * max(1.0, float(b.abs().max())), n
    assert set(g_t) == set(g_r)
    for k in g_r:
        err, sc = float((g_t[k] - g_r[k]).abs().max()), float(g_r[k].abs().max())
        assert err <= 1e-12 * sc or (sc == 0.0 and err == 0.0), (k, err, sc)


# the shapes of the GPU tests: both units-per-CTA values and the full-grid sizes, one k-chunk (H = 16), two and three batch tiles
HEADROOM_CASES = [(16, 33, 17, False), (528, 33, 17, False), (544, 33, 17, False), (1056, 65, 17, False), (208, 1, 17, False),
                  (16, 33, 17, True), (544, 33, 17, True), (1056, 33, 17, True)]


def _headroom(stats, case, film, tag, grads=True):
    out64, g64 = f3.run(*case, stats, film=film, grads=grads)
    for gemm in (False, True):
        out32, g32 = f3.run(*case, stats, dtype=torch.float32, film=film, gemm=gemm, grads=grads)
        fn, fe = _worst(f3.forward_errors(out32, out64))
        msg = f"  [{tag} gemm mode {int(gemm)}] float32 forward worst {fn} {fe:.2e} ({f3.FP32_FWD_TOL / max(fe, 1e-30):.1f}x headroom)"
        assert 4 * fe <= f3.FP32_FWD_TOL, (tag, gemm, fn, fe)
        if grads:
            tol = f3.FP32_GEMM_GRAD_TOL if gemm else f3.FP32_GRAD_TOL
            gn, ge = _worst(f3.grad_errors(g32, g64))
            msg += f"  gradient worst {gn} {ge:.2e} ({tol / max(ge, 1e-30):.1f}x headroom)"
            assert 4 * ge <= tol, (tag, gemm, gn, ge)
        print(msg)


@pytest.mark.parametrize("H,B,T,film", HEADROOM_CASES)
def test_float32_has_4x_headroom(stats, H, B, T, film):
    _headroom(stats, _case(H, B, T, 64, seed=7, film=film), film, f"{'film ' if film else ''}H{H} B{B} T{T}")


def test_float32_has_4x_headroom_training_shape(stats):
    """B = 32, T = 256, H = 1024: forward and full BPTT of the normal decoder, forward of the FiLM decoder."""
    _headroom(stats, _case(1024, 32, 256, 64, seed=7), False, "H1024 B32 T256")
    _headroom(stats, _case(1024, 32, 256, 64, seed=8, film=True), True, "film H1024 B32 T256", grads=False)


@pytest.fixture(scope="module")
def fault_base(stats):
    res = {}
    for film in (False, True):
        case = _case(512, 33, 17, 64, seed=2024, film=film)
        res[film] = case, f3.run(*case, stats, film=film)
    return res


@pytest.mark.parametrize("fault", f3.PERTURBATIONS)
def test_bounds_catch_small_kernel_faults(stats, fault_base, fault):
    """H = 512 (U = 4, 128 CTAs), B = 33 (two batch tiles), T = 17: each modelled fault moves some output group or some gradient of the
    fault-free restatement by more than its bound (the looser mode-1 gradient bound).  Also printed: whether the older bounds -- 2e-4
    forward / 3e-4 max-abs gradient for the normal decoder, 2e-3 forward / 2e-3 rel-L2 gradient for FiLM -- would have caught it."""
    film = fault.startswith("film")
    case, (out0, g0) = fault_base[film]
    out, g = f3.run(*case, stats, film=film, perturb=fault)
    fn, fe = _worst(f3.forward_errors(out, out0))
    gn, ge = _worst(f3.grad_errors(g, g0))
    rl = max(f3.rel_l2(g[k], g0[k]) for k in g0)
    if film:
        old = fe > f3.OLD_FILM_TOL or rl > f3.OLD_FILM_TOL
    else:
        old = fe > f3.OLD_FWD_TOL or ge > f3.OLD_GRAD_TOL
    print(f"  [{fault}] forward worst {fn} {fe:.2e} (bound {f3.FP32_FWD_TOL:.0e})  gradient worst {gn} {ge:.2e} "
          f"(bound {f3.FP32_GEMM_GRAD_TOL:.0e}), rel-L2 {rl:.2e}  caught by the older bounds: {old}")
    assert fe > f3.FP32_FWD_TOL or ge > f3.FP32_GEMM_GRAD_TOL, (fault, fn, fe, gn, ge)
