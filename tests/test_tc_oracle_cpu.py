"""CPU checks of oracle/tc_oracle.py, the bf16-operand-matched restatement of the tensor-core decoder engine:
(1) without rounding it IS the reference decoder (outputs and every gradient equal model_oracle's in float64);
(2) the tolerances tests/test_tc_engine_gpu.py asserts against it catch small kernel faults that the fp32-oracle tolerances miss;
(3) the library's tc size functions and ops.tc_eligible agree with the documented hidden-size rule.  No GPU involved."""
import numpy as np
import pytest
import torch

from oracle import model_oracle as mo
from oracle import tc_oracle as tco
from tests._util import NAMES, ensure_built, run_with_grads, tt
from zeggs_b200 import synth


def _case(H, B, T, Z, seed):
    P = synth.make_params(H=H, Z=Z, seed=seed, with_style=False)
    win = tt(synth.make_pose_windows(B, T, seed=seed))
    rs = np.random.RandomState(seed)
    speech = torch.from_numpy(rs.randn(B, T, 64) * 0.5)
    style = torch.from_numpy(rs.randn(B, T, Z))
    cot = [torch.from_numpy(rs.randn(*win[n].shape)) for n in NAMES]
    return P, win, speech, style, cot


@pytest.mark.parametrize("H", [64, 384])
@pytest.mark.parametrize("T", [1, 2, 9])
@pytest.mark.parametrize("Z", [64, 9])
def test_unrounded_tc_oracle_is_the_reference_decoder(H, T, Z):
    """bf16=False: the folded restatement (fold matrix, cfold, root rows, hoisted cond product, split layer-2 adjoint) reproduces
    model_oracle.decoder_forward and its autograd to 1e-9 relative -- outputs per group and every parameter / speech / style gradient."""
    case = _case(H, 3, T, Z, seed=40 + H + T + Z)
    out_r, g_r = run_with_grads(mo.decoder_forward, *case)
    out_t, g_t = run_with_grads(tco.decoder_forward_tc, *case, bf16=False)
    for n, a, b in zip(NAMES, out_t, out_r):
        assert a.shape == b.shape, n
        assert float((a - b).abs().max()) <= 1e-9 * max(1.0, float(b.abs().max())), n
    assert set(g_t) == set(g_r)
    for k in g_r:
        a, b = g_t[k], g_r[k]
        err, sc = float((a - b).abs().max()), float(b.abs().max())
        if T == 1:                          # a one-frame window is the given pose: nothing reaches it
            assert sc == 0.0 and err == 0.0, k
        assert err <= 1e-9 * max(sc, 1e-30) or (sc == 0.0 and err == 0.0), (k, err, sc)


def _worst(out, grads, out_ref, grads_ref):
    fe = tco.forward_errors(out, out_ref)
    ge = {k: tco.rel_l2(grads[k], grads_ref[k]) for k in grads_ref}
    return max(fe.items(), key=lambda kv: kv[1]), max(ge.items(), key=lambda kv: kv[1])


@pytest.fixture(scope="module")
def sensitivity_base():
    case = _case(384, 4, 17, 64, seed=2024)
    return case, run_with_grads(tco.decoder_forward_tc, *case, bf16=True)


@pytest.mark.parametrize("fault", list(tco.PERTURBATIONS) + ["no_rounding"])
def test_tc_tolerances_catch_small_kernel_faults(sensitivity_base, fault):
    """H = 384, B = 4, T = 17: each modelled fault moves some output group by more than TC_FWD_TOL or some gradient by more than
    TC_GRAD_TOL (relative L2) away from the fault-free bf16 restatement.  The printout also shows the fault against the fp32-oracle
    tolerances of the older tensor-core tests, which most of these faults pass."""
    case, (out0, g0) = sensitivity_base
    kw = dict(bf16=False) if fault == "no_rounding" else dict(bf16=True, perturb=fault)
    out, g = run_with_grads(tco.decoder_forward_tc, *case, **kw)
    (fn, fe), (gn, ge) = _worst(out, g, out0, g0)
    print(f"  [{fault}] worst forward {fn} {fe:.3e} (tol {tco.TC_FWD_TOL:.1e}, fp32-oracle tol {tco.FP32_ORACLE_FWD_TOL:.0e})  "
          f"worst gradient {gn} {ge:.3e} (tol {tco.TC_GRAD_TOL:.1e}, fp32-oracle tol {tco.FP32_ORACLE_GRAD_TOL:.0e})  "
          f"caught by the fp32-oracle tolerances: {fe > tco.FP32_ORACLE_FWD_TOL or ge > tco.FP32_ORACLE_GRAD_TOL}")
    assert fe > tco.TC_FWD_TOL or ge > tco.TC_GRAD_TOL, (fault, fn, fe, gn, ge)


@pytest.fixture(scope="module")
def lib():
    ensure_built()
    from zeggs_b200 import _lib
    return _lib.lib()


def test_tc_eligibility_rule_is_one_rule(lib):
    """ops.tc_eligible and the library's forward / backward pack sizes agree with H % 128 == 0 and 384 <= H <= 1024 (no compute calls)."""
    from zeggs_b200 import ops
    for S, Z in ((64, 64), (64, 9)):
        for H in range(64, 1088 + 1, 64):
            rule = H % 128 == 0 and 384 <= H <= 1024
            got = (ops.tc_eligible(H, S, Z), lib.zeggs_decoder_packed_tc_bytes(H, S, Z) > 0,
                   lib.zeggs_decoder_packed_bwd_tc_bytes(H, S, Z) > 0, lib.zeggs_decoder_tc_workspace_bytes(H, S, Z) > 0,
                   lib.zeggs_decoder_bwd_tc_workspace_bytes(H, S, Z) > 0)
            assert got == (rule,) * 5, (H, S, Z, got)
    assert lib.zeggs_decoder_packed_tc_bytes(256, 64, 64) == 0 and lib.zeggs_decoder_packed_bwd_tc_bytes(256, 64, 64) == 0
