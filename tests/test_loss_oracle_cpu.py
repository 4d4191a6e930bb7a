"""CPU checks behind tests/test_loss_gpu.py, the training-loss kernel's oracle test.  No GPU involved.

(1) model_oracle.loss_residuals is what train_losses takes |.| of: in float64 its weighted means give the 17 terms to 1e-12.
(2) The sign-aware gradient comparison (tests/_util.loss_ambiguous_frames): at the training shape the fp32 oracle, standing in
    for an exact fp32 kernel, passes it at the GPU test's tolerance but fails a plain whole-tensor comparison even at the old 3e-4
    bound, because some residuals within rounding of zero take the other sign.  So the mask is needed.
(3) Small modelled kernel faults (one term's gradient scaled by 1 +- 1% or 0.1%, its value unchanged) fail the new tolerance;
    most pass the old 3e-4 bound.
(4) TrainStep's parent-array check rejects the trees the loss kernel cannot walk."""
import numpy as np
import pytest
import torch

from oracle import model_oracle as mo
from tests._util import loss_ambiguous_frames, loss_case, masked_grad_errors, oracle_loss_grads
from tests.test_loss_gpu import EXCLUDED_MAX, GRAD_TOL      # clean-frame gradient error / tensor max, on the shipped tree
from zeggs_b200 import synth

OLD_GRAD_TOL = 3e-4      # the earlier whole-tensor bound


def _shipped():
    st = synth.load_stats()
    return np.asarray(st["parents"]), float(st["dt"])


@pytest.mark.parametrize("B,T", [(2, 2), (5, 33)])
def test_residual_means_are_the_train_loss_terms(B, T):
    parents, dt = _shipped()
    O, W, gaze, _, _ = loss_case(B, T, seed=3 + T, copy_frame0=True)
    O, W, gaze = [o.double() for o in O], [w.double() for w in W], gaze.double()
    _, L = mo.train_losses(O, W, gaze, parents, dt)
    R = mo.loss_residuals(O, W, gaze, parents, dt)
    assert set(R) == set(mo.LOSS_NAMES) == set(mo.LOSS_WEIGHTS)
    for k in mo.LOSS_NAMES:
        assert R[k].dtype == torch.float64
        assert R[k].shape[:2] == (B, T - 1 if k in mo.DIFF_TERMS else T), k
        got = mo.LOSS_WEIGHTS[k] * float(R[k].abs().mean())
        assert abs(got - float(L[k])) <= 1e-12 * abs(float(L[k])), (k, got, float(L[k]))


def test_fp32_oracle_needs_the_sign_aware_comparison():
    """B=32, T=256 (the training shape), frame 0 copied from the ground truth as the decoder returns it."""
    parents, dt = _shipped()
    B, T = 32, 256
    O, W, gaze, mu, lv = loss_case(B, T, seed=41, copy_frame0=True)
    _, _, g64 = oracle_loss_grads(O, W, gaze, parents, dt, mu, lv)
    _, _, g32 = oracle_loss_grads(O, W, gaze, parents, dt, mu, lv, dtype=torch.float32)
    amb_y, amb_rot = loss_ambiguous_frames(O, W, gaze, parents, dt)
    frac = max(float(amb_y.float().mean()), float(amb_rot.float().mean()))
    masked = masked_grad_errors(g32, g64, amb_y, amb_rot)
    none = torch.zeros(B, T, dtype=torch.bool)
    whole = masked_grad_errors(g32, g64, none, none)
    print(f"  excluded {amb_y.float().mean():.3f} (dRootRot {amb_rot.float().mean():.3f}); clean-frame worst "
          f"{max(masked.values()):.2e} ({max(masked, key=masked.get)}); whole-tensor worst {max(whole.values()):.2e} "
          f"({max(whole, key=whole.get)})")
    assert frac <= EXCLUDED_MAX
    assert max(masked.values()) <= GRAD_TOL
    assert max(whole.values()) > OLD_GRAD_TOL


def _faulty_loss(scale):
    """train_losses restated on loss_residuals, with term k's gradient scaled by scale[k] and its value unchanged."""
    def fn(O, W, gaze, parents, dt, mu, lv, iteration):
        R = mo.loss_residuals(O, W, gaze, parents, dt)
        L = {}
        for k in mo.LOSS_NAMES:
            r = R[k]
            if k in scale:
                d = (scale[k] - 1.0) * r
                r = r + d - d.detach()
            L[k] = mo.LOSS_WEIGHTS[k] * r.abs().mean()
        kl, kw = mo.compute_kl_div(mu, lv, iteration)
        L["kl_div"] = kw * kl
        return sum(L.values()) / 18.0, L
    return fn


FAULTS = {"root_pos x0.99": {"root_pos": 0.99}, "gaze x0.99": {"gaze": 0.99}, "gaze x0.999": {"gaze": 0.999},
          "ldvt x0.99": {"ldvt": 0.99}, "cvrt x1.01": {"cvrt": 1.01}}


@pytest.fixture(scope="module")
def fault_base():
    parents, dt = _shipped()
    O, W, gaze, mu, lv = loss_case(5, 33, seed=41)
    amb = loss_ambiguous_frames(O, W, gaze, parents, dt)
    _, _, g = oracle_loss_grads(O, W, gaze, parents, dt, mu, lv)
    _, _, g_same = oracle_loss_grads(O, W, gaze, parents, dt, mu, lv, loss_fn=_faulty_loss({}))
    return (O, W, gaze, parents, dt, mu, lv), amb, g, g_same


def test_restated_loss_without_fault_is_the_oracle(fault_base):
    _, amb, g, g_same = fault_base
    e = masked_grad_errors(g_same, g, *amb)
    assert max(e.values()) <= 1e-12, e


def _fault_error(fault_base, name):
    case, amb, g, _ = fault_base
    _, _, gf = oracle_loss_grads(*case, loss_fn=_faulty_loss(FAULTS[name]))
    e = masked_grad_errors(gf, g, *amb)
    worst = max(e.values())
    print(f"  [{name}] worst clean-frame gradient error {worst:.2e} ({max(e, key=e.get)}); new tol {GRAD_TOL:.1e}, "
          f"old tol {OLD_GRAD_TOL:.0e}")
    return worst


@pytest.mark.parametrize("fault", list(FAULTS))
def test_modelled_fault_fails_the_new_tolerance(fault_base, fault):
    """B=5, T=33: a 1% (gaze: 0.1%) error in one term's gradient scale moves some clean-frame gradient by more than GRAD_TOL of its max."""
    assert _fault_error(fault_base, fault) > GRAD_TOL


def test_old_bound_missed_most_modelled_faults(fault_base):
    assert sum(_fault_error(fault_base, f) <= OLD_GRAD_TOL for f in FAULTS) >= 2


def test_parents_validation_accepts_trees():
    from zeggs_b200.train import check_parents
    shipped, _ = _shipped()
    got = check_parents(shipped)
    assert got.dtype == np.int32 and np.array_equal(got, shipped)
    assert np.array_equal(check_parents(np.arange(-1, 74)), np.arange(-1, 74))     # a 75-deep chain
    assert np.array_equal(check_parents([-1] + [0] * 74), [-1] + [0] * 74)         # a star


BAD_PARENTS = {
    "too_short": list(range(-1, 73)),
    "too_long": list(range(-1, 75)),
    "root_has_a_parent": [0] + list(range(0, 74)),
    "cycle": [-1, 2, 1] + list(range(2, 74)),
    "self_parent": [-1, 1] + list(range(1, 74)),
    "forward_reference": [-1, 5] + list(range(1, 74)),
    "out_of_range": [-1] + list(range(0, 73)) + [75],
    "second_root": [-1, -1] + list(range(1, 74)),
    "not_integers": [-1] + [0.5] * 74,
    "two_dimensional": [[p] for p in range(-1, 74)],
}


@pytest.mark.parametrize("name", list(BAD_PARENTS))
def test_parents_validation_rejects(name):
    from zeggs_b200.train import check_parents
    with pytest.raises(ValueError):
        check_parents(BAD_PARENTS[name])


def test_train_step_rejects_bad_parents_before_touching_anything():
    """TrainStep checks the skeleton first: the networks (None here) and the device are never reached."""
    from zeggs_b200.train import TrainStep
    for name in ("cycle", "out_of_range"):
        with pytest.raises(ValueError):
            TrainStep(None, None, None, {}, BAD_PARENTS[name], 1.0 / 60.0)
