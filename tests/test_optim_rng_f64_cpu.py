"""CPU (no GPU): the bounds tests/test_optim_rng_f64_gpu.py holds the RAdam kernel to admit the reference's own fp32 arithmetic
(oracle/model_oracle.radam_step on fp32 tensors) with >= 4x headroom and reject every modelled kernel fault
(tests/_optim_rng_cases.py); the numpy restatement of the counter-based draws (oracle/rng_oracle.py) agrees with a plain-int
statement of the same generator, and its masks and normals have the distributions they stand for."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import rng_oracle as ro
from tests import _optim_rng_cases as oc

HEADROOM = 4.0


def _grid(b1, b2, step_fn):
    """Worst ratio of step_fn over the one-step grid at (b1, b2): every step, grad_scale, eps and lr, on a mixed state and on a
    state with p = 0 -> (ratio, case)."""
    out = (0.0, None)
    for seed, p_zero in ((1, False), (2, True)):
        st = oc.make_state(oc.GRID_N, seed, p_zero)
        for step in oc.STEPS:
            for gs in oc.GRAD_SCALES:
                for eps in oc.EPSS:
                    for lr in oc.LRS:
                        hp = (step, lr, b1, b2, eps, gs)
                        ref = oc.oracle_step(*st, *hp)
                        with np.errstate(all="ignore"):
                            r = oc.worst(oc.step_ratios(step_fn(st, *hp), ref, st, *hp))
                        if not r <= out[0]:
                            out = (r, (p_zero, *hp))
    return out


# ---------------------------------------------------------------------------------------------- RAdam bounds admit fp32
@pytest.mark.parametrize("betas", oc.BETAS, ids=str)
def test_reference_fp32_meets_one_step_bounds(betas):
    r, case = _grid(*betas, oc.reference_fp32_step)
    print(f"  [reference fp32, betas {betas}] worst {r:.3g} of the bound at (p=0, step, lr, b1, b2, eps, gs) = {case}")
    assert r * HEADROOM <= 1.0, case


@pytest.mark.parametrize("betas", oc.BETAS, ids=str)
def test_kernel_arithmetic_meets_one_step_bounds(betas):
    """The kernel's own fp32 arithmetic (betas and 1 - beta as the host's doubles, rounded once) with the same headroom."""
    r, case = _grid(*betas, oc.emulate_step)
    print(f"  [kernel arithmetic, betas {betas}] worst {r:.3g} of the bound at {case}")
    assert r * HEADROOM <= 1.0, case


@pytest.fixture(scope="module")
def traj():
    g = oc.traj_grads()
    return g, oc.traj_oracle(g)


@pytest.mark.parametrize("arith", ["reference", "kernel"])
def test_fp32_meets_trajectory_bounds(traj, arith):
    g, ref = traj
    upd = oc.traj_fp32(g, oc.reference_fp32_step if arith == "reference" else oc.emulate_step)
    r = oc.traj_ratios(upd, ref)
    t = int(torch.argmax(r)) + 1
    print(f"  [{arith} fp32 trajectory] worst {float(r.max()):.3g} of the bound at step {t}; at steps 6 / 100 / 1000 / 1200: "
          f"{float(r[5]):.3g} / {float(r[99]):.3g} / {float(r[999]):.3g} / {float(r[-1]):.3g}")
    assert float(r.max()) * HEADROOM <= 1.0, t


# ---------------------------------------------------------------------------------------------- faults break a bound
@pytest.mark.parametrize("fault", list(oc.FAULTS))
def test_fault_breaks_a_bound(traj, fault):
    worst = 0.0
    for b1, b2 in oc.BETAS:
        r, case = _grid(b1, b2, lambda *a: oc.emulate_step(*a, fault=fault))
        worst = max(worst, r)
    g, ref = traj
    with np.errstate(all="ignore"):
        tr = oc.traj_ratios(oc.traj_fp32(g, lambda *a: oc.emulate_step(*a, fault=fault)), ref)
    bad = (tr > 1.0).nonzero().flatten() + 1
    print(f"  [fault {fault}: {oc.FAULTS[fault]}] one step: worst {worst:.3g} of the bound; trajectory: {len(bad)} steps break it"
          + (f" ({int(bad[0])} .. {int(bad[-1])})" if len(bad) else ""))
    assert worst > 1.0 or len(bad) > 0


def test_parent_arithmetic_breaks_the_adaptive_steps():
    """The kernel before the fix (1.0f - (float)beta2) against the bounds at beta2 = 0.999: every adaptive step of the one-step
    grid with p = 0 fails, and so do the trajectory's steps from the switch at step 6 on."""
    st = oc.make_state(oc.GRID_N, 2, p_zero=True)
    for step in oc.STEPS[5:]:
        hp = (step, 1e-4, 0.9, 0.999, 1e-5, 1.0)
        r = oc.step_ratios(oc.emulate_step(st, *hp, fault="parent"), oc.oracle_step(*st, *hp), st, *hp)
        assert r["p"][0] > 1.0, step
    g = oc.traj_grads(steps=200)
    tr = oc.traj_ratios(oc.traj_fp32(g, lambda *a: oc.emulate_step(*a, fault="parent")), oc.traj_oracle(g))
    assert float(tr[:5].max()) <= 1.0 and bool((tr[5:50] > 1.0).all())


# ---------------------------------------------------------------------------------------------- the RNG restatement
SEEDS = [0, 1, 2 ** 62 - 1, 2 ** 64 - 1, 0x243F6A8885A308D3]


def test_restatement_equals_plain_int_generator():
    idx = np.concatenate([np.arange(300), np.array([2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1, 2 ** 32, 2 ** 40 + 7])]).astype(np.uint64)
    for s in SEEDS:
        assert ro.mix_u32(s, idx).tolist() == [ro.mix_u32_int(s, int(i)) for i in idx], s
        for salt in (1, 2, 3, 4, 17):
            assert ro.device_seed(s, salt) == ro.device_seed_int(s, salt), (s, salt)
    # Box-Muller inputs: u1 and the angle from the plain-int words, rounded to float32 step by step
    seed = ro.device_seed_int(7, 3)
    u1, ang = ro.box_muller_inputs(41, seed)
    for k in range(21):
        a, b = np.float32(ro.mix_u32_int(seed, 2 * k)), np.float32(ro.mix_u32_int(seed, 2 * k + 1))
        assert u1[k] == np.float32((a + np.float32(1.0)) * np.float32(2.0 ** -32))
        assert ang[k] == np.float32(np.float32(6.2831855) * np.float32(b * np.float32(2.0 ** -32)))
    # thresholds and scales of the mask
    assert ro.threshold(0.0) == 0 and ro.threshold(0.5) == 2 ** 31 and ro.threshold(0.99999994) == 4294967040
    assert ro.threshold(0.1) == int(np.float32(0.1) * np.float32(2.0 ** 32))
    assert ro.keep_scale(0.99999994) == np.float32(2.0 ** 24)


@pytest.mark.parametrize("p", [0.1, 0.2, 0.5])
def test_masks_keep_fraction_and_independence(p):
    """Keep fraction 1 - p within 5 sigma; no correlation (|r| <= 5 / sqrt(n)) across salts, consecutive seed words (steps) and
    adjacent indices."""
    n, t = 1 << 20, 123456789
    keep = lambda t_, salt: (ro.dropout_mask_dev(n, p, t_, salt) > 0).astype(np.float64)
    a = keep(t, 1)
    frac = a.mean()
    print(f"  [p {p}] keep fraction {frac:.6f} (1 - p = {1 - p}, sigma {math.sqrt(p * (1 - p) / n):.2e})")
    assert abs(frac - (1 - p)) <= 5 * math.sqrt(p * (1 - p) / n)
    lim = 5 / math.sqrt(n)
    for tag, b in (("salt", keep(t, 2)), ("step", keep(t + 1, 1)), ("host seed", (ro.dropout_mask(n, p, t) > 0).astype(float))):
        r = np.corrcoef(a, b)[0, 1]
        print(f"  [p {p}] correlation across {tag}: {r:.2e}")
        assert abs(r) <= lim, tag
    r = np.corrcoef(a[:-1], a[1:])[0, 1]
    assert abs(r) <= lim


def test_normals_distribution():
    """KS against N(0, 1), variance and excess kurtosis within 5 sigma of 1 and 0, each pair (2i, 2i + 1) and consecutive seed
    words uncorrelated, and no draw beyond the tail limit sqrt(64 ln 2)."""
    n = 1 << 22
    x = ro.randn_dev(n, 99, 3)
    ks = stats.kstest(x, "norm")
    var, kurt = x.var(), stats.kurtosis(x)
    pair = np.corrcoef(x[0::2], x[1::2])[0, 1]
    step = np.corrcoef(x, ro.randn_dev(n, 100, 3))[0, 1]
    print(f"  [normals] mean {x.mean():.2e} var {var:.5f} excess kurtosis {kurt:.4f} KS p {ks.pvalue:.3f} pair corr {pair:.2e} "
          f"step corr {step:.2e} max |x| {np.abs(x).max():.3f}")
    assert ks.pvalue > 1e-3
    assert abs(x.mean()) <= 5 / math.sqrt(n) and abs(var - 1) <= 5 * math.sqrt(2 / n) and abs(kurt) <= 5 * math.sqrt(24 / n)
    assert abs(pair) <= 5 / math.sqrt(n / 2) and abs(step) <= 5 / math.sqrt(n)
    assert np.abs(x).max() <= ro.TAIL


def test_tail_limit():
    """The smallest u1 is 2^-32, so |x| <= sqrt(-2 ln 2^-32) = sqrt(64 ln 2) = 6.660...: a true normal exceeds it with probability
    2.7e-11, about once per 1400 training steps' worth of 25.5 M draws -- torch.randn can, these draws cannot."""
    u1 = np.float32((np.float32(0.0) + np.float32(1.0)) * np.float32(2.0 ** -32))
    assert math.isclose(math.sqrt(-2 * math.log(float(u1))), ro.TAIL, rel_tol=1e-15)
    assert abs(ro.TAIL - 6.6604) < 1e-3
    assert math.isclose(2 * stats.norm.sf(ro.TAIL), 2.7e-11, rel_tol=0.05)
