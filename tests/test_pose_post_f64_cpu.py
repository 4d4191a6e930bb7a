"""CPU (no GPU): the pose -> BVH post-step's float64 restatement (tests/_pose_cases.py) equals oracle/pose_oracle.py (float32,
pinned against the reference) on well-conditioned inputs; the kernel's float32 arithmetic (pose_oracle, and the restatement in
float32) meets every bound tests/test_pose_post_f64_gpu.py holds the kernel to, with >= 4x headroom; each modelled fault breaks
a bound; and the same for quaternion -> Euler degrees ('zyx', 'xzy')."""
import numpy as np
import pytest

from oracle import pose_oracle as po
from tests import _pose_cases as pc

HEADROOM = 4.0
CAL_SHAPES = pc.SHAPES


def _print(tag, r):
    for k, v in r.items():
        print(f"  [{tag}] {k}: {v:.3g} of its bound")


def test_euler_conventions_round_trip():
    """euler_quat inverts quat.to_euler's formulas for both orders, so the kernel's angles can be turned back into rotations."""
    q = pc.random_quats((500,), np.random.RandomState(0))
    for order in ("zyx", "xzy"):
        assert pc.qdist(pc.euler_quat(pc.to_euler(q, order), order), q).max() <= 1e-13, order


def test_float64_restatement_equals_pose_oracle_on_well_conditioned_input():
    """Orthonormal unit-scale ltxy, re-base on with the identity start pose (what pose_oracle does): the float64 restatement and
    the float32 oracle agree to float32 rounding, and the float32 restatement equals the oracle bit for bit."""
    c = pc.pose_case(3, 20, 75, seed=1, skew=False)
    p64, e64, _ = pc.run_post(c)
    p32, e32, _ = pc.run_post(c, np.float32)
    for n in range(3):
        pos, eul = po.pose_to_bvh_channels(c["root_pos"][n], c["root_rot"][n], c["lpos"][n], c["ltxy"][n])
        assert np.array_equal(pos, p32[n]) and np.array_equal(eul, np.degrees(e32[n]))
        assert np.abs(pos - p64[n]).max() <= 1e-6 * max(1.0, np.abs(p64[n]).max())
        d = pc.qdist(pc.euler_quat(np.radians(eul.astype(np.float64))), pc.euler_quat(e64[n]))
        assert d[np.abs(np.degrees(e64[n][..., 1])) < 90.0 - pc.LOCK_DEG].max() <= 1e-5


@pytest.mark.parametrize("shape", CAL_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_float32_meets_the_bounds_with_headroom(shape):
    """The kernel's float32 arithmetic against float64 on every case family of the GPU sweep at this shape."""
    worst = {}
    for special in (False, True):
        for rebase, start in ((True, False), (True, True), (False, False)):
            c = pc.pose_case(*shape, seed=sum(shape) + (not special), special=special, rebase=rebase, start=start)
            r = pc.ratios(c["ltxy"], c["lpos"], *pc.run_post(c, np.float32), pc.run_post(c))
            for k, v in r.items():
                worst[k] = max(worst.get(k, 0.0), v)
    _print(f"float32 {shape}", worst)
    assert max(worst.values()) * HEADROOM <= 1.0, worst


def test_cases_reach_every_branch_and_lock():
    """The special rotations drive each branch of the matrix -> quaternion conversion, the trace within 1e-6 of 0, ties, and
    pitch within 0.6 degrees of lock (with some within 0.05 degrees, where only the pitch is held)."""
    m = pc.qmat(pc.special_rotations())
    t = np.trace(m, axis1=-2, axis2=-1)
    cx = (m[:, 0, 0] > m[:, 1, 1]) & (m[:, 0, 0] > m[:, 2, 2])
    cy = m[:, 1, 1] > m[:, 2, 2]
    branch = np.where(t > 0, 0, np.where(cx, 1, np.where(cy, 2, 3)))
    assert set(branch.tolist()) == {0, 1, 2, 3}
    assert np.sum(np.abs(t) <= 1e-6) >= 10
    pitch = np.degrees(pc.euler_zyx(pc.special_rotations())[:, 1])
    assert np.sum(np.abs(pitch) >= 90 - pc.UNDETERMINED_DEG) >= 6 and np.sum(np.abs(np.abs(pitch) - 89.9) < 1e-6) >= 6


FAULT_SHAPE = (3, 241, 75)


@pytest.mark.parametrize("fault", list(pc.FAULTS))
def test_fault_breaks_a_bound(fault):
    c = pc.pose_case(*FAULT_SHAPE, seed=5, special=True)
    r = pc.ratios(c["ltxy"], c["lpos"], *pc.run_post(c, np.float32, fault), pc.run_post(c))
    broken = {k: v for k, v in r.items() if v > 1.0}
    print(f"  [fault {fault}: {pc.FAULTS[fault]}] breaks " + ", ".join(f"{k} ({v:.3g})" for k, v in broken.items()))
    assert broken


# ---------------------------------------------------------------------------------------------- quat -> Euler
@pytest.mark.parametrize("order", ["zyx", "xzy"])
def test_quat_to_euler_restatement_meets_the_bounds(order):
    """The float64 restatement's own angles rebuild the input rotation to the rotation bound, computed in long double as a check
    of the per-angle bound too."""
    q = pc.q2e_quats(4000, 3)
    e = pc.to_euler(q, order)
    r = pc.q2e_ratio(q, e, order)
    el = pc.to_euler(q.astype(np.longdouble), order).astype(np.float64)
    r["per angle vs long double"] = float((np.abs(pc.wrap(e - el)).max(-1) / pc.Q2E_TOL).max())
    _print(f"float64 to_euler {order}", r)
    assert max(r.values()) * HEADROOM <= 1.0


def test_quat_to_euler_fault_breaks_a_bound():
    q = pc.q2e_quats(4000, 3)
    r = pc.q2e_ratio(q, pc.to_euler(q, "xzy", fault="xzy_as_zyx"), "xzy")
    _print(f"fault xzy_as_zyx: {pc.Q2E_FAULTS['xzy_as_zyx']}", r)
    assert max(r.values()) > 1.0
