"""GPU: the pose -> BVH post-step (csrc/pose_post.cu, zeggs_pose_to_bvh_channels) through ops.pose_to_bvh_channels(...,
want_lrot=True) against the float64 restatement of tests/_pose_cases.py, and quaternion -> Euler degrees (csrc/dataset.cu,
zeggs_quat_to_euler_deg) against its float64 restatement.

* Post-step bounds (kappa = 1 / sin of the angle between the input x and y): joints j >= 1 keep lpos bit for bit; root
  positions <= 2e-6 max(1, max |ref| of the clip); the rotations the Euler angles stand for <= 5e-5 kappa max(1, 0.2 /
  cos(pitch)) apart below 89.95 degrees of pitch; per angle <= 5e-5 kappa / cos(pitch) where |pitch| <= 80 degrees; the pitch
  within 0.6 degrees of lock <= 2e-3 sqrt(kappa); lrot <= 5e-5 kappa up to sign, the sign the float64 one wherever every
  branch selector clears 1e-5.
* Cases: every branch of the matrix -> quaternion conversion, trace within 1e-6 of 0, 180-degree turns about x, y, z and oblique
  axes, diagonal ties, pitch 0, +-45, +-89.9 and +-90 degrees; ltxy scaled 1e-3 .. 1e3 and skewed down to 1 degree; (N, T, J) =
  (1, 1, 1), (1, 2, 75), (3, 241, 75) with a first frame per clip, (2, 9, 128) and (3, 3600, 75) (810 000 elements, so the
  grid-stride loop runs twice); re-base on and off; the identity start pose and a nontrivial one.
* Bitwise: want_lrot on and off give the same positions and angles; each clip of a batch equals the clip alone.
* quat_to_euler_deg, 'zyx' and 'xzy', on quaternions of norm 1e-3 .. 1e3, some next to gimbal lock: rotation distance <= 1e-12
  rad (<= 1e-7 within 0.6 degrees of lock), per angle <= 1e-12 / cos(pitch) where |pitch| <= 80 degrees; n = 0, 1, and past the
  kernel's grid of 132 * 32 * 256 threads.
tests/test_pose_post_f64_cpu.py shows the kernel's float32 arithmetic meets these bounds with >= 4x headroom and that each
modelled fault breaks one.
"""
import numpy as np
import pytest
import torch

from tests import _pose_cases as pc
from tests._util import ensure_built

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


def _kernel(dev, c, want_lrot=True, clips=slice(None)):
    from zeggs_b200 import ops
    t = lambda k: torch.from_numpy(np.ascontiguousarray(c[k][clips])).to(dev)
    out = ops.pose_to_bvh_channels(t("root_pos"), t("root_rot"), t("lpos"), t("ltxy"), c["start_position"], c["start_rotation"],
                                   rebase=c["rebase"], want_lrot=want_lrot)
    return [o.cpu().numpy() for o in out]


def _report(tag, r):
    for k, v in r.items():
        print(f"  [{tag}] {k}: {v:.3g} of its bound")
    bad = {k: v for k, v in r.items() if not v <= 1.0}
    assert not bad, (tag, bad)


@pytest.mark.parametrize("start", [False, True], ids=["identity_start", "start_pose"])
@pytest.mark.parametrize("rebase", [True, False], ids=["rebase", "no_rebase"])
@pytest.mark.parametrize("shape", pc.SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_post_step_against_float64(dev, shape, rebase, start):
    if start and not rebase:
        pytest.skip("the start pose only applies when re-basing")
    c = pc.pose_case(*shape, seed=sum(shape), special=True, rebase=rebase, start=start)
    pos, eul, lrot = _kernel(dev, c)
    _report(f"{shape} rebase={rebase} start={start}", pc.ratios(c["ltxy"], c["lpos"], pos, np.radians(eul.astype(np.float64)),
                                                                 lrot, pc.run_post(c)))
    pos2, eul2 = _kernel(dev, c, want_lrot=False)
    assert np.array_equal(pos2.view(np.uint32), pos.view(np.uint32)) and np.array_equal(eul2.view(np.uint32), eul.view(np.uint32))
    if shape[0] > 1 and shape[0] * shape[1] * shape[2] < 500000:
        for n in range(shape[0]):
            pn, en, ln = _kernel(dev, c, clips=slice(n, n + 1))
            for a, b in ((pn, pos[n:n + 1]), (en, eul[n:n + 1]), (ln, lrot[n:n + 1])):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), n


# ---------------------------------------------------------------------------------------------- quat -> Euler degrees
def _q2e(dev, q, order):
    from zeggs_b200 import ops
    return np.radians(ops.quat_to_euler_deg(torch.from_numpy(q).to(dev), order).cpu().numpy())


@pytest.mark.parametrize("n", [0, 1, 4000, 132 * 32 * 256 + 4099])
@pytest.mark.parametrize("order", ["zyx", "xzy"])
def test_quat_to_euler_deg_against_float64(dev, order, n):
    q = pc.q2e_quats(n, seed=n % 97)
    e = _q2e(dev, q, order)
    assert e.shape == (n, 3)
    if n:
        _report(f"quat_to_euler_deg {order} n{n}", pc.q2e_ratio(q, e, order))
