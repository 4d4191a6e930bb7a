"""Cases and a float64 restatement of the pose -> BVH post-step (csrc/pose_post.cu, zeggs_pose_to_bvh_channels) and of
quaternion -> Euler degrees (csrc/dataset.cu, zeggs_quat_to_euler_deg).

* `post(..., dtype)`: orthogonalise from x and y, the four-branch matrix -> quaternion of quat.py, the root re-base on each
  clip's first frame with the start pose (or none), the root transform folded into joint 0 and 'zyx' Euler angles.  In float64
  it is the reference for the GPU sweep; in float32 it is the kernel's arithmetic (equal to oracle/pose_oracle.py, which is
  pinned against the reference) and sets the bounds; with `fault` it models kernel mistakes the bounds must reject.
* `to_euler(q, order)`: quat.normalize then quat.to_euler for 'zyx' and 'xzy', float64.
* `euler_quat`: the unit quaternion an Euler triple stands for, to rebuild a rotation from the kernel's angles in float64.
  'zyx' angles [z, y, x] are qz qy qx; 'xzy' angles [x, y, z] are qy qz qx (what quat.to_euler's formulas invert).
* Bounds, with kappa = 1 / sin(angle between the input x and y vectors) and pitch the asin angle of the float64 reference.
  The rotation distance is between the rotations the kernel's and the reference's Euler angles stand for (the reference's
  quaternion need not be unit: at scales near 1e-3 the 1e-10 of txform.py's normalisation is no longer negligible), and
  <= ROT_TOL kappa max(1, LOCK_SLOPE / cos(pitch)) wherever |pitch| < 89.95 degrees; per Euler angle where |pitch| <= 80
  degrees <= ROT_TOL kappa / cos(pitch); the pitch itself within 0.6 degrees of gimbal lock <= PITCH_LOCK_TOL sqrt(kappa); lrot
  <= ROT_TOL kappa up to sign; root positions <= POS_RTOL max(1, max |ref| of the clip); positions of joints j >= 1 bitwise
  equal to lpos; every output finite.
  Toward gimbal lock the yaw and roll formulas divide rounding noise by cos(pitch) in the reference's own float32 arithmetic, so
  the rebuilt rotation is only as good as u / cos(pitch) there (LOCK_SLOPE: up to 24 u / cos(pitch) on ltxy scaled near 1e-3,
  where the 1e-10 of txform.py leaves the frame slightly non-orthonormal).  Within 0.05 degrees (cos(pitch) below about
  sqrt(u)) float32 cannot tell the pitch from 90 degrees and the reference's yaw and roll are rounding noise: there only the
  pitch is held, to about sqrt(kappa u) (PITCH_LOCK_TOL).
"""
import numpy as np

ROT_TOL = 5e-5                   # rad, times kappa
LOCK_SLOPE = 0.2                 # the rotation bound grows as ROT_TOL kappa LOCK_SLOPE / cos(pitch) past 78 degrees of pitch
PITCH_LOCK_TOL = 2e-3            # rad, times sqrt(kappa): |pitch| within LOCK_DEG of 90 degrees
LOCK_DEG = 0.6
UNDETERMINED_DEG = 0.05          # within this of 90 degrees float32 cannot tell the pitch from 90: yaw and roll are not checked
PER_ANGLE_MAX_PITCH = 80.0       # degrees: the per-angle bound applies below this pitch
POS_RTOL = 2e-6
SIGN_CLEAR = 1e-5                # lrot's sign is checked where every branch selector clears this
Q2E_TOL, Q2E_LOCK_TOL = 1e-12, 1e-7   # quat_to_euler_deg: rotation distance away from / within LOCK_DEG of gimbal lock

FAULTS = {
    "rows_for_cols": "the orthogonalised axes taken as the matrix's rows (the inverse rotation)",
    "branch_order": "the y-diagonal branch tested before the x-diagonal one",
    "rebase_clip0": "every clip re-based on clip 0's first frame",
    "no_root_fold": "the root transform not folded into joint 0",
    "zyx_as_xyz": "the 'zyx' angles emitted in x, y, z order",
}
Q2E_FAULTS = {"xzy_as_zyx": "'xzy' computed with the 'zyx' formulas"}


# ---------------------------------------------------------------------------------------------- quaternion algebra
def qmul(x, y):
    """quat.py:17-25 (w first), in the dtype of its arguments."""
    x0, x1, x2, x3 = x[..., 0:1], x[..., 1:2], x[..., 2:3], x[..., 3:4]
    y0, y1, y2, y3 = y[..., 0:1], y[..., 1:2], y[..., 2:3], y[..., 3:4]
    return np.concatenate([y0 * x0 - y1 * x1 - y2 * x2 - y3 * x3, y0 * x1 + y1 * x0 - y2 * x3 + y3 * x2,
                           y0 * x2 + y1 * x3 + y2 * x0 - y3 * x1, y0 * x3 - y1 * x2 + y2 * x1 + y3 * x0], axis=-1)


def qmul_vec(q, v):
    """quat.py:36-38: the cross products in float64, whatever q's dtype."""
    u = q[..., 1:].astype(np.float64)
    t = 2.0 * np.cross(u, v.astype(np.float64))
    return v.astype(np.float64) + q[..., 0:1].astype(np.float64) * t + np.cross(u, t)


def qinv(q):
    return q * np.array([1, -1, -1, -1], dtype=q.dtype)


def axis_quat(angle, axis):
    q = np.zeros(np.shape(angle) + (4,))
    q[..., 0] = np.cos(np.asarray(angle) / 2)
    q[..., 1 + axis] = np.sin(np.asarray(angle) / 2)
    return q


def euler_quat(e, order="zyx"):
    """Unit float64 quaternion of Euler radians e [..., 3] in the convention quat.to_euler(order) returns."""
    e = np.asarray(e, dtype=np.float64)
    if order == "zyx":
        return qmul(qmul(axis_quat(e[..., 0], 2), axis_quat(e[..., 1], 1)), axis_quat(e[..., 2], 0))
    return qmul(qmul(axis_quat(e[..., 1], 1), axis_quat(e[..., 2], 2)), axis_quat(e[..., 0], 0))


def qdist(a, b):
    """Geodesic distance in rad between the rotations of quaternions a and b (normalised here), float64."""
    a = np.asarray(a, np.float64) / np.linalg.norm(np.asarray(a, np.float64), axis=-1, keepdims=True)
    b = np.asarray(b, np.float64) / np.linalg.norm(np.asarray(b, np.float64), axis=-1, keepdims=True)
    r = qmul(qinv(a), b)
    return 2.0 * np.arctan2(np.linalg.norm(r[..., 1:], axis=-1), np.abs(r[..., 0]))


def qmat(q):
    """Rotation matrix of unit quaternions [..., 4] -> [..., 3, 3] (columns are the rotated x, y, z axes)."""
    w, x, y, z = (q[..., i] for i in range(4))
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


# ---------------------------------------------------------------------------------------------- the post-step
def orthogonalize(xy, dtype, fault=None):
    """txform.py:23-34: xy [..., 2, 3] -> matrices whose COLUMNS are the normalised x, y = z x x, z = x x y."""
    xy = np.asarray(xy).astype(dtype)
    eps = dtype(1e-10)
    x = xy[..., 0, :]
    z = np.cross(x, xy[..., 1, :])
    y = np.cross(z, x)
    n = lambda v: v / (np.sqrt(np.sum(v * v, axis=-1, keepdims=True)) + eps)
    return np.stack([n(x), n(y), n(z)], axis=-2 if fault == "rows_for_cols" else -1)


def quat_from_matrix(m, fault=None):
    """quat.py:166-206, the four-branch form with eps 1e-10, in m's dtype."""
    dt = m.dtype.type
    eps, one, two, q4 = dt(1e-10), dt(1), dt(2), dt(0.25)
    e = lambda i, j: m[..., i, j]
    t = e(0, 0) + e(1, 1) + e(2, 2)
    s = dt(0.5) / np.sqrt(np.maximum(t + one, eps))
    b0 = np.stack([q4 / s, s * (e(2, 1) - e(1, 2)), s * (e(0, 2) - e(2, 0)), s * (e(1, 0) - e(0, 1))], -1)
    s0 = two * np.sqrt(np.maximum(one + e(0, 0) - e(1, 1) - e(2, 2), eps))
    b1 = np.stack([(e(2, 1) - e(1, 2)) / s0, s0 * q4, (e(0, 1) + e(1, 0)) / s0, (e(0, 2) + e(2, 0)) / s0], -1)
    s1 = two * np.sqrt(np.maximum(one + e(1, 1) - e(0, 0) - e(2, 2), eps))
    b2 = np.stack([(e(0, 2) - e(2, 0)) / s1, (e(0, 1) + e(1, 0)) / s1, s1 * q4, (e(1, 2) + e(2, 1)) / s1], -1)
    s2 = two * np.sqrt(np.maximum(one + e(2, 2) - e(0, 0) - e(1, 1), eps))
    b3 = np.stack([(e(1, 0) - e(0, 1)) / s2, (e(0, 2) + e(2, 0)) / s2, (e(1, 2) + e(2, 1)) / s2, s2 * q4], -1)
    cx = (e(0, 0) > e(1, 1)) & (e(0, 0) > e(2, 2))
    cy = e(1, 1) > e(2, 2)
    if fault == "branch_order":
        return np.where((t > 0)[..., None], b0, np.where(cy[..., None], b2, np.where(cx[..., None], b1, b3)))
    return np.where((t > 0)[..., None], b0, np.where(cx[..., None], b1, np.where(cy[..., None], b2, b3)))


def branch_margin(m):
    """Smallest distance of a branch selector of quat_from_matrix from its decision: |trace|, |m00 - m11|, |m00 - m22|,
    |m11 - m22| (float64 matrices)."""
    d = lambda i, j: m[..., i, i] - m[..., j, j]
    t = m[..., 0, 0] + m[..., 1, 1] + m[..., 2, 2]
    return np.minimum(np.minimum(np.abs(t), np.abs(d(0, 1))), np.minimum(np.abs(d(0, 2)), np.abs(d(1, 2))))


def euler_zyx(q):
    """quat.py:111-119 (no normalisation), radians."""
    x0, x1, x2, x3 = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    c = q.dtype.type
    return np.stack([np.arctan2(c(2) * (x0 * x3 + x1 * x2), c(1) - c(2) * (x2 * x2 + x3 * x3)),
                     np.arcsin(np.clip(c(2) * (x0 * x2 - x3 * x1), c(-1), c(1))),
                     np.arctan2(c(2) * (x0 * x1 + x2 * x3), c(1) - c(2) * (x1 * x1 + x2 * x2))], -1)


def post(root_pos, root_rot, lpos, ltxy, start_position=(0, 0, 0), start_rotation=(1, 0, 0, 0), rebase=True,
         dtype=np.float64, fault=None):
    """[N, T, ...] pose arrays -> (positions [N,T,J,3], euler radians [N,T,J,3] in 'zyx' channel order, lrot [N,T,J,4]) in
    `dtype`.  float32 follows the kernel's arithmetic (the root composition's cross products in float64, as quat.py does)."""
    dt = np.dtype(dtype).type
    rp, rq, lp = (np.asarray(a).astype(dt) for a in (root_pos, root_rot, lpos))
    lrot = quat_from_matrix(orthogonalize(ltxy, dt, fault), fault)
    if rebase:
        first = slice(0, 1) if fault == "rebase_clip0" else slice(None)
        p0, q0 = rp[first, 0:1], rq[first, 0:1]
        oi = qinv(q0)
        sp = np.asarray(start_position, dtype=np.float64)
        sr = np.asarray(start_rotation).astype(dt)
        rpos = qmul_vec(oi, rp - p0)
        rrot = qmul(oi, rq)
        rpos = qmul_vec(np.broadcast_to(sr, rrot.shape), rpos) + sp
        rrot = qmul(np.broadcast_to(sr, rrot.shape), rrot)
    else:
        rpos, rrot = rp.astype(np.float64), rq
    pos = lp.copy()
    rot = lrot.copy()
    if fault != "no_root_fold":
        pos[:, :, 0] = (qmul_vec(rrot, lp[:, :, 0]) + rpos).astype(dt)
        rot[:, :, 0] = qmul(rrot, lrot[:, :, 0])
    e = euler_zyx(rot)
    if fault == "zyx_as_xyz":
        e = e[..., ::-1]
    return pos, e, rot


def kappa(ltxy):
    """1 / sin(angle between the input x and y vectors), float64."""
    xy = np.asarray(ltxy, np.float64)
    x, y = xy[..., 0, :], xy[..., 1, :]
    c = np.linalg.norm(np.cross(x, y), axis=-1)
    return np.linalg.norm(x, axis=-1) * np.linalg.norm(y, axis=-1) / c


# ---------------------------------------------------------------------------------------------- checks against the bounds
def wrap(d):
    return (d + np.pi) % (2.0 * np.pi) - np.pi


def ratios(ltxy, lpos, pos, eul, lrot, ref, pos_is_bitwise=True):
    """Worst ratio to each bound of (pos, eul radians, lrot) against the float64 reference `ref` = post(..., float64).
    -> dict name: ratio (inf where a bitwise check fails)."""
    rpos, reul, rrot = ref
    k = kappa(ltxy)
    pitch = reul[..., 1]
    cosp = np.cos(pitch)
    out = {}
    if pos_is_bitwise:
        same = np.array_equal(np.asarray(pos)[:, :, 1:].view(np.uint32), np.asarray(lpos, np.float32)[:, :, 1:].view(np.uint32))
        out["joints>=1 positions bitwise"] = 0.0 if same else np.inf
    scale = np.maximum(1.0, np.abs(rpos[:, :, 0]).reshape(rpos.shape[0], -1).max(axis=1))[:, None, None]
    out["root position"] = float((np.abs(np.asarray(pos, np.float64)[:, :, 0] - rpos[:, :, 0]) / (POS_RTOL * scale)).max())
    d = qdist(euler_quat(np.asarray(eul, np.float64)), euler_quat(reul))
    lock = np.abs(np.degrees(pitch)) >= 90.0 - LOCK_DEG
    determined = np.abs(np.degrees(pitch)) < 90.0 - UNDETERMINED_DEG
    out["rotation"] = float((d / (ROT_TOL * k * np.maximum(1.0, LOCK_SLOPE / cosp)))[determined].max())
    if lock.any():
        dp = np.abs(np.asarray(eul, np.float64)[..., 1] - pitch)
        out["pitch at lock"] = float((dp / (PITCH_LOCK_TOL * np.sqrt(k)))[lock].max())
    out["finite"] = 0.0 if np.all(np.isfinite(eul)) and np.all(np.isfinite(pos)) else np.inf
    sel = np.abs(np.degrees(pitch)) <= PER_ANGLE_MAX_PITCH
    da = np.abs(wrap(np.asarray(eul, np.float64) - reul)).max(axis=-1)
    out["per angle"] = float((da[sel] / (ROT_TOL * k[sel] / cosp[sel])).max()) if sel.any() else 0.0
    g = np.asarray(lrot, np.float64)
    dq = np.minimum(np.abs(g - rrot).max(-1), np.abs(g + rrot).max(-1))
    out["lrot up to sign"] = float((dq / (ROT_TOL * k)).max())
    m = orthogonalize(ltxy, np.float64)
    clear = branch_margin(m) > SIGN_CLEAR
    flipped = np.abs(g - rrot).max(-1) > np.abs(g + rrot).max(-1)
    out["lrot sign where the branch is clear"] = np.inf if np.any(flipped[:, :, 1:] & clear[:, :, 1:]) else 0.0
    return out


# ---------------------------------------------------------------------------------------------- cases
def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def special_rotations():
    """Unit float64 quaternions that drive each branch of quat_from_matrix on purpose and the Euler edges: trace well above 0,
    trace within +-1e-6 of 0, 180-degree turns about x, y, z and oblique axes (and axes near x tilted toward y, where the y
    branch would be inaccurate), diagonal ties, and pitch at 0, +-45, +-89.9 and exactly +-90 degrees."""
    qs = [np.array([1.0, 0, 0, 0]), euler_quat([0.3, -0.2, 0.1])]                         # trace 3, trace well above 0
    for ax in [(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1), (1, -2, 3), (1, 1e-3, 0),
               (1, 1e-3, 1e-4), (1e-3, 1, 0), (2e-3, 0, 1), (1, 1, 1e-3)]:
        qs.append(np.concatenate([[0.0], _unit(np.array(ax, float))]))                   # 180 degrees: trace -1
    for ax in [(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1), (1, -1, 2)]:                   # 120-degree class: trace 0 (and +-1e-6)
        for dtr in (0.0, 1e-6, -1e-6, 3e-7):
            ang = np.arccos((dtr - 1.0) / 2.0)
            qs.append(axis_angle(_unit(np.array(ax, float)), ang))
    for ax in [(1, 1, 0), (1, 0, 1), (0, 1, 1)]:                                         # ties between two diagonals
        for ang in (np.pi, 2.5, 2.0):
            qs.append(axis_angle(_unit(np.array(ax, float)), ang))
    for p in (0.0, 45.0, -45.0, 89.9, -89.9, 90.0, -90.0, 89.5, -89.99):
        for yaw, roll in ((0.0, 0.0), (0.7, -1.9), (-2.5, 2.9)):
            qs.append(euler_quat([yaw, np.radians(p), roll]))
    return np.stack(qs)


def axis_angle(axis, ang):
    return np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * np.asarray(axis, float)])


def random_quats(shape, rs):
    return _unit(rs.randn(*shape, 4))


def ltxy_from_quats(q, rs, scale=None, skew_deg=None):
    """float32 ltxy [..., 2, 3] whose orthogonalised frame is q: x = s_x R e_x, y = s_y (cos a R e_x + sin a R e_y) with the
    angle a between them (90 degrees when skew_deg is None) and positive scales s."""
    R = qmat(q)
    ex, ey = R[..., :, 0], R[..., :, 1]
    shp = q.shape[:-1]
    sx = np.ones(shp) if scale is None else scale(shp)
    sy = np.ones(shp) if scale is None else scale(shp)
    a = np.full(shp, np.pi / 2) if skew_deg is None else np.radians(skew_deg(shp))
    x = sx[..., None] * ex
    y = sy[..., None] * (np.cos(a)[..., None] * ex + np.sin(a)[..., None] * ey)
    return np.stack([x, y], axis=-2).astype(np.float32)


def pose_case(N, T, J, seed, special=False, rebase=True, start=False, skew=True):
    """One post-step call: dict of float32 arrays root_pos [N,T,3], root_rot [N,T,4] (unit, each clip its own first frame),
    lpos [N,T,J,3], ltxy [N,T,J,2,3], plus start_position / start_rotation / rebase.  special: the special rotations are laid
    over every third (clip, frame, joint) from the first, with orthonormal x and y (at scales near 1e-3 the 1e-10 of txform.py
    makes the frame non-orthonormal, which would blur the edges these rotations are there to reach).  skew: every other ltxy
    scaled by 1e-3 .. 1e3 and, on a third of them, skewed down to 1 degree between x and y."""
    rs = np.random.RandomState(seed)
    q = random_quats((N, T, J), rs)
    if skew:
        scale = lambda shp: 10.0 ** rs.uniform(-3, 3, shp)
        skew_deg = lambda shp: np.where(rs.rand(*shp) < 1 / 3, 10.0 ** rs.uniform(0, np.log10(90), shp), 90.0)
        ltxy = ltxy_from_quats(q, rs, scale, skew_deg)
    else:
        ltxy = ltxy_from_quats(q, rs)
    if special:                               # every third element from the first, with orthonormal unit-scale x and y
        sq = special_rotations()
        k = min(len(sq), N * T * J)
        idx = np.arange(k) * 3 if N * T * J >= 3 * len(sq) else np.arange(k)
        q.reshape(-1, 4)[idx] = sq[:k]
        ltxy.reshape(-1, 2, 3)[idx] = ltxy_from_quats(sq[:k], rs)
    rq = random_quats((N, T), rs)
    rq = (rq / np.linalg.norm(rq, axis=-1, keepdims=True)).astype(np.float32)
    rp = (rs.randn(N, T, 3) * np.array([80.0, 10.0, 80.0]) + np.array([0.0, 95.0, 0.0])).astype(np.float32)
    lpos = (rs.randn(N, T, J, 3) * 10.0).astype(np.float32)
    sp = (12.5, -3.0, 140.25) if start else (0.0, 0.0, 0.0)
    sr = tuple(_unit(np.array([0.9, 0.1, -0.3, 0.2])).astype(np.float32).tolist()) if start else (1.0, 0.0, 0.0, 0.0)
    return dict(root_pos=rp, root_rot=rq, lpos=lpos, ltxy=ltxy, start_position=sp, start_rotation=sr, rebase=rebase)


def run_post(case, dtype=np.float64, fault=None):
    return post(case["root_pos"], case["root_rot"], case["lpos"], case["ltxy"], case["start_position"], case["start_rotation"],
                case["rebase"], dtype, fault)


# (N, T, J) shapes of the sweep; the last is 810 000 joints x frames, past one grid of 132 * 16 * 256 = 540 672 threads
SHAPES = [(1, 1, 1), (1, 2, 75), (3, 241, 75), (2, 9, 128), (3, 3600, 75)]


# ---------------------------------------------------------------------------------------------- quat -> Euler
def to_euler(q, order, fault=None):
    """quat.normalize (quat.py:92-93, eps 0) then quat.to_euler(order), float64 radians."""
    q = np.asarray(q, np.float64)
    x = q / (np.sqrt(np.sum(q * q, axis=-1, keepdims=True)) + 0.0)
    if order == "zyx" or fault == "xzy_as_zyx":
        return euler_zyx(x)
    x0, x1, x2, x3 = x[..., 0], x[..., 1], x[..., 2], x[..., 3]
    return np.stack([np.arctan2(2.0 * (x1 * x0 - x2 * x3), -x1 * x1 + x2 * x2 - x3 * x3 + x0 * x0),
                     np.arctan2(2.0 * (x2 * x0 - x1 * x3), x1 * x1 - x2 * x2 - x3 * x3 + x0 * x0),
                     np.arcsin(np.clip(2.0 * (x1 * x2 + x3 * x0), -1.0, 1.0))], -1)


def euler_pitch_index(order):
    return 1 if order == "zyx" else 2


def q2e_quats(n, seed, near_lock=True):
    """float64 non-unit quaternions [n, 4], norms 1e-3 .. 1e3; with near_lock, a quarter lie within 1e-3 .. 0.5 degrees of
    gimbal lock for 'zyx' and a quarter for 'xzy'."""
    rs = np.random.RandomState(seed)
    q = random_quats((n,), rs)
    if near_lock and n >= 4:
        k = n // 4
        off = np.radians(10.0 ** rs.uniform(-3, np.log10(0.5), 2 * k)) * np.where(rs.rand(2 * k) < 0.5, 1, -1)
        pitch = np.sign(off) * (np.pi / 2) - off
        a, c = rs.uniform(-np.pi, np.pi, (2, 2 * k))
        q[:k] = euler_quat(np.stack([a[:k], pitch[:k], c[:k]], -1), "zyx")
        q[k:2 * k] = euler_quat(np.stack([a[k:], c[k:], pitch[k:]], -1), "xzy")
    return q * (10.0 ** rs.uniform(-3, 3, n))[:, None]


def q2e_ratio(q, e_rad, order):
    """Worst ratios of Euler radians e_rad against the float64 restatement: rotation distance (<= Q2E_TOL, <= Q2E_LOCK_TOL
    within LOCK_DEG of lock) and per angle (<= Q2E_TOL / cos(pitch) where |pitch| <= 80 degrees)."""
    ref = to_euler(q, order)
    p = ref[..., euler_pitch_index(order)]
    lock = np.abs(np.degrees(p)) >= 90.0 - LOCK_DEG
    d = qdist(euler_quat(e_rad, order), q)
    tol = np.where(lock, Q2E_LOCK_TOL, Q2E_TOL)
    sel = np.abs(np.degrees(p)) <= PER_ANGLE_MAX_PITCH
    da = np.abs(wrap(e_rad - ref)).max(-1)
    return {"rotation": float((d / tol).max()) if d.size else 0.0,
            "per angle": float((da[sel] / (Q2E_TOL / np.cos(p[sel]))).max()) if sel.any() else 0.0}
