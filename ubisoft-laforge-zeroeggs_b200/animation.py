"""BVH in, pose features out: the data-format edge in front of the accelerated path (numpy; the MOTION numbers parse on the device).

Mirrors what the reference does to a style example / first-pose BVH before the networks see it:
  ZEGGS/anim/bvh.py:4-134        load(): HIERARCHY + MOTION text -> rotations (degrees, file channel order), positions, offsets, ...
  ZEGGS/data_pipeline.py:89-180  preprocess_animation(): FK, ground-projected root (Spine2) facing the Hips' forward axis, median gaze
                                 target 100 units ahead of the Head, root-relative joint 0, finite-difference velocities (helical
                                 angular velocities), rotated x/y axes (ltxy)
so that generate_gesture() runs with nothing but this package.  float64 throughout (the reference mixes float32 / float64);
parity with the reference's own functions is checked at 1e-4 * max(1, |ref|) (tests/test_animation_cpu.py, golden generate_e2e.npz)."""
import re

import numpy as np

POSE_KEYS = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt"]
_AXIS = {"x": np.array([1.0, 0.0, 0.0]), "y": np.array([0.0, 1.0, 0.0]), "z": np.array([0.0, 0.0, 1.0])}
_CHAN = {"Xrotation": "x", "Yrotation": "y", "Zrotation": "z"}


# ---------------------------------------------------------------------------------------------- BVH text
def load_bvh(path):
    """-> dict(rotations [T,J,3] deg, positions [T,J,3], offsets [J,3], parents [J], names, order, frametime), like bvh.py:load.
    The MOTION block is parsed on the device when the library and a CUDA device are available (bit-identical to the host parse, which
    decides every case the device parser leaves to it), on the host otherwise."""
    got = _load_bvh_device(path) if _device_parse_available() else None
    if got is not None:
        header, data = got
        return _assemble(path, header, data)
    with open(path, "r") as f:
        lines = iter(f.read().split("\n"))
    header = _parse_header(lines)
    nframes = header[-1]
    rows = [r for r in lines if r.strip()]
    data = np.array([np.array(r.split(), dtype=np.float64) for r in rows[:nframes]]) if nframes else np.zeros((0, 0))
    return _assemble(path, header, data)


def _parse_header(lines):
    """HIERARCHY of a BVH file from an iterator over its lines; consumes them up to the "Frame Time:" line.
    -> (names, offsets, parents, chans, order, frametime, nframes)"""
    names, offsets, parents, chans = [], [], [], []
    stack, order, frametime, nframes = [], None, None, None
    in_end = False
    for line in lines:
        ln = line.strip()
        if not ln or ln == "HIERARCHY":
            continue
        tok = ln.split()
        if tok[0] in ("ROOT", "JOINT"):
            names.append(tok[1]); offsets.append([0.0, 0.0, 0.0]); parents.append(stack[-1] if stack else -1); chans.append(0)
            stack.append(len(names) - 1)
        elif tok[0] == "End":
            in_end = True
        elif tok[0] == "}":
            if in_end:
                in_end = False
            else:
                stack.pop()
        elif tok[0] == "OFFSET":
            if not in_end:
                offsets[stack[-1]] = [float(v) for v in tok[1:4]]
        elif tok[0] == "CHANNELS":
            n = int(tok[1])
            chans[stack[-1]] = n
            rot = tok[2:2 + n][-3:] if n in (3, 6) else tok[5:8]
            if order is None and all(c in _CHAN for c in rot):
                order = "".join(_CHAN[c] for c in rot)
        elif tok[0] == "Frames:":
            nframes = int(tok[1])
        elif tok[0] == "Frame" and tok[1] == "Time:":
            frametime = float(tok[2])
            break
    return names, offsets, parents, chans, order, frametime, nframes


def _assemble(path, header, data):
    """MOTION values data [T, C] (float64, file channel order) + header -> the load_bvh dict."""
    names, offsets, parents, chans, order, frametime, _ = header
    J = len(names)
    T = data.shape[0]
    off = np.asarray(offsets, dtype=np.float64)
    positions = np.repeat(off[None], T, axis=0)
    rotations = np.zeros((T, J, 3))
    col = 0
    for j in range(J):
        n = chans[j]
        if n == 3:
            rotations[:, j] = data[:, col:col + 3]
        elif n == 6:
            positions[:, j] = data[:, col:col + 3]
            rotations[:, j] = data[:, col + 3:col + 6]
        else:
            raise ValueError(f"{path}: joint {names[j]} has {n} channels (3 or 6 supported)")
        col += n
    return dict(rotations=rotations.astype(np.float32), positions=positions.astype(np.float32), offsets=off.astype(np.float32),
                parents=np.asarray(parents, dtype=np.int32), names=names, order=order or "zyx", frametime=frametime)


# MOTION tokens the device leaves to the host (not on the exact fast path) are filled here one by one; with more than this many, the
# whole block is parsed on the host
MAX_FLAGGED_TOKENS = 1 << 16
_LINE_BREAK = re.compile(rb"\r\n|\r|\n")
_TOKEN = re.compile(rb"[^ \t\n\r\x0b\x0c\x1c-\x1f]+")


def _device_parse_available():
    import torch
    from . import _lib
    if not torch.cuda.is_available():
        return False
    try:
        _lib.lib()
    except _lib.ZeggsError:
        return False
    return True


def _header_lines(buf, state):
    """The lines of an ASCII file as Python's universal-newline read + split("\\n") gives them; state["next"] = where the text after
    the last line handed out starts.  A non-ASCII byte raises UnicodeDecodeError."""
    pos = 0
    for m in _LINE_BREAK.finditer(buf):
        state["next"] = m.end()
        yield buf[pos:m.start()].tobytes().decode("ascii")
        pos = m.end()
    state["next"] = len(buf)
    yield buf[pos:].tobytes().decode("ascii")


def _load_bvh_device(path):
    """-> (header, data [T, C] float64) with the MOTION block parsed by zeggs_bvh_parse_motion, or None when the host parser must
    decide: non-ASCII text, no frames, a joint with other than 3 or 6 channels, a block of 2 GB or more, no rows, a row whose token
    count is not C, a token numpy rejects, or more tokens off the fast path than MAX_FLAGGED_TOKENS."""
    import ctypes as C
    import os
    import torch
    from . import _lib
    n = os.path.getsize(path)
    host = torch.empty(n, dtype=torch.uint8, pin_memory=True)
    buf = host.numpy()
    with open(path, "rb") as f:
        if f.readinto(memoryview(buf)) != n:
            return None
    state = {}
    try:
        header = _parse_header(_header_lines(memoryview(buf), state))
    except UnicodeDecodeError:
        return None
    chans, frametime, nframes = header[3], header[5], header[6]
    if frametime is None or not nframes or nframes < 0 or not chans or any(c not in (3, 6) for c in chans):
        return None
    start, ncol = state["next"], sum(chans)
    if n - start >= 1 << 31:
        return None
    dev = torch.device("cuda", torch.cuda.current_device())
    text = torch.empty(n - start, dtype=torch.uint8, device=dev)
    text.copy_(host[start:], non_blocking=True)
    out = torch.empty((nframes, ncol), dtype=torch.float64, device=dev)
    flagged = torch.empty((MAX_FLAGGED_TOKENS, 2), dtype=torch.int64, device=dev)
    status = torch.empty(3, dtype=torch.int32, device=dev)
    l = _lib.lib()
    ws = torch.empty(int(l.zeggs_bvh_parse_motion_workspace_size(n - start, nframes)), dtype=torch.uint8, device=dev)
    a = _lib.BvhParseArgs(n_bytes=n - start, n_frames=nframes, C=ncol, max_flagged=MAX_FLAGGED_TOKENS, text=text.data_ptr(),
                          out=out.data_ptr(), flagged=flagged.data_ptr(), status=status.data_ptr(), workspace=ws.data_ptr(),
                          workspace_bytes=ws.numel())
    _lib.check(l.zeggs_bvh_parse_motion(C.byref(a), _lib.stream_ptr()), "zeggs_bvh_parse_motion")
    rows, nflag, bad = (int(v) for v in status.cpu())
    if bad or rows == 0 or nflag > MAX_FLAGGED_TOKENS:
        return None
    data = out[:rows].cpu().numpy()
    if nflag:
        block, flat = memoryview(buf)[start:], data.reshape(-1)
        for idx, off in flagged[:nflag].cpu().numpy():
            tok = _TOKEN.match(block, int(off)).group().decode("ascii")
            try:
                flat[idx] = np.array([tok], dtype=np.float64)[0]           # the host parse's own conversion of this token
            except ValueError:
                return None
    return header, data


# ---------------------------------------------------------------------------------------------- quaternions (w first)
def q_mul(a, b):
    aw, ax, ay, az = np.moveaxis(a, -1, 0)
    bw, bx, by, bz = np.moveaxis(b, -1, 0)
    return np.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], axis=-1)


def q_inv(a):
    return a * np.array([1.0, -1.0, -1.0, -1.0])


def q_rot(q, v):
    u = q[..., 1:]
    t = 2.0 * np.cross(u, v)
    return v + q[..., :1] * t + np.cross(u, t)


def q_from_euler_deg(e, order):
    half = np.radians(e) * 0.5
    qs = []
    for i, c in enumerate(order):
        qs.append(np.concatenate([np.cos(half[..., i:i + 1]), np.sin(half[..., i:i + 1]) * _AXIS[c]], axis=-1))
    return q_mul(qs[0], q_mul(qs[1], qs[2]))


def q_unroll(q):
    """Flip signs frame to frame so consecutive quaternions stay in one hemisphere (quat.py:130-136)."""
    q = q.copy()
    for t in range(1, len(q)):
        flip = np.sum(q[t] * q[t - 1], axis=-1) < 0.0
        q[t][flip] = -q[t][flip]
    return q


def q_positive(q):
    return np.where(q[..., :1] > 0.0, q, -q)


def q_to_helical(q, eps=1e-5):
    n = np.linalg.norm(q[..., 1:], axis=-1, keepdims=True)
    half = np.where(n < eps, np.ones_like(n), np.arctan2(n, q[..., :1]) / np.where(n < eps, 1.0, n))
    return 2.0 * half * q[..., 1:]


def q_between(a, b):
    return np.concatenate([np.sqrt(np.sum(a * a, -1) * np.sum(b * b, -1))[..., None] + np.sum(a * b, -1)[..., None], np.cross(a, b)], axis=-1)


def fk(lrot, lpos, parents):
    grot, gpos = [lrot[:, 0]], [lpos[:, 0]]
    for j in range(1, len(parents)):
        p = int(parents[j])
        gpos.append(q_rot(grot[p], lpos[:, j]) + gpos[p])
        grot.append(q_mul(grot[p], lrot[:, j]))
    return np.stack(grot, axis=1), np.stack(gpos, axis=1)


def _diff_with_extrapolated_first(x, dt, fn=None):
    """v[1:] = d/dt, v[0] = v[1] - (v[3] - v[2])  (data_pipeline.py:143-160)."""
    v = np.zeros_like(x[..., :3]) if fn is not None else np.zeros_like(x)
    v[1:] = (fn(x[1:], x[:-1]) if fn is not None else (x[1:] - x[:-1])) / dt
    v[0] = v[1] - (v[3] - v[2])
    return v


def preprocess_animation(anim):
    """data_pipeline.py:89-180 -> dict with the 8 pose tensors + gaze_pos / gaze_dir (float32, the reference's shapes)."""
    names = list(anim["names"])
    parents = anim["parents"]
    dt = float(anim["frametime"])
    lrot = q_unroll(q_from_euler_deg(np.asarray(anim["rotations"], dtype=np.float64), anim["order"]))
    lpos = np.asarray(anim["positions"], dtype=np.float64).copy()
    T = len(lrot)
    if T < 4:
        raise ValueError("preprocess_animation needs at least 4 frames (the first velocity is extrapolated from frames 1..3)")
    grot, gpos = fk(lrot, lpos, parents)
    ground = np.array([1.0, 0.0, 1.0])
    root_pos = gpos[:, names.index("Spine2")] * ground
    fwd = q_rot(grot[:, names.index("Hips")], _AXIS["z"][None]) * ground
    fwd /= np.linalg.norm(fwd, axis=-1, keepdims=True)
    root_rot = q_between(np.repeat(_AXIS["z"][None], T, axis=0), fwd)
    root_rot /= np.linalg.norm(root_rot, axis=-1, keepdims=True)
    look = q_rot(grot[:, names.index("Head")], _AXIS["z"][None]) * ground
    look /= np.linalg.norm(look, axis=-1, keepdims=True)
    gaze_pos = np.repeat(np.median(root_pos + 100.0 * look, axis=0)[None], T, axis=0)
    inv_root = q_inv(root_rot)
    gaze_dir = q_rot(inv_root, gaze_pos - root_pos)
    lrot[:, 0] = q_mul(inv_root, lrot[:, 0])
    lpos[:, 0] = q_rot(inv_root, lpos[:, 0] - root_pos)
    ang = lambda a, b: q_to_helical(q_positive(q_mul(a, q_inv(b))))
    lvel = _diff_with_extrapolated_first(lpos, dt)
    lvrt = _diff_with_extrapolated_first(lrot, dt, ang)
    prev_inv = np.concatenate([inv_root[:1], inv_root[:-1]], axis=0)          # frame 0 uses its own rotation (:155-160)
    root_vrt = q_rot(prev_inv, _diff_with_extrapolated_first(root_rot, dt, ang))
    root_vel = q_rot(prev_inv, _diff_with_extrapolated_first(root_pos, dt))
    ltxy = np.stack([q_rot(lrot, _AXIS["x"]), q_rot(lrot, _AXIS["y"])], axis=-2)
    f = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return dict(root_pos=f(root_pos), root_rot=f(root_rot), root_vel=f(root_vel), root_vrt=f(root_vrt), lpos=f(lpos), lrot=f(lrot),
                ltxy=f(ltxy), lvel=f(lvel), lvrt=f(lvrt), gaze_pos=f(gaze_pos), gaze_dir=f(gaze_dir))


def trim(anim, start_end):
    """Frame range cut applied to the RAW animation before feature extraction (generate.py:196-203)."""
    if start_end is None:
        return anim
    out = dict(anim)
    out["rotations"] = anim["rotations"][start_end[0]:start_end[1]]
    out["positions"] = anim["positions"][start_end[0]:start_end[1]]
    return out
