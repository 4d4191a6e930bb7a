"""BVH text writer for generated motion.  The values come from the device post-step (ops.pose_to_bvh_channels: the numbers the
reference's utils.write_bvh hands to anim/bvh.py:save, ZEGGS/utils.py:47-87); this module only lays them out as text in the same
file layout (HIERARCHY with OFFSET = first-frame local positions, root with 6 channels, joints with 3 rotation channels in `order`,
MOTION with one line per frame in depth-first joint order, anim/bvh.py:136-219).  Host-side file formatting: outside the
accelerated path, kept so the drop-in needs nothing from the reference tree to write its result."""
import numpy as np

_CH = {"x": "Xrotation", "y": "Yrotation", "z": "Zrotation"}


def _walk(parents):
    """Depth-first joint order with, for every joint, its children in index order (the order bvh.py:save visits them)."""
    children = [[] for _ in parents]
    for i, p in enumerate(parents):
        if i != 0 and p >= 0:
            children[p].append(i)
    return children


def save_bvh(filename, positions, rotations_deg, parents, names=None, order="zyx", frametime=1.0 / 60.0, offsets=None):
    """positions [T,J,3] (joint 0 = root trajectory), rotations_deg [T,J,3] in `order`; offsets [J,3] gives every OFFSET (default: the
    first frame of positions)."""
    positions = np.asarray(positions)
    rotations_deg = np.asarray(rotations_deg)
    parents = [int(p) for p in parents]
    J = len(parents)
    names = list(names) if names is not None else [f"joint_{i}" for i in range(J)]
    children = _walk(parents)
    offsets = positions[0] if offsets is None else np.asarray(offsets)
    rot_names = " ".join(_CH[c] for c in order)
    lines, seq = [], []

    def emit(i, tabs, root):
        seq.append(i)
        t = "\t" * tabs
        lines.append(f"{t}{'ROOT' if root else 'JOINT'} {names[i]}\n{t}{{\n")
        t1 = t + "\t"
        lines.append("%sOFFSET %f %f %f\n" % ((t1,) + tuple(float(v) for v in offsets[i])))
        if root:
            lines.append(f"{t1}CHANNELS 6 Xposition Yposition Zposition {rot_names} \n")
        else:
            lines.append(f"{t1}CHANNELS 3 {rot_names}\n")
        for c in children[i]:
            emit(c, tabs + 1, False)
        if not children[i] and not root:
            lines.append(f"{t1}End Site\n{t1}{{\n{t1}\tOFFSET %f %f %f\n{t1}}}\n" % (0.0, 0.0, 0.0))
        lines.append(f"{t}}}\n")

    emit(0, 0, True)
    T = rotations_deg.shape[0]
    cols = [positions[:, 0, :]] + [rotations_deg[:, j, :] for j in seq]
    table = np.concatenate(cols, axis=1).astype(np.float64)
    with open(filename, "w") as f:
        f.write("HIERARCHY\n")
        f.writelines(lines)
        f.write("MOTION\n")
        f.write("Frames: %i\n" % T)
        f.write("Frame Time: %f\n" % frametime)
        fmt = " ".join(["%f"] * table.shape[1]) + " \n"
        f.writelines(fmt % tuple(row) for row in table)
