"""BVH text writer for generated motion.  The values come from the device post-step (ops.pose_to_bvh_channels: the numbers the
reference's utils.write_bvh hands to anim/bvh.py:save, ZEGGS/utils.py:47-87); this module only lays them out as text in the same
file layout (HIERARCHY with OFFSET = first-frame local positions, root with 6 channels, joints with 3 rotation channels in `order`,
MOTION with one line per frame in depth-first joint order, anim/bvh.py:136-219), so the drop-in needs nothing from the reference tree to
write its result.  With CUDA tensors the MOTION rows are formatted on the device (zeggs_bvh_format_motion, byte-identical); with numpy
arrays, on the host as below."""
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
    on_device = _is_cuda(positions) and _is_cuda(rotations_deg)
    if not on_device:
        positions = np.asarray(positions)
        rotations_deg = np.asarray(rotations_deg)
    parents = [int(p) for p in parents]
    J = len(parents)
    names = list(names) if names is not None else [f"joint_{i}" for i in range(J)]
    children = _walk(parents)
    if offsets is None:
        offsets = positions[0].cpu().numpy() if on_device else positions[0]
    else:
        offsets = np.asarray(offsets)
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
    block = _format_motion_device(positions, rotations_deg, seq) if on_device else None
    if on_device and block is None:
        positions, rotations_deg = positions.cpu().numpy(), rotations_deg.cpu().numpy()
    table = _motion_table(positions, rotations_deg, seq) if block is None else None
    with open(filename, "w") as f:
        f.write("HIERARCHY\n")
        f.writelines(lines)
        f.write("MOTION\n")
        f.write("Frames: %i\n" % T)
        f.write("Frame Time: %f\n" % frametime)
        if block is not None:
            f.flush()
            f.buffer.write(block)
        else:
            f.writelines(_row_format(table.shape[1]) % tuple(row) for row in table)


def _motion_table(positions, rotations_deg, seq):
    cols = [positions[:, 0, :]] + [rotations_deg[:, j, :] for j in seq]
    return np.concatenate(cols, axis=1).astype(np.float64)


def _row_format(ncol):
    return " ".join(["%f"] * ncol) + " \n"


def _is_cuda(x):
    return getattr(x, "is_cuda", False) is True


# values too large for the device's 128-bit "%f" (|v| >= 2^128 / 10^6) are formatted here, row by row; with more than this many the
# whole block is formatted on the host
MAX_FLAGGED_VALUES = 1 << 12


def _format_motion_device(positions, rotations_deg, seq):
    """MOTION rows of CUDA tensors positions / rotations_deg [T,J,3] by zeggs_bvh_format_motion -> a bytes-like block, or None when
    the host writer must do it (shapes it does not cover, or more than MAX_FLAGGED_VALUES values beyond the 128-bit path)."""
    import ctypes as C
    import torch
    from . import _lib
    T, J = int(rotations_deg.shape[0]), int(rotations_deg.shape[1])
    if positions.shape != rotations_deg.shape or rotations_deg.dim() != 3 or rotations_deg.shape[2] != 3 or len(seq) != J:
        return None
    if positions.device != rotations_deg.device:
        return None
    if positions.dtype == rotations_deg.dtype == torch.float32:
        f64 = 0
    else:
        f64 = 1
        positions, rotations_deg = positions.to(torch.float64), rotations_deg.to(torch.float64)
    positions, rotations_deg = positions.contiguous(), rotations_deg.contiguous()
    dev = positions.device
    l = _lib.lib()
    with torch.cuda.device(dev):
        out = torch.empty(int(l.zeggs_bvh_format_motion_max_size(T, J)), dtype=torch.uint8, device=dev)
        row_start = torch.empty(T + 1, dtype=torch.int64, device=dev)
        flagged = torch.empty(MAX_FLAGGED_VALUES, dtype=torch.int64, device=dev)
        status = torch.empty(2, dtype=torch.int64, device=dev)
        seq_dev = torch.tensor(seq, dtype=torch.int32).to(dev)
        ws = torch.empty(int(l.zeggs_bvh_format_motion_workspace_size(T, J)), dtype=torch.uint8, device=dev)
        a = _lib.BvhFormatArgs(T=T, J=J, in_f64=f64, max_flagged=MAX_FLAGGED_VALUES, positions=positions.data_ptr(),
                               rotations=rotations_deg.data_ptr(), seq=seq_dev.data_ptr(), out=out.data_ptr(), out_capacity=out.numel(),
                               row_start=row_start.data_ptr(), flagged=flagged.data_ptr(), status=status.data_ptr(),
                               workspace=ws.data_ptr(), workspace_bytes=ws.numel())
        _lib.check(l.zeggs_bvh_format_motion(C.byref(a), _lib.stream_ptr()), "zeggs_bvh_format_motion")
        total, nflag = (int(v) for v in status.cpu())
        if nflag > MAX_FLAGGED_VALUES:
            return None
        block = torch.empty(total, dtype=torch.uint8, pin_memory=True)
        block.copy_(out[:total])
        if not nflag:
            return block.numpy()
        # rows holding a value beyond the 128-bit path: the device left them incomplete, the host writes them whole
        ncol = 3 + 3 * J
        bad = sorted({int(i) // ncol for i in flagged[:nflag].cpu().numpy()})
        starts = row_start.cpu().numpy()
        text, parts, pos = block.numpy(), [], 0
        for t in bad:
            table = _motion_table(positions[t:t + 1].cpu().numpy(), rotations_deg[t:t + 1].cpu().numpy(), seq)
            parts += [text[pos:starts[t]].tobytes(), (_row_format(ncol) % tuple(table[0])).encode("ascii")]
            pos = starts[t + 1]
        parts.append(text[pos:].tobytes())
        return b"".join(parts)
