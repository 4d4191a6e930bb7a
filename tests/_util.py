import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

NAMES = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt"]


def ensure_built():
    import __graft_entry__ as g
    g.build()


def tt(d, device=None):
    return {k: torch.from_numpy(np.asarray(v)).to(device) if device else torch.from_numpy(np.asarray(v)) for k, v in d.items()}


def stats_tensors(device=None):
    from zeggs_b200 import synth
    st = synth.load_stats()
    out = {k: torch.as_tensor(st[k], dtype=torch.float32) for k in
           ("audio_input_mean", "audio_input_std", "anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")}
    if device:
        out = {k: v.to(device) for k, v in out.items()}
    out["parents"] = torch.as_tensor(st["parents"])
    out["dt"] = float(st["dt"])
    return out


def make_decoder(P, H, S=64, Z=64, device="cuda"):
    from zeggs_b200 import modules
    dec = modules.Decoder(1134, 1131, S, Z, H, 2)
    dec.load_state_dict({k[len("decoder."):]: torch.from_numpy(v) for k, v in P.items() if k.startswith("decoder.")})
    return dec.to(device).eval()


def report(name, got, ref):
    got = got.detach().float().cpu()
    ref = ref.detach().float().cpu()
    err = float((got - ref).abs().max())
    scale = float(ref.abs().max())
    print(f"  [{name}] max-abs err {err:.3e} (ref max {scale:.3e})")
    return err, scale


# ---------------------------------------------------------------------------------------------- training loss
LOSS_KL_ITER = 7000           # kl_weight(7000) = 0.076: below the 0.2 clip, so a wrong weight shows


def loss_case(B, T, seed, copy_frame0=False, Z=64):
    """Inputs of one training-loss call, fp32 on the CPU: O (decoder output) and W (ground truth) as lists in NAMES order,
    the ground truth's gaze_pos, mu and logvar [B,Z].  copy_frame0: O's frame 0 is W's, as the decoder returns it."""
    from zeggs_b200 import synth
    O = tt(synth.make_pose_windows(B, T, seed=seed))
    W = tt(synth.make_pose_windows(B, T, seed=seed + 1))
    if copy_frame0:
        for k in NAMES:
            O[k][:, 0] = W[k][:, 0]
    rs = np.random.RandomState(seed)
    mu = torch.from_numpy(rs.randn(B, Z).astype(np.float32))
    lv = torch.from_numpy((rs.randn(B, Z) * 0.3).astype(np.float32))
    return [O[k] for k in NAMES], [W[k] for k in NAMES], W["gaze_pos"], mu, lv


def oracle_loss_grads(O, W, gaze, parents, dt, mu=None, lv=None, dtype=torch.float64, loss_fn=None):
    """model_oracle.train_losses (or loss_fn with its signature) in `dtype` and its autograd -> (total, {term: value},
    {pose name / "mu" / "logvar": gradient of the total})."""
    from oracle import model_oracle as mo
    Ot = [o.to(dtype).requires_grad_(True) for o in O]
    leaves = list(Ot)
    if mu is not None:
        mu, lv = mu.to(dtype).requires_grad_(True), lv.to(dtype).requires_grad_(True)
        leaves += [mu, lv]
    total, L = (loss_fn or mo.train_losses)(Ot, [w.to(dtype) for w in W], gaze.to(dtype), parents, dt, mu, lv, LOSS_KL_ITER)
    gs = torch.autograd.grad(total, leaves)
    names = NAMES + (["mu", "logvar"] if mu is not None else [])
    return float(total.detach()), {k: float(v.detach()) for k, v in L.items()}, dict(zip(names, gs))


def loss_ambiguous_frames(O, W, gaze, parents, dt):
    """Frames whose loss gradient an fp32 implementation may legitimately get wrong -> (mask for dY and dRootPos, mask for
    dRootRot), bool [B,T].  Every gradient element is a weighted sum of sign(residual); a residual within rounding of zero
    can take either sign in fp32.  A residual is ambiguous if 0 < |r64| <= 16 x (the largest |r_fp32 - r64| of its channel
    over the case); an exact float64 zero comes from bitwise-equal inputs, which fp32 also maps to 0.  dY / dRootPos of frame
    f depend on f's direct residuals and the difference residuals f-1 and f; dRootRot of f also on frame f+1's direct residuals
    (its world root velocities rotate by f's rotation)."""
    from oracle import model_oracle as mo
    r64 = mo.loss_residuals([o.double() for o in O], [w.double() for w in W], gaze.double(), parents, dt)
    r32 = mo.loss_residuals([o.float() for o in O], [w.float() for w in W], gaze.float(), parents, dt)
    B, T = O[0].shape[:2]
    direct = torch.zeros(B, T, dtype=torch.bool)
    diff = torch.zeros(B, T - 1, dtype=torch.bool)
    for k, a in r64.items():
        margin = 16.0 * (r32[k].double() - a).abs().flatten(0, 1).amax(dim=0)
        amb = ((a != 0) & (a.abs() <= margin)).flatten(2).any(dim=2)
        if k in mo.DIFF_TERMS:
            diff |= amb
        else:
            direct |= amb
    y = direct.clone()
    y[:, 1:] |= diff
    y[:, :-1] |= diff
    rot = y.clone()
    rot[:, :-1] |= direct[:, 1:]
    return y, rot


def unpack_pose_grad(dY, dRootPos, dRootRot):
    """The loss kernel's gradients (dY packed like train.pack_pose) -> {pose name: gradient} with the pose tensors' shapes."""
    B, T = dY.shape[:2]
    nj = 75
    sizes = [("root_vel", (3,)), ("root_vrt", (3,)), ("lpos", (nj, 3)), ("ltxy", (nj, 2, 3)), ("lvel", (nj, 3)), ("lvrt", (nj, 3))]
    out, o = dict(root_pos=dRootPos, root_rot=dRootRot), 0
    for n, shp in sizes:
        k = int(np.prod(shp))
        out[n] = dY[..., o:o + k].reshape(B, T, *shp)
        o += k
    return out


def masked_grad_errors(got, ref, amb_y, amb_rot):
    """Per pose gradient: the largest |got - ref| over the frames the masks leave in, relative to max |ref| over all frames.
    Asserts that every element of `got`, excluded frames included, is finite."""
    res = {}
    for n in NAMES:
        g, r = got[n].detach().double().cpu(), ref[n].detach().double().cpu()
        assert g.shape == r.shape, n
        assert bool(torch.isfinite(g).all()), n
        keep = ~(amb_rot if n == "root_rot" else amb_y)
        err = float((g - r).abs()[keep].max()) if bool(keep.any()) else 0.0
        res[n] = err / max(float(r.abs().max()), 1e-30)
    return res


def run_with_grads(fn, P, win, speech, style, cot, **kw):
    """float64 forward of fn (model_oracle.decoder_forward signature) + autograd of sum(out * cot) -> (outputs, {name: gradient}).
    Gradients the outputs do not depend on are zero."""
    st = stats_tensors()
    Pt = {k: torch.from_numpy(v).double().requires_grad_(k.startswith("decoder.")) for k, v in P.items()}
    sp, sy = speech.double().requires_grad_(True), style.double().requires_grad_(True)
    out = fn(Pt, *[win[n][:, 0].double() for n in NAMES], win["gaze_pos"].double(), sp, sy,
             *[st[k].double() for k in ("anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")], st["dt"], **kw)
    keys = sorted(k for k in Pt if k.startswith("decoder."))
    leaves = [Pt[k] for k in keys] + [sp, sy]
    loss = sum((o * c.double()).sum() for o, c in zip(out, cot))
    if loss.requires_grad:
        gs = torch.autograd.grad(loss, leaves, allow_unused=True)
    else:
        gs = [None] * len(leaves)
    grads = {k: (g if g is not None else torch.zeros_like(x)) for k, g, x in zip(keys + ["speech", "style"], gs, leaves)}
    return [o.detach() for o in out], grads
