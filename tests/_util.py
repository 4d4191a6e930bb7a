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
