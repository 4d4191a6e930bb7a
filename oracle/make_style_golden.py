"""Generate the goldens of the StyleEncoder variants beyond the shipped attn + VAE by running the UNMODIFIED reference (imported
from /root/reference via oracle/ref_shim.py) on seeded synthetic inputs:

    tests/golden/style_gru.npz          the reference's StyleEncoder alone: type 'gru' with the VAE on and off, type 'attn' without it
    tests/golden/train_gru_h64.npz      whole train step (loss, 18 terms, gradients), GRU style encoder with the VAE, H = 64
    tests/golden/train_gru_h384.npz     the same without the VAE, H = 384 (tensor-core engine eligible)

Run in the dev container (the reference tree does not exist on the GPU box):
    python -m oracle.make_style_golden [style_gru] [gru_h64] [gru_h384]
Weights are regenerated from zeggs_b200.synth.make_params(seed, style_type=...) on both sides; the train-step goldens use the same
inputs, seeds and file layout as oracle/make_golden.py's train_h*.npz.
"""
import os

import numpy as np
import torch

from oracle import ref_shim
from oracle.make_golden import GOLD, ref_train_losses, stats_t, tt
from zeggs_b200 import synth

POSE = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt"]
LOSS_KEYS = ["loss_root_pos", "loss_root_rot", "loss_root_vel", "loss_root_vrt", "loss_lpos", "loss_lrot", "loss_lvel", "loss_lvrt",
             "loss_cpos", "loss_crot", "loss_cvel", "loss_cvrt", "loss_ldvl", "loss_ldvt", "loss_cdvl", "loss_cdvt", "loss_gaze",
             "loss_kl_div"]

# style encoders alone: tag -> (type, use_vae, style hidden, B, T_ex, param seed)
STYLE_CASES = {
    "gru_vae_h64_t16": ("gru", True, 64, 2, 16, 31), "gru_novae_h64_t16": ("gru", False, 64, 2, 16, 32),
    "gru_vae_h64_t33": ("gru", True, 64, 2, 33, 33), "gru_novae_h64_t33": ("gru", False, 64, 2, 33, 34),
    "gru_vae_h512_t256": ("gru", True, 512, 2, 256, 35), "gru_novae_h512_t256": ("gru", False, 512, 2, 256, 36),
    "attn_novae_h64_t16": ("attn", False, 64, 2, 16, 37),
}
# train steps: tag -> (H, B, T, T_ex, style type, use_vae)
TRAIN_CASES = {"gru_h64": (64, 2, 6, 16, "gru", True), "gru_h384": (384, 4, 12, 24, "gru", False)}


def write_style_golden(Z=64, temperature=1.3):
    """The reference's own StyleEncoder, eval mode, on synth weights (synth.make_params(style_type=..., style_hidden=...,
    style_embed=2Z or Z, seed)) and a normalised synth example; VAE noise injected (eps) into the reference's re-parameterisation
    line.  Stored per case: the outputs and the parameter gradients of sum(out * cotangent) -- elementwise up to 4096 elements, as
    norms otherwise.  Also the state-dict keys and shapes of the v1-sized GRU encoders (StyleEncoder(1134, 512, 64, type='gru'))."""
    m = ref_shim.ref_modules()
    _, _, i_mu, i_sd, _, _, _, _ = stats_t()
    out = {"Z": Z, "temperature": temperature}
    for tag, (typ, vae, Hs, B, T_ex, seed) in STYLE_CASES.items():
        E = 2 * Z if vae else Z
        P = synth.make_params(H=64, seed=seed, style_hidden=Hs, style_embed=E, style_type=typ)
        net = m.StyleEncoder(synth.P_IN, Hs, Z, type=typ, use_vae=vae)
        net.load_state_dict({k[len("style_encoder."):]: torch.from_numpy(v) for k, v in P.items() if k.startswith("style_encoder.")})
        net.eval()
        x = (torch.from_numpy(synth.make_style_example(B, T_ex, seed=seed)) - i_mu) / i_sd
        rs = np.random.RandomState(seed)
        eps = rs.randn(B, Z).astype(np.float32)
        enc = net.encoder(x)
        if vae:                                             # modules.py:291-302 with eps injected
            mu, logvar = enc[:, :Z], enc[:, Z:]
            outs = [mu + torch.from_numpy(eps) * (torch.exp(0.5 * logvar) / temperature), mu, logvar]
        else:                                               # modules.py:303-304
            outs = [enc]
        cots = [rs.randn(*o.shape).astype(np.float32) for o in outs]
        names = [n for n, _ in net.named_parameters()]
        grads = torch.autograd.grad(sum((o * torch.from_numpy(c)).sum() for o, c in zip(outs, cots)), list(net.parameters()))
        rec = dict(type=typ, use_vae=vae, H=Hs, B=B, T_ex=T_ex, param_seed=seed, eps=eps)
        for n, o, c in zip(("z", "mu", "logvar"), outs, cots):
            rec[n] = o.detach().numpy(); rec["cot_" + n] = c
        for n, gr in zip(names, grads):
            rec["gradnorm." + n] = np.float64(gr.double().norm().item())
            if gr.numel() <= 4096:
                rec["grad." + n] = gr.numpy()
        out.update({f"{tag}.{k}": v for k, v in rec.items()})
    for vae in (True, False):
        sd = m.StyleEncoder(synth.P_IN, 512, 64, type="gru", use_vae=vae).state_dict()
        out[f"keys_vae{int(vae)}"] = np.array(list(sd.keys()))
        out[f"shapes_vae{int(vae)}"] = np.array([list(v.shape) + [0] * (3 - v.dim()) for v in sd.values()], dtype=np.int64)
    np.savez_compressed(os.path.join(GOLD, "style_gru.npz"), **out)
    print("style_gru golden written:", os.path.getsize(os.path.join(GOLD, "style_gru.npz")), "bytes")


def write_train_golden(tag, S=64, Z=64):
    """The reference's train-step forward (eval mode, injected VAE eps where there is a VAE) and its own loss lines
    (train.py:277-421; without the VAE mu = logvar = None, so the KL term is 0 and the sum is still / 18), then autograd."""
    H, B, T, T_ex, style_type, use_vae = TRAIN_CASES[tag]
    P = synth.make_params(H=H, seed=11, style_type=style_type, style_embed=2 * Z if use_vae else Z)
    m = ref_shim.ref_modules()
    se, de = m.SpeechEncoder(synth.N_AUDIO, S, S), m.Decoder(synth.P_IN, synth.P_OUT, S, Z, H, 2)
    st = m.StyleEncoder(synth.P_IN, 512, Z, type=style_type, use_vae=use_vae)
    Pt = tt(P)
    for net, pre in ((se, "speech_encoder."), (de, "decoder."), (st, "style_encoder.")):
        net.load_state_dict({k[len(pre):]: v for k, v in Pt.items() if k.startswith(pre)})
        net.eval()
    win = synth.make_pose_windows(B, T, seed=5)
    audio = synth.make_audio_features(B, T, seed=5)
    style_ex = synth.make_style_example(B, T_ex, seed=5)
    eps = np.random.RandomState(3).randn(B, Z).astype(np.float32)
    a_mu, a_sd, i_mu, i_sd, o_mu, o_sd, parents, dt = stats_t()
    W = tt(win)
    speech = se((torch.from_numpy(audio) - a_mu) / a_sd)
    enc = st.encoder((torch.from_numpy(style_ex) - i_mu) / i_sd)
    if use_vae:
        mu, logvar = enc[:, :Z], enc[:, Z:]
        z = mu + torch.from_numpy(eps) * torch.exp(0.5 * logvar)
    else:
        z, mu, logvar = enc, None, None
    O = de(W["root_pos"][:, 0], W["root_rot"][:, 0], W["root_vel"][:, 0], W["root_vrt"][:, 0], W["lpos"][:, 0],
           W["ltxy"][:, 0], W["lvel"][:, 0], W["lvrt"][:, 0], W["gaze_pos"], speech, z.unsqueeze(1).repeat((1, T, 1)),
           parents, i_mu, i_sd, o_mu, o_sd, dt)
    ns = {"O_" + n: o for n, o in zip(POSE, O)}
    ns.update({"W_" + n: W[n] for n in POSE})
    ns.update(W_gaze_pos=W["gaze_pos"], parents=parents, dt=dt, mu=mu, logvar=logvar, iteration=9000)
    env = ref_train_losses(ns)
    loss = env["loss"]
    nets = (("speech_encoder.", se), ("decoder.", de), ("style_encoder.", st))
    names = [pre + n for pre, net in nets for n, _ in net.named_parameters()]
    grads = torch.autograd.grad(loss, [p for _, net in nets for p in net.parameters()])
    d = dict(H=H, B=B, T=T, T_ex=T_ex, param_seed=11, input_seed=5, eps=eps, iteration=9000, style_type=style_type, use_vae=use_vae,
             speech=speech.detach().numpy(), z=z.detach().numpy(), loss=np.float64(loss.item()))
    if use_vae:
        d.update(mu=mu.detach().numpy(), logvar=logvar.detach().numpy())
    for n, o in zip(POSE, O):
        d["O_" + n] = o.detach().numpy()
    for k in LOSS_KEYS:
        d[k] = np.float64(float(env[k]))
    d.update({"grad." + n: x.detach().numpy() for n, x in zip(names, grads) if x.numel() <= 4096})
    d.update({"gradnorm." + n: np.float64(x.double().norm().item()) for n, x in zip(names, grads)})
    np.savez_compressed(os.path.join(GOLD, f"train_{tag}.npz"), **d)
    print(tag, "loss", loss.item())


def main(only=None):
    os.makedirs(GOLD, exist_ok=True)
    torch.manual_seed(0)
    for tag in only or ["style_gru"] + list(TRAIN_CASES):
        if tag == "style_gru":
            write_style_golden()
        else:
            write_train_golden(tag)


if __name__ == "__main__":
    import sys
    main(only=sys.argv[1:] or None)
