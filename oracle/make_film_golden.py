"""Write tests/golden/train_film_h64.npz and train_film_h128.npz by running the UNMODIFIED reference's Decoder(rnn_cond="film")
(imported through oracle/ref_shim.py) in a whole train step: the window forward, the reference's own loss lines and autograd.
Same layout as the train_h* goldens of oracle/make_golden.py (weights regenerated from zeggs_b200.synth.make_params(seed,
rnn_cond="film") on both sides, inputs from their seeds, outputs / loss terms / gradients stored).

Run where the reference tree is readable:
    python -m oracle.make_film_golden
"""
import os

import numpy as np
import torch

from oracle import make_golden as mg
from oracle import ref_shim
from zeggs_b200 import synth

# tag: (H, B, T, T_ex); B, T != 3: the reference's dim-less torch.cross in its loss differs from the last-dim cross there
FILM_CASES = {"film_h64": (64, 4, 17, 16), "film_h128": (128, 4, 17, 16)}


def write_film_golden(tag):
    H, B, T, T_ex = FILM_CASES[tag]
    P = synth.make_params(H=H, seed=11, rnn_cond="film")
    m = ref_shim.ref_modules()
    se, st = m.SpeechEncoder(synth.N_AUDIO, 64, 64), m.StyleEncoder(synth.P_IN, 512, 64, type="attn", use_vae=True)
    de = m.Decoder(synth.P_IN, synth.P_OUT, 64, 64, H, 2, rnn_cond="film")
    Pt = mg.tt(P)
    for pre, net in (("speech_encoder.", se), ("decoder.", de), ("style_encoder.", st)):
        net.load_state_dict({k[len(pre):]: v for k, v in Pt.items() if k.startswith(pre)})
        net.eval()
    win = synth.make_pose_windows(B, T, seed=5)
    audio = synth.make_audio_features(B, T, seed=5)
    style_ex = synth.make_style_example(B, T_ex, seed=5)
    eps = np.random.RandomState(3).randn(B, 64).astype(np.float32)
    speech, (z, mu, logvar), O, env = mg.ref_forward_train(se, st, de, win, audio, style_ex, eps, iteration=9000)
    loss = env["loss"]
    params = list(se.parameters()) + list(de.parameters()) + list(st.parameters())
    names = (["speech_encoder." + n for n, _ in se.named_parameters()] + ["decoder." + n for n, _ in de.named_parameters()] +
             ["style_encoder." + n for n, _ in st.named_parameters()])
    grads = torch.autograd.grad(loss, params)
    d = dict(H=H, B=B, T=T, T_ex=T_ex, param_seed=11, input_seed=5, eps=eps, iteration=9000, rnn_cond="film",
             speech=speech.detach().numpy(), z=z.detach().numpy(), mu=mu.detach().numpy(), logvar=logvar.detach().numpy(),
             loss=np.float64(loss.item()))
    for n, o in zip(["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt"], O):
        d["O_" + n] = o.detach().numpy()
    for k in ["loss_root_pos", "loss_root_rot", "loss_root_vel", "loss_root_vrt", "loss_lpos", "loss_lrot", "loss_lvel", "loss_lvrt",
              "loss_cpos", "loss_crot", "loss_cvel", "loss_cvrt", "loss_ldvl", "loss_ldvt", "loss_cdvl", "loss_cdvt", "loss_gaze",
              "loss_kl_div"]:
        d[k] = np.float64(float(env[k]))
    d.update({"grad." + n: x.detach().numpy() for n, x in zip(names, grads) if x.numel() <= 4096})
    d.update({"gradnorm." + n: np.float64(x.double().norm().item()) for n, x in zip(names, grads)})
    np.savez_compressed(os.path.join(mg.GOLD, f"train_{tag}.npz"), **d)
    print(tag, "loss", loss.item())


if __name__ == "__main__":
    torch.set_num_threads(8)
    for tag in FILM_CASES:
        write_film_golden(tag)
