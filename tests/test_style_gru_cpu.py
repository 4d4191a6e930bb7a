"""StyleEncoder type 'gru' and use_vae=False (modules.py:278-343) without a GPU: the parameter containers against the reference's
state-dict layout, whole-module pickles, and the oracle restatement against what the unmodified reference computed
(tests/golden/style_gru.npz, tests/golden/train_gru_*.npz; oracle/make_style_golden.py)."""
import io
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import model_oracle as mo, style_oracle as so
from tests._util import NAMES, tt
from zeggs_b200 import synth


def _style_params(g, tag):
    typ, vae = str(g[tag + ".type"]), bool(g[tag + ".use_vae"])
    Z = int(g["Z"])
    P = synth.make_params(H=64, seed=int(g[tag + ".param_seed"]), style_hidden=int(g[tag + ".H"]), style_embed=2 * Z if vae else Z,
                          style_type=typ)
    return typ, vae, {k: torch.from_numpy(v).requires_grad_(True) for k, v in P.items() if k.startswith("style_encoder.")}


@pytest.mark.parametrize("use_vae", [True, False])
def test_gru_style_encoder_has_the_reference_state_dict(golden_dir, use_vae):
    from zeggs_b200 import modules
    g = np.load(os.path.join(golden_dir, "style_gru.npz"))
    enc = modules.StyleEncoder(1134, 512, 64, type="gru", use_vae=use_vae)
    sd = enc.state_dict()
    keys = [str(k) for k in g[f"keys_vae{int(use_vae)}"]]
    assert list(sd.keys()) == keys
    for k, shp in zip(keys, g[f"shapes_vae{int(use_vae)}"]):
        assert tuple(sd[k].shape) == tuple(int(s) for s in shp if s), k
    assert sum(p.numel() for p in enc.parameters()) == (5_812_352 if use_vae else 5_746_752)
    assert enc.encoder_type == "gru"
    assert len(enc._weights()) == len(list(enc.parameters()))


def test_gru_train_setup_parameter_count():
    """v1 sizes with the GRU style encoder: 29,250,027 trainable parameters (25,543,147 with attn)."""
    from zeggs_b200 import train
    opts = {"speech_encoder": {"nhidden": 64, "speech_encoding_size": 64},
            "style_encoder": {"nhidden": 512, "style_encoding_size": 64, "type": "gru", "use_vae": True},
            "decoder": {"nhidden": 1024}}
    dims = {"num_audio_features": 81, "pose_input_size": 1134, "pose_output_size": 1131}
    nets = train.build_networks(opts, dims, "example", 9, "cpu")
    assert sum(p.numel() for n in nets for p in n.parameters()) == 29_250_027
    opts["style_encoder"]["type"] = "attn"
    nets = train.build_networks(opts, dims, "example", 9, "cpu")
    assert sum(p.numel() for n in nets for p in n.parameters()) == 25_543_147


def test_unknown_style_encoder_type_raises():
    from zeggs_b200 import _lib, modules
    with pytest.raises(_lib.ZeggsError):
        modules.StyleEncoder(1134, 512, 64, type="lstm", use_vae=True)


@pytest.mark.parametrize("use_vae", [True, False])
def test_gru_style_encoder_whole_module_pickle_round_trip(use_vae):
    """torch.save(module) as train.py:482-509 writes it round-trips; the reference's pickles name the classes modules.StyleEncoder /
    modules.StyleEncoderGRU, which resolve to ours with this package registered as `modules` (generate.load_networks does so)."""
    import sys
    from zeggs_b200 import modules
    enc = modules.StyleEncoder(1134, 64, 64, type="gru", use_vae=use_vae)
    buf = io.BytesIO()
    torch.save(enc, buf)
    buf.seek(0)
    got = torch.load(buf, weights_only=False)
    assert type(got) is modules.StyleEncoder and type(got.encoder) is modules.StyleEncoderGRU
    assert got.use_vae == use_vae and got.encoder_type == "gru"
    saved = sys.modules.get("modules")
    sys.modules["modules"] = modules
    try:
        up = pickle.Unpickler(io.BytesIO(b""))
        assert up.find_class("modules", "StyleEncoder") is modules.StyleEncoder
        assert up.find_class("modules", "StyleEncoderGRU") is modules.StyleEncoderGRU
    finally:
        if saved is not None:
            sys.modules["modules"] = saved
        else:
            del sys.modules["modules"]
    for (k, a), (k2, b) in zip(enc.state_dict().items(), got.state_dict().items()):
        assert k == k2 and torch.equal(a, b)


@pytest.mark.parametrize("tag", ["gru_vae_h64_t16", "gru_novae_h64_t16", "gru_vae_h64_t33", "gru_novae_h64_t33", "gru_vae_h512_t256",
                                 "gru_novae_h512_t256", "attn_novae_h64_t16"])
def test_style_encoder_oracle_matches_reference_golden(golden_dir, tag):
    """Forward <= 1e-5 * max(1, |ref|); parameter gradients of the stored cotangent: elementwise 2e-4 of max|ref| where stored,
    norms within 2e-4 relative."""
    g = np.load(os.path.join(golden_dir, "style_gru.npz"))
    typ, vae, Pt = _style_params(g, tag)
    st = synth.load_stats()
    B, T = int(g[tag + ".B"]), int(g[tag + ".T_ex"])
    f = lambda k: torch.as_tensor(st[k], dtype=torch.float32)
    x = (torch.from_numpy(synth.make_style_example(B, T, seed=int(g[tag + ".param_seed"]))) - f("anim_input_mean")) / f("anim_input_std")
    outs = so.style_encoder(Pt, x, eps=torch.from_numpy(g[tag + ".eps"]), temperature=float(g["temperature"]), use_vae=vae, type=typ)
    outs = [o for o in outs if o is not None]
    names = ["z", "mu", "logvar"][:len(outs)]
    for n, o in zip(names, outs):
        ref = g[f"{tag}.{n}"]
        assert np.max(np.abs(o.detach().numpy() - ref)) <= 1e-5 * max(1.0, float(np.abs(ref).max())), n
    keys = sorted(Pt)
    grads = torch.autograd.grad(sum((o * torch.from_numpy(g[f"{tag}.cot_{n}"])).sum() for n, o in zip(names, outs)),
                                [Pt[k] for k in keys])
    for k, gr in zip(keys, grads):
        name = k[len("style_encoder."):]
        ref_n = float(g[f"{tag}.gradnorm.{name}"])
        assert abs(float(gr.double().norm()) - ref_n) <= 2e-4 * max(ref_n, 1e-6), k
        if f"{tag}.grad.{name}" in g.files:
            ref = g[f"{tag}.grad.{name}"]
            assert np.max(np.abs(gr.numpy() - ref)) <= 2e-4 * max(1e-6, float(np.abs(ref).max())), k
    if typ == "gru":        # only output[:, -1] is consumed: the reverse direction's W_hh multiplies h = 0
        assert float(g[f"{tag}.gradnorm.encoder.rnn_layer.weight_hh_l0_reverse"]) == 0.0


@pytest.mark.parametrize("tag", ["gru_h64", "gru_h384"])
def test_train_step_oracle_with_gru_style_encoder_matches_reference_golden(golden_dir, tag):
    g = np.load(os.path.join(golden_dir, f"train_{tag}.npz"))
    H, B, T, T_ex = int(g["H"]), int(g["B"]), int(g["T"]), int(g["T_ex"])
    vae = bool(g["use_vae"])
    P = tt(synth.make_params(H=H, seed=int(g["param_seed"]), style_type=str(g["style_type"]), style_embed=128 if vae else 64))
    for v in P.values():
        v.requires_grad_(True)
    st = synth.load_stats()
    f = lambda k: torch.as_tensor(st[k], dtype=torch.float32)
    seed = int(g["input_seed"])
    win = tt(synth.make_pose_windows(B, T, seed=seed))
    audio = torch.from_numpy(synth.make_audio_features(B, T, seed=seed))
    style_ex = torch.from_numpy(synth.make_style_example(B, T_ex, seed=seed))
    speech = mo.speech_encoder(P, (audio - f("audio_input_mean")) / f("audio_input_std"))
    z, mu, logvar = so.style_encoder(P, (style_ex - f("anim_input_mean")) / f("anim_input_std"), eps=torch.from_numpy(g["eps"]),
                                     use_vae=vae, type="gru")
    assert np.max(np.abs(z.detach().numpy() - g["z"])) <= 5e-6
    O = mo.decoder_forward(P, *[win[n][:, 0] for n in NAMES], win["gaze_pos"], speech, z.unsqueeze(1).repeat(1, T, 1),
                           f("anim_input_mean"), f("anim_input_std"), f("anim_output_mean"), f("anim_output_std"), float(st["dt"]))
    loss, terms = mo.train_losses(O, [win[n] for n in NAMES], win["gaze_pos"], st["parents"], float(st["dt"]), mu, logvar,
                                  int(g["iteration"]))
    assert abs(loss.item() - float(g["loss"])) <= 1e-5 * abs(float(g["loss"]))
    assert ("kl_div" in terms) == vae and (vae or float(g["loss_kl_div"]) == 0.0)
    names = list(P.keys())
    grads = torch.autograd.grad(loss, [P[k] for k in names])
    for k, gr in zip(names, grads):
        ref_n = float(g["gradnorm." + k])
        assert abs(float(gr.double().norm()) - ref_n) <= 2e-4 * max(ref_n, 1e-6), k
        if "grad." + k in g.files:
            assert np.max(np.abs(gr.numpy() - g["grad." + k])) <= 2e-4 * max(1e-6, float(np.max(np.abs(g["grad." + k])))), k
