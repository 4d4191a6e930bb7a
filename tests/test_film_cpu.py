"""CPU: the FiLM-conditioned decoder (rnn_cond "film") -- the oracle against the reference goldens (tests/golden/train_film_*.npz,
written by oracle/make_film_golden.py), the module's state-dict layout and pickles against the reference's, the C ABI mirrors, and
the FiLM kernels' register / spill report."""
import ctypes
import io
import os
import pickle
import re
import subprocess

import numpy as np
import pytest
import torch

from tests._util import NAMES, tt
from oracle import film_oracle as fo
from oracle import ref_shim
from oracle import model_oracle as mo
from zeggs_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run_oracle(g):
    """The whole train-step forward of the golden's case through the oracle, with the FiLM decoder."""
    H, B, T, T_ex = int(g["H"]), int(g["B"]), int(g["T"]), int(g["T_ex"])
    P = tt(synth.make_params(H=H, seed=int(g["param_seed"]), rnn_cond="film"))
    for v in P.values():
        v.requires_grad_(True)
    st = synth.load_stats()
    f = lambda k: torch.as_tensor(st[k], dtype=torch.float32)
    win = tt(synth.make_pose_windows(B, T, seed=int(g["input_seed"])))
    audio = torch.from_numpy(synth.make_audio_features(B, T, seed=int(g["input_seed"])))
    style_ex = torch.from_numpy(synth.make_style_example(B, T_ex, seed=int(g["input_seed"])))
    speech = mo.speech_encoder(P, (audio - f("audio_input_mean")) / f("audio_input_std"))
    z, mu, logvar = mo.style_encoder(P, (style_ex - f("anim_input_mean")) / f("anim_input_std"), eps=torch.from_numpy(g["eps"]))
    O = fo.decoder_forward_film(P, *[win[n][:, 0] for n in NAMES], win["gaze_pos"], speech, z.unsqueeze(1).repeat(1, T, 1),
                                f("anim_input_mean"), f("anim_input_std"), f("anim_output_mean"), f("anim_output_std"), float(st["dt"]))
    loss, terms = mo.train_losses(O, [win[n] for n in NAMES], win["gaze_pos"], st["parents"], float(st["dt"]), mu, logvar,
                                  int(g["iteration"]))
    return P, O, loss, terms


@pytest.mark.parametrize("tag", ["film_h64", "film_h128"])
def test_film_oracle_matches_reference_golden(golden_dir, tag):
    """Forward outputs, loss, the 18 terms and every parameter gradient, to the tolerances the train_h64 oracle check uses."""
    g = np.load(os.path.join(golden_dir, f"train_{tag}.npz"))
    P, O, loss, terms = _run_oracle(g)
    for n, o in zip(NAMES, O):
        ref = g["O_" + n]
        assert np.max(np.abs(o.detach().numpy() - ref)) <= 2e-5 * max(1.0, float(np.max(np.abs(ref)))), n
    assert abs(loss.item() - float(g["loss"])) <= 1e-5 * abs(float(g["loss"]))
    assert len(terms) == 18
    for k, v in terms.items():
        assert abs(float(v) - float(g["loss_" + k])) <= 2e-5 * max(1e-3, abs(float(g["loss_" + k]))), k
    names = list(P.keys())
    grads = torch.autograd.grad(loss, [P[k] for k in names], allow_unused=True)
    assert any(k.startswith("decoder.recurrent_decoder.gammas_predictor") for k in names)
    for k, gr in zip(names, grads):
        ref_n = float(g["gradnorm." + k])
        assert gr is not None, k
        assert abs(float(gr.double().norm()) - ref_n) <= 2e-4 * max(ref_n, 1e-6), k
        if "grad." + k in g.files:
            assert np.max(np.abs(gr.numpy() - g["grad." + k])) <= 2e-4 * max(1e-6, float(np.max(np.abs(g["grad." + k])))), k


def _reference_film_shapes(H, S, Z):
    """State-dict keys and shapes of the reference's Decoder(rnn_cond="film") (modules.py:11-45, 188-212, 230-236), written out."""
    A = 1134 + S
    d, c = "recurrent_decoder.", "cell_state_encoder."
    shapes = {d + "gammas_predictor.linear_layer.weight": (2 * H, Z), d + "gammas_predictor.linear_layer.bias": (2 * H,),
              d + "betas_predictor.linear_layer.weight": (2 * H, Z), d + "betas_predictor.linear_layer.bias": (2 * H,),
              d + "layer0.weight": (H, A), d + "layer0.bias": (H,),
              d + "layer2.weight": (H, H), d + "layer2.bias": (H,), d + "layer3.weight": (1131, H), d + "layer3.bias": (1131,),
              c + "layer0.weight": (H, 1134 + Z), c + "layer0.bias": (H,), c + "layer1.weight": (H, H), c + "layer1.bias": (H,),
              c + "layer2.weight": (2 * H, H), c + "layer2.bias": (2 * H,)}
    for l, K in ((0, A + H), (1, H)):
        shapes.update({d + f"layer1.weight_ih_l{l}": (3 * H, K), d + f"layer1.weight_hh_l{l}": (3 * H, H),
                       d + f"layer1.bias_ih_l{l}": (3 * H,), d + f"layer1.bias_hh_l{l}": (3 * H,)})
    return shapes


@pytest.mark.parametrize("H,S,Z", [(64, 64, 64), (1024, 64, 64), (96, 32, 16)])
def test_film_decoder_state_dict_matches_reference(H, S, Z):
    from zeggs_b200 import modules
    dec = modules.Decoder(1134, 1131, S, Z, H, 2, rnn_cond="film")
    got = {k: tuple(v.shape) for k, v in dec.state_dict().items()}
    assert got == _reference_film_shapes(H, S, Z)
    assert dec.film and (dec.hidden_size, dec.speech_encoding_size, dec.style_encoding_size) == (H, S, Z)
    assert len(dec._weights()) == len(list(dec.parameters())) == 24
    assert {id(p) for p in dec._weights()} == {id(p) for p in dec.parameters()}
    P = synth.make_params(H=H, S=S, Z=Z, seed=3, rnn_cond="film", with_style=False)
    assert {k[len("decoder."):]: v.shape for k, v in P.items() if k.startswith("decoder.")} == got


def test_unknown_rnn_cond_raises():
    from zeggs_b200 import _lib, modules
    with pytest.raises(_lib.ZeggsError, match="rnn_cond"):
        modules.Decoder(1134, 1131, 64, 64, 64, 2, rnn_cond="films")


@pytest.mark.skipif(not os.path.isdir(ref_shim.REF_ZEGGS), reason="needs the reference tree")
def test_reference_pickled_film_decoder_unpickles_into_our_class():
    """A whole-module pickle of the reference's FiLM decoder (what generate.py:130-138 loads) becomes our Decoder with the FiLM
    container: same tensors, rnn_cond recognised from the class."""
    from zeggs_b200 import modules
    ref = ref_shim.ref_modules()
    torch.manual_seed(0)
    rdec = ref.Decoder(1134, 1131, 64, 64, 64, 2, rnn_cond="film")
    buf = io.BytesIO()
    torch.save(rdec, buf)

    class _Into(pickle.Unpickler):
        def find_class(self, module, name):
            return getattr(modules, name) if module == "modules" else super().find_class(module, name)

    buf.seek(0)
    dec = torch.load(buf, weights_only=False, pickle_module=type("pm", (), {"Unpickler": _Into, "load": pickle.load}))
    assert type(dec) is modules.Decoder and isinstance(dec.recurrent_decoder, modules.RecurrentDecoderFiLM)
    assert dec.film and dec.hidden_size == 64 and dec.speech_encoding_size == 64 and dec.style_encoding_size == 64
    ref_sd = rdec.state_dict()
    for k, v in dec.state_dict().items():
        assert torch.equal(v, ref_sd[k]), k


def test_film_struct_mirrors_match_library():
    from zeggs_b200 import _lib
    l = _lib.lib()
    for name in ("zeggs_decoder_film_fwd_args", "zeggs_decoder_film_bwd_args"):
        mirror = _lib.struct_mirrors()[name]
        assert l.zeggs_struct_size(name.encode()) == ctypes.sizeof(mirror) > 0, name
    assert _lib.DecoderFilmFwdArgs.dec.offset == 0 and _lib.DecoderFilmBwdArgs.dec.offset == 0
    assert l.zeggs_decoder_packed_film_bytes(64, 64, 64) > l.zeggs_decoder_packed_bytes(64, 64, 64) > 0
    assert l.zeggs_decoder_film_workspace_bytes(3, 17, 64, 64, 64, 1) > l.zeggs_decoder_workspace_bytes(3, 17, 64, 64, 64, 1)
    assert l.zeggs_decoder_packed_film_bytes(1064, 64, 64) == 0


def test_film_kernels_compile_for_sm90a_without_spills(tmp_path):
    """-Xptxas -v of the two sources that hold the FiLM recurrences: every kernel, FiLM variants included, with no spill."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("needs nvcc")
    csrc = os.path.join(ROOT, "ubisoft-laforge-zeroeggs_b200", "csrc")
    seen = set()
    for src in ("decoder_fwd.cu", "decoder_bwd.cu"):
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                            "-Xptxas", "-v", "-c", os.path.join(csrc, src), "-o", str(tmp_path / (src + ".o"))],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        fn = None
        for line in r.stderr.splitlines():
            m = re.search(r"Compiling entry function '(\S+)'", line)
            if m:
                fn = m.group(1)
                seen.add(fn)
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m:
                assert m.group(1) == "0" and m.group(2) == "0", (fn, line)
    for k in ("decoder_fwd_kernelILi4ELb1E", "decoder_fwd_kernelILi8ELb1E", "decoder_bwd_kernelILi4ELb1E", "decoder_bwd_kernelILi8ELb1E",
              "pack_film_kernel", "pack_film_bwd_kernel", "colsum_ld_kernel", "film_style0_kernel"):
        assert any(k in s for s in seen), k
