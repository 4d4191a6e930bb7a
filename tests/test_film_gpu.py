"""GPU: the FiLM-conditioned decoder (rnn_cond "film") on the fp32 engine -- window forward and every gradient against the oracle
(oracle/film_oracle.py, evaluated in float64 on the CPU), the one-call backward against the two-phase form, TrainStep against
the reference goldens (tests/golden/train_film_*.npz) and its graph replay / concurrent lanes against eager / one stream, and the
tensor-core engine's refusal.

Tolerances: the fp32 engine's bounds of oracle/fp32_oracle.py -- forward FP32_FWD_TOL x max(1, max|ref|) per pose-channel group,
gradients max-abs FP32_GEMM_GRAD_TOL x max|ref| (GEMM mode 1); train step as the fp32-engine rows of the train_h64 / train_h128 golden
test (gemm mode 0)."""
import os

import numpy as np
import pytest
import torch

from oracle.fp32_oracle import FP32_FWD_TOL, FP32_GEMM_GRAD_TOL
from tests._util import NAMES, ensure_built, stats_tensors, tt
from tests.test_gpu_parity import _batch, _load

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


@pytest.fixture
def engine(dev):
    from zeggs_b200 import ops
    prev, prev_mode = ops.DECODER_ENGINE, ops.GEMM_MODE
    yield ops
    ops.set_decoder_engine(prev)
    ops.set_gemm_mode(prev_mode)


def _film_decoder(P, H, dev):
    from zeggs_b200 import modules
    return _load(modules.Decoder(1134, 1131, 64, 64, H, 2, rnn_cond="film"), P, "decoder.", dev)


def _window_inputs(B, T, seed, dev):
    from zeggs_b200 import synth
    W = tt(synth.make_pose_windows(B, T, seed=seed), dev)
    rs = np.random.RandomState(seed + 1)
    speech = torch.from_numpy(rs.randn(B, T, 64).astype(np.float32)).to(dev)
    # a style that changes every frame: the predictors' rows must be those of frame t, not of another frame
    style = torch.from_numpy(rs.randn(B, T, 64).astype(np.float32)).to(dev)
    return W, speech, style


def _oracle(P, W, speech, style, st, dev):
    from oracle import film_oracle as fo
    d = lambda t: t.detach().to("cpu", torch.float64)
    Pd = {k: d(torch.from_numpy(v)) for k, v in P.items() if k.startswith("decoder.")}
    return Pd, lambda Pd_, sp, sy: fo.decoder_forward_film(
        Pd_, *[d(W[n][:, 0]) for n in NAMES], d(W["gaze_pos"]), sp, sy, d(st["anim_input_mean"]), d(st["anim_input_std"]),
        d(st["anim_output_mean"]), d(st["anim_output_std"]), st["dt"])


def _ours(dec, W, speech, style, st, dev):
    f = lambda k: st[k].to(dev)
    return dec(*[W[n][:, 0] for n in NAMES], W["gaze_pos"], speech, style, st["parents"], f("anim_input_mean"), f("anim_input_std"),
               f("anim_output_mean"), f("anim_output_std"), st["dt"])


@pytest.mark.parametrize("H", [64, 128, 1024])
@pytest.mark.parametrize("B,T", [(1, 1), (1, 2), (7, 9), (32, 256), (33, 9)])
def test_film_window_forward_vs_oracle(dev, engine, H, B, T):
    from zeggs_b200 import synth
    engine.set_decoder_engine("auto")          # "auto" runs a FiLM decoder on the fp32 engine
    P = synth.make_params(H=H, seed=21, rnn_cond="film", with_style=False)
    dec = _film_decoder(P, H, dev).eval()
    st = stats_tensors()
    W, speech, style = _window_inputs(B, T, 4, dev)
    with torch.no_grad():
        got = _ours(dec, W, speech, style, st, dev)
        Pd, run = _oracle(P, W, speech, style, st, dev)
        ref = run(Pd, speech.cpu().double(), style.cpu().double())
    worst = 0.0
    for n, o, r in zip(NAMES, got, ref):
        err = float((o.cpu().double() - r).abs().max()) / max(1.0, float(r.abs().max()))
        worst = max(worst, err)
        assert err <= FP32_FWD_TOL, (n, err)
    print(f"  H={H} B={B} T={T}: worst per-group error {worst:.3e} ({worst / FP32_FWD_TOL:.3f} of the bound)")


@pytest.mark.parametrize("H", [64, 128, 1024])
@pytest.mark.parametrize("B,T", [(5, 8), (33, 6)])
def test_film_gradients_vs_oracle_autograd(dev, engine, H, B, T):
    """Every parameter gradient, dSpeech and dStyle of a random linear functional of the window's outputs, with a per-frame style;
    B = 33 runs the BPTT over two batch tiles, the second with one real sample."""
    from zeggs_b200 import synth
    engine.set_decoder_engine("fp32")
    P = synth.make_params(H=H, seed=22, rnn_cond="film", with_style=False)
    dec = _film_decoder(P, H, dev).train()
    st = stats_tensors()
    W, speech, style = _window_inputs(B, T, 6, dev)
    speech.requires_grad_(True)
    style.requires_grad_(True)
    got = _ours(dec, W, speech, style, st, dev)
    g = torch.Generator(device="cpu").manual_seed(5)
    R = [torch.randn(o.shape, generator=g).to(dev) for o in got]
    loss = sum((o * r).sum() for o, r in zip(got, R))
    names = [k for k, _ in dec.named_parameters()]
    grads = torch.autograd.grad(loss, list(dec.parameters()) + [speech, style])
    Pd, run = _oracle(P, W, speech, style, st, dev)
    for v in Pd.values():
        v.requires_grad_(True)
    sp, sy = speech.detach().cpu().double().requires_grad_(True), style.detach().cpu().double().requires_grad_(True)
    ref_out = run(Pd, sp, sy)
    ref_loss = sum((o * r.cpu().double()).sum() for o, r in zip(ref_out, R))
    keys = ["decoder." + k for k in names]
    ref = torch.autograd.grad(ref_loss, [Pd[k] for k in keys] + [sp, sy])
    bad, worst = [], 0.0
    for n, a, b in zip(names + ["dSpeech", "dStyle"], grads, ref):
        e = float((a.cpu().double() - b).abs().max()) / max(float(b.abs().max()), 1e-30)
        worst = max(worst, e)
        if not e <= FP32_GEMM_GRAD_TOL:
            bad.append((n, e))
    print(f"  H={H} B={B} T={T}: worst gradient max-abs / max|ref| {worst:.3e} ({worst / FP32_GEMM_GRAD_TOL:.3f} of the bound)")
    assert not bad, bad


def test_film_two_phase_backward_matches_one_call(dev, engine):
    from zeggs_b200 import ops, synth
    engine.set_decoder_engine("fp32")
    H, B, T = 128, 6, 10
    P = synth.make_params(H=H, seed=23, rnn_cond="film", with_style=False)
    dec = _film_decoder(P, H, dev)
    st = stats_tensors(dev)
    W, speech, style = _window_inputs(B, T, 8, dev)
    stats = (st["anim_input_mean"], st["anim_input_std"], st["anim_output_mean"], st["anim_output_std"])
    from zeggs_b200.train import pack_pose
    pose0 = pack_pose(*[W[n] for n in NAMES[2:]])[:, 0]
    Y, rp, rq, state = ops.decoder_window_forward(dec, W["root_pos"][:, 0], W["root_rot"][:, 0], pose0, W["gaze_pos"], speech, style,
                                                  stats, st["dt"], save=True)
    g = torch.Generator(device="cpu").manual_seed(9)
    dY, dRp, dRq = (torch.randn(t.shape, generator=g).to(dev) for t in (Y, rp, rq))
    one = ops.decoder_window_backward(dec, state, dY, dRp, dRq)
    one = [t.clone() for t in one[0]] + [one[1].clone(), one[2].clone()]
    grads, dS, dZ, finish = ops.decoder_window_backward(dec, state, dY, dRp, dRq, split=True)
    finish()
    torch.cuda.synchronize()
    for a, b in zip(one, list(grads) + [dS, dZ]):
        assert torch.equal(a, b)


def test_film_rejects_tensor_core_engine(dev, engine):
    from zeggs_b200 import _lib, synth
    engine.set_decoder_engine("tc")
    P = synth.make_params(H=384, seed=24, rnn_cond="film", with_style=False)
    dec = _film_decoder(P, 384, dev)
    st = stats_tensors()
    W, speech, style = _window_inputs(2, 4, 10, dev)
    with pytest.raises(_lib.ZeggsError, match="FiLM"):
        with torch.no_grad():
            _ours(dec, W, speech, style, st, dev)


def test_film_unsupported_hidden_size_raises(dev, engine):
    from zeggs_b200 import _lib, synth
    engine.set_decoder_engine("fp32")
    P = synth.make_params(H=1064, seed=25, rnn_cond="film", with_style=False)
    dec = _film_decoder(P, 1064, dev)
    st = stats_tensors()
    W, speech, style = _window_inputs(1, 3, 11, dev)
    with pytest.raises(_lib.ZeggsError, match="hidden size 1064"):
        with torch.no_grad():
            _ours(dec, W, speech, style, st, dev)


def test_film_generate_gesture_stitch_vs_oracle(dev, engine, tmp_path):
    """generate_gesture() from whole-module pickles with a FiLM decoder, two example styles stitched (the style changes halfway through
    the 240 generated frames), against the oracle's FiLM window (float64) on the same speech encoding, style rows and first pose, put
    through the same pose -> BVH channel step and BVH writer: BVH positions <= 1e-3 (cm), Euler angles <= 5e-3 degrees, as the normal
    decoder's end-to-end row."""
    import json
    import shutil
    from pathlib import Path
    from oracle import film_oracle as fo
    from tests import _fixtures as fx
    from zeggs_b200 import animation, audio, bvhio, generate, modules, ops, synth
    engine.set_decoder_engine("auto")
    H = 128
    P = synth.make_params(H=H, seed=26, rnn_cond="film")
    net = tmp_path / "net"; net.mkdir()
    se = _load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", "cpu")
    torch.save(se, net / "speech_encoder.pt")
    torch.save(_load(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), P, "style_encoder.", "cpu"), net / "style_encoder.pt")
    torch.save(_film_decoder(P, H, "cpu"), net / "decoder.pt")
    data = tmp_path / "data"; data.mkdir()
    stats = synth.load_stats()
    np.savez(data / "stats.npz", **{k: stats[k] for k in ("audio_input_mean", "audio_input_std", "anim_input_mean", "anim_input_std",
                                                         "anim_output_mean", "anim_output_std")})
    shutil.copy(os.path.join(fx.DATA, "data_definition_v1.json"), data / "data_definition.json")
    conf = json.load(open(os.path.join(fx.DATA, "data_pipeline_conf_v1.json")))
    conf["audio_conf"]["normalize_loudness"] = False
    json.dump(conf, open(data / "data_pipeline_conf.json", "w"))
    bvh_path = Path(fx.make_synthetic_bvh(str(tmp_path / "style.bvh")))
    wav_path = Path(fx.make_wav(str(tmp_path / "speech.wav")))
    res = tmp_path / "res"
    final = generate.generate_gesture(wav_path, [(bvh_path, (10, 300)), (bvh_path, None)], net, data, res, style_encoding_type="example",
                                      blend_type="stitch", blend_ratio=[0.5, 0.5], file_name="out", temperature=1e6, seed=1234)
    T = final.shape[1]
    assert T == 240 and not torch.equal(final[0, 0], final[0, -1]), "the stitched style must change over the window"
    b = animation.load_bvh(str(res / "out.bvh"))
    # the oracle's inputs: the speech encoding generate_gesture computed, its style rows, the first pose of the last style example
    from scipy.io import wavfile
    fs, pcm = wavfile.read(str(wav_path))
    wav = torch.from_numpy(generate._decode_16k(wav_path, fs, pcm))
    feats = audio.preprocess_audio(wav, 60, T, conf["audio_conf"], conf.get("audio_feature_type", ["mel_spec", "energy"]), device=dev)
    f = lambda k: torch.as_tensor(stats[k], dtype=torch.float32, device=dev)
    se = se.to(dev).eval()
    with torch.no_grad():
        speech = se((feats[None] - f("audio_input_mean")) / f("audio_input_std"))
    a = animation.preprocess_animation(animation.trim(animation.load_bvh(str(bvh_path)), None))
    d = lambda x: torch.as_tensor(np.asarray(x)).to("cpu", torch.float64)
    Pd = {k: d(v) for k, v in P.items() if k.startswith("decoder.")}
    fp = [d(a[k][0])[None] for k in NAMES]
    with torch.no_grad():
        O = fo.decoder_forward_film(Pd, *fp, d(a["gaze_pos"][0]).reshape(1, 1, 3).repeat(1, T, 1), d(speech.cpu()), d(final.cpu()),
                                    d(stats["anim_input_mean"]), d(stats["anim_input_std"]), d(stats["anim_output_mean"]),
                                    d(stats["anim_output_std"]), float(stats["dt"]))
    V = {k: o.float().to(dev) for k, o in zip(NAMES, O)}
    pos, eul = ops.pose_to_bvh_channels(V["root_pos"], V["root_rot"], V["lpos"], V["ltxy"], (0.0, 0.0, 0.0), (1.0, 0.0, 0.0, 0.0))
    details = json.load(open(data / "data_definition.json"))
    bvhio.save_bvh(str(tmp_path / "oracle.bvh"), pos[0].cpu().numpy(), eul[0].cpu().numpy(), details["parents"], details["bone_names"],
                   "zyx", details["dt"])                 # what generate_gesture writes: root trajectory, frame-0 offsets, rotations
    r = animation.load_bvh(str(tmp_path / "oracle.bvh"))
    e_pos = float(np.abs(b["positions"].astype(np.float64) - r["positions"]).max())
    e_eul = float(np.abs(b["rotations"].astype(np.float64) - r["rotations"]).max())
    print(f"  stitch: BVH positions max-abs {e_pos:.3e} cm, Euler {e_eul:.3e} deg")
    assert e_pos <= 1e-3 and e_eul <= 5e-3


def _film_step(dev, H, seed, **kw):
    from zeggs_b200 import modules, synth
    from zeggs_b200.train import TrainStep
    P = synth.make_params(H=H, seed=seed, rnn_cond="film")
    se = _load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", dev)
    st = _load(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), P, "style_encoder.", dev)
    de = _film_decoder(P, H, dev)
    stats = synth.load_stats()
    return TrainStep(se, de, st, stats, stats["parents"], float(stats["dt"]), **kw)


@pytest.mark.parametrize("tag", ["film_h64", "film_h128"])
def test_film_train_step_vs_reference_golden(dev, golden_dir, engine, tag):
    """Whole step (encoders -> FiLM decoder -> loss -> backward, eval-mode dropout, injected VAE eps) against the reference's loss, 18
    terms and gradients: loss 2e-5, terms 3e-5, gradient norms 5e-4 relative, stored gradients max-abs 5e-4 of max|ref| (gemm mode 0)."""
    engine.set_decoder_engine("fp32")
    engine.set_gemm_mode(0)
    g = np.load(os.path.join(golden_dir, f"train_{tag}.npz"))
    H, B, T, T_ex = int(g["H"]), int(g["B"]), int(g["T"]), int(g["T_ex"])
    step = _film_step(dev, H, int(g["param_seed"]))
    step.iteration = int(g["iteration"])
    step.optimizer.zero_grad()
    loss = step.forward_backward(_batch(dev, B, T, T_ex, int(g["input_seed"])), eps=torch.from_numpy(g["eps"]).to(dev), train_mode=False)
    torch.cuda.synchronize()
    print(f"  loss {loss.item():.6f} vs golden {float(g['loss']):.6f}")
    assert abs(loss.item() - float(g["loss"])) <= 2e-5 * abs(float(g["loss"]))
    terms = step.terms.cpu().numpy()
    names = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "lrot", "lvel", "lvrt", "cpos", "crot", "cvel", "cvrt",
             "ldvl", "ldvt", "cdvl", "cdvt", "gaze", "kl_div"]
    for i, n in enumerate(names):
        ref = float(g["loss_" + n])
        assert abs(terms[1 + i] - ref) <= 3e-5 * max(1e-3, abs(ref)), (n, terms[1 + i], ref)
    bad = []
    for prefix, net in (("speech_encoder.", step.se), ("decoder.", step.dec), ("style_encoder.", step.st)):
        for k, p in net.named_parameters():
            ref_n = float(g["gradnorm." + prefix + k])
            got_n = float(p.grad.double().norm())
            if not abs(got_n - ref_n) <= 5e-4 * max(ref_n, 1e-7):
                bad.append((prefix + k, got_n, ref_n))
            if "grad." + prefix + k in g.files:
                ref = g["grad." + prefix + k]
                if not float(np.abs(p.grad.cpu().numpy() - ref).max()) <= 5e-4 * max(float(np.abs(ref).max()), 1e-7):
                    bad.append((prefix + k, "elementwise"))
    assert not bad, bad


def test_film_graph_replay_and_lanes_match_eager_single_stream(dev, engine, monkeypatch):
    """TrainStep with a FiLM decoder: graph-captured steps with concurrent lanes, eager steps with lanes, and graph steps on one
    stream give identical losses and parameters after 4 steps (the flat gradient includes the FiLM predictors)."""
    engine.set_decoder_engine("auto")
    res = {}
    for mode, lanes in (("graph", "1"), ("eager", "1"), ("graph", "0")):
        monkeypatch.setenv("ZEGGS_LANES", lanes)
        torch.manual_seed(321)
        step = _film_step(dev, 128, 79, lr=1e-3, use_graph=True)
        if mode == "eager":
            step.graph_min_seen = 10 ** 9
        losses = [float(step.step(_batch(dev, 4, 16, 24, 90 + it)).item()) for it in range(4)]
        torch.cuda.synchronize()
        if mode == "graph":
            assert len(step._graphs) == 1
        pg = step.dec.recurrent_decoder.gammas_predictor.linear_layer.weight
        res[(mode, lanes)] = (losses, step.optimizer.flat_param.clone(), pg.detach().clone())
        del step
    for k, v in res.items():
        print(f"  {k}: losses {v[0]}")
    ref = res[("graph", "1")]
    assert not torch.equal(ref[2], torch.from_numpy(
        __import__("zeggs_b200.synth", fromlist=["x"]).make_params(H=128, seed=79, rnn_cond="film")
        ["decoder.recurrent_decoder.gammas_predictor.linear_layer.weight"]).to(dev)), "the predictors were not trained"
    assert np.allclose(res[("eager", "1")][0], ref[0], rtol=1e-6, atol=0)          # as the normal decoder's graph-vs-eager row
    assert float((res[("eager", "1")][1] - ref[1]).abs().max()) <= 1e-7
    assert res[("graph", "0")][0] == ref[0]                                          # lanes only reorder independent work
    assert float((res[("graph", "0")][1] - ref[1]).abs().max()) == 0.0
