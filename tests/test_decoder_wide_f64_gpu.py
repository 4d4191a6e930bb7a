"""Decoders wider than 1056 hidden units on the fp32 engine (16 units per CTA, two 8-unit passes per stage, H % 16 == 0 up to 2112)
against the float64 oracle (model_oracle / film_oracle through autograd), at the bounds of oracle/fp32_oracle.py as
tests/test_decoder_fp32_f64_gpu.py applies them (tests/test_decoder_wide_cpu.py shows float32 arithmetic meets them with 4x headroom
at H = 2112 and that faults in one 16-unit CTA break them).

Covered: the forward at every new hidden size; forward and full BPTT (every parameter gradient, dSpeech, dStyle) at H in
{1072, 1536, 2048, 2112} x B in {1, 32, 33} in GEMM modes 0 and 1, and the mode-1 fallback to the SIMT weight-gradient kernels when the
split-bf16 histories do not fit the scratch buffer; the FiLM decoder at 1072 and 2112; the largest batch one call takes at H = 2112 and
the error one sample more gets; TrainStep at H = 1536 (graph replay against eager launches, concurrent lanes against one stream); and
train() with a 1536-wide decoder whose checkpoints generate_gesture() loads, its BVH against the float64 oracle window."""
import json
import os
import random
import shutil
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import model_oracle as mo
from tests._util import NAMES
from tests.test_decoder_fp32_f64_gpu import (_bwd_smem, _case, _check, _hist_bytes, _max_batch, _reference, _run_gpu, dev, ops,  # noqa: F401
                                             private_lane)
from tests.test_gpu_parity import _batch, _load

pytestmark = pytest.mark.gpu

WIDE_H = list(range(1072, 2112 + 1, 16))


@pytest.mark.parametrize("H", WIDE_H)
def test_forward_every_wide_hidden_size(dev, ops, H):
    case = _case(H, 3, 5, 64, seed=9000 + H)
    got, _ = _run_gpu(dev, *case, grads=False)
    ref, _ = _reference(*case, grads=False)
    _check(f"fwd H{H} B3 T5", got, ref)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("B", [1, 32, 33])
@pytest.mark.parametrize("H", [1072, 1536, 2048, 2112])
def test_forward_backward_wide(dev, ops, H, B, mode):
    """H = 1072: 67 CTAs, two 16-row tiles of layer-2 / x_pose-gradient rows per CTA; 2112: 132 CTAs, one tile.  B = 33: two batch
    tiles, the second with one real sample.  GEMM mode 1 runs the split-bf16 weight-gradient GEMMs, mode 0 the SIMT kernels."""
    ops.set_gemm_mode(mode)
    case = _case(H, B, 9, 64, seed=9100 + H + B)
    got, g = _run_gpu(dev, *case)
    ref, g_ref = _reference(*case)
    _check(f"H{H} B{B} T9 gemm mode {mode}", got, ref, g, g_ref, gemm_mode=mode)


@pytest.mark.parametrize("H", [1536, 2112])
def test_simt_weight_gradient_fallback(dev, ops, private_lane, H):
    """GEMM mode 1 on a lane whose scratch buffer is one 256-byte block short of the split-bf16 histories: the weight gradients fall
    back to the SIMT k-major kernels, as they do whenever the histories, which grow with H, exceed the lane's scratch buffer."""
    ops.set_gemm_mode(1)
    B, T = 32, 9
    need = _hist_bytes(H, B, T, 64, 64)
    buf = torch.empty(need, dtype=torch.uint8, device=dev)
    case = _case(H, B, T, 64, seed=9200 + H)
    with private_lane(buf, need - 256):
        got, g = _run_gpu(dev, *case)
    ref, g_ref = _reference(*case)
    _check(f"SIMT fallback H{H} B{B} T{T}", got, ref, g, g_ref, gemm_mode=1)


@pytest.mark.parametrize("H", [1072, 2112])
@pytest.mark.parametrize("B,T", [(1, 9), (33, 9)])
def test_film_wide(dev, ops, H, B, T):
    case = _case(H, B, T, 64, seed=9300 + H + B, film=True)
    got, g = _run_gpu(dev, *case, film=True)
    ref, g_ref = _reference(*case, film=True)
    _check(f"film H{H} B{B} T{T}", got, ref, g, g_ref)


def _fwd_smem_u16(nbt):
    """fwd_smem_bytes<16> (csrc/decoder_fwd.cu): the stage buffers and reduction tile of one 8-unit pass, gi0p for all 16 units of each batch tile."""
    stg = 16 * 48 + 1024
    return (8 * 2 * stg + 8 * 48 * 32 + nbt * 3 * 16 * 32 + 6 * 32) * 4


def test_largest_batch_at_2112_and_one_more(dev, ops):
    """At H = 2112 the forward's shared memory bounds one call (352 samples on the H100; the BPTT's own bound is higher, so the forward
    is the limit of a training call too): the largest batch runs forward and backward and matches the oracle; one sample more is
    refused with a ZeggsError naming the limit, with and without the backward.  It must take the 32-sample training batch."""
    from zeggs_b200 import _lib
    H = 2112
    cap = torch.cuda.get_device_properties(dev).shared_memory_per_block_optin
    b_fwd = _max_batch(_fwd_smem_u16, cap)
    b_bwd = _max_batch(lambda n: _bwd_smem(H, 16, n), cap)
    print(f"  H{H} U16: largest batch forward {b_fwd}, backward {b_bwd} ({cap} bytes of shared memory per block)")
    assert 32 <= b_fwd <= b_bwd
    case = _case(H, b_fwd, 2, 64, seed=9400)
    got, g = _run_gpu(dev, *case)
    ref, g_ref = _reference(*case)
    _check(f"largest batch H{H} B{b_fwd} T2", got, ref, g, g_ref)
    for grads in (False, True):
        with pytest.raises(_lib.ZeggsError, match=f"at most {b_fwd} samples"):
            _run_gpu(dev, *_case(H, b_fwd + 1, 2, 64, seed=9401), grads=grads)


# ---------------------------------------------------------------------------------------------------------- end to end
def _step(dev, H, seed, **kw):
    from zeggs_b200 import modules, synth
    from zeggs_b200.train import TrainStep
    P = synth.make_params(H=H, seed=seed)
    se = _load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", dev)
    st = _load(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), P, "style_encoder.", dev)
    de = _load(modules.Decoder(1134, 1131, 64, 64, H, 2), P, "decoder.", dev)
    stats = synth.load_stats()
    return TrainStep(se, de, st, stats, stats["parents"], float(stats["dt"]), **kw)


def test_train_step_graph_and_lanes_at_1536(dev, ops, monkeypatch):
    """TrainStep with a 1536-wide decoder ("auto" runs it on the fp32 engine), B = 32: graph-captured steps with concurrent lanes, eager
    steps with lanes, and graph steps on one stream give the same losses and parameters after 3 steps (as the FiLM decoder's row)."""
    ops.set_decoder_engine("auto")
    res = {}
    for mode, lanes in (("graph", "1"), ("eager", "1"), ("graph", "0")):
        monkeypatch.setenv("ZEGGS_LANES", lanes)
        torch.manual_seed(322)
        step = _step(dev, 1536, 81, lr=1e-3, use_graph=True)
        if mode == "eager":
            step.graph_min_seen = 10 ** 9
        losses = [float(step.step(_batch(dev, 32, 16, 24, 190 + it)).item()) for it in range(3)]
        torch.cuda.synchronize()
        if mode == "graph":
            assert len(step._graphs) == 1
        res[(mode, lanes)] = (losses, step.optimizer.flat_param.clone())
        del step
    for k, v in res.items():
        print(f"  {k}: losses {v[0]}")
    ref = res[("graph", "1")]
    assert all(np.isfinite(ref[0]))
    assert np.allclose(res[("eager", "1")][0], ref[0], rtol=1e-6, atol=0)
    assert float((res[("eager", "1")][1] - ref[1]).abs().max()) <= 1e-7
    assert res[("graph", "0")][0] == ref[0]
    assert float((res[("graph", "0")][1] - ref[1]).abs().max()) == 0.0


def test_train_then_generate_gesture_at_1536(dev, ops, tmp_path):
    """train() for 3 iterations on a synthetic processed set with net_opt.decoder.nhidden = 1536 writes checkpoints; generate_gesture()
    loads them and its BVH matches the float64 oracle window of the trained decoder on the same speech encoding, style rows and first
    pose, through the same pose -> BVH channel step: positions <= 1e-3 cm, Euler angles <= 5e-3 degrees (the FiLM generate row)."""
    from tests import _fixtures as fx
    from zeggs_b200 import animation, audio, bvhio, generate, synth
    from zeggs_b200.train import train
    H = 1536
    ddef, dproc = fx.make_dataset_files(str(tmp_path))
    to = dict(seed=21, use_gpu=True, resume=False, learning_rate=1e-3, learning_rate_decay=0.999, eps=1e-5, niterations=3 / 1000.0,
              batchsize=32, window=64, style_encoding_type="example", generate_samples_step=1000, use_tensorboard=False,
              decoder_engine="auto", cuda_graph=True, device_dataset=True)
    no = dict(speech_encoder=dict(nhidden=64, speech_encoding_size=64),
              style_encoder=dict(nhidden=512, style_encoding_size=64, example_length=64, type="attn", use_vae=True),
              decoder=dict(nhidden=H))
    state = random.getstate()
    random.seed(0)
    try:
        train(str(tmp_path / "models"), str(tmp_path / "logs"), dproc, ddef, to, no)
    finally:
        random.setstate(state)
    net = tmp_path / "models"
    dec = torch.load(net / "decoder.pt", map_location="cpu", weights_only=False)
    assert dec.recurrent_decoder.layer0.weight.shape[0] == H
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
    b = animation.load_bvh(str(res / "out.bvh"))
    from scipy.io import wavfile
    fs, pcm = wavfile.read(str(wav_path))
    wav = torch.from_numpy(generate._decode_16k(wav_path, fs, pcm))
    feats = audio.preprocess_audio(wav, 60, T, conf["audio_conf"], conf.get("audio_feature_type", ["mel_spec", "energy"]), device=dev)
    f = lambda k: torch.as_tensor(stats[k], dtype=torch.float32, device=dev)
    se = torch.load(net / "speech_encoder.pt", map_location="cpu", weights_only=False).to(dev).eval()
    with torch.no_grad():
        speech = se((feats[None] - f("audio_input_mean")) / f("audio_input_std"))
    a = animation.preprocess_animation(animation.trim(animation.load_bvh(str(bvh_path)), None))
    d = lambda x: torch.as_tensor(np.asarray(x)).to("cpu", torch.float64)
    Pd = {"decoder." + k: d(v) for k, v in dec.state_dict().items()}
    fp = [d(a[k][0])[None] for k in NAMES]
    with torch.no_grad():
        O = mo.decoder_forward(Pd, *fp, d(a["gaze_pos"][0]).reshape(1, 1, 3).repeat(1, T, 1), d(speech.cpu()), d(final.cpu()),
                               d(stats["anim_input_mean"]), d(stats["anim_input_std"]), d(stats["anim_output_mean"]),
                               d(stats["anim_output_std"]), float(stats["dt"]))
    V = {k: o.float().to(dev) for k, o in zip(NAMES, O)}
    pos, eul = ops.pose_to_bvh_channels(V["root_pos"], V["root_rot"], V["lpos"], V["ltxy"], (0.0, 0.0, 0.0), (1.0, 0.0, 0.0, 0.0))
    details = json.load(open(data / "data_definition.json"))
    bvhio.save_bvh(str(tmp_path / "oracle.bvh"), pos[0].cpu().numpy(), eul[0].cpu().numpy(), details["parents"], details["bone_names"],
                   "zyx", details["dt"])
    r = animation.load_bvh(str(tmp_path / "oracle.bvh"))
    e_pos = float(np.abs(b["positions"].astype(np.float64) - r["positions"]).max())
    e_eul = float(np.abs(b["rotations"].astype(np.float64) - r["rotations"]).max())
    print(f"  H{H} train -> generate: BVH positions max-abs {e_pos:.3e} cm, Euler {e_eul:.3e} deg")
    assert e_pos <= 1e-3 and e_eul <= 5e-3
