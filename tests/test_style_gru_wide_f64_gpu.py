"""GPU: GRU style encoders wider than 1056 hidden units (16 units per CTA, W_hh read from L2 per K chunk; H % 16 == 0 up to 2112)
against the float64 oracle, at the bounds of tests/test_style_gru_f64_gpu.py (tests/test_style_gru_wide_cpu.py shows float32 meets them
with >= 4x headroom at H = 2112 and that faults of the wide path break them).  Cases and oracles: tests/_gru_cases.py; the float64
oracle runs on the device here, so the 2112-wide cases take seconds.

Outputs are held to 2e-5 x max(1, |ref|) in GEMM mode 0, where every product around the recurrence is fp32 SIMT and the kernels' own
error shows (2e-6 .. 3e-6 at these widths on the H100).  In mode 1 the convolutions, input projections and projection run as split-bf16
tensor-core products (~1e-5 relative each); at B = 65 their error alone reaches 2e-5 at every width from 1072 up, so mode-1 outputs get
the mode-1 forward bound of tests/test_style_gru_gpu.py, 1e-4.  Gradient bounds are those of tests/test_style_gru_f64_gpu.py in every
setting.

* The forward at every new hidden size (66: 1072 .. 2112), B = 3, T = 5, GEMM modes 0 and 1.
* Forward and backward at H in {1072, 1360, 1376, 1536, 2112} x B in {1, 32, 33, 65} (T = 17, VAE), and T in {1, 2} at B in {1, 33}
  without the VAE, each in three settings (mode 0, mode 1, mode 1 + fast_wgrad).  3H = 4080 at 1360 and 4128 at 1376: the bias
  gradients are one column-sum launch below 4096 columns and two slabs above.
* The largest batch one call takes at H = 2112 (1792) against the oracle; one sample more is refused before any launch.
* W_hh at 4- and 8-byte offsets from 16-byte alignment, as TrainStep's flat parameter buffer places it.
* Generation: B = 1, T = 3600, H = 2112, forward, no eps.
* TrainStep with a 1536-wide GRU style encoder (VAE, tensor-core decoder engine): graph replay against eager launches, concurrent lanes
  against one stream.
* generate_gesture from whole-module pickles with a 2112-wide GRU style encoder without the VAE, and train() with a 1536-wide one whose
  checkpoints generate_gesture loads.
"""
import json
import os
import random
import shutil
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import _encoder_cases as ec
from tests import _gru_cases as gc
from tests._util import report, stats_tensors
from tests.test_gpu_parity import _batch, _load
from tests.test_style_gru_f64_gpu import SETTINGS, _report, _run_gpu, dev, setting  # noqa: F401

pytestmark = pytest.mark.gpu

WIDE_H = list(range(1072, 2112 + 1, 16))
EDGE_H = [1072, 1360, 1376, 1536, 2112]
CASES = {
    **{f"H{H}_B{B}_T17_vae": dict(B=B, T=17, H=H) for H in EDGE_H for B in (1, 32, 33, 65)},
    **{f"H{H}_B{B}_T{T}_novae": dict(B=B, T=T, H=H, vae=False) for H in EDGE_H for B in (1, 33) for T in (1, 2)},
}
MAX_B = 1792            # at every H > 1056: the BPTT's 16-unit carry of 56 batch tiles in 227 KB of shared memory
MODE1_FWD_TOL = 1e-4    # outputs through split-bf16 products (tests/test_style_gru_gpu.py)


def _errors(setting_name, *args, **kw):
    """gc.errors with the output bound of the setting."""
    errs = gc.errors(*args, **kw)
    if setting_name == "mode0":
        return errs
    return [(n, e, MODE1_FWD_TOL if b == gc.FWD_TOL and "out" in n else b) for n, e, b in errs]


@pytest.fixture
def on_device(dev, monkeypatch):
    """The float64 oracle and restatement of tests/_gru_cases.py on the device: their parameter leaves and a case's tensors move there."""
    leaves = ec._leaves
    monkeypatch.setattr(ec, "_leaves", lambda P, dtype, grads: {k: v.to(dev).detach().requires_grad_(grads)
                                                                for k, v in leaves(P, dtype, False).items()})

    def move(case):
        to = lambda t: None if t is None else t.to(dev)
        return SimpleNamespace(**dict(vars(case), x=to(case.x), eps=to(case.eps),
                                      cots=None if case.cots is None else [to(c) for c in case.cots]))
    return move


def _margined(P, case):
    """gc.margined_params with the float64 internals on the device."""
    P = dict(P)
    for site, bkey in gc.RELU_SITES:
        P[gc._SE + bkey] = np.zeros_like(P[gc._SE + bkey])
        z = gc._internals(P, case, torch.float64)[site].cpu()
        z = z.reshape(-1, z.shape[-1])
        std = z.std(0) if z.shape[0] > 1 else z.std().expand(z.shape[1])
        b = -z.max(0).values - gc.GATE_GAP * std
        b[0::2] = (-z.min(0).values + gc.GATE_GAP * std)[0::2]
        P[gc._SE + bkey] = b.float().numpy()
    return P


_oracles = {}


def _oracle(case, on_device, key):
    """Cached per case: (natural parameters, margined parameters, natural outputs, margined outputs, gradients, matched gradients, keys the
    matched oracle rounded)."""
    if key not in _oracles:
        _oracles.clear()
        c = on_device(case)
        P = gc.gru_params(case.H, case.E)
        Pm = _margined(P, c)
        nat_o = gc.run_oracle(P, c)[0]
        o, g = gc.run_oracle(Pm, c)
        _, mg, opts = gc.run_restated(Pm, c, matched=True)
        _oracles[key] = (P, Pm, nat_o, o, g, mg, {r[0] for r in opts.rounded})
    return _oracles[key]


def _check(tag, case, oracle, setting_name, dev):
    P, Pm, nat_o, o, g, mg, rounded = oracle
    fast = setting_name == "mode1_fast_wgrad"
    errs = [(f"natural {n}", e, b) for n, e, b in _errors(setting_name, _run_gpu(P, case, dev, False)[0], None, nat_o, None)]
    go, gg = _run_gpu(Pm, case, dev, True)
    errs += _errors(setting_name, go, gg, o, mg if fast else g, rounded if fast else ())
    assert float(gg[gc.W_HH_R].abs().max()) == 0.0
    _report(tag, errs)


@pytest.mark.parametrize("H", WIDE_H)
def test_forward_at_every_wide_hidden_size(dev, setting, on_device, H):
    case = gc.sweep_case(H)
    P = gc.gru_params(H, case.E)
    ref = gc.run_oracle(P, on_device(case))[0]
    for name in ("mode0", "mode1"):
        setting(name)
        _report(f"H{H} B3 T5 {name}", _errors(name, _run_gpu(P, case, dev, False)[0], None, ref, None))


@pytest.mark.parametrize("name", SETTINGS)
@pytest.mark.parametrize("cid", list(CASES))
def test_wide_gru_style_encoder_vs_float64(dev, setting, on_device, cid, name):
    setting(name)
    kw = dict(CASES[cid])
    case = gc.gru_case(seed=10000 * kw["B"] + 10 * kw["T"] + kw["H"], **kw)
    _check(f"{cid} {name}", case, _oracle(case, on_device, cid), name, dev)


def test_largest_batch_at_2112_and_one_more(dev, setting, on_device):
    from zeggs_b200 import _lib, modules
    H = 2112
    l = _lib.lib()
    assert l.zeggs_style_enc_gru_workspace_bytes(MAX_B, 2, 1134, H, 128, 1) > 0
    assert l.zeggs_style_enc_gru_workspace_bytes(MAX_B + 1, 2, 1134, H, 128, 1) == 0
    setting("mode0")
    case = gc.gru_case(B=MAX_B, T=2, H=H, seed=2112)
    _check(f"H{H} B{MAX_B} T2 (largest batch)", case, _oracle(case, on_device, "largest"), "mode0", dev)
    _oracles.clear()
    mod = modules.StyleEncoder(1134, H, 64, type="gru", use_vae=True).to(dev)
    x = torch.zeros(MAX_B + 1, 2, 1134, device=dev)
    torch.cuda.synchronize()
    launches = l.zeggs_launch_count()
    with pytest.raises(_lib.ZeggsError, match=f"at most {MAX_B} samples"):
        mod(x, 1.0, eps=torch.zeros(MAX_B + 1, 64, device=dev))
    assert l.zeggs_launch_count() == launches


@pytest.mark.parametrize("name", ["mode0", "mode1"])
def test_generation_forward_at_2112(dev, setting, on_device, name):
    setting(name)
    case = gc.gru_case(B=1, T=3600, H=2112, grads=False, eps=False, seed=3600)
    if "gen" not in _oracles:
        _oracles.clear()
        P = gc.gru_params(case.H, case.E)
        _oracles["gen"] = (P, gc.run_oracle(P, on_device(case))[0])
    P, ref = _oracles["gen"]
    _report(f"H2112 B1 T3600 gen {name}", _errors(name, _run_gpu(P, case, dev, False)[0], None, ref, None))


@pytest.mark.parametrize("offset", [1, 2])
def test_unaligned_w_hh(dev, setting, on_device, monkeypatch, offset):
    """W_hh as a view `offset` floats into a buffer (TrainStep's flat parameters put it at any 4-byte offset): forward and backward at
    H = 2112, B = 33, T = 17 in mode 0 match the oracle."""
    import tests.test_style_gru_f64_gpu as sg
    setting("mode0")
    case = gc.gru_case(B=33, T=17, H=2112, seed=77 + offset)
    make = sg._module

    def shifted(P, case, dev):
        mod = make(P, case, dev)
        w = mod.encoder.rnn_layer.weight_hh_l0
        buf = torch.empty(w.numel() + offset, device=dev)
        buf[offset:].copy_(w.data.reshape(-1))
        w.data = buf[offset:].view(w.shape)
        assert w.data_ptr() % 16 == 4 * offset
        return mod
    monkeypatch.setattr(sg, "_module", shifted)
    _check(f"H2112 B33 T17 W_hh at +{4 * offset} B", case, _oracle(case, on_device, f"unaligned{offset}"), "mode0", dev)


# ---------------------------------------------------------------------------------------------------------- end to end
def _step(dev, Hs, seed, **kw):
    from zeggs_b200 import modules, synth
    from zeggs_b200.train import TrainStep
    P = synth.make_params(H=512, seed=seed, style_hidden=Hs, style_type="gru")
    se = _load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", dev)
    st = _load(modules.StyleEncoder(1134, Hs, 64, type="gru", use_vae=True), P, "style_encoder.", dev)
    de = _load(modules.Decoder(1134, 1131, 64, 64, 512, 2), P, "decoder.", dev)
    stats = synth.load_stats()
    return TrainStep(se, de, st, stats, stats["parents"], float(stats["dt"]), **kw)


def test_train_step_graph_and_lanes_with_a_1536_wide_gru_style_encoder(dev, monkeypatch):
    """B = 32, tensor-core decoder engine: graph-captured steps with concurrent lanes, eager steps with lanes, and graph steps on one
    stream give the same losses and parameters after 3 steps."""
    from zeggs_b200 import ops
    prev = ops.DECODER_ENGINE
    ops.set_decoder_engine("tc")
    res = {}
    try:
        for mode, lanes in (("graph", "1"), ("eager", "1"), ("graph", "0")):
            monkeypatch.setenv("ZEGGS_LANES", lanes)
            torch.manual_seed(422)
            step = _step(dev, 1536, 82, lr=1e-3, use_graph=True)
            if mode == "eager":
                step.graph_min_seen = 10 ** 9
            losses = [float(step.step(_batch(dev, 32, 16, 24, 290 + it)).item()) for it in range(3)]
            torch.cuda.synchronize()
            if mode == "graph":
                assert len(step._graphs) == 1
            res[(mode, lanes)] = (losses, step.optimizer.flat_param.clone())
            del step
    finally:
        ops.set_decoder_engine(prev)
    for k, v in res.items():
        print(f"  {k}: losses {v[0]}")
    ref = res[("graph", "1")]
    assert all(np.isfinite(ref[0]))
    assert np.allclose(res[("eager", "1")][0], ref[0], rtol=1e-6, atol=0)
    assert float((res[("eager", "1")][1] - ref[1]).abs().max()) <= 1e-7
    assert res[("graph", "0")][0] == ref[0]
    assert float((res[("graph", "0")][1] - ref[1]).abs().max()) == 0.0


def _data_dir(tmp_path):
    from tests import _fixtures as fx
    from zeggs_b200 import synth
    data = tmp_path / "data"; data.mkdir()
    stats = synth.load_stats()
    np.savez(data / "stats.npz", **{k: stats[k] for k in ("audio_input_mean", "audio_input_std", "anim_input_mean", "anim_input_std",
                                                         "anim_output_mean", "anim_output_std")})
    shutil.copy(os.path.join(fx.DATA, "data_definition_v1.json"), data / "data_definition.json")
    shutil.copy(os.path.join(fx.DATA, "data_pipeline_conf_v1.json"), data / "data_pipeline_conf.json")
    return data, Path(fx.make_synthetic_bvh(str(tmp_path / "style.bvh"))), Path(fx.make_wav(str(tmp_path / "speech.wav")))


def test_generate_gesture_with_a_2112_wide_gru_checkpoint(dev, tmp_path):
    """Whole-module pickles with a 2112-wide GRU style encoder without the VAE: generate_gesture writes the BVH, and its style encoding
    matches the float64 oracle on the same example features (<= 1e-4 x max(1, |ref|))."""
    from oracle import style_oracle as so
    from zeggs_b200 import animation, generate, modules, synth
    Hs = 2112
    P = synth.make_params(H=256, seed=44, style_hidden=Hs, style_type="gru", style_embed=64)
    net = tmp_path / "net"; net.mkdir()
    torch.save(_load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", "cpu"), net / "speech_encoder.pt")
    torch.save(_load(modules.StyleEncoder(1134, Hs, 64, type="gru", use_vae=False), P, "style_encoder.", "cpu"), net / "style_encoder.pt")
    torch.save(_load(modules.Decoder(1134, 1131, 64, 64, 256, 2), P, "decoder.", "cpu"), net / "decoder.pt")
    data, bvh_path, wav_path = _data_dir(tmp_path)
    res = tmp_path / "res"
    enc = generate.generate_gesture(wav_path, [(bvh_path, (10, 300))], net, data, res, file_name="out", use_gpu=True)
    b = animation.load_bvh(str(res / "out.bvh"))
    assert np.all(np.isfinite(b["positions"])) and b["positions"].shape[0] == enc.shape[1]
    z = enc[0, 0]
    a = animation.preprocess_animation(animation.trim(animation.load_bvh(str(bvh_path)), (10, 300)))
    n = len(a["root_vel"])
    vec = np.concatenate([a[k].reshape(n, -1) for k in ("root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt")]
                         + [np.zeros((n, 3), np.float32)], axis=1)
    st = stats_tensors()
    ex = (torch.as_tensor(vec, dtype=torch.float32) - st["anim_input_mean"]) / st["anim_input_std"]
    Pd = {k: torch.from_numpy(np.asarray(v)).double().to(dev) for k, v in P.items() if k.startswith("style_encoder.")}
    with torch.no_grad():
        ref, _, _ = so.style_encoder(Pd, ex[None].double().to(dev), use_vae=False, type="gru")
    err, sc = report("generate gru H2112 z", z[None].cpu(), ref.cpu())
    assert err <= 1e-4 * max(1.0, sc)


def test_train_then_generate_with_a_1536_wide_gru_style_encoder(dev, tmp_path):
    """train() for 3 iterations with net_opt.style_encoder = {type: "gru", nhidden: 1536, use_vae: true} writes checkpoints whose style
    encoder is 1536 wide; generate_gesture loads them and writes a finite BVH."""
    from tests import _fixtures as fx
    from zeggs_b200 import animation, generate
    from zeggs_b200.train import train
    ddef, dproc = fx.make_dataset_files(str(tmp_path))
    to = dict(seed=21, use_gpu=True, resume=False, learning_rate=1e-3, learning_rate_decay=0.999, eps=1e-5, niterations=3 / 1000.0,
              batchsize=32, window=64, style_encoding_type="example", generate_samples_step=1000, use_tensorboard=False,
              decoder_engine="auto", cuda_graph=True, device_dataset=True)
    no = dict(speech_encoder=dict(nhidden=64, speech_encoding_size=64),
              style_encoder=dict(nhidden=1536, style_encoding_size=64, example_length=64, type="gru", use_vae=True),
              decoder=dict(nhidden=512))
    state = random.getstate()
    random.seed(0)
    try:
        train(str(tmp_path / "models"), str(tmp_path / "logs"), dproc, ddef, to, no)
    finally:
        random.setstate(state)
    net = tmp_path / "models"
    st = torch.load(net / "style_encoder.pt", map_location="cpu", weights_only=False)
    assert st.encoder.rnn_layer.weight_hh_l0.shape == (3 * 1536, 1536)
    assert all(bool(torch.isfinite(p).all()) for p in st.parameters())
    data, bvh_path, wav_path = _data_dir(tmp_path)
    conf = json.load(open(data / "data_pipeline_conf.json"))
    conf["audio_conf"]["normalize_loudness"] = False
    json.dump(conf, open(data / "data_pipeline_conf.json", "w"))
    res = tmp_path / "res"
    enc = generate.generate_gesture(wav_path, [(bvh_path, (10, 300))], net, data, res, file_name="out", use_gpu=True)
    b = animation.load_bvh(str(res / "out.bvh"))
    assert bool(torch.isfinite(enc).all()) and np.all(np.isfinite(b["positions"]))
