"""GPU: the GRU style encoder (zeggs_style_enc_gru_fwd / _bwd) and the attn encoder without the VAE, against oracle autograd and the
reference goldens (tests/golden/style_gru.npz, train_gru_*.npz), inside TrainStep (CUDA graphs, lanes) and in generate_gesture.

Tolerances: forward z / mu / logvar <= 2e-5 (fp32 SIMT GEMMs, gemm mode 0) or 1e-4 (tensor-core split-bf16, mode 1) x max(1, |ref|);
gradients as _grad_close of test_gpu_parity.py.  The long example (B = 1, T_ex = 3600, forward only, default mode 1):
<= 1e-4 x max(1, |ref|)."""
import os

import numpy as np
import pytest
import torch

from tests._util import NAMES, ensure_built, report, stats_tensors, tt
from tests.test_gpu_parity import _batch, _grad_close, _load

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


@pytest.fixture
def gemm_mode(dev):
    from zeggs_b200 import ops

    def set_mode(m):
        ops.set_gemm_mode(m)
    yield set_mode
    set_mode(1)


@pytest.fixture
def decoder_engine(dev):
    from zeggs_b200 import ops
    prev = ops.DECODER_ENGINE
    yield ops.set_decoder_engine
    ops.set_decoder_engine(prev)


def _gru_params(Hs, use_vae, seed):
    from zeggs_b200 import synth
    return synth.make_params(H=64, seed=seed, style_hidden=Hs, style_embed=128 if use_vae else 64, style_type="gru")


def _gru_encoder(P, Hs, use_vae, dev):
    from zeggs_b200 import modules
    return _load(modules.StyleEncoder(1134, Hs, 64, type="gru", use_vae=use_vae), P, "style_encoder.", dev)


def _example(B, T, seed):
    from zeggs_b200 import synth
    st = stats_tensors()
    return (torch.from_numpy(synth.make_style_example(B, T, seed=seed)) - st["anim_input_mean"]) / st["anim_input_std"]


_ORACLE = {}


def _oracle(B, T, use_vae):
    """oracle autograd of sum(out * cot) (cached: shared by both GEMM modes)."""
    key = (B, T, use_vae)
    if key not in _ORACLE:
        from oracle import style_oracle as so
        P = _gru_params(512, use_vae, 100 + T)
        x = _example(B, T, seed=B + T)
        rs = np.random.RandomState(B * 100 + T)
        eps = torch.from_numpy(rs.randn(B, 64).astype(np.float32))
        Pt = {k: v.clone().requires_grad_(True) for k, v in tt(P).items() if k.startswith("style_encoder.")}
        ref = [r for r in so.style_encoder(Pt, x, eps=eps, temperature=1.3, use_vae=use_vae, type="gru") if r is not None]
        cots = [torch.from_numpy(rs.randn(*r.shape).astype(np.float32)) for r in ref]
        keys = sorted(Pt)
        g_ref = torch.autograd.grad(sum((r * c).sum() for r, c in zip(ref, cots)), [Pt[k] for k in keys])
        _ORACLE[key] = (P, x, eps, [r.detach() for r in ref], cots, keys, g_ref)
    return _ORACLE[key]


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("use_vae", [True, False])
@pytest.mark.parametrize("B,T", [(2, 16), (3, 33), (32, 512)])
def test_gru_style_encoder_fwd_bwd_vs_oracle(dev, gemm_mode, B, T, use_vae, mode):
    gemm_mode(mode)
    P, x, eps, ref, cots, keys, g_ref = _oracle(B, T, use_vae)
    enc = _gru_encoder(P, 512, use_vae, dev)
    out = [o for o in enc(x.to(dev), 1.3, eps=eps.to(dev)) if o is not None]
    assert len(out) == len(ref)
    named = dict(enc.named_parameters())
    g_got = torch.autograd.grad(sum((o * c.to(dev)).sum() for o, c in zip(out, cots)), [named[k[len("style_encoder."):]] for k in keys])
    for n, o, r in zip(("z", "mu", "logvar"), out, ref):
        err, sc = report(f"gru fwd B{B} T{T} vae{int(use_vae)} mode{mode} {n}", o, r)
        assert err <= (2e-5 if mode == 0 else 1e-4) * max(1.0, sc), n
    bad = []
    for k, a, b in zip(keys, g_got, g_ref):
        _grad_close(f"gru bwd {k}", a, b, mode, bad)
    assert not bad, bad
    # the reverse direction's W_hh multiplied h = 0: exactly zero gradient, as the reference's autograd gives
    assert float(g_got[keys.index("style_encoder.encoder.rnn_layer.weight_hh_l0_reverse")].abs().max()) == 0.0


def test_gru_style_encoder_long_example_T3600(dev):
    """Inference feeds the whole style clip: B = 1, T_ex = 3600 (60 s), forward only, default GEMM mode, against the oracle's full
    bidirectional scan."""
    from oracle import style_oracle as so
    P = _gru_params(512, True, 3600)
    x = _example(1, 3600, seed=3600)
    with torch.no_grad():
        ref = so.style_encoder(tt(P), x, eps=torch.zeros(1, 64), use_vae=True, type="gru")
        enc = _gru_encoder(P, 512, True, dev).eval()
        out = enc(x.to(dev), 1.0, eps=torch.zeros(1, 64, device=dev))
    for n, o, r in zip(("z", "mu", "logvar"), out, ref):
        err, sc = report(f"gru T3600 {n}", o, r)
        assert err <= 1e-4 * max(1.0, sc), n


@pytest.mark.parametrize("tag", ["gru_vae_h64_t16", "gru_novae_h64_t16", "gru_vae_h64_t33", "gru_novae_h64_t33", "gru_vae_h512_t256",
                                 "gru_novae_h512_t256", "attn_novae_h64_t16"])
def test_style_encoder_vs_reference_golden(dev, golden_dir, gemm_mode, tag):
    """The reference's own StyleEncoder outputs and parameter gradients (fp32 SIMT GEMMs): forward <= 2e-5 x max(1, |ref|), stored
    gradients max-abs <= 3e-4 of max|ref|, gradient norms within 5e-4 relative."""
    gemm_mode(0)
    from zeggs_b200 import modules, synth
    g = np.load(os.path.join(golden_dir, "style_gru.npz"))
    typ, vae, Hs, Z = str(g[tag + ".type"]), bool(g[tag + ".use_vae"]), int(g[tag + ".H"]), int(g["Z"])
    seed, B, T = int(g[tag + ".param_seed"]), int(g[tag + ".B"]), int(g[tag + ".T_ex"])
    P = synth.make_params(H=64, seed=seed, style_hidden=Hs, style_embed=2 * Z if vae else Z, style_type=typ)
    enc = _load(modules.StyleEncoder(1134, Hs, Z, type=typ, use_vae=vae), P, "style_encoder.", dev).eval()
    x = _example(B, T, seed).to(dev)
    out = [o for o in enc(x, float(g["temperature"]), eps=torch.from_numpy(g[tag + ".eps"]).to(dev)) if o is not None]
    names = ["z", "mu", "logvar"][:len(out)]
    for n, o in zip(names, out):
        err, sc = report(f"{tag} {n}", o, torch.from_numpy(g[f"{tag}.{n}"]))
        assert err <= 2e-5 * max(1.0, sc), n
    params = list(enc.named_parameters())
    grads = torch.autograd.grad(sum((o * torch.from_numpy(g[f"{tag}.cot_{n}"]).to(dev)).sum() for n, o in zip(names, out)),
                                [p for _, p in params])
    bad = []
    for (k, _), gr in zip(params, grads):
        ref_n = float(g[f"{tag}.gradnorm.{k}"])
        got_n = float(gr.double().norm())
        if not abs(got_n - ref_n) <= 5e-4 * max(ref_n, 1e-7):
            bad.append((k, "norm", got_n, ref_n))
        if f"{tag}.grad.{k}" in g.files:
            ref = g[f"{tag}.grad.{k}"]
            if not float(np.abs(gr.cpu().numpy() - ref).max()) <= 3e-4 * max(float(np.abs(ref).max()), 1e-7):
                bad.append((k, "elementwise"))
    assert not bad, bad


# ---------------------------------------------------------------------------------------------- TrainStep
def _make_gru_step(dev, H, param_seed, use_vae, style_type="gru", **kw):
    from zeggs_b200 import modules, synth
    from zeggs_b200.train import TrainStep
    P = synth.make_params(H=H, seed=param_seed, style_type=style_type, style_embed=128 if use_vae else 64)
    se = _load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", dev)
    st = _load(modules.StyleEncoder(1134, 512, 64, type=style_type, use_vae=use_vae), P, "style_encoder.", dev)
    de = _load(modules.Decoder(1134, 1131, 64, 64, H, 2), P, "decoder.", dev)
    stats = synth.load_stats()
    return TrainStep(se, de, st, stats, stats["parents"], float(stats["dt"]), **kw), P


def _golden_step(dev, golden_dir, tag):
    g = np.load(os.path.join(golden_dir, f"train_{tag}.npz"))
    H, B, T, T_ex = int(g["H"]), int(g["B"]), int(g["T"]), int(g["T_ex"])
    step, _ = _make_gru_step(dev, H, int(g["param_seed"]), bool(g["use_vae"]))
    step.iteration = int(g["iteration"])
    batch = _batch(dev, B, T, T_ex, int(g["input_seed"]))
    step.optimizer.zero_grad()
    loss = step.forward_backward(batch, eps=torch.from_numpy(g["eps"]).to(dev), train_mode=False)
    torch.cuda.synchronize()
    return g, step, loss


@pytest.mark.parametrize("mode", [0, 1])
def test_train_step_gru_vae_fp32_engine_vs_reference_golden(dev, golden_dir, gemm_mode, decoder_engine, mode):
    """train_gru_h64 (GRU encoder with the VAE, fp32 recurrence engine), tolerances of test_train_step_loss_and_gradients_vs_reference_golden:
    loss 2e-5 / 2e-4 relative, terms 3e-5 / 5e-4, gradient norms 5e-4 / 3e-3, stored gradients max-abs 5e-4 / rel-L2 3e-3."""
    gemm_mode(mode)
    decoder_engine("fp32")
    g, step, loss = _golden_step(dev, golden_dir, "gru_h64")
    terms = step.terms.cpu().numpy()
    print(f"  loss {loss.item():.6f} vs golden {float(g['loss']):.6f}")
    assert abs(loss.item() - float(g["loss"])) <= (2e-5 if mode == 0 else 2e-4) * abs(float(g["loss"]))
    names = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "lrot", "lvel", "lvrt", "cpos", "crot", "cvel", "cvrt",
             "ldvl", "ldvt", "cdvl", "cdvt", "gaze", "kl_div"]
    for i, n in enumerate(names):
        ref = float(g["loss_" + n])
        assert abs(terms[1 + i] - ref) <= (3e-5 if mode == 0 else 5e-4) * max(1e-3, abs(ref)), (n, terms[1 + i], ref)
    bad = []
    for prefix, net in (("speech_encoder.", step.se), ("decoder.", step.dec), ("style_encoder.", step.st)):
        for k, p in net.named_parameters():
            ref_n = float(g["gradnorm." + prefix + k])
            got_n = float(p.grad.double().norm())
            if not abs(got_n - ref_n) <= (5e-4 if mode == 0 else 3e-3) * max(ref_n, 1e-7):
                bad.append((prefix + k, got_n, ref_n))
            if "grad." + prefix + k in g.files:
                ref = g["grad." + prefix + k]
                d = p.grad.cpu().numpy() - ref
                if mode == 0:
                    if not float(np.abs(d).max()) <= 5e-4 * max(float(np.abs(ref).max()), 1e-7):
                        bad.append((prefix + k, "elementwise", float(np.abs(d).max())))
                elif not float(np.linalg.norm(d)) <= 3e-3 * max(float(np.linalg.norm(ref)), 1e-9):
                    bad.append((prefix + k, "relL2", float(np.linalg.norm(d))))
    assert not bad, bad


def test_train_step_gru_no_vae_tc_engine_vs_reference_golden(dev, golden_dir, decoder_engine):
    """train_gru_h384 (GRU encoder without the VAE: KL term 0, sum still / 18) on the tensor-core engine, tolerances of
    test_train_step_tc_engine_vs_reference_golden: loss 5e-3 relative, terms 3e-2, gradient norms 5e-2, stored gradients rel-L2 6e-2."""
    decoder_engine("tc")
    g, step, loss = _golden_step(dev, golden_dir, "gru_h384")
    assert step.dec.__dict__.get("_zeggs_packed_tc") is not None, "the tensor-core engine did not run"
    terms = step.terms.cpu().numpy()
    rel = abs(loss.item() - float(g["loss"])) / abs(float(g["loss"]))
    names = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "lrot", "lvel", "lvrt", "cpos", "crot", "cvel", "cvrt",
             "ldvl", "ldvt", "cdvl", "cdvt", "gaze", "kl_div"]
    worst_t = max(abs(terms[1 + i] - float(g["loss_" + n])) / max(1e-3, abs(float(g["loss_" + n]))) for i, n in enumerate(names))
    assert terms[18] == 0.0
    bad, worst_n, worst_e = [], 0.0, 0.0
    for prefix, net in (("speech_encoder.", step.se), ("decoder.", step.dec), ("style_encoder.", step.st)):
        for k, p in net.named_parameters():
            ref_n = float(g["gradnorm." + prefix + k])
            r = abs(float(p.grad.double().norm()) - ref_n) / max(ref_n, 1e-7)
            worst_n = max(worst_n, r)
            if r > 5e-2:
                bad.append((prefix + k, "norm", r))
            if "grad." + prefix + k in g.files:
                ref = g["grad." + prefix + k]
                e = float(np.linalg.norm(p.grad.cpu().numpy() - ref)) / max(float(np.linalg.norm(ref)), 1e-9)
                worst_e = max(worst_e, e)
                if e > 6e-2:
                    bad.append((prefix + k, "relL2", e))
    print(f"  [gru_h384 tc] loss rel {rel:.3e}, worst term {worst_t:.3e}, worst grad-norm {worst_n:.3e}, worst stored-grad {worst_e:.3e}")
    assert rel <= 5e-3 and worst_t <= 3e-2
    assert not bad, bad


@pytest.mark.parametrize("use_vae", [True, False])
def test_gru_graph_replayed_train_steps_match_eager_launches(dev, decoder_engine, use_vae):
    """TrainStep(use_graph=True) with the GRU style encoder: step 1 eager, step 2 captured + replayed, steps 3-5 replayed, against the
    same steps launched eagerly: losses and parameters after 5 steps identical."""
    decoder_engine("tc")
    res = {}
    for mode in ("graph", "eager"):
        torch.manual_seed(123)
        step, _ = _make_gru_step(dev, 384, 79, use_vae, lr=1e-3, use_graph=True)
        if mode == "eager":
            step.graph_min_seen = 10 ** 9
        losses = [float(step.step(_batch(dev, 4, 16, 24, 50 + it)).item()) for it in range(5)]
        torch.cuda.synchronize()
        if mode == "graph":
            assert step.use_graph and len(step._graphs) == 1, "the CUDA-graph path did not run"
        res[mode] = (losses, step.optimizer.flat_param.clone())
        del step
    print("  graph losses", res["graph"][0]); print("  eager losses", res["eager"][0])
    assert all(np.isfinite(res["graph"][0]))
    assert res["graph"][0] == res["eager"][0]
    assert float((res["graph"][1] - res["eager"][1]).abs().max()) == 0.0


@pytest.mark.parametrize("style_type,use_vae", [("gru", True), ("gru", False), ("attn", False)])
def test_style_variants_concurrent_lanes_match_single_stream_step(dev, decoder_engine, monkeypatch, style_type, use_vae):
    """The style encoder's forward / backward on the 'style' lane (next to the speech encoder and the decoder's phase-2 weight
    gradients) against the same steps on one stream: identical losses and parameters."""
    decoder_engine("tc")
    res = {}
    for lanes in ("1", "0"):
        monkeypatch.setenv("ZEGGS_LANES", lanes)
        torch.manual_seed(321)
        step, _ = _make_gru_step(dev, 384, 80, use_vae, style_type=style_type, lr=1e-3, use_graph=True)
        assert step.lanes == (lanes == "1")
        losses = [float(step.step(_batch(dev, 4, 16, 24, 70 + it)).item()) for it in range(4)]
        torch.cuda.synchronize()
        res[lanes] = (losses, step.optimizer.flat_param.clone())
        del step
    print("  lanes  losses", res["1"][0]); print("  serial losses", res["0"][0])
    assert all(np.isfinite(res["1"][0]))
    assert res["1"][0] == res["0"][0]
    assert float((res["1"][1] - res["0"][1]).abs().max()) == 0.0


# ---------------------------------------------------------------------------------------------- generate_gesture
def test_generate_gesture_with_gru_checkpoint_without_vae(dev, tmp_path):
    """A GRU / no-VAE checkpoint (whole-module pickles) through generate_gesture: the BVH is written, the returned encoding is the
    style encoder's z broadcast over the clip, and z matches the oracle on the same example features (<= 1e-4 x max(1, |ref|))."""
    import json
    import shutil
    from pathlib import Path
    from oracle import style_oracle as so
    from tests import _fixtures as fx
    from zeggs_b200 import animation, generate, modules, synth
    H = 256
    P = synth.make_params(H=H, seed=43, style_type="gru", style_embed=64)
    net = tmp_path / "net"; net.mkdir()
    torch.save(_load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", "cpu"), net / "speech_encoder.pt")
    torch.save(_load(modules.StyleEncoder(1134, 512, 64, type="gru", use_vae=False), P, "style_encoder.", "cpu"), net / "style_encoder.pt")
    torch.save(_load(modules.Decoder(1134, 1131, 64, 64, H, 2), P, "decoder.", "cpu"), net / "decoder.pt")
    data = tmp_path / "data"; data.mkdir()
    stats = synth.load_stats()
    np.savez(data / "stats.npz", **{k: stats[k] for k in ("audio_input_mean", "audio_input_std", "anim_input_mean", "anim_input_std",
                                                         "anim_output_mean", "anim_output_std")})
    shutil.copy(os.path.join(fx.DATA, "data_definition_v1.json"), data / "data_definition.json")
    shutil.copy(os.path.join(fx.DATA, "data_pipeline_conf_v1.json"), data / "data_pipeline_conf.json")
    bvh_path = Path(fx.make_synthetic_bvh(str(tmp_path / "style.bvh")))
    wav_path = Path(fx.make_wav(str(tmp_path / "speech.wav")))
    res = tmp_path / "res"
    enc = generate.generate_gesture(wav_path, [(bvh_path, (10, 300))], net, data, res, file_name="out", use_gpu=True)
    assert (res / "out.bvh").exists() and (res / "out.wav").exists()
    b = animation.load_bvh(str(res / "out.bvh"))
    assert np.all(np.isfinite(b["positions"])) and b["positions"].shape[0] == enc.shape[1]
    z = generate.generate_gesture(None, [(bvh_path, (10, 300))], net, data, None)
    assert tuple(z.shape) == (1, 64) and tuple(enc.shape) == (1, enc.shape[1], 64)
    assert torch.equal(enc[0, 0], z[0]) and torch.equal(enc[0, -1], z[0])
    a = animation.preprocess_animation(animation.trim(animation.load_bvh(str(bvh_path)), (10, 300)))
    n = len(a["root_vel"])
    vec = np.concatenate([a[k].reshape(n, -1) for k in ("root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt")]
                         + [np.zeros((n, 3), np.float32)], axis=1)
    st = stats_tensors()
    ex = (torch.as_tensor(vec, dtype=torch.float32) - st["anim_input_mean"]) / st["anim_input_std"]
    with torch.no_grad():
        ref, _, _ = so.style_encoder(tt(P), ex[None], use_vae=False, type="gru")
    err, sc = report("generate gru z", z, ref)
    assert err <= 1e-4 * max(1.0, sc)
