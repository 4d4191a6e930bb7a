"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle and the committed reference goldens.  The GEMM front end has its
own float64 tests: tests/test_gemm_f64_gpu.py.

Tolerances (stated per SURVEY.md 8d):
  mel features            abs <= 2e-4 on the ln-domain 80-mel + energy features (fp32 FFT vs the f64 reference)
  decoder fp32 path       against the float64 oracle, the bounds of oracle/fp32_oracle.py: per-pose-channel max-abs
                          <= FP32_FWD_TOL * max(1, max|ref|) (de-normalised units), free-running; gradients max-abs
                          <= FP32_GEMM_GRAD_TOL * max|ref| (GEMM mode 1); reference goldens (fp32) 2e-4
"""
import os

import numpy as np
import pytest
import torch

from tests._util import NAMES, ensure_built, make_decoder, report, stats_tensors, tt

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


def test_normalize_rows_is_bit_identical_to_the_two_tensor_ops(dev):
    """zeggs_normalize_rows against (x - mean) / std (train.py:232-234): same fp32 subtract + IEEE divide -> identical bits."""
    from zeggs_b200 import ops
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(3, 37, 1134, generator=g) * 7).to(dev)
    mean = torch.randn(1134, generator=g).to(dev)
    std = (torch.rand(1134, generator=g) + 0.05).to(dev)
    assert torch.equal(ops.normalize_rows(x, mean, std), (x - mean) / std)


# ---------------------------------------------------------------------------------------------- mel
@pytest.mark.parametrize("hop", [200, 160])
def test_mel_against_reference_golden(dev, golden_dir, hop):
    from zeggs_b200 import audio
    g = np.load(os.path.join(golden_dir, "mel_small.npz"))
    wav = torch.from_numpy(g["wav"]).to(dev)
    fe = audio.MelFrontEnd(dev, hop_length=hop)
    n60 = g[f"feat_hop{hop}"].shape[1]
    mel, feat = fe.forward(wav, 60, n60, want_mel=True, want_feat=True)
    err, _ = report(f"mel[0,1] hop{hop}", mel, torch.from_numpy(g[f"mel_hop{hop}"]))
    assert err <= 1e-4
    err, _ = report(f"feat hop{hop}", feat, torch.from_numpy(g[f"feat_hop{hop}"]))
    assert err <= 2e-4


def test_mel_long_clips_against_oracle(dev):
    from oracle import mel_oracle
    from zeggs_b200 import audio, synth
    wav = synth.make_waveforms(3, 160000, seed=5)
    wav[2, 50000:90000] = 0.0
    fe = audio.MelFrontEnd(dev)
    _, feat = fe.forward(torch.from_numpy(wav).to(dev), 60, 600)
    for i in range(3):
        ref = mel_oracle.preprocess_audio(wav[i], 60, 600)
        err, _ = report(f"feat clip{i}", feat[i], torch.from_numpy(ref))
        assert err <= 2e-4
    # drop-in surface (numpy in -> numpy out), ragged length
    from oracle.make_golden import audio_params
    x = wav[0, :12345]
    n60 = int(round(60.0 * len(x) / 16000))
    got = audio.preprocess_audio(x, 60, n60, audio_params(200), ["mel_spec", "energy"])
    ref = mel_oracle.preprocess_audio(x, 60, n60)
    assert got.dtype == np.float32 and got.shape == ref.shape
    assert np.abs(got - ref).max() <= 2e-4


# ---------------------------------------------------------------------------------------------- decoder
def _decoder_case(dev, H, B, T, seed, P=None, speech=None, style=None, ref_dtype=torch.float32):
    from oracle import model_oracle as mo
    from zeggs_b200 import synth
    st = stats_tensors()
    P = P or synth.make_params(H=H, seed=seed, with_style=False)
    win = tt(synth.make_pose_windows(B, T, seed=seed))
    rs = np.random.RandomState(seed)
    if speech is None:
        speech = torch.from_numpy((rs.randn(B, T, 64) * 0.5).astype(np.float32))
        style = torch.from_numpy(rs.randn(B, 1, 64).astype(np.float32)).repeat(1, T, 1)
    with torch.no_grad():
        d = lambda x: x.to(ref_dtype)
        ref = mo.decoder_forward({k: d(v) for k, v in tt(P).items()}, *[d(win[n][:, 0]) for n in NAMES], d(win["gaze_pos"]), d(speech),
                                 d(style), *[d(st[k]) for k in ("anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")],
                                 st["dt"])
        dec = make_decoder(P, H, device=dev)
        out = dec(*[win[n][:, 0].to(dev) for n in NAMES], win["gaze_pos"].to(dev), speech.to(dev), style.to(dev),
                  st["parents"], st["anim_input_mean"].to(dev), st["anim_input_std"].to(dev),
                  st["anim_output_mean"].to(dev), st["anim_output_std"].to(dev), st["dt"])
    torch.cuda.synchronize()
    return out, ref


@pytest.mark.parametrize("H,B,T", [(64, 2, 6), (128, 4, 9), (128, 40, 5), (512, 16, 12), (1024, 32, 8), (1024, 1, 40)])
def test_decoder_forward_vs_oracle(dev, H, B, T):
    from oracle.fp32_oracle import FP32_FWD_TOL
    out, ref = _decoder_case(dev, H, B, T, seed=100 + H + B, ref_dtype=torch.float64)
    assert len(out) == 8
    for n, o, r in zip(NAMES, out, ref):
        assert tuple(o.shape) == tuple(r.shape), n
        err = float((o.cpu().double() - r).abs().max())
        sc = float(r.abs().max())
        print(f"  [decoder H{H} B{B} T{T} {n}] max-abs err {err:.3e} (ref max {sc:.3e}), {err / max(1.0, sc) / FP32_FWD_TOL:.3f} of the bound")
        assert err <= FP32_FWD_TOL * max(1.0, sc), n


@pytest.mark.parametrize("tag", ["h64", "h128"])
def test_decoder_forward_vs_reference_golden(dev, golden_dir, tag):
    from zeggs_b200 import synth
    g = np.load(os.path.join(golden_dir, f"train_{tag}.npz"))
    H, B, T = int(g["H"]), int(g["B"]), int(g["T"])
    P = synth.make_params(H=H, seed=int(g["param_seed"]))
    st = stats_tensors(dev)
    win = tt(synth.make_pose_windows(B, T, seed=int(g["input_seed"])), dev)
    dec = make_decoder(P, H, device=dev)
    speech = torch.from_numpy(g["speech"]).to(dev)
    style = torch.from_numpy(g["z"]).to(dev).unsqueeze(1).repeat(1, T, 1)
    with torch.no_grad():
        out = dec(*[win[n][:, 0] for n in NAMES], win["gaze_pos"], speech, style, st["parents"], st["anim_input_mean"],
                  st["anim_input_std"], st["anim_output_mean"], st["anim_output_std"], st["dt"])
    for n, o in zip(NAMES, out):
        ref = torch.from_numpy(g["O_" + n])
        err, sc = report(f"decoder golden {tag} {n}", o, ref)
        assert err <= 2e-4 * max(1.0, sc), n


# ---------------------------------------------------------------------------------------------- decoder backward (BPTT)
@pytest.mark.parametrize("H,B,T", [(64, 2, 6), (128, 4, 9), (128, 40, 4), (512, 16, 6), (1024, 32, 5)])
def test_decoder_backward_vs_oracle_autograd(dev, H, B, T):
    """GEMM mode 1 (the default): every gradient max-abs <= FP32_GEMM_GRAD_TOL * max|ref| against float64 autograd."""
    from oracle import model_oracle as mo
    from oracle.fp32_oracle import FP32_GEMM_GRAD_TOL
    from zeggs_b200 import synth
    seed = 300 + H + B
    st = stats_tensors()
    P = synth.make_params(H=H, seed=seed, with_style=False)
    win = tt(synth.make_pose_windows(B, T, seed=seed))
    rs = np.random.RandomState(seed)
    speech = torch.from_numpy((rs.randn(B, T, 64) * 0.5).astype(np.float32))
    style = torch.from_numpy(rs.randn(B, T, 64).astype(np.float32))
    cot = [torch.from_numpy(rs.randn(*win[n].shape).astype(np.float32)) for n in NAMES]
    # oracle (CPU autograd, float64)
    d = lambda x: x.double()
    Pt = {k: d(v).requires_grad_(True) for k, v in tt(P).items() if k.startswith("decoder.")}
    sp_o, sy_o = d(speech).requires_grad_(True), d(style).requires_grad_(True)
    ref = mo.decoder_forward(Pt, *[d(win[n][:, 0]) for n in NAMES], d(win["gaze_pos"]), sp_o, sy_o, d(st["anim_input_mean"]),
                             d(st["anim_input_std"]), d(st["anim_output_mean"]), d(st["anim_output_std"]), st["dt"])
    loss_o = sum((o * d(c)).sum() for o, c in zip(ref, cot))
    keys = sorted(Pt.keys())
    g_ref = torch.autograd.grad(loss_o, [Pt[k] for k in keys] + [sp_o, sy_o])
    # CUDA path
    dec = make_decoder(P, H, device=dev).train()
    sp_g, sy_g = speech.to(dev).requires_grad_(True), style.to(dev).requires_grad_(True)
    out = dec(*[win[n][:, 0].to(dev) for n in NAMES], win["gaze_pos"].to(dev), sp_g, sy_g, st["parents"],
              st["anim_input_mean"].to(dev), st["anim_input_std"].to(dev), st["anim_output_mean"].to(dev),
              st["anim_output_std"].to(dev), st["dt"])
    loss_g = sum((o * c.to(dev)).sum() for o, c in zip(out, cot))
    named = dict(dec.named_parameters())
    g_got = torch.autograd.grad(loss_g, [named[k[len("decoder."):]] for k in keys] + [sp_g, sy_g])
    torch.cuda.synchronize()
    assert abs(loss_g.item() - loss_o.item()) <= 1e-4 * max(1.0, abs(loss_o.item()))
    bad = []
    for k, a, b in zip(keys + ["speech", "style"], g_got, g_ref):
        err, sc = float((a.cpu().double() - b).abs().max()), float(b.abs().max())
        print(f"  [bwd H{H} B{B} T{T} {k}] max-abs err {err:.3e} (ref max {sc:.3e}), {err / max(sc, 1e-30) / FP32_GEMM_GRAD_TOL:.3f} of the bound")
        if not err <= FP32_GEMM_GRAD_TOL * sc:
            bad.append((k, err, sc))
    assert not bad, bad


# ---------------------------------------------------------------------------------------------- encoders
def _load(mod, P, prefix, dev):
    mod.load_state_dict({k[len(prefix):]: torch.from_numpy(v) for k, v in P.items() if k.startswith(prefix)})
    return mod.to(dev)


@pytest.fixture
def gemm_mode(dev):
    """Select the GEMM engine for one test and restore the default (1 = tensor-core split-bf16) afterwards."""
    from zeggs_b200 import ops

    def set_mode(m):
        ops.set_gemm_mode(m)
    yield set_mode
    set_mode(1)


def _grad_close(name, got, ref, mode, bad):
    """mode 0 (fp32 SIMT): max-abs 3e-4 of max|ref|.  mode 1 (tensor-core split-bf16, ~1e-5 relative products): relative L2 error
    <= 3e-2 -- a ReLU/ELU gate whose pre-activation is within 1e-5 of zero can legitimately flip (about one element per
    100k), which moves the affected rows by O(1) of their size but leaves the L2 error small (on the smallest case, 32
    rows, ONE flip is 1.5-2.6e-2 of a bias-gradient norm; which element flips depends on the summation order, e.g. split-K).
    The backward algebra itself is pinned by mode 0 and the GEMM by test_gemm_f32_front_end_tcgen05 (4e-5)."""
    err, sc = report(name, got, ref)
    if mode == 0:
        if not err <= 3e-4 * max(sc, 1e-6):
            bad.append((name, err, sc))
    else:
        num = float((got.detach().cpu().double() - ref.double()).norm())
        den = float(ref.double().norm())
        if not num <= 3e-2 * max(den, 1e-9):
            bad.append((name, "relL2", num / max(den, 1e-30)))


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("B,T,train", [(2, 6, False), (3, 40, True), (4, 97, True)])
def test_speech_encoder_fwd_bwd(dev, gemm_mode, B, T, train, mode):
    """fp32 SIMT engine: abs <= 1e-5 forward, 3e-4 max-abs gradients; tensor-core split-bf16 engine: abs <= 1e-4 forward, rel-L2
    2e-3 gradients -- vs oracle autograd with the same injected dropout masks."""
    gemm_mode(mode)
    from oracle import model_oracle as mo
    from zeggs_b200 import modules, synth
    P = synth.make_params(H=64, seed=21)
    rs = np.random.RandomState(B * 100 + T)
    x = torch.from_numpy(rs.randn(B, T, 81).astype(np.float32))
    masks = None
    if train:
        masks = [torch.from_numpy(((rs.rand(B, T, 64) >= 0.2) / 0.8).astype(np.float32)) for _ in range(2)]
    cot = torch.from_numpy(rs.randn(B, T, 64).astype(np.float32))
    Pt = {k: v.clone().requires_grad_(True) for k, v in tt(P).items() if k.startswith("speech_encoder.")}
    ref = mo.speech_encoder(Pt, x, None if masks is None else [m.transpose(1, 2) for m in masks])
    keys = sorted(Pt)
    g_ref = torch.autograd.grad((ref * cot).sum(), [Pt[k] for k in keys])
    enc = _load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", dev)
    enc.train(train)
    out = enc(x.to(dev), None if masks is None else [m.to(dev) for m in masks])
    named = dict(enc.named_parameters())
    g_got = torch.autograd.grad((out * cot.to(dev)).sum(), [named[k[len("speech_encoder."):]] for k in keys])
    err, sc = report(f"speech fwd B{B} T{T}", out, ref)
    assert err <= (1e-5 if mode == 0 else 1e-4) * max(1.0, sc)
    bad = []
    for k, a, b in zip(keys, g_got, g_ref):
        _grad_close(f"speech bwd {k}", a, b, mode, bad)
    assert not bad, bad


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("B,T,train", [(2, 16, False), (3, 33, True), (2, 130, True)])
def test_style_encoder_fwd_bwd(dev, gemm_mode, B, T, train, mode):
    """(z, mu, logvar): abs <= 2e-5 (fp32 SIMT engine) / 1e-4 (tensor-core split-bf16); gradients as in _grad_close --
    vs oracle autograd with injected eps and dropout masks."""
    gemm_mode(mode)
    from oracle import model_oracle as mo
    from zeggs_b200 import modules, synth
    P = synth.make_params(H=64, seed=22)
    st = stats_tensors()
    rs = np.random.RandomState(B * 100 + T)
    x = (torch.from_numpy(synth.make_style_example(B, T, seed=B + T)) - st["anim_input_mean"]) / st["anim_input_std"]
    eps = torch.from_numpy(rs.randn(B, 64).astype(np.float32))
    masks = None
    if train:
        mk = lambda shape, p: torch.from_numpy(((rs.rand(*shape) >= p) / (1 - p)).astype(np.float32))
        masks = dict(c1=mk((B, T, 512), 0.2), c2=mk((B, T, 128), 0.2), attn=mk((B, 4, T, T), 0.1), ao=mk((B, T, 128), 0.1),
                     ff=mk((B, T, 128), 0.1))
    cots = [torch.from_numpy(rs.randn(B, 64).astype(np.float32)) for _ in range(3)]
    Pt = {k: v.clone().requires_grad_(True) for k, v in tt(P).items() if k.startswith("style_encoder.")}
    ref = mo.style_encoder(Pt, x, eps=eps, temperature=1.3, masks=masks)
    keys = sorted(Pt)
    g_ref = torch.autograd.grad(sum((r * c).sum() for r, c in zip(ref, cots)), [Pt[k] for k in keys])
    enc = _load(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), P, "style_encoder.", dev)
    enc.train(train)
    out = enc(x.to(dev), 1.3, eps=eps.to(dev), masks=None if masks is None else {k: v.to(dev) for k, v in masks.items()})
    named = dict(enc.named_parameters())
    g_got = torch.autograd.grad(sum((o * c.to(dev)).sum() for o, c in zip(out, cots)),
                                [named[k[len("style_encoder."):]] for k in keys])
    for n, o, r in zip(("z", "mu", "logvar"), out, ref):
        err, sc = report(f"style fwd B{B} T{T} {n}", o, r)
        assert err <= (2e-5 if mode == 0 else 1e-4) * max(1.0, sc), n
    bad = []
    for k, a, b in zip(keys, g_got, g_ref):
        _grad_close(f"style bwd {k}", a, b, mode, bad)
    assert not bad, bad


# ---------------------------------------------------------------------------------------------- loss / optimizer / train step
def _make_step(dev, H, param_seed):
    from zeggs_b200 import modules, synth
    from zeggs_b200.train import TrainStep
    P = synth.make_params(H=H, seed=param_seed)
    se = _load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", dev)
    st = _load(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), P, "style_encoder.", dev)
    de = _load(modules.Decoder(1134, 1131, 64, 64, H, 2), P, "decoder.", dev)
    stats = synth.load_stats()
    return TrainStep(se, de, st, stats, stats["parents"], float(stats["dt"])), P


def _batch(dev, B, T, T_ex, seed):
    from zeggs_b200 import synth
    b = tt(synth.make_pose_windows(B, T, seed=seed), dev)
    b["audio"] = torch.from_numpy(synth.make_audio_features(B, T, seed=seed)).to(dev)
    b["style"] = torch.from_numpy(synth.make_style_example(B, T_ex, seed=seed)).to(dev)
    return b


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("tag", ["h64", "h128"])
def test_train_step_loss_and_gradients_vs_reference_golden(dev, golden_dir, gemm_mode, tag, mode):
    """Whole step body (encoders -> decoder -> FK loss -> backward) against the reference's own loss / gradients
    (golden written by oracle/make_golden.py from the unmodified reference, eval-mode dropout, injected VAE eps)."""
    gemm_mode(mode)
    g = np.load(os.path.join(golden_dir, f"train_{tag}.npz"))
    H, B, T, T_ex = int(g["H"]), int(g["B"]), int(g["T"]), int(g["T_ex"])
    step, P = _make_step(dev, H, int(g["param_seed"]))
    step.iteration = int(g["iteration"])
    batch = _batch(dev, B, T, T_ex, int(g["input_seed"]))
    step.optimizer.zero_grad()
    loss = step.forward_backward(batch, eps=torch.from_numpy(g["eps"]).to(dev), train_mode=False)
    torch.cuda.synchronize()
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


def test_fused_radam_vs_reference_golden(dev, golden_dir):
    from zeggs_b200.optimizers import RAdam
    g = np.load(os.path.join(golden_dir, "radam.npz"))
    p = torch.nn.Parameter(torch.from_numpy(g["p0"].copy()).to(dev))
    opt = RAdam([p], lr=1e-4, eps=1e-5)
    for i in range(g["grads"].shape[0]):
        opt.zero_grad()
        p.grad.copy_(torch.from_numpy(g["grads"][i]).to(dev))
        opt.step()
        assert np.abs(p.detach().cpu().numpy() - g["traj"][i]).max() <= 2e-7, i


# ---------------------------------------------------------------------------------------------- inference path (config 1)
def test_generate_motion_end_to_end_vs_oracle(dev):
    """WAV samples -> mel -> SpeechEncoder -> StyleEncoder (example) -> free-running decoder (B=1, 3 s clip), eval mode.
    Per-pose-channel max-abs <= 5e-4 * max(1, max|ref|) in de-normalised units (default tensor-core split-bf16 encoders,
    fp32 recurrence)."""
    from oracle import mel_oracle, model_oracle as mo
    from zeggs_b200 import generate, modules, synth
    H = 1024
    P = synth.make_params(H=H, seed=77)
    st = synth.load_stats()
    nets = dict(speech_encoder=_load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", dev).eval(),
                style_encoder=_load(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), P, "style_encoder.", dev).eval(),
                decoder=_load(modules.Decoder(1134, 1131, 64, 64, H, 2), P, "decoder.", dev).eval())
    wav = synth.make_waveforms(1, 48000, seed=9)[0]
    ex = synth.make_style_example(1, 200, seed=9)[0]
    win = synth.make_pose_windows(1, 2, seed=9)
    fp = {k: win[k][0, 0] for k in NAMES}
    from oracle.make_golden import audio_params
    eps = np.zeros((1, 64), np.float32)
    out, z = generate.generate_motion(nets, st, audio_params(200), wav, ex, fp, win["gaze_pos"][0, 0], float(st["dt"]),
                                      temperature=1.0, eps=torch.zeros(1, 64, device=dev), device=dev)
    torch.cuda.synchronize()
    # oracle chain
    f = lambda k: torch.as_tensor(st[k], dtype=torch.float32)
    T = 180
    Pt = tt(P)
    with torch.no_grad():
        feat = torch.from_numpy(mel_oracle.preprocess_audio(wav, 60, T))[None]
        sp = mo.speech_encoder(Pt, (feat - f("audio_input_mean")) / f("audio_input_std"))
        zz, mu, lv = mo.style_encoder(Pt, (torch.from_numpy(ex)[None] - f("anim_input_mean")) / f("anim_input_std"), eps=torch.from_numpy(eps))
        gaze = torch.from_numpy(win["gaze_pos"][0, 0]).reshape(1, 1, 3).repeat(1, T, 1)
        ref = mo.decoder_forward(Pt, *[torch.from_numpy(fp[k])[None] for k in NAMES], gaze, sp, zz.unsqueeze(1).repeat(1, T, 1),
                                 f("anim_input_mean"), f("anim_input_std"), f("anim_output_mean"), f("anim_output_std"), float(st["dt"]))
    err, sc = report("generate z", z, zz)
    assert err <= 1e-4 * max(1.0, sc)
    for n, o, r in zip(NAMES, out, ref):
        assert tuple(o.shape) == tuple(r.shape)
        err, sc = report(f"generate {n}", o, r)
        assert err <= 5e-4 * max(1.0, sc), n


def test_checkpoint_round_trip_whole_module_pickles(dev, tmp_path):
    """train.py:482-509 / generate.py:130-138 artefact format: torch.save(module) -> load_networks -> same outputs."""
    from zeggs_b200 import generate, modules, synth
    P = synth.make_params(H=64, seed=5)
    dec = _load(modules.Decoder(1134, 1131, 64, 64, 64, 2), P, "decoder.", dev).eval()
    se = _load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", dev).eval()
    torch.save(dec, tmp_path / "decoder.pt"); torch.save(se, tmp_path / "speech_encoder.pt")
    nets = generate.load_networks(tmp_path, dev, with_style=False)
    x = torch.randn(2, 9, 81, device=dev)
    with torch.no_grad():
        assert torch.equal(nets["speech_encoder"](x), se(x))
    assert nets["decoder"].hidden_size == 64


# ---------------------------------------------------------------------------------------------- tensor-core recurrence engine
@pytest.fixture
def decoder_engine():
    from zeggs_b200 import ops

    def set_engine(name):
        ops.set_decoder_engine(name)
    yield set_engine
    ops.set_decoder_engine("fp32")


@pytest.mark.parametrize("H,B,T", [(384, 4, 9), (512, 16, 40), (1024, 32, 24), (1024, 7, 64), (512, 40, 10), (1024, 3, 2)])
def test_decoder_forward_tc_engine_vs_oracle(dev, decoder_engine, H, B, T):
    """tensor-core recurrence (bf16 MMA operands, fp32 accumulate/state): free-running per-pose-channel max-abs
    <= 2e-2 * max(1, max|ref|) in de-normalised units (bf16 operand rounding, 2^-9 relative, compounds over the window)."""
    decoder_engine("tc")
    out, ref = _decoder_case(dev, H, B, T, seed=500 + H + B)
    for n, o, r in zip(NAMES, out, ref):
        err, sc = report(f"decoder[tc] H{H} B{B} T{T} {n}", o, r)
        assert torch.isfinite(o).all()
        assert err <= 2e-2 * max(1.0, sc), n


@pytest.mark.parametrize("H,B,T", [(512, 16, 12), (1024, 32, 10)])
def test_decoder_training_with_tc_forward(dev, decoder_engine, H, B, T):
    """Forward on the tensor-core engine (saved fp32 activations) + BPTT kernel: gradients vs oracle autograd, relative L2 <= 3e-2
    (mixed-precision training numerics: the backward differentiates the bf16-operand forward)."""
    from oracle import model_oracle as mo
    from zeggs_b200 import synth
    decoder_engine("tc")
    seed = 700 + H
    st = stats_tensors()
    P = synth.make_params(H=H, seed=seed, with_style=False)
    win = tt(synth.make_pose_windows(B, T, seed=seed))
    rs = np.random.RandomState(seed)
    speech = torch.from_numpy((rs.randn(B, T, 64) * 0.5).astype(np.float32))
    style = torch.from_numpy(rs.randn(B, T, 64).astype(np.float32))
    cot = [torch.from_numpy(rs.randn(*win[n].shape).astype(np.float32)) for n in NAMES]
    Pt = {k: v.clone().requires_grad_(True) for k, v in tt(P).items() if k.startswith("decoder.")}
    ref = mo.decoder_forward(Pt, *[win[n][:, 0] for n in NAMES], win["gaze_pos"], speech, style, st["anim_input_mean"],
                             st["anim_input_std"], st["anim_output_mean"], st["anim_output_std"], st["dt"])
    keys = sorted(Pt.keys())
    g_ref = torch.autograd.grad(sum((o * c).sum() for o, c in zip(ref, cot)), [Pt[k] for k in keys])
    dec = make_decoder(P, H, device=dev).train()
    out = dec(*[win[n][:, 0].to(dev) for n in NAMES], win["gaze_pos"].to(dev), speech.to(dev), style.to(dev), st["parents"],
              st["anim_input_mean"].to(dev), st["anim_input_std"].to(dev), st["anim_output_mean"].to(dev),
              st["anim_output_std"].to(dev), st["dt"])
    named = dict(dec.named_parameters())
    g_got = torch.autograd.grad(sum((o * c.to(dev)).sum() for o, c in zip(out, cot)), [named[k[len("decoder."):]] for k in keys])
    bad = []
    for k, a, b in zip(keys, g_got, g_ref):
        num = float((a.cpu().double() - b.double()).norm()); den = float(b.double().norm())
        print(f"  [tc-train H{H} {k}] relL2 {num / max(den, 1e-30):.3e}")
        if not num <= 3e-2 * max(den, 1e-9):
            bad.append((k, num / max(den, 1e-30)))
    assert not bad, bad


def test_full_size_window_engines_agree_and_are_deterministic(dev, decoder_engine):
    """BASELINE.json config 2 at the reference-actual size (B=32, T=256, H=1024), too large for the CPU oracle in a unit test:
    (1) the tensor-core engine run twice is bit-identical (fixed summation orders, no atomics on the data path);
    (2) it agrees with the fp32 SIMT engine -- itself pinned to the oracle at <= 2e-4 on the small cases above -- within the
    stated bf16-operand tolerance over the whole 256-frame free-running window: per-pose-channel max-abs <= 5e-2 * max(1, |ref|);
    (3) frame 0 of every output is the given first pose (modules.py:153-162)."""
    from zeggs_b200 import synth
    H, B, T = 1024, 32, 256
    st = stats_tensors()
    P = synth.make_params(H=H, seed=77, with_style=False)
    win = tt(synth.make_pose_windows(B, T, seed=78))
    rs = np.random.RandomState(79)
    speech = torch.from_numpy((rs.randn(B, T, 64) * 0.5).astype(np.float32)).to(dev)
    style = torch.from_numpy(rs.randn(B, 1, 64).astype(np.float32)).repeat(1, T, 1).to(dev)
    dec = make_decoder(P, H, device=dev)
    args = [win[n][:, 0].to(dev) for n in NAMES] + [win["gaze_pos"].to(dev), speech, style, st["parents"]] + \
           [st[k].to(dev) for k in ("anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")] + [st["dt"]]
    outs = {}
    with torch.no_grad():
        for name in ("tc", "tc2", "fp32"):
            decoder_engine("tc" if name.startswith("tc") else "fp32")
            outs[name] = [o.clone() for o in dec(*args)]
    torch.cuda.synchronize()
    for n, a, b, r in zip(NAMES, outs["tc"], outs["tc2"], outs["fp32"]):
        assert torch.equal(a, b), f"{n}: tensor-core engine not deterministic"
        assert torch.isfinite(a).all()
        err, sc = report(f"full-size tc vs fp32 {n}", a, r)
        assert err <= 5e-2 * max(1.0, sc), n
        assert torch.equal(a[:, 0].cpu(), win[n][:, 0]), f"{n}: frame 0 must be the given pose"


def test_full_size_train_step_engines_agree(dev, decoder_engine):
    """Whole train step at the bench size (B=32, T=256, H=1024, T_ex=384): loss and every parameter-gradient norm of the
    tensor-core engine against the fp32 SIMT engine (same dropout masks / VAE noise via the same torch seed):
    loss within 1e-2 relative, gradient norms within 6e-2 relative (bf16 operands over 255 recurrent steps)."""
    B, T, T_ex, H = 32, 256, 384, 1024
    res = {}
    for eng in ("fp32", "tc"):
        decoder_engine(eng)
        step, P = _make_step(dev, H, 1234)
        batch = _batch(dev, B, T, T_ex, 5)
        torch.manual_seed(11); torch.cuda.manual_seed(11)
        step.optimizer.zero_grad()
        loss = step.forward_backward(batch)
        torch.cuda.synchronize()
        norms = {}
        for prefix, net in (("speech_encoder.", step.se), ("decoder.", step.dec), ("style_encoder.", step.st)):
            for k, p in net.named_parameters():
                norms[prefix + k] = float(p.grad.double().norm())
        res[eng] = (float(loss.item()), norms)
        del step
        torch.cuda.empty_cache()
    l0, l1 = res["fp32"][0], res["tc"][0]
    print(f"  full-size loss fp32 {l0:.5f} tc {l1:.5f}")
    assert np.isfinite(l1) and abs(l1 - l0) <= 1e-2 * abs(l0)
    bad = [(k, res["tc"][1][k], v) for k, v in res["fp32"][1].items() if not abs(res["tc"][1][k] - v) <= 6e-2 * max(v, 1e-7)]
    assert not bad, bad


def test_label_style_z9_engines_agree(dev, decoder_engine):
    """configs_v2 geometry (one-hot label style, Z = 9 -> odd W_ih0 row stride A + H): the tensor-core engine against the fp32
    SIMT engine, window outputs <= 2e-2 * max(1, |ref|), parameter / speech gradient norms within 2e-2 relative."""
    from zeggs_b200 import modules, synth
    H, B, T, Z = 512, 4, 6, 9
    st = stats_tensors()
    torch.manual_seed(3)
    dec = modules.Decoder(1134, 1131, 64, Z, H, 2).to(dev)
    win = tt(synth.make_pose_windows(B, T, seed=3))
    speech = (torch.randn(B, T, 64) * 0.5).to(dev).requires_grad_(True)
    style = torch.zeros(B, T, Z)
    style[:, :, 2] = 1.0
    res = {}
    for eng in ("fp32", "tc"):
        decoder_engine(eng)
        for p in dec.parameters():
            p.grad = None
        speech.grad = None
        out = dec(*[win[n][:, 0].to(dev) for n in NAMES], win["gaze_pos"].to(dev), speech, style.to(dev), st["parents"],
                  *[st[k].to(dev) for k in ("anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")], st["dt"])
        sum((o * o).sum() for o in out).backward()
        torch.cuda.synchronize()
        res[eng] = ([o.detach().clone() for o in out], float(torch.cat([p.grad.flatten() for p in dec.parameters()]).norm()),
                    float(speech.grad.norm()))
    for n, a, b in zip(NAMES, res["tc"][0], res["fp32"][0]):
        err, sc = report(f"z9 tc vs fp32 {n}", a, b)
        assert err <= 2e-2 * max(1.0, sc), n
    assert abs(res["tc"][1] - res["fp32"][1]) <= 2e-2 * res["fp32"][1]
    assert abs(res["tc"][2] - res["fp32"][2]) <= 2e-2 * res["fp32"][2]


# ---------------------------------------------------------------------------------------------- round 2: the benchmarked engine pinned to the oracle / reference
def test_tc_engine_request_is_strict(dev, decoder_engine):
    """An explicit 'tc' request on an ineligible hidden size raises (it never silently runs the fp32 engine); 'auto' falls back."""
    from zeggs_b200 import _lib
    decoder_engine("tc")
    with pytest.raises(_lib.ZeggsError):
        _decoder_case(dev, 128, 2, 4, seed=1)
    decoder_engine("auto")
    out, ref = _decoder_case(dev, 128, 2, 4, seed=1)
    for n, o, r in zip(NAMES, out, ref):
        err, sc = report(f"auto->fp32 H128 {n}", o, r)
        assert err <= 2e-4 * max(1.0, sc)


def _channel_table(tag, out, ref, frames=None):
    """Per-pose-channel-group max-abs error table (de-normalised units), optionally per frame range; returns {name: (err, scale)}."""
    res = {}
    for n, o, r in zip(NAMES, out, ref):
        o, r = o.detach().float().cpu(), r.detach().float().cpu()
        if frames is not None:
            o, r = o[:, frames[0]:frames[1]], r[:, frames[0]:frames[1]]
        res[n] = (float((o - r).abs().max()), float(r.abs().max()))
        print(f"  [{tag}] {n:9s} max-abs err {res[n][0]:.3e}  ref max {res[n][1]:.3e}  rel-to-max(1,ref) {res[n][0] / max(1.0, res[n][1]):.3e}")
    return res


# tolerances of the tensor-core (bf16 operand) recurrence against the fp32 CPU oracle, as fractions of max(1, max|ref|) per pose-channel
# group, free running (errors feed back through the pose): stated in DESIGN.md 2
TC_TOL_WINDOW = 1e-2        # B=32, T=256 training window
TC_TOL_LONG = 2e-2          # T=3600 (60 s) generation


def test_full_size_tc_forward_vs_oracle(dev, decoder_engine):
    """BASELINE config 2, reference-actual size (B=32, T=256, H=1024): the tensor-core engine against the CPU oracle's forward
    (oracle/model_oracle.decoder_forward, modules.py:47-162), per-pose-channel table printed and asserted."""
    decoder_engine("tc")
    out, ref = _decoder_case(dev, 1024, 32, 256, seed=2024)
    res = _channel_table("full-size tc vs ORACLE", out, ref)
    _channel_table("full-size tc vs ORACLE, frames 0..64", out, ref, frames=(0, 64))
    for n, (err, sc) in res.items():
        assert err <= TC_TOL_WINDOW * max(1.0, sc), n
    decoder_engine("fp32")
    out32, _ = _decoder_case(dev, 1024, 32, 256, seed=2024)
    res32 = _channel_table("full-size fp32 engine vs ORACLE", out32, ref)
    for n, (err, sc) in res32.items():
        assert err <= 2e-3 * max(1.0, sc), n


@pytest.mark.parametrize("tag", ["h384", "h1024"])
def test_train_step_tc_engine_vs_reference_golden(dev, golden_dir, decoder_engine, tag):
    """The whole step body on the TENSOR-CORE engine (H >= 384: U=4/G=96 at H=384, U=8/G=128 -- the bench geometry -- at H=1024)
    against the unmodified reference's loss, 18 terms and gradients (oracle/make_golden.py): loss within 5e-3 relative, terms
    within 3e-2, gradient norms within 5e-2, stored gradient tensors rel-L2 <= 6e-2 (bf16 MMA operands; encoders' weight
    gradients single-pass bf16)."""
    decoder_engine("tc")
    g = np.load(os.path.join(golden_dir, f"train_{tag}.npz"))
    H, B, T, T_ex = int(g["H"]), int(g["B"]), int(g["T"]), int(g["T_ex"])
    step, P = _make_step(dev, H, int(g["param_seed"]))
    step.iteration = int(g["iteration"])
    batch = _batch(dev, B, T, T_ex, int(g["input_seed"]))
    step.optimizer.zero_grad()
    loss = step.forward_backward(batch, eps=torch.from_numpy(g["eps"]).to(dev), train_mode=False)
    torch.cuda.synchronize()
    assert step.dec.__dict__.get("_zeggs_packed_tc") is not None, "the tensor-core engine did not run"
    terms = step.terms.cpu().numpy()
    rel = abs(loss.item() - float(g["loss"])) / abs(float(g["loss"]))
    print(f"  [{tag} tc] loss {loss.item():.6f} vs reference golden {float(g['loss']):.6f}  rel {rel:.3e}")
    names = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "lrot", "lvel", "lvrt", "cpos", "crot", "cvel", "cvrt",
             "ldvl", "ldvt", "cdvl", "cdvt", "gaze", "kl_div"]
    worst_t = 0.0
    for i, n in enumerate(names):
        ref = float(g["loss_" + n])
        worst_t = max(worst_t, abs(terms[1 + i] - ref) / max(1e-3, abs(ref)))
    worst_n, worst_e, bad = 0.0, 0.0, []
    for prefix, net in (("speech_encoder.", step.se), ("decoder.", step.dec), ("style_encoder.", step.st)):
        for k, p in net.named_parameters():
            ref_n = float(g["gradnorm." + prefix + k])
            got_n = float(p.grad.double().norm())
            r = abs(got_n - ref_n) / max(ref_n, 1e-7)
            worst_n = max(worst_n, r)
            if r > 5e-2:
                bad.append((prefix + k, "norm", got_n, ref_n))
            if "grad." + prefix + k in g.files:
                ref = g["grad." + prefix + k]
                e = float(np.linalg.norm(p.grad.cpu().numpy() - ref)) / max(float(np.linalg.norm(ref)), 1e-9)
                worst_e = max(worst_e, e)
                if e > 6e-2:
                    bad.append((prefix + k, "relL2", e))
    print(f"  [{tag} tc] worst loss-term rel {worst_t:.3e}, worst grad-norm rel {worst_n:.3e}, worst stored-grad relL2 {worst_e:.3e}")
    assert rel <= 5e-3
    assert worst_t <= 3e-2
    assert not bad, bad


def test_long_clip_drift_T3600(dev, decoder_engine):
    """BASELINE config 5 horizon (60 s = 3600 frames, H=1024): (a) tc engine vs the CPU oracle at B=2, (b) tc vs the fp32 engine at
    B=64 (two 32-sample tiles).  Free running for 3599 bf16-operand steps; per-pose-channel max-abs over the whole clip and
    over the first 600 frames printed; asserted against TC_TOL_LONG."""
    decoder_engine("tc")
    out, ref = _decoder_case(dev, 1024, 2, 3600, seed=3600)
    _channel_table("T3600 B2 tc vs ORACLE, frames 0..600", out, ref, frames=(0, 600))
    res = _channel_table("T3600 B2 tc vs ORACLE", out, ref)
    for o in out:
        assert torch.isfinite(o).all()
    from zeggs_b200 import synth
    st = stats_tensors()
    H, B, T = 1024, 64, 3600
    P = synth.make_params(H=H, seed=88, with_style=False)
    win = tt(synth.make_pose_windows(B, 2, seed=88))
    rs = np.random.RandomState(88)
    speech = torch.from_numpy((rs.randn(B, T, 64) * 0.5).astype(np.float32)).to(dev)
    style = torch.from_numpy(rs.randn(B, 1, 64).astype(np.float32)).repeat(1, T, 1).to(dev)
    gaze = win["gaze_pos"][:, :1].repeat(1, T, 1).to(dev)
    dec = make_decoder(P, H, device=dev)
    args = [win[n][:, 0].to(dev) for n in NAMES] + [gaze, speech, style, st["parents"]] + \
           [st[k].to(dev) for k in ("anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")] + [st["dt"]]
    outs = {}
    with torch.no_grad():
        for eng in ("tc", "fp32"):
            decoder_engine(eng)
            outs[eng] = [o.clone() for o in dec(*args)]
    torch.cuda.synchronize()
    res64 = _channel_table("T3600 B64 tc vs fp32 engine", outs["tc"], outs["fp32"])
    for n, (err, sc) in list(res.items()) + list(res64.items()):
        assert err <= TC_TOL_LONG * max(1.0, sc), n


def _v1_weights(golden_dir):
    """The shipped v1 networks, derived by build() into oracle/_ref/ from the original tree (oracle/ref_data.py)."""
    from oracle import ref_data
    W = ref_data.load_v1_weights()
    if W is None:
        pytest.skip("oracle/_ref/ holds no v1 networks (build() found no original tree to derive them from)")
    return W


def test_v1_pretrained_weights_vs_reference_golden(dev, golden_dir, decoder_engine):
    """The shipped, TRAINED v1 weights (larger gates, saturating GRUs) through the CUDA path -- SpeechEncoder, StyleEncoder and the
    decoder on both engines -- against outputs the unmodified reference produced from the pickles (tests/golden/v1_pretrained.npz)."""
    import json
    from zeggs_b200 import modules, synth
    P = _v1_weights(golden_dir)
    g = np.load(os.path.join(golden_dir, "v1_pretrained.npz"))
    B, T, T_ex, seed, H = int(g["B"]), int(g["T"]), int(g["T_ex"]), int(g["input_seed"]), int(g["H"])
    st = stats_tensors(dev)
    se = _load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", dev).eval()
    sty = _load(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), P, "style_encoder.", dev).eval()
    de = _load(modules.Decoder(1134, 1131, 64, 64, H, 2), P, "decoder.", dev).eval()
    win = tt(synth.make_pose_windows(B, T, seed=seed), dev)
    audio = torch.from_numpy(synth.make_audio_features(B, T, seed=seed)).to(dev)
    ex = torch.from_numpy(synth.make_style_example(B, T_ex, seed=seed)).to(dev)
    record = {}
    with torch.no_grad():
        speech = se((audio - st["audio_input_mean"]) / st["audio_input_std"])
        z, mu, logvar = sty((ex - st["anim_input_mean"]) / st["anim_input_std"], 1.0, eps=torch.zeros(B, 64, device=dev))
        err_s, sc_s = report("v1 speech encoder", speech, torch.from_numpy(g["speech"]))
        err_m, sc_m = report("v1 style mu", mu, torch.from_numpy(g["mu"]))
        record["speech"] = [err_s, sc_s]; record["mu"] = [err_m, sc_m]
        assert err_s <= 2e-4 * max(1.0, sc_s) and err_m <= 2e-4 * max(1.0, sc_m)
        ref = [torch.from_numpy(g["O_" + n]) for n in NAMES]
        sp_ref = torch.from_numpy(g["speech"]).to(dev)
        sy_ref = torch.from_numpy(g["mu"]).to(dev).unsqueeze(1).repeat(1, T, 1)
        for eng, tol in (("fp32", 1e-3), ("tc", TC_TOL_WINDOW)):
            decoder_engine(eng)
            out = de(*[win[n][:, 0] for n in NAMES], win["gaze_pos"], sp_ref, sy_ref, st["parents"], st["anim_input_mean"],
                     st["anim_input_std"], st["anim_output_mean"], st["anim_output_std"], st["dt"])
            res = _channel_table(f"v1 weights, {eng} engine vs REFERENCE", out, ref)
            record[eng] = {n: list(v) for n, v in res.items()}
            for n, (err, sc) in res.items():
                assert err <= tol * max(1.0, sc), (eng, n)
    os.makedirs(os.path.join(os.path.dirname(os.path.dirname(golden_dir)), "gpurun_out"), exist_ok=True)
    with open(os.path.join(os.path.dirname(os.path.dirname(golden_dir)), "gpurun_out", "v1_pretrained_parity.json"), "w") as f:
        json.dump(record, f, indent=1)


def test_short_training_curve_tc_tracks_fp32(dev, decoder_engine):
    """Convergence evidence for training on the tensor-core engine: 40 optimizer steps from the same initial weights, batches,
    dropout masks and VAE noise (same torch seed) on both engines at H=384, lr=1e-3: the loss curves stay within 2 % of each other
    at every step and both decrease."""
    curves = {}
    for eng in ("fp32", "tc"):
        decoder_engine(eng)
        step, P = _make_step(dev, 384, 4321)
        for gr in step.optimizer.param_groups:
            gr["lr"] = 1e-3
        torch.manual_seed(7); torch.cuda.manual_seed(7)
        losses = []
        for it in range(40):
            batch = _batch(dev, 8, 24, 32, 1000 + it % 4)
            losses.append(float(step.step(batch).item()))
        curves[eng] = losses
        del step
    a, b = np.array(curves["fp32"]), np.array(curves["tc"])
    print("  fp32 curve", np.round(a[::5], 4)); print("  tc   curve", np.round(b[::5], 4))
    assert np.all(np.isfinite(b))
    assert np.max(np.abs(a - b) / np.abs(a)) <= 2e-2
    assert a[-4:].mean() < a[:4].mean() and b[-4:].mean() < b[:4].mean()


def test_graph_replayed_train_steps_match_eager_launches(dev, decoder_engine):
    """TrainStep(use_graph=True): step 1 eager, step 2 captured + replayed, steps 3-5 replayed -- against the same steps launched
    eagerly (same device-side dropout/VAE seeds, same RAdam device counters): losses and parameters after 5 steps identical."""
    from zeggs_b200 import modules, synth
    from zeggs_b200.train import TrainStep
    decoder_engine("tc")
    res = {}
    for mode in ("graph", "eager"):
        torch.manual_seed(123)
        P = synth.make_params(H=384, seed=77)
        se = _load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", dev)
        st = _load(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), P, "style_encoder.", dev)
        de = _load(modules.Decoder(1134, 1131, 64, 64, 384, 2), P, "decoder.", dev)
        stats = synth.load_stats()
        step = TrainStep(se, de, st, stats, stats["parents"], float(stats["dt"]), lr=1e-3, use_graph=True)
        if mode == "eager":
            step.graph_min_seen = 10 ** 9
        losses = []
        for it in range(5):
            losses.append(float(step.step(_batch(dev, 4, 16, 24, 50 + it)).item()))
        torch.cuda.synchronize()
        if mode == "graph":
            assert step.use_graph and len(step._graphs) == 1, "the CUDA-graph path did not run"
            assert step.graph_launches > 0
        res[mode] = (losses, step.optimizer.flat_param.clone(), int(step.optimizer.step_dev.item()), step.optimizer._step)
        del step
    print("  graph losses", res["graph"][0]); print("  eager losses", res["eager"][0])
    assert res["graph"][2] == 5 and res["graph"][3] == 5 and res["eager"][2] == 5
    assert np.allclose(res["graph"][0], res["eager"][0], rtol=1e-6, atol=0)
    assert float((res["graph"][1] - res["eager"][1]).abs().max()) <= 1e-7


def test_concurrent_lanes_match_single_stream_step(dev, decoder_engine, monkeypatch):
    """TrainStep with the concurrent lanes (encoders side by side; encoders' backward next to the decoder's phase-2 weight gradients,
    each lane with its own stream and GEMM scratch) against the same calls issued in the same order on ONE stream: every kernel is
    deterministic and the lanes only reorder independent work, so losses and parameters must be identical.  Both runs use the
    two-phase decoder backward; test_two_phase_decoder_backward_matches_one_call pins it to the one-call form."""
    from zeggs_b200 import modules, synth
    from zeggs_b200.train import TrainStep
    decoder_engine("tc")
    res = {}
    for lanes in ("1", "0"):
        monkeypatch.setenv("ZEGGS_LANES", lanes)
        torch.manual_seed(321)
        P = synth.make_params(H=384, seed=78)
        se = _load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", dev)
        st = _load(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), P, "style_encoder.", dev)
        de = _load(modules.Decoder(1134, 1131, 64, 64, 384, 2), P, "decoder.", dev)
        stats = synth.load_stats()
        step = TrainStep(se, de, st, stats, stats["parents"], float(stats["dt"]), lr=1e-3, use_graph=True)
        assert step.lanes == (lanes == "1")
        losses = [float(step.step(_batch(dev, 4, 16, 24, 70 + it)).item()) for it in range(4)]
        torch.cuda.synchronize()
        res[lanes] = (losses, step.optimizer.flat_param.clone())
        del step
    print("  lanes  losses", res["1"][0]); print("  serial losses", res["0"][0])
    assert res["1"][0] == res["0"][0]
    assert float((res["1"][1] - res["0"][1]).abs().max()) == 0.0


@pytest.mark.parametrize("engine,H", [("tc", 384), ("fp32", 128)])
def test_two_phase_decoder_backward_matches_one_call(dev, decoder_engine, engine, H):
    """ops.decoder_window_backward in one call and in two phases (split=True, then finish()) on the same saved forward: every decoder
    parameter gradient, dSpeech and dStyle bitwise equal, on both engines."""
    from zeggs_b200 import ops, synth
    from zeggs_b200.train import POSE_KEYS, pack_pose
    decoder_engine(engine)
    B, T = 4, 16
    P = synth.make_params(H=H, seed=82, with_style=False)
    dec = make_decoder(P, H, device=dev).train()
    win = tt(synth.make_pose_windows(B, T, seed=82), dev)
    rs = np.random.RandomState(82)
    randn = lambda *shape: torch.from_numpy(rs.randn(*shape).astype(np.float32)).to(dev)
    st = stats_tensors(dev)
    stats = [st[k] for k in ("anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")]
    W = [win[k] for k in POSE_KEYS]
    WY = pack_pose(*W[2:])
    Y, rp, rq, state = ops.decoder_window_forward(dec, W[0][:, 0], W[1][:, 0], WY[:, 0], win["gaze_pos"], 0.5 * randn(B, T, 64),
                                                  randn(B, T, 64), stats, st["dt"], save=True)
    assert state[0].engine == (1 if engine == "tc" else 0)
    cot = (randn(*Y.shape), randn(*rp.shape), randn(*rq.shape))
    grads, dSpeech, dStyle = ops.decoder_window_backward(dec, state, *cot)
    one = [*grads, dSpeech, dStyle]
    grads, dSpeech, dStyle, finish = ops.decoder_window_backward(dec, state, *cot, split=True)
    finish()
    two = [*grads, dSpeech, dStyle]
    torch.cuda.synchronize()
    assert float(one[0].abs().max()) > 0 and float(one[-1].abs().max()) > 0
    bad = [n for n, a, b in zip(ops._DEC_GRAD_NAMES + ["dSpeech", "dStyle"], one, two) if not torch.equal(a, b)]
    assert not bad, bad


# ---------------------------------------------------------------------------------------------- loudness normalisation + int16 decode (SURVEY 8f row 4)
def test_loudness_gain_and_normalised_features_vs_oracle(dev):
    """zeggs_loudness_gain (BS.1770 K-weighting + gating on the device) against oracle/loudness_oracle.py (restated pyloudnorm 0.1.0,
    parity unpinned): integrated loudness within 1e-3 LU, gain within 2e-4 relative; preprocess_audio(normalize_loudness=True) and
    int16 PCM input against the oracle chain (gain * wav -> mel), abs <= 3e-4 on the features."""
    from oracle import loudness_oracle as lo, mel_oracle
    from oracle.make_golden import audio_params
    from zeggs_b200 import audio, synth
    wav = synth.make_waveforms(4, 160000, seed=12)
    wav[1] *= 0.05                       # a quiet clip: gain > 1
    wav[2, 30000:110000] = 0.0           # a long silent stretch: blocks below the absolute gate
    wav[3] = np.clip(wav[3] * 3.0, -1, 1)
    meter = audio.LoudnessMeter(dev, 16000)
    gain, lufs = meter.gain(torch.from_numpy(wav).to(dev), want_lufs=True)
    for i in range(4):
        ref_l = lo.integrated_loudness(wav[i], 16000)
        ref_g = lo.loudness_gain(wav[i], 16000)
        print(f"  clip {i}: LUFS {float(lufs[i]):.5f} vs oracle {ref_l:.5f}; gain {float(gain[i]):.6f} vs {ref_g:.6f}")
        assert abs(float(lufs[i]) - ref_l) <= 1e-3
        assert abs(float(gain[i]) - ref_g) <= 2e-4 * ref_g
    # ragged length (27 gating blocks, last block clamped) through the drop-in surface, float and int16 input
    x = wav[0, :48123]
    n60 = int(round(60.0 * len(x) / 16000))
    p = audio_params(200); p.normalize_loudness = True
    ref = mel_oracle.preprocess_audio((lo.normalize_loudness(x, 16000)).astype(np.float64), 60, n60)
    got = audio.preprocess_audio(x, 60, n60, p, ["mel_spec", "energy"])
    err = float(np.abs(got - ref).max()); print(f"  normalised features max-abs err {err:.3e}")
    assert err <= 3e-4
    x16 = np.round(x * 32767.0).astype(np.int16)
    xf = (x16 / 32768.0).astype(np.float32)                                   # audio_files.py:211-236
    ref16 = mel_oracle.preprocess_audio((lo.normalize_loudness(xf, 16000)).astype(np.float64), 60, n60)
    got16 = audio.preprocess_audio(x16, 60, n60, p, ["mel_spec", "energy"])
    err = float(np.abs(got16 - ref16).max()); print(f"  int16 PCM normalised features max-abs err {err:.3e}")
    assert err <= 3e-4


# ---------------------------------------------------------------------------------------------- pose -> BVH channels (8f row 3) and generate_gesture end to end
def test_pose_to_bvh_channels_vs_reference_golden(dev, golden_dir):
    """zeggs_pose_to_bvh_channels against what the reference's generate.py:389-406 + utils.write_bvh hand to bvh.save
    (tests/golden/pose_post.npz): positions <= 2e-5 * max(1,|ref|), Euler angles <= 5e-3 degrees, local quaternions <= 1e-5."""
    from zeggs_b200 import ops
    g = np.load(os.path.join(golden_dir, "pose_post.npz"))
    t = lambda k: torch.from_numpy(g[k]).to(dev)
    pos, eul, lrot = ops.pose_to_bvh_channels(t("root_pos"), t("root_rot"), t("lpos"), t("ltxy"), want_lrot=True)
    for n in range(2):
        e, sc = report(f"bvh positions clip{n}", pos[n], torch.from_numpy(g[f"positions{n}"]))
        assert e <= 2e-5 * max(1.0, sc)
        e, _ = report(f"bvh euler deg clip{n}", eul[n], torch.from_numpy(g[f"rotations{n}"]))
        assert e <= 5e-3
        q_ref = torch.from_numpy(g[f"lrot{n}"])
        e, _ = report(f"lrot clip{n} (joints 1..)", lrot[n, :, 1:], q_ref[:, 1:])
        assert e <= 1e-5


@pytest.mark.parametrize("loud", [0, 1])
def test_generate_gesture_end_to_end_vs_reference_golden(dev, golden_dir, tmp_path, loud):
    """generate_gesture() -- the reference's call surface -- on the synthetic BVH + int16 WAV of tests/_fixtures.py against the BVH
    the UNMODIFIED reference wrote for the same files and weights (tests/golden/generate_e2e.npz, CPU run in the dev container):
    one example style, two styles blended 'add', two styles 'stitch'; with loudness normalisation off (pure reference arithmetic)
    and on (reference + oracle-backed pyloudnorm stub; that third-party step is parity-unpinned).  fp32 recurrence engine,
    240 free-running frames: BVH positions <= 1e-3 (absolute, cm), Euler angles <= 5e-3 degrees, style encodings <= 1e-4."""
    import json
    import shutil
    from pathlib import Path
    from tests import _fixtures as fx
    from zeggs_b200 import animation, generate, modules, synth
    g = np.load(os.path.join(golden_dir, "generate_e2e.npz"))
    H = int(g["H"])
    P = synth.make_params(H=H, seed=int(g["param_seed"]))
    net = tmp_path / "net"; net.mkdir()
    torch.save(_load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", "cpu"), net / "speech_encoder.pt")
    torch.save(_load(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), P, "style_encoder.", "cpu"), net / "style_encoder.pt")
    torch.save(_load(modules.Decoder(1134, 1131, 64, 64, H, 2), P, "decoder.", "cpu"), net / "decoder.pt")
    data = tmp_path / "data"; data.mkdir()
    stats = synth.load_stats()
    np.savez(data / "stats.npz", **{k: stats[k] for k in ("audio_input_mean", "audio_input_std", "anim_input_mean", "anim_input_std",
                                                         "anim_output_mean", "anim_output_std")})
    shutil.copy(os.path.join(fx.DATA, "data_definition_v1.json"), data / "data_definition.json")
    conf = json.load(open(os.path.join(fx.DATA, "data_pipeline_conf_v1.json")))
    conf["audio_conf"]["normalize_loudness"] = bool(loud)
    json.dump(conf, open(data / "data_pipeline_conf.json", "w"))
    bvh_path = Path(fx.make_synthetic_bvh(str(tmp_path / "style.bvh")))
    wav_path = Path(fx.make_wav(str(tmp_path / "speech.wav")))
    cases = dict(one=dict(styles=[(bvh_path, (10, 300))]),
                 add=dict(styles=[(bvh_path, (10, 300)), (bvh_path, (150, 400))], blend_type="add", blend_ratio=[0.25, 0.75]),
                 stitch=dict(styles=[(bvh_path, (10, 300)), (bvh_path, None)], blend_type="stitch", blend_ratio=[0.5, 0.5]))
    for name, kw in cases.items():
        res = tmp_path / f"res_{name}"
        enc = generate.generate_gesture(wav_path, network_path=net, data_path=data, results_path=res, style_encoding_type="example",
                                        file_name="out", first_pose=None, temperature=1e6, seed=1234, use_gpu=True, **kw)
        assert (res / "out.wav").exists()
        b = animation.load_bvh(str(res / "out.bvh"))
        tag = f"loud{loud}_{name}"
        e, sc = report(f"{tag} encoding", enc, torch.from_numpy(g[tag + "_encoding"]))
        assert tuple(enc.shape) == tuple(g[tag + "_encoding"].shape) and e <= 1e-4 * max(1.0, sc)
        e, sc = report(f"{tag} BVH positions", torch.from_numpy(b["positions"]), torch.from_numpy(g[tag + "_positions"]))
        assert e <= 1e-3
        e, _ = report(f"{tag} BVH euler degrees", torch.from_numpy(b["rotations"]), torch.from_numpy(g[tag + "_rotations"]))
        assert e <= 5e-3
    if not loud:
        enc = generate.generate_gesture(None, [(bvh_path, (10, 300))], net, data, None, temperature=1e6)
        e, sc = report("embedding-only call", enc, torch.from_numpy(g["embedding_only"]))
        assert tuple(enc.shape) == (1, 64) and e <= 1e-4 * max(1.0, sc)


# ---------------------------------------------------------------------------------------------- device-resident window supplier (8f row 2)
def _synthetic_processed_data(tmp_path):
    import json
    from zeggs_b200 import synth
    from zeggs_b200.data import KEYS
    st = synth.load_stats()
    rs = np.random.RandomState(3)
    N = 900
    data = {"X_audio_features": rs.randn(N, 81).astype(np.float32)}
    win = synth.make_pose_windows(1, N, seed=4)
    for k in KEYS:
        data["Y_" + k] = win[k][0]
    ranges = np.array([[0, 300], [300, 420], [420, 900]], dtype=np.int64)       # a short range exercises the clamping / tail repeat
    data.update(ranges_train=ranges, ranges_valid=ranges[:1], ranges_train_labels=np.array([0, 2, 1]), ranges_valid_labels=np.array([0]))
    for k in ("audio_input_mean", "audio_input_std", "anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std"):
        data[k] = st[k]
    np.savez(tmp_path / "processed_data.npz", **data)
    with open(tmp_path / "data_definition.json", "w") as f:
        json.dump(dict(bone_names=[f"b{i}" for i in range(75)], label_names=["Neutral", "Happy", "Sad"],
                       parents=[int(p) for p in st["parents"]], dt=float(st["dt"])), f)
    return tmp_path / "data_definition.json", tmp_path / "processed_data.npz"


@pytest.mark.parametrize("window,ex_len,style", [(64, 128, "example"), (100, 200, "example"), (64, 64, "example"), (64, 128, "label")])
def test_device_window_gather_is_bit_identical_to_host_supplier(dev, tmp_path, window, ex_len, style):
    """zeggs_window_gather (data in HBM, one launch per batch) against WindowDataset.sample_host_batch -- itself checked against the
    reference's SGDataset in tests/test_dataset_vs_reference.py -- for the same seed: every tensor of the batch bit-identical."""
    from zeggs_b200.data import DeviceWindowDataset, WindowDataset
    ddef, dproc = _synthetic_processed_data(tmp_path)
    host = WindowDataset(ddef, dproc, window, style, ex_len, seed=9)
    devd = DeviceWindowDataset(ddef, dproc, window, style, ex_len, seed=9, device=dev)
    for _ in range(3):
        hb = host.sample_host_batch(7)
        db = devd.sample_batch(7)
        torch.cuda.synchronize()
        assert set(hb) == set(db)
        for k in hb:
            assert tuple(hb[k].shape) == tuple(db[k].shape), k
            assert torch.equal(hb[k], db[k].cpu()), k


def test_two_fast_wgrad_contexts_do_not_share_state(dev):
    """The GEMM front end takes its scratch buffer and weight-gradient setting from the caller's zeggs_ctx: two GEMM mode 1 contexts
    that differ only in fast_wgrad, used alternately on two streams for a weight-gradient layout product (C = A[K,M]^T B[K,N]), give
    each its own numerics (split-bf16 ~fp32 vs one bf16 pass), with no library-global setter involved."""
    import ctypes as C
    from zeggs_b200 import _lib
    g = torch.Generator().manual_seed(3)
    M, N, K = 256, 384, 512
    A, B = torch.randn(K, M, generator=g).to(dev), torch.randn(K, N, generator=g).to(dev)
    ref = A.double().T @ B.double()
    bufs = [torch.empty(64 << 20, dtype=torch.uint8, device=dev) for _ in range(2)]
    ctxs = [_lib.Ctx(scratch=bufs[i].data_ptr(), scratch_bytes=bufs[i].numel(), gemm_mode=1, fast_wgrad=i) for i in (0, 1)]
    streams = [torch.cuda.Stream(dev), torch.cuda.Stream(dev)]
    outs = [torch.empty(M, N, device=dev) for _ in range(2)]
    torch.cuda.synchronize()
    for rep in range(3):
        for i in (0, 1):
            _lib.check(_lib.lib().zeggs_gemm_f32_ctx(C.addressof(ctxs[i]), 1, M, N, K, A.data_ptr(), M, B.data_ptr(), N, None, outs[i].data_ptr(), N,
                                                     0, 0, streams[i].cuda_stream), "zeggs_gemm_f32_ctx")
    torch.cuda.synchronize()
    e0 = float((outs[0].double() - ref).abs().max() / ref.abs().max())
    e1 = float((outs[1].double() - ref).abs().max() / ref.abs().max())
    print(f"  ctx0 (split-bf16, fast_wgrad 0) rel err {e0:.2e}; ctx1 (one bf16 pass, fast_wgrad 1) rel err {e1:.2e}")
    assert e0 <= 2e-5 and 1e-4 <= e1 <= 2e-2

