"""Training monitoring on the GPU: TrainStep.evaluate (forward-only loss on held-out windows) against the CPU oracle and free of
side effects, the device validation batches against the host supplier, and train() end to end writing per-iteration snapshots,
sample animations and the validation-loss log without changing the training trajectory."""
import json
import os
import random

import numpy as np
import pytest
import torch

from tests._util import ensure_built, tt
from tests.test_validation_cpu import RANGES_TRAIN, RANGES_VALID, make_files

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


@pytest.fixture
def decoder_engine(dev):
    from zeggs_b200 import ops
    prev = ops.DECODER_ENGINE
    yield ops.set_decoder_engine
    ops.set_decoder_engine(prev)


def _load(mod, P, prefix, dev):
    mod.load_state_dict({k[len(prefix):]: torch.from_numpy(v) for k, v in P.items() if k.startswith(prefix)})
    return mod.to(dev)


def _make_step(dev, H, style, seed=5, use_graph=False):
    from zeggs_b200 import modules, synth
    from zeggs_b200.train import TrainStep
    Z = 64 if style == "example" else 3
    P = synth.make_params(H=H, Z=Z, seed=seed, with_style=(style == "example"))
    se = _load(modules.SpeechEncoder(81, 64, 64), P, "speech_encoder.", dev)
    st = _load(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), P, "style_encoder.", dev) if style == "example" else None
    de = _load(modules.Decoder(1134, 1131, 64, Z, H, 2), P, "decoder.", dev)
    stats = synth.load_stats()
    return TrainStep(se, de, st, stats, stats["parents"], float(stats["dt"]), lr=1e-3, use_graph=use_graph, eval_seed=9), P


def _batch(dev, B, T, T_ex, seed, style="example"):
    from zeggs_b200 import synth
    b = tt(synth.make_pose_windows(B, T, seed=seed), dev)
    b["audio"] = torch.from_numpy(synth.make_audio_features(B, T, seed=seed)).to(dev)
    if style == "example":
        b["style"] = torch.from_numpy(synth.make_style_example(B, T_ex, seed=seed)).to(dev)
    else:
        lab = torch.zeros(B, 3)
        lab[torch.arange(B), torch.arange(B) % 3] = 1.0
        b["style"] = lab.to(dev)
    return b


@pytest.mark.parametrize("style", ["example", "label"])
@pytest.mark.parametrize("engine,H", [("fp32", 64), ("tc", 384)])
def test_evaluate_vs_oracle_loss(dev, decoder_engine, engine, H, style):
    """evaluate() against OracleTrainer.loss (eval mode, same injected VAE noise, same kl_weight(iteration)): the total and the 18
    terms within the tolerances of the whole-step loss in test_gpu_parity.py (split-bf16 GEMMs; bf16 recurrence operands on tc)."""
    from oracle.train_oracle import OracleTrainer
    from zeggs_b200 import synth
    decoder_engine(engine)
    step, P = _make_step(dev, H, style)
    step.iteration = 7000                     # kl_weight(7000) = 0.076: below the 0.2 clip
    batch = _batch(dev, 4, 16, 24, 31, style)
    eps = torch.from_numpy(np.random.RandomState(2).randn(4, 64).astype(np.float32))
    terms = step.evaluate(batch, eps=eps.to(dev) if style == "example" else None).cpu().numpy()
    if engine == "tc":
        assert step.dec.__dict__.get("_zeggs_packed_tc") is not None, "the tensor-core engine did not run"
    oracle = OracleTrainer(P, synth.load_stats(), label_style=(style == "label"))
    oracle.it = step.iteration
    with torch.no_grad():
        loss, ref = oracle.loss({k: v.cpu() for k, v in batch.items()}, eps_vae=eps if style == "example" else None)
    loss = float(loss)
    names = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "lrot", "lvel", "lvrt", "cpos", "crot", "cvel", "cvrt",
             "ldvl", "ldvt", "cdvl", "cdvt", "gaze", "kl_div"]
    ref_terms = [float(ref.get(n, 0.0)) for n in names]              # no KL term without a style encoder
    print(f"  [{engine} {style}] total {terms[0]:.6f} vs oracle {loss:.6f}")
    tol_total, tol_term = (2e-4, 5e-4) if engine == "fp32" else (5e-3, 3e-2)
    assert abs(terms[0] - loss) <= tol_total * abs(loss)
    for i, (n, r) in enumerate(zip(names, ref_terms)):
        assert abs(terms[1 + i] - r) <= tol_term * max(1e-3, abs(r)), (n, terms[1 + i], r)
    if style == "label":
        assert terms[18] == 0.0


def _snapshot(step):
    o, dev = step.optimizer, step.dev
    return dict(grad=o.flat_grad.clone(), param=o.flat_param.clone(), m=o.exp_avg.clone(), v=o.exp_avg_sq.clone(),
                step_dev=o.step_dev.clone(), hyper=o.hyper.clone(), _step=o._step, it=step.iteration, terms=step.terms.clone(),
                seed=step.seed.t.clone() if step.seed is not None else None, cpu=torch.get_rng_state(), cuda=torch.cuda.get_rng_state(dev),
                np=np.random.get_state()[1].copy(), py=random.getstate())


def _same(a, b):
    for k in a:
        x, y = a[k], b[k]
        if isinstance(x, torch.Tensor):
            assert torch.equal(x, y), k
        elif isinstance(x, np.ndarray):
            assert np.array_equal(x, y), k
        else:
            assert x == y, k


@pytest.mark.parametrize("engine,H", [("fp32", 64), ("tc", 384)])
def test_evaluate_is_side_effect_free(dev, decoder_engine, engine, H):
    """evaluate() between training steps: optimizer buffers, iteration, the step's loss vector, the dropout DeviceSeed and every
    global generator bitwise unchanged; two calls give bitwise-equal terms; an eager step and graph-replayed steps taken after it
    give losses and parameters bitwise equal to the same steps without it."""
    decoder_engine(engine)
    vb = _batch(dev, 4, 16, 24, 90)
    runs = {}
    for with_eval in (True, False):
        torch.manual_seed(11)
        step, _ = _make_step(dev, H, "example", seed=6, use_graph=True)
        losses = []
        for it in range(6):
            if with_eval and it in (2, 3, 5):
                before = _snapshot(step)
                t1 = step.evaluate(vb)
                t2 = step.evaluate(vb)
                torch.cuda.synchronize()
                assert torch.equal(t1, t2)
                assert bool(torch.isfinite(t1).all())
                _same(before, _snapshot(step))
            b = _batch(dev, 4, 16, 24, 60 + it)
            if it == 4:                                               # an eager step (injected VAE noise) after evaluate()
                eps = torch.from_numpy(np.random.RandomState(it).randn(4, 64).astype(np.float32)).to(dev)
                losses.append(float(step.step(b, eps=eps).item()))
            else:
                losses.append(float(step.step(b).item()))
        torch.cuda.synchronize()
        assert step.use_graph and len(step._graphs) == 1, "the CUDA-graph path did not run"
        runs[with_eval] = (losses, step.optimizer.flat_param.clone())
        del step
    print("  with evaluate   ", runs[True][0]); print("  without evaluate", runs[False][0])
    assert runs[True][0] == runs[False][0]
    assert torch.equal(runs[True][1], runs[False][1])


def test_evaluate_sees_the_weights_a_replay_wrote(dev, decoder_engine):
    """After graph-replayed steps, evaluate() runs on the updated parameters: equal to a fresh TrainStep built on a copy of them."""
    decoder_engine("tc")
    torch.manual_seed(12)
    step, P = _make_step(dev, 384, "example", seed=7, use_graph=True)
    vb = _batch(dev, 4, 16, 24, 91)
    t0 = step.evaluate(vb).clone()
    for it in range(4):
        step.step(_batch(dev, 4, 16, 24, 40 + it))
    t1 = step.evaluate(vb)
    fresh, _ = _make_step(dev, 384, "example", seed=7)
    fresh.optimizer.flat_param.copy_(step.optimizer.flat_param)
    fresh.iteration = step.iteration
    t2 = fresh.evaluate(vb)
    torch.cuda.synchronize()
    assert len(step._graphs) == 1
    assert not torch.equal(t0, t1)
    assert torch.equal(t1, t2)


@pytest.mark.parametrize("style", ["example", "label"])
def test_device_validation_batches_match_host_supplier(dev, tmp_path, style):
    from zeggs_b200.data import DeviceWindowDataset, WindowDataset
    ddef, dproc = make_files(str(tmp_path))
    host = WindowDataset(ddef, dproc, 64, style, 128, seed=3)
    devd = DeviceWindowDataset(ddef, dproc, 64, style, 128, seed=3, device=dev)
    devd.example_window_length = host.example_window_length = 100   # the per-iteration length does not reach validation
    assert np.array_equal(host.valid_starts, devd.valid_starts) and len(host.valid_starts) >= 5
    state = devd.rs.get_state()[1].copy()
    for idx in (np.arange(0, 4), np.arange(4, len(host.valid_starts)), np.array([len(host.valid_starts) - 1, 0])):
        hb, db = host.valid_host_batch(idx), devd.valid_batch(idx)
        torch.cuda.synchronize()
        assert set(hb) == set(db)
        for k in hb:
            assert tuple(hb[k].shape) == tuple(db[k].shape), k
            assert torch.equal(hb[k], db[k].cpu()), k
    assert np.array_equal(state, devd.rs.get_state()[1])


# ---------------------------------------------------------------------------------------------- train() end to end
def _options(seed, gss, niter_total):
    train_options = dict(seed=seed, use_gpu=True, resume=False, learning_rate=1e-3, learning_rate_decay=0.999, eps=1e-5,
                         niterations=niter_total / 1000.0, batchsize=4, window=64, style_encoding_type="example",
                         generate_samples_step=gss, use_tensorboard=False, decoder_engine="fp32", cuda_graph=True, device_dataset=True)
    network_options = dict(speech_encoder=dict(nhidden=64, speech_encoding_size=64),
                           style_encoder=dict(nhidden=512, style_encoding_size=64, example_length=64, type="attn", use_vae=True),
                           decoder=dict(nhidden=64))
    return train_options, network_options


def _run_train(base, ddef, dproc, gss, n):
    from zeggs_b200.train import train
    models, logs = os.path.join(base, "models"), os.path.join(base, "logs")
    to, no = _options(21, gss, n)
    state = random.getstate()
    random.seed(0)            # train() draws the per-iteration example length from Python's generator, unseeded (train.py:228-229)
    try:
        train(models, logs, dproc, ddef, to, no)
    finally:
        random.setstate(state)
    return models, logs


def _final_params(models):
    from zeggs_b200.generate import load_networks
    nets = load_networks(models, "cpu")
    return {f"{n}.{k}": v for n, m in nets.items() for k, v in m.state_dict().items()}


def _expected_samples(seed, its, n_train, n_valid, Z=64):
    """(iteration, split, i, range index) in the order train() draws them from RandomState(seed)."""
    rs, out = np.random.RandomState(seed), []
    for it in its:
        for split, n in (("train", n_train), ("valid", n_valid)):
            if n == 0:
                continue
            for i in range(3):
                out.append((it, split, i, int(rs.randint(n))))
                rs.randn(1, Z)
    return out


def _oracle_channels(raw, s, e):
    from oracle import pose_oracle as po
    rp, rq, lp, xy = raw["Y_root_pos"][s:e], raw["Y_root_rot"][s:e], raw["Y_lpos"][s:e], raw["Y_ltxy"][s:e]
    lrot = po.quat_from_xform(po.orthogonalize_from_xy(xy))
    pos, rot = lp.copy(), lrot.copy()
    pos[:, 0] = po.quat_mul_vec(rq, lp[:, 0]) + rp
    rot[:, 0] = po.quat_mul(rq, lrot[:, 0])
    return pos, np.degrees(po.to_euler_zyx(rot))


def test_train_writes_snapshots_samples_and_validation_log(dev, tmp_path, decoder_engine):
    from zeggs_b200 import animation
    from zeggs_b200.generate import load_networks
    ddef, dproc = make_files(str(tmp_path / "data"))
    raw = dict(np.load(dproc))
    labels = json.load(open(ddef))["label_names"]
    n_it = 6
    models, logs = _run_train(str(tmp_path / "a"), ddef, dproc, 2, n_it)
    its = [2, 4, 6]
    for it in its:
        d = os.path.join(models, str(it))
        assert sorted(os.listdir(d)) == ["checkpoints.pt", "decoder.pt", "speech_encoder.pt", "style_encoder.pt"]
        nets = load_networks(d, dev)
        assert set(nets) == {"speech_encoder", "decoder", "style_encoder"}
        assert torch.load(os.path.join(d, "checkpoints.pt"), weights_only=False)["iteration"] == it
    samples = os.path.join(logs, "samples")
    files = sorted(os.listdir(samples))
    assert len(files) == 12 * len(its)
    for it, split, i, ri in _expected_samples(21, its, len(RANGES_TRAIN), len(RANGES_VALID)):
        ranges = RANGES_TRAIN if split == "train" else RANGES_VALID
        lab = labels[int(raw[f"ranges_{split}_labels"][ri])]
        s, e = ranges[ri][0], min(ranges[ri][0] + 1800, ranges[ri][1])
        for kind in ("ground", "predict"):
            name = f"iteration_{it}_{split}_{kind}_{i}_{lab}.bvh"
            assert name in files, name
            a = animation.load_bvh(os.path.join(samples, name))
            assert a["rotations"].shape == (e - s, 75, 3) and a["order"] == "zyx"
            assert np.all(np.isfinite(a["rotations"])) and np.all(np.isfinite(a["positions"]))
            if kind == "ground":
                pos, eul = _oracle_channels(raw, s, e)
                assert np.abs(a["positions"][:, 0] - pos[:, 0]).max() <= 1e-3 * max(1.0, np.abs(pos[:, 0]).max())
                assert np.allclose(a["offsets"][1:], pos[0, 1:], atol=1e-5 * max(1.0, np.abs(pos).max()))
                qa = animation.q_from_euler_deg(a["rotations"].astype(np.float64), "zyx")
                qo = animation.q_from_euler_deg(eul.astype(np.float64), "zyx")
                assert (1.0 - np.abs((qa * qo).sum(-1))).max() <= 1e-6
    lines = open(os.path.join(logs, "valid_loss.jsonl")).read().strip().split("\n")
    assert len(lines) == len(its)
    for it, ln in zip(its, lines):
        rec = json.loads(ln)
        assert rec["iteration"] == it and rec["windows"] > 0 and np.isfinite(rec["train_loss"])
        assert len(rec["valid"]) == 19 and all(np.isfinite(v) for v in rec["valid"].values())
    # the monitoring does not touch the training trajectory
    models_b, _ = _run_train(str(tmp_path / "b"), ddef, dproc, 10 ** 6, n_it)
    pa, pb = _final_params(models), _final_params(models_b)
    assert set(pa) == set(pb)
    for k in pa:
        assert torch.equal(pa[k], pb[k]), k


def test_train_without_validation_split_writes_training_samples_only(dev, tmp_path, decoder_engine):
    ddef, dproc = make_files(str(tmp_path / "data"), with_valid=False)
    models, logs = _run_train(str(tmp_path / "a"), ddef, dproc, 2, 2)
    files = sorted(os.listdir(os.path.join(logs, "samples")))
    assert len(files) == 6 and all("_train_" in f for f in files)
    assert not os.path.exists(os.path.join(logs, "valid_loss.jsonl"))
    assert sorted(os.listdir(os.path.join(models, "2"))) == ["checkpoints.pt", "decoder.pt", "speech_encoder.pt", "style_encoder.pt"]
