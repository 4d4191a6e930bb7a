"""TensorBoard logs of train() without a device: the hyper-parameter flattening against the reference's helpers.flatten_dict on its
shipped configs, TensorBoardLog read back from its event files (tags, sub-runs, steps, values bitwise, hparams), and the error a
missing tensorboard package gives."""
import json
import os
import sys

import numpy as np
import pytest

from oracle import ref_shim
from zeggs_b200 import _lib
from zeggs_b200.train import TERM_NAMES, TensorBoardLog, flatten_options

NET_OPT = dict(decoder=dict(nhidden=64, num_rnn_layers=2, rnn_cond="normal"), speech_encoder=dict(nhidden=64, speech_encoding_size=64),
               style_encoder=dict(nhidden=512, style_encoding_size=64, example_length=64, type="attn", use_vae=True))
TRAIN_OPT = dict(niterations=0.25, batchsize=4, learning_rate=1e-3, resume=False, seed=21, use_tensorboard=True, style_encoding_type="example")


def scalar_events(tb_dir):
    """{(run, tag): [(step, value), ...]} over every event file under tb_dir, duplicates kept, in file order; run is the
    sub-directory relative to tb_dir ("" for tb_dir itself)."""
    from tensorboard.backend.event_processing.event_file_loader import LegacyEventFileLoader
    out = {}
    for root, _, files in sorted(os.walk(tb_dir)):
        run = os.path.relpath(root, tb_dir)
        run = "" if run == "." else run
        for f in sorted(files):
            if ".tfevents." not in f:
                continue
            for ev in LegacyEventFileLoader(os.path.join(root, f)).Load():
                for v in ev.summary.value:
                    if v.HasField("simple_value"):
                        out.setdefault((run, v.tag), []).append((ev.step, v.simple_value))
    return out


def loss_series(tb_dir, prefix="losses"):
    """{TERM_NAMES entry: [(step, value), ...]} as TensorBoardLog lays out `prefix`: the total in tb_dir itself, each of the 18 terms
    in its own sub-run."""
    ev = scalar_events(tb_dir)
    out = {"total": ev.get(("", f"{prefix}/total_loss"), [])}
    for n in TERM_NAMES[1:]:
        out[n] = ev.get((f"{prefix}_losses_loss_{n}", f"{prefix}/losses"), [])
    return out


def hparams_of(tb_dir):
    """{name: value} of the hparams session-start record under tb_dir (exactly one expected)."""
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    from tensorboard.plugins.hparams import plugin_data_pb2
    found = []
    for root, _, files in os.walk(tb_dir):
        if not any(".tfevents." in f for f in files):
            continue
        ea = EventAccumulator(root)
        ea.Reload()
        try:
            contents = ea.PluginTagToContent("hparams").values()
        except KeyError:                   # a run without hparams data
            continue
        for content in contents:
            d = plugin_data_pb2.HParamsPluginData.FromString(content)
            if d.HasField("session_start_info"):
                found.append({k: v.WhichOneof("kind") and getattr(v, v.WhichOneof("kind")) for k, v in d.session_start_info.hparams.items()})
    assert len(found) == 1, found
    return found[0]


@pytest.mark.skipif(not ref_shim.available(), reason="needs the reference tree")
@pytest.mark.parametrize("config", ["configs_v1.json", "configs_v2.json"])
def test_hparams_flattening_matches_reference(config):
    ref_shim.install()
    import helpers                       # ZEGGS/helpers.py
    with open(os.path.join(ref_shim.REF_ROOT, "configs", config)) as f:
        cfg = json.load(f)
    want = helpers.flatten_dict(cfg["net_opt"])
    want.update(helpers.flatten_dict(cfg["train_opt"]))
    got = flatten_options(cfg["net_opt"])
    got.update(flatten_options(cfg["train_opt"]))
    assert got == want
    assert got["decoder_nhidden"] == 1024 and got["style_encoder_use_vae"] is True and got["use_tensorboard"] is True
    deep = dict(a=dict(b=dict(c=1, d=dict(e="x")), f=2.5), g=dict(), h=[1, 2])
    assert flatten_options(deep) == helpers.flatten_dict(deep) == {"a_b_c": 1, "a_b_d_e": "x", "a_f": 2.5, "h": [1, 2]}


def test_writer_round_trip(tmp_path):
    """Rows written in two blocks come back from the event files: the total under losses/total_loss, the 18 terms as the sub-runs
    losses_losses_loss_<name> with tag losses/losses, every step 0..n-1 exactly once, every value bitwise the row's float32."""
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    n = 23
    rs = np.random.RandomState(4)
    rows = (rs.randn(n, 19) * np.logspace(-6, 2, 19)).astype(np.float32)
    rows[3, 18] = 0.0                                  # the KL term without a VAE
    tb_dir = tmp_path / "tb"
    tb = TensorBoardLog(tb_dir, NET_OPT, TRAIN_OPT)
    tb.write("losses", np.arange(0, 10), rows[:10])
    tb.write("losses", np.arange(10, n), rows[10:])
    tb.write("valid", [20], rows[None, 5].astype(np.float64))
    tb.close()
    runs = sorted(d for d in os.listdir(tb_dir) if d.startswith("losses_losses_"))
    assert runs == sorted(f"losses_losses_loss_{k}" for k in TERM_NAMES[1:])
    ser = loss_series(str(tb_dir))
    for j, name in enumerate(TERM_NAMES):
        steps = [s for s, _ in ser[name]]
        assert sorted(steps) == list(range(n)), name
        for s, v in ser[name]:
            assert np.float32(v).tobytes() == rows[s, j].tobytes(), (name, s)
    val = loss_series(str(tb_dir), "valid")
    for j, name in enumerate(TERM_NAMES):
        assert [(s, np.float32(v)) for s, v in val[name]] == [(20, rows[5, j])], name
    ea = EventAccumulator(str(tb_dir))
    ea.Reload()
    assert "losses/total_loss" in ea.Tags()["scalars"]
    assert [e.step for e in ea.Scalars("losses/total_loss")] == list(range(n))
    ea = EventAccumulator(str(tb_dir / "losses_losses_loss_gaze"))
    ea.Reload()
    assert [np.float32(e.value) for e in ea.Scalars("losses/losses")] == list(rows[:, 17])
    h = hparams_of(str(tb_dir))
    want = flatten_options(NET_OPT)
    want.update(flatten_options(TRAIN_OPT))
    assert set(h) == set(want)
    assert h["decoder_nhidden"] == 64 and h["style_encoder_type"] == "attn"
    assert h["use_tensorboard"] == 1.0                 # add_hparams stores a bool as a number, as in the reference's run


def test_missing_tensorboard_is_an_error_before_any_work(monkeypatch, tmp_path):
    from zeggs_b200.train import train
    monkeypatch.setitem(sys.modules, "torch.utils.tensorboard", None)        # import of it raises ImportError
    opts = dict(TRAIN_OPT, use_gpu=True)
    with pytest.raises(_lib.ZeggsError, match="tensorboard"):
        train(tmp_path / "models", tmp_path / "logs", tmp_path / "missing.npz", tmp_path / "missing.json", opts, NET_OPT)
    assert not os.path.exists(tmp_path / "logs")
