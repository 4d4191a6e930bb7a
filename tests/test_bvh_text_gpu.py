"""BVH MOTION text on the device (csrc/bvh_text.cu) against the host code it stands in for: load_bvh arrays bit-identical to the host
parse (dtype included) on well-formed, unusual and malformed blocks, save_bvh bytes identical to the host writer, and the three callers
(generate_gesture, write_samples, data_pipeline) writing the same files with the device entry points as without them."""
import os
import shutil
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import _fixtures as fx
from tests._util import ensure_built

pytestmark = pytest.mark.gpu

KEYS = ("rotations", "positions", "offsets", "parents", "names", "order", "frametime")


@pytest.fixture(scope="module", autouse=True)
def built():
    ensure_built()


def _host_only(monkeypatch):
    from zeggs_b200 import animation, bvhio
    monkeypatch.setattr(animation, "_device_parse_available", lambda: False)
    monkeypatch.setattr(bvhio, "_format_motion_device", lambda *a, **k: None)


def _load_both(path, monkeypatch, expect_device=True):
    from zeggs_b200 import animation
    assert animation._device_parse_available()
    assert (animation._load_bvh_device(str(path)) is not None) == expect_device
    dev = animation.load_bvh(str(path))
    with monkeypatch.context() as m:
        _host_only(m)
        host = animation.load_bvh(str(path))
    return dev, host


def _assert_same(a, b):
    for k in KEYS:
        if isinstance(a[k], np.ndarray):
            assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k], equal_nan=True), k
            assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k           # -0.0 and NaN payloads too
        else:
            assert a[k] == b[k], k


def _rewrite_motion(src, dst, fn, header_fn=None):
    text = open(src).read()
    head, motion = text.split("Frame Time:", 1)
    ft, rows = motion.split("\n", 1)
    head = header_fn(head) if header_fn else head
    with open(dst, "wb") as f:
        f.write((head + "Frame Time:" + ft + "\n").encode("ascii") + fn(rows))


@pytest.fixture(scope="module")
def fixture_bvh(tmp_path_factory):
    return fx.make_synthetic_bvh(str(tmp_path_factory.mktemp("bvh") / "s.bvh"))


# ---------------------------------------------------------------------------------------------- parser
def test_fixture_and_150s_take_parse_bit_identical(fixture_bvh, tmp_path, monkeypatch):
    _assert_same(*_load_both(fixture_bvh, monkeypatch))
    long = fx.make_synthetic_bvh(str(tmp_path / "long.bvh"), frames=9000, seed=5)     # 150 s at 60 fps, 75 joints
    dev, host = _load_both(long, monkeypatch)
    assert dev["rotations"].shape == (9000, 75, 3)
    _assert_same(dev, host)


@pytest.mark.parametrize("variant", ["crlf", "cr", "tabs", "blank_lines", "more_rows", "fewer_rows", "signs_exponents"])
def test_unusual_layouts_parse_bit_identical(fixture_bvh, tmp_path, monkeypatch, variant):
    rows = open(fixture_bvh).read().split("Frame Time:", 1)[1].split("\n", 1)[1].split("\n")
    body = [r for r in rows if r.strip()]
    p = tmp_path / "v.bvh"
    if variant == "crlf":
        fn = lambda r: r.replace("\n", "\r\n").encode()
        _rewrite_motion(fixture_bvh, p, fn, header_fn=lambda h: h.replace("\n", "\r\n"))
    elif variant == "cr":
        _rewrite_motion(fixture_bvh, p, lambda r: r.replace("\n", "\r").encode())
    elif variant == "tabs":
        _rewrite_motion(fixture_bvh, p, lambda r: "\n".join("\t" + x.replace(" ", "\t \x0b", 7) + "\x0c" for x in body).encode())
    elif variant == "blank_lines":
        _rewrite_motion(fixture_bvh, p, lambda r: "\n\n  \t\n".join(body[:50]).encode() + b"\n \r\n\x1c\n" + "\n".join(body[50:]).encode())
    elif variant == "more_rows":
        _rewrite_motion(fixture_bvh, p, lambda r: "\n".join(body + body[:17]).encode())
    elif variant == "fewer_rows":
        _rewrite_motion(fixture_bvh, p, lambda r: "\n".join(body[:-33]).encode())
    else:
        rs = np.random.RandomState(3)
        def sgn(x):
            toks = x.split()
            out = [("+" + t if not t.startswith("-") and rs.rand() < 0.3 else t) for t in toks]
            out = [("%.5e" % float(t)) if rs.rand() < 0.2 else t for t in out]
            out = [("." + t[2:] if t.startswith("0.") else t) for t in out]
            return " ".join(out)
        _rewrite_motion(fixture_bvh, p, lambda r: "\n".join(sgn(x) for x in body).encode())
    dev, host = _load_both(p, monkeypatch)
    if variant == "more_rows":
        assert dev["rotations"].shape[0] == len(body)
    if variant == "fewer_rows":
        assert dev["rotations"].shape[0] == len(body) - 33
    _assert_same(dev, host)


def test_flagged_tokens_filled_on_the_host_and_overflow(tmp_path, monkeypatch):
    from zeggs_b200 import animation
    d = fx.skeleton()
    rs = np.random.RandomState(9)
    for frames, name in ((40, "some"), (600, "overflow")):       # most of 600 x 228 %.17g tokens are off the fast path
        src = fx.make_synthetic_bvh(str(tmp_path / f"{name}_src.bvh"), frames=frames)
        vals = rs.randn(frames, 228) * 10.0 ** rs.uniform(-6, 4, (frames, 228))
        if name == "some":
            vals[0, :6] = [np.nan, np.inf, -np.inf, 1e300, -0.0, 5e-324]
        def rows(_):
            out = []
            for t, v in enumerate(vals):
                toks = ["%.17g" % x if (name == "overflow" or (t * 228 + c) % 11 == 0) else "%f" % x for c, x in enumerate(v)]
                out.append(" ".join(toks))
            if name == "some":
                out[1] = out[1].replace(out[1].split()[3], "1_5", 1)
            return "\n".join(out).encode()
        p = tmp_path / f"{name}.bvh"
        _rewrite_motion(src, p, rows)
        assert len(d["parents"]) == 75
        dev, host = _load_both(p, monkeypatch, expect_device=(name == "some"))
        _assert_same(dev, host)
    assert animation.MAX_FLAGGED_TOKENS < 600 * 228 // 2


def test_wrong_token_count_raises_the_host_error(fixture_bvh, tmp_path, monkeypatch):
    from zeggs_b200 import animation
    p = tmp_path / "bad.bvh"
    _rewrite_motion(fixture_bvh, p, lambda r: r.replace("\n", " 1.0\n", 1).encode())
    with pytest.raises(Exception) as dev_err:
        animation.load_bvh(str(p))
    with monkeypatch.context() as m:
        _host_only(m)
        with pytest.raises(Exception) as host_err:
            animation.load_bvh(str(p))
    assert type(dev_err.value) is type(host_err.value) and str(dev_err.value) == str(host_err.value)
    q = tmp_path / "bad_token.bvh"
    _rewrite_motion(fixture_bvh, q, lambda r: r.replace(r.split()[0], "abc", 1).encode())          # same token count, not a number
    with pytest.raises(Exception) as dev_err:
        animation.load_bvh(str(q))
    with monkeypatch.context() as m:
        _host_only(m)
        with pytest.raises(Exception) as host_err:
            animation.load_bvh(str(q))
    assert type(dev_err.value) is type(host_err.value) and str(dev_err.value) == str(host_err.value)


def test_non_ascii_block_takes_the_host_path(fixture_bvh, tmp_path, monkeypatch):
    p = tmp_path / "nbsp.bvh"
    _rewrite_motion(fixture_bvh, p, lambda r: r.replace(" ", "\u00a0", 5).encode("utf-8"))       # NBSP: whitespace to str.split()
    dev, host = _load_both(p, monkeypatch, expect_device=False)
    _assert_same(dev, host)


# ---------------------------------------------------------------------------------------------- writer
def _save_both(tmp_path, pos, rot, parents, names=None, order="zyx", dt=1 / 60, offsets=None, tag="w"):
    from zeggs_b200 import bvhio
    a, b = tmp_path / f"{tag}_dev.bvh", tmp_path / f"{tag}_host.bvh"
    bvhio.save_bvh(str(a), torch.from_numpy(pos).cuda(), torch.from_numpy(rot).cuda(), parents, names, order, dt, offsets)
    bvhio.save_bvh(str(b), pos, rot, parents, names, order, dt, offsets)
    return a.read_bytes(), b.read_bytes()


def test_save_generated_60s_clip_byte_identical(tmp_path):
    from zeggs_b200 import ops, synth
    d = fx.skeleton()
    win = synth.make_pose_windows(1, 3600, seed=12)
    t = {k: torch.from_numpy(win[k]).cuda() for k in ("root_pos", "root_rot", "lpos", "ltxy")}
    pos, eul = ops.pose_to_bvh_channels(t["root_pos"], t["root_rot"], t["lpos"], t["ltxy"], (0.0, 0.0, 0.0), (1.0, 0.0, 0.0, 0.0))
    a, b = _save_both(tmp_path, pos[0].cpu().numpy(), eul[0].cpu().numpy(), d["parents"], d["bone_names"], dt=d["dt"])
    assert len(a) > 3600 * 228 * 8 and a == b


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_save_edge_values_byte_identical(tmp_path, dtype):
    d = fx.skeleton()
    rs = np.random.RandomState(4)
    T = 64
    pos = (rs.randn(T, 75, 3) * 10.0 ** rs.uniform(-8, 7, (T, 75, 3))).astype(dtype)
    rot = (rs.randn(T, 75, 3) * 180).astype(dtype)
    edges = [1 / 128, 3 / 128, -1 / 128, -0.0, -1e-9, np.nan, np.inf, -np.inf, 2.5e-6, 0.0, -5e-45, 1e-7]
    rot.reshape(-1)[:len(edges)] = edges
    pos[5:8, 0] = 3.4e32 if dtype == np.float64 else 3.0e38       # beyond the 128-bit path in float32, near its edge in float64
    pos[9, 0, 1] = 1e300 if dtype == np.float64 else 3.4e38
    a, b = _save_both(tmp_path, pos, rot, d["parents"], d["bone_names"], dt=d["dt"], tag=np.dtype(dtype).name)
    assert a == b


# ---------------------------------------------------------------------------------------------- callers
def test_data_pipeline_outputs_byte_identical(tmp_path, monkeypatch):
    from tests import _pipeline_inputs as pin
    from zeggs_b200.data_pipeline import data_pipeline
    g = pin.load_golden()
    pin.write_inputs(g, str(tmp_path))
    data_pipeline(pin.conf_for(str(tmp_path), "dev"), label_names=pin.data_definition(g)["label_names"])
    with monkeypatch.context() as m:
        _host_only(m)
        data_pipeline(pin.conf_for(str(tmp_path), "host"), label_names=pin.data_definition(g)["label_names"])
    seen = 0
    for d, _, fns in os.walk(tmp_path / "dev"):
        for fn in fns:
            if fn == "data_pipeline_conf.json":
                continue
            pa = os.path.join(d, fn)
            pb = os.path.join(str(tmp_path / "host"), os.path.relpath(pa, str(tmp_path / "dev")))
            if fn.endswith(".npz"):
                with np.load(pa) as x, np.load(pb) as y:
                    assert sorted(x.files) == sorted(y.files)
                    for k in x.files:
                        assert x[k].dtype == y[k].dtype and np.array_equal(x[k], y[k]), (fn, k)
            else:
                assert open(pa, "rb").read() == open(pb, "rb").read(), fn
            seen += fn.endswith(".bvh")
    assert seen > 0


def _generate_setup(tmp_path):
    import json
    from zeggs_b200 import modules, synth
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "generate_e2e.npz"))
    H = int(g["H"])
    P = synth.make_params(H=H, seed=int(g["param_seed"]))

    def load(mod, prefix):
        mod.load_state_dict({k[len(prefix):]: torch.from_numpy(v) for k, v in P.items() if k.startswith(prefix)})
        return mod

    net = tmp_path / "net"; net.mkdir()
    torch.save(load(modules.SpeechEncoder(81, 64, 64), "speech_encoder."), net / "speech_encoder.pt")
    torch.save(load(modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=True), "style_encoder."), net / "style_encoder.pt")
    torch.save(load(modules.Decoder(1134, 1131, 64, 64, H, 2), "decoder."), net / "decoder.pt")
    data = tmp_path / "data"; data.mkdir()
    stats = synth.load_stats()
    np.savez(data / "stats.npz", **{k: stats[k] for k in ("audio_input_mean", "audio_input_std", "anim_input_mean", "anim_input_std",
                                                         "anim_output_mean", "anim_output_std")})
    shutil.copy(os.path.join(fx.DATA, "data_definition_v1.json"), data / "data_definition.json")
    conf = json.load(open(os.path.join(fx.DATA, "data_pipeline_conf_v1.json")))
    conf["audio_conf"]["normalize_loudness"] = False
    json.dump(conf, open(data / "data_pipeline_conf.json", "w"))
    return net, data


def test_generate_gesture_output_byte_identical(tmp_path, monkeypatch):
    from zeggs_b200 import generate
    net, data = _generate_setup(tmp_path)
    bvh = Path(fx.make_synthetic_bvh(str(tmp_path / "style.bvh")))
    wav = Path(fx.make_wav(str(tmp_path / "speech.wav"), seconds=10.0))

    def run(res):
        enc = generate.generate_gesture(wav, [(bvh, (10, 300)), (bvh, None)], net, data, res, style_encoding_type="example",
                                        blend_type="stitch", blend_ratio=[0.5, 0.5], file_name="out", temperature=1e6, seed=1234,
                                        first_pose=bvh, use_gpu=True)
        return enc.cpu(), (res / "out.bvh").read_bytes()

    e_dev, b_dev = run(tmp_path / "dev")
    with monkeypatch.context() as m:
        _host_only(m)
        e_host, b_host = run(tmp_path / "host")
    assert torch.equal(e_dev, e_host)
    assert b_dev.count(b"\n") > 600 and b_dev == b_host


def test_write_samples_files_byte_identical(tmp_path, monkeypatch):
    """train()'s sample animations: every save_bvh call of write_samples gets CUDA tensors and writes the bytes the host writer
    writes for the same values."""
    import random
    from tests.test_validation_cpu import make_files
    from zeggs_b200 import bvhio
    from zeggs_b200.train import train
    real, calls = bvhio.save_bvh, []

    def spy(filename, positions, rotations_deg, *args, **kw):
        assert positions.is_cuda and rotations_deg.is_cuda
        real(filename, positions, rotations_deg, *args, **kw)
        ref = str(filename) + ".host"
        real(ref, positions.cpu().numpy(), rotations_deg.cpu().numpy(), *args, **kw)
        calls.append((open(filename, "rb").read(), open(ref, "rb").read()))

    monkeypatch.setattr(bvhio, "save_bvh", spy)
    ddef, dproc = make_files(str(tmp_path / "data"))
    to = dict(seed=21, use_gpu=True, resume=False, learning_rate=1e-3, learning_rate_decay=0.999, eps=1e-5, niterations=2 / 1000.0,
              batchsize=4, window=64, style_encoding_type="example", generate_samples_step=1, use_tensorboard=False,
              decoder_engine="fp32", cuda_graph=False, device_dataset=True)
    no = dict(speech_encoder=dict(nhidden=64, speech_encoding_size=64),
              style_encoder=dict(nhidden=512, style_encoding_size=64, example_length=64, type="attn", use_vae=True),
              decoder=dict(nhidden=64))
    state = random.getstate()
    random.seed(0)
    try:
        train(str(tmp_path / "models"), str(tmp_path / "logs"), dproc, ddef, to, no)
    finally:
        random.setstate(state)
    assert len(calls) >= 6
    for a, b in calls:
        assert a == b
