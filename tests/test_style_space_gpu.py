"""GPU: the style embedding space.  zeggs_embedding_moments (csrc/style_space.cu) against float64 on the host, and
zeggs_b200.style_space.build() on a dataset made by the data pipeline from synthetic 75-joint takes, against the float64 style
oracle (oracle/style_oracle.py).

* Moments: N in {1, 2, 31, 32, 33, 255, 256, 257, 4097} x Z in {1, 9, 64, 128, 512} x G in {1, 19}, and N = 1 000 003 at
  Z in {1, 9, 64}; rows with a common offset of 1e3 and a spread of 1e-3; with G = 19 group 1 has no rows (count 0, sum 0).
  Bounds: tests/test_style_space_cpu.py (float64 summation error; the restated kernel meets them with >= 4x headroom there).
  Two calls give the same bits.
* build(): attn with the VAE, attn without it, gru with the VAE (GEMM mode 0): every embedding row within 2e-5 * max(1, |ref|) of
  the float64 oracle on its window; centroids, mean and covariance within the moment bounds of float64 numpy over the returned
  embeddings; two builds save identical bytes; a label with no windows has no centroid.
* The command line writes the space, and a vector from it drives generate_gesture to a BVH.
* The shipped v1 network (oracle/_ref/, skipped when build() could not derive it): generate_gesture given space.embedding(...)
  writes the same BVH as given that vector directly, and returns it as the style encoding.
* A checkpoint without a style encoder (the label-based model) is refused before any launch.
"""
import json
import os

import numpy as np
import pytest
import torch

from tests._util import ensure_built
from tests.test_style_space_cpu import moment_bounds, moment_case

pytestmark = pytest.mark.gpu

FWD_TOL = 2e-5
LABELS = ["Neutral", "Happy", "Sad"]
L_TEST = 64


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


def _check_moments(X, g, G, dev, tag):
    from zeggs_b200 import ops
    Xd, gd = torch.from_numpy(X).to(dev), torch.from_numpy(g).to(dev)
    out1 = ops.embedding_moments(Xd, gd, G)
    out2 = ops.embedding_moments(Xd, gd, G)
    for a, b in zip(out1, out2):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes(), f"{tag}: two calls differ"      # bits, NaN included
    mean, cov, gsum, cnt = (t.cpu().numpy() for t in out1)
    X64 = X.astype(np.float64)
    N = X.shape[0]
    rm = X64.mean(0)
    bm, bc, bcen = moment_bounds(X, g, G, rm)
    rat = [float(np.max(np.abs(mean - rm) / bm))]
    assert np.array_equal(cnt, np.bincount(g, minlength=G))
    if N > 1:
        d = X64 - rm
        rc = (d.T @ d) / (N - 1)
        rat.append(float(np.max(np.abs(cov - rc) / bc)))
        assert np.array_equal(cov, cov.T)
    else:
        assert np.all(np.isnan(cov))          # 0 / 0, as numpy.cov with one row
    for k in range(G):
        if cnt[k]:
            rat.append(float(np.max(np.abs(gsum[k] / cnt[k] - X64[g == k].mean(0)) / bcen[k])))
        else:
            assert not gsum[k].any()
    print(f"STYLE_SPACE_MOMENTS {tag} worst ratio to bound {max(rat):.3e}")
    assert max(rat) <= 1.0, (tag, rat)
    return max(rat)


MOMENT_CASES = [(N, Z, G) for N in (1, 2, 31, 32, 33, 255, 256, 257, 4097) for Z in (1, 9, 64, 128, 512) for G in (1, 19)]
MOMENT_CASES += [(1_000_003, Z, 19) for Z in (1, 9, 64)]


@pytest.mark.parametrize("N,Z,G", MOMENT_CASES)
def test_embedding_moments_match_float64(dev, N, Z, G):
    X, g = moment_case(N, Z, G)
    if G > 1 and N >= 2:
        assert not np.any(g == 1)
    _check_moments(X, g, G, dev, f"N={N} Z={Z} G={G}")


@pytest.mark.parametrize("N,Z", [(257, 9), (4097, 64), (1_000_003, 9)])
def test_embedding_moments_large_common_offset(dev, N, Z):
    X, g = moment_case(N, Z, 19, seed=5, offset=1e3, spread=1e-3)
    _check_moments(X, g, 19, dev, f"offset N={N} Z={Z}")


def test_embedding_moments_refusals(dev):
    from zeggs_b200 import _lib, ops
    l = _lib.lib()
    assert l.zeggs_embedding_moments_workspace_size(0, 9, 1) == 0
    assert l.zeggs_embedding_moments_workspace_size(5, 0, 1) == 0
    assert l.zeggs_embedding_moments_workspace_size(5, 9, 129) == 0
    assert l.zeggs_embedding_moments_workspace_size(5, 9, 128) > 0
    X = torch.zeros((5, 9), device=dev)
    n0 = l.zeggs_launch_count()
    with pytest.raises(_lib.ZeggsError, match=r"G = 129 groups \(1\.\.128\)"):
        ops.embedding_moments(X, torch.zeros(5, dtype=torch.int32, device=dev), 129)
    with pytest.raises(_lib.ZeggsError, match="group ids"):
        ops.embedding_moments(X, torch.full((5,), 3, dtype=torch.int32, device=dev), 3)
    with pytest.raises(_lib.ZeggsError, match="N = 0 rows"):
        ops.embedding_moments(X[:0], torch.zeros(0, dtype=torch.int32, device=dev), 1)
    assert l.zeggs_launch_count() == n0


# ------------------------------------------------------------------ build() on a pipeline-built dataset

@pytest.fixture(scope="module")
def dataset(dev, tmp_path_factory):
    """Four synthetic 75-joint takes through the data pipeline: Neutral, Happy, Neutral for training, Sad held out (so Sad has no
    training windows)."""
    from tests import _fixtures as fx
    from tests import _pipeline_inputs as pin
    from zeggs_b200.data_pipeline import data_pipeline
    base = tmp_path_factory.mktemp("style_space_set")
    (base / "original").mkdir()
    rows = []
    for k, style in enumerate(["Neutral", "Happy", "Neutral", "Sad"]):
        fx.make_synthetic_bvh(str(base / "original" / f"t{k}.bvh"), frames=420, seed=60 + k)
        fx.make_wav(str(base / "original" / f"t{k}.wav"), seconds=7.0, seed=70 + k)
        (base / "original" / f"t{k}.csv").write_text("#,Name,Start,End\nR1,S,0:00.000,0:06.900\n")
        rows.append(f"t{k}.wav,10:00:00:00,,,,t{k}.fbx,10:00:00:00,,,,{style},1,10:00:00:10,10:00:06:50,t{k}.bvh,{'TRUE' if k == 3 else 'FALSE'}")
    cols = "audio_filename,audio_start_time,audio_end_time,audio_duration,audio_clap_time,anim_fbx_file,anim_start_time,anim_end_time," \
           "anim_duration,anim_clap_time,style,capture_session,acting_start_time,acting_end_time,anim_bvh,validation"
    (base / "info.csv").write_text(cols + "\n" + "\n".join(rows) + "\n")
    data_pipeline(pin.conf_for(str(base)), label_names=LABELS)
    return base


def _nets(base, name, type, vae):
    """Freshly initialised whole-module pickles of the three networks (style hidden 64, Z = 64), as train() saves them."""
    from zeggs_b200 import modules
    d = base / name
    d.mkdir(parents=True, exist_ok=True)
    torch.manual_seed(sum(name.encode()))
    torch.save(modules.SpeechEncoder(81, 64, 64), d / "speech_encoder.pt")
    torch.save(modules.Decoder(1134, 1131, 64, 64, 64, 2), d / "decoder.pt")
    torch.save(modules.StyleEncoder(1134, 64, 64, type=type, use_vae=vae), d / "style_encoder.pt")
    return d


@pytest.fixture
def gemm_mode0():
    from zeggs_b200 import ops
    ops.set_gemm_mode(0)
    yield
    ops.set_gemm_mode(1)


def _oracle_embeddings(space, net_dir, data_dir, type, vae):
    """Each window's example built on the host (WindowDataset._example_vec), normalised in float32 with stats.npz, through the float64
    oracle -> [N, Z]."""
    from oracle import style_oracle
    from zeggs_b200 import data
    enc = torch.load(net_dir / "style_encoder.pt", map_location="cpu", weights_only=False)
    P = {"style_encoder." + k: v.double() for k, v in enc.state_dict().items()}
    ds = data.WindowDataset(str(data_dir / "data_definition.json"), str(data_dir / "processed_data.npz"), L_TEST, "example", L_TEST)
    st = np.load(data_dir / "stats.npz")
    m, s = torch.as_tensor(st["anim_input_mean"], dtype=torch.float32), torch.as_tensor(st["anim_input_std"], dtype=torch.float32)
    x = torch.stack([(ds._example_vec(int(w), int(w) + L_TEST, L_TEST) - m) / s for w in space.window_start])
    with torch.no_grad():
        z, mu, _ = style_oracle.style_encoder(P, x.double(), use_vae=vae, type=type)
    return (mu if vae else z).numpy()


@pytest.mark.parametrize("type,vae", [("attn", True), ("attn", False), ("gru", True)])
def test_build_matches_float64_oracle(dev, dataset, tmp_path, gemm_mode0, type, vae):
    from zeggs_b200 import _lib, data, style_space
    net = _nets(tmp_path, f"{type}_{vae}", type, vae)
    ddir = dataset / "processed"
    space = style_space.build(net, ddir, example_length=L_TEST, batch=7, device=dev)
    ds = data.WindowDataset(str(ddir / "data_definition.json"), str(ddir / "processed_data.npz"), L_TEST, "example", L_TEST)
    starts, ri, lab = style_space.example_windows(ds.ranges, ds.labels, L_TEST)
    assert np.array_equal(space.window_start, starts) and np.array_equal(space.range_index, ri) and np.array_equal(space.labels, lab)
    N = len(starts)
    assert N >= 8 and space.embeddings.shape == (N, 64) and space.embeddings.dtype == np.float32
    ref = _oracle_embeddings(space, net, ddir, type, vae)
    err = np.abs(space.embeddings - ref).max(1) / np.maximum(1.0, np.abs(ref).max(1))
    print(f"STYLE_SPACE_BUILD {type} vae={vae} N={N} worst row error {err.max():.3e}")
    assert err.max() <= FWD_TOL
    # the statistics against float64 numpy over the returned embeddings
    E = space.embeddings.astype(np.float64)
    rm = E.mean(0)
    bm, bc, bcen = moment_bounds(space.embeddings, space.labels, len(LABELS), rm)
    assert np.all(np.abs(space.mean - rm) <= bm)
    assert np.all(np.abs(space.cov - np.cov(E, rowvar=False)) <= bc)
    assert space.counts == {n: int(np.count_nonzero(space.labels == i)) for i, n in enumerate(LABELS)}
    assert space.counts["Sad"] == 0 and set(space.centroids) == {"Neutral", "Happy"}
    for i, n in enumerate(LABELS[:2]):
        assert np.all(np.abs(space.centroids[n] - E[space.labels == i].mean(0)) <= bcen[i])
    with pytest.raises(_lib.ZeggsError, match="no windows"):
        space.embedding("Sad")
    assert np.allclose(space.components @ np.diag(space.variances) @ space.components.T, space.cov, atol=1e-12 * np.abs(space.cov).max())


def test_two_builds_save_identical_bytes(dev, dataset, tmp_path):
    from zeggs_b200 import style_space
    net = _nets(tmp_path, "attn_twice", "attn", True)
    for name in ("a.npz", "b.npz"):
        style_space.build(net, dataset / "processed", splits=("train", "valid"), example_length=L_TEST, device=dev).save(tmp_path / name)
    assert (tmp_path / "a.npz").read_bytes() == (tmp_path / "b.npz").read_bytes()
    assert style_space.load(tmp_path / "a.npz").counts["Sad"] > 0


def test_command_line_writes_a_space_that_drives_generation(dev, dataset, tmp_path, capsys):
    from tests import _fixtures as fx
    from zeggs_b200 import generate, style_space
    out = tmp_path / "run"
    net = _nets(out, "saved_models", "attn", True)
    opts = {"paths": {"base_path": str(dataset), "path_processed_data": "processed", "output_dir": str(out), "models_dir": None},
            "net_opt": {"style_encoder": {"example_length": L_TEST}}}
    (out / "options.json").write_text(json.dumps(opts))
    style_space.main(["-o", str(out / "options.json"), "--out", str(tmp_path / "style_space.npz")])
    table = capsys.readouterr().out
    assert "Neutral" in table and "Sad" in table and "total" in table
    space = style_space.load(tmp_path / "style_space.npz")
    assert space.example_length == L_TEST and space.network_path == str(net)
    wav = fx.make_wav(str(tmp_path / "speech.wav"), seconds=2.0, seed=81)
    bvh = dataset / "original" / "t0.bvh"
    res = tmp_path / "res"
    generate.generate_gesture(wav, [(space.embedding("Happy"), "happy")], net, dataset / "processed", res, first_pose=str(bvh),
                              file_name="happy")
    assert (res / "happy.bvh").stat().st_size > 0


def test_v1_network_generates_from_a_space_vector(dev, dataset, tmp_path):
    from oracle import ref_data
    from tests import _fixtures as fx
    from zeggs_b200 import generate, style_space
    v1 = ref_data.saved_models_dir()
    if not os.path.exists(os.path.join(v1, "style_encoder.pt")):
        pytest.skip("the shipped v1 network was not derived into oracle/_ref/ by build()")
    space = style_space.build(v1, dataset / "processed", device=dev)
    assert space.example_length == 256 and space.Z == 64 and len(space.labels) >= 2
    vec = space.embedding("Happy", {0: 1.5})
    wav = fx.make_wav(str(tmp_path / "speech.wav"), seconds=2.0, seed=82)
    bvh = str(dataset / "original" / "t1.bvh")
    a = generate.generate_gesture(wav, [(vec, "x")], v1, dataset / "processed", tmp_path / "a", first_pose=bvh, file_name="x")
    b = generate.generate_gesture(wav, [(np.array(vec.tolist(), np.float32), "x")], v1, dataset / "processed", tmp_path / "b",
                                  first_pose=bvh, file_name="x")
    assert (tmp_path / "a" / "x.bvh").read_bytes() == (tmp_path / "b" / "x.bvh").read_bytes()
    enc = a.cpu().numpy().reshape(-1, 64)
    assert np.array_equal(enc, np.broadcast_to(vec, enc.shape))
    assert torch.equal(a, b)


def test_checkpoint_without_style_encoder_is_refused_before_any_launch(dev, dataset, tmp_path):
    from zeggs_b200 import _lib, style_space
    net = _nets(tmp_path, "label_model", "attn", True)
    os.remove(net / "style_encoder.pt")
    l = _lib.lib()
    n0 = l.zeggs_launch_count()
    with pytest.raises(_lib.ZeggsError, match="no style_encoder.pt"):
        style_space.build(net, dataset / "processed", device=dev)
    assert l.zeggs_launch_count() == n0
