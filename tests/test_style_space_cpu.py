"""CPU companion of tests/test_style_space_gpu.py: the style embedding space (zeggs_b200.style_space) and its moments kernel
(csrc/style_space.cu, zeggs_embedding_moments) without a device.

* A float64 restatement of the kernel's arithmetic -- two passes, the header's slices, row order inside a slice, slice order across
  them, groups in order for the mean -- against numpy.cov and per-group means (1e-13 of the largest entry).
* The GPU tests' bounds, stated from float64 summation error (u = 2^-53; the factor 2 also covers the host oracle's own error):
    mean[c]          2 (N + 2) u sum_r |x_rc| / N
    centroid[g, c]   2 (n_g + 2) u sum_{r in g} |x_rc| / n_g
    cov[i, j]        2 ((N + 4) u sum_r |d_ri| |d_rj| + N dm_i dm_j) / (N - 1),  d = x - mean, dm = the mean's bound
  The restatement meets them with >= 4x headroom against an 80-bit reference, and two modelled kernel faults exceed them: the
  covariance divided by N instead of N - 1, and the last slice's covariance partial dropped.
* StyleSpace.embedding() arithmetic, the eigenvector sign rule, the window tiling, save / load byte identity and every refusal.
"""
import json

import numpy as np
import pytest

U = 2.0 ** -53


def slicing(N, Z):
    """(slices, rows per slice) of zeggs_embedding_moments (include/zeggs_b200.h)."""
    nb = -(-Z // 64)
    tiles = nb * (nb + 1) // 2
    s0 = min(-(-N // 256), max(1, 512 // tiles))
    R = -(-N // s0)
    return -(-N // R), R


def _seq_sum(a):
    """Sum along axis 0 in index order (np.sum is pairwise; cumsum is sequential)."""
    return np.cumsum(a, axis=0)[-1] if len(a) else np.zeros(a.shape[1:])


def restated_moments(X, g, G, fault=None):
    """The kernel's arithmetic in float64 -> (mean, cov, group_sum, group_count).  fault: None, "divide_by_n" or "drop_last_partial"."""
    X = np.asarray(X, np.float64)
    N, Z = X.shape
    S, R = slicing(N, Z)
    part, cnt = np.zeros((S, G, Z)), np.zeros((S, G), np.int64)
    for s in range(S):
        xs, gs = X[s * R:(s + 1) * R], g[s * R:(s + 1) * R]
        for k in range(G):
            part[s, k] = _seq_sum(xs[gs == k])
            cnt[s, k] = int(np.count_nonzero(gs == k))
    gsum = _seq_sum(part)
    mean = _seq_sum(gsum) / N
    pc = []
    for s in range(S):
        d = X[s * R:(s + 1) * R] - mean
        pc.append(_seq_sum(d[:, :, None] * d[:, None, :]))
    if fault == "drop_last_partial":
        pc = pc[:-1]
    tot = _seq_sum(np.array(pc).reshape(-1, Z, Z))
    cov = tot / (N if fault == "divide_by_n" else N - 1)
    cov = np.triu(cov) + np.triu(cov, 1).T          # both triangles from the upper entry, as the kernel writes them
    return mean, cov, gsum, cnt.sum(0)


def moment_bounds(X, g, G, mean_ref):
    """The bounds above -> (mean [Z], cov [Z, Z], centroid [G, Z]; rows of empty groups are 0)."""
    X = np.asarray(X, np.float64)
    N = X.shape[0]
    ax = np.abs(X)
    b_mean = 2 * (N + 2) * U * ax.sum(0) / N
    d = np.abs(X - mean_ref)
    b_cov = 2 * ((N + 4) * U * (d.T @ d) + N * np.outer(b_mean, b_mean)) / max(N - 1, 1)
    b_cen = np.zeros((G, X.shape[1]))
    for k in range(G):
        n = int(np.count_nonzero(g == k))
        if n:
            b_cen[k] = 2 * (n + 2) * U * ax[g == k].sum(0) / n
    return b_mean, b_cov, b_cen


def moment_case(N, Z, G, seed=0, offset=None, spread=None):
    """Seeded float32 rows: column means in [-2, 2] and unit spread, or a common offset with a small spread; with G > 1 group 1 is
    left empty."""
    rs = np.random.RandomState(seed + 7 * N + Z)
    if offset is None:
        X = rs.randn(N, Z) + rs.uniform(-2, 2, size=(1, Z))
    else:
        X = offset + spread * rs.randn(N, Z)
    g = rs.randint(0, G, size=N).astype(np.int32)
    if G > 1:
        g[g == 1] = 0
    return X.astype(np.float32), g


def _ld_reference(X, g, G):
    """80-bit (numpy longdouble) mean, covariance and per-group means: the 'exact' side of the headroom check."""
    Xl = np.asarray(X, np.longdouble)
    N = Xl.shape[0]
    mean = Xl.sum(0) / N
    d = Xl - mean
    cov = (d.T @ d) / (N - 1)
    cen = np.array([Xl[g == k].sum(0) / max(1, np.count_nonzero(g == k)) for k in range(G)])
    return mean, cov, cen


def _ratios(got, ref, bounds):
    mean, cov, gsum, cnt = got
    rm, rc, rcen = ref
    bm, bc, bcen = bounds
    nz = cnt > 0
    cen = gsum[nz] / cnt[nz][:, None]
    return (float(np.max(np.abs(mean - rm) / bm)), float(np.max(np.abs(cov - rc) / bc)),
            float(np.max(np.abs(cen - rcen[nz]) / bcen[nz])))


BOUND_CASES = [(2, 9, 1, None), (33, 9, 19, None), (257, 64, 19, None), (4097, 64, 19, None), (1000, 128, 1, None),
               (4097, 9, 1, (1e3, 1e-3))]


@pytest.mark.parametrize("N,Z,G,off", BOUND_CASES)
def test_restated_kernel_meets_the_gpu_bounds_with_headroom_and_faults_exceed_them(N, Z, G, off):
    X, g = moment_case(N, Z, G, offset=None if off is None else off[0], spread=None if off is None else off[1])
    ref = _ld_reference(X, g, G)
    bounds = moment_bounds(X, g, G, np.asarray(ref[0], np.float64))
    ok = _ratios(restated_moments(X, g, G), ref, bounds)
    assert max(ok) <= 0.25, ok
    for fault in ("divide_by_n", "drop_last_partial"):
        r = _ratios(restated_moments(X, g, G, fault), ref, bounds)
        assert r[1] > 1.0, (fault, r)


@pytest.mark.parametrize("N,Z,G", [(2, 1, 1), (31, 9, 19), (257, 64, 19), (4097, 9, 1)])
def test_two_pass_restatement_matches_numpy(N, Z, G):
    X, g = moment_case(N, Z, G, seed=3)
    mean, cov, gsum, cnt = restated_moments(X, g, G)
    X64 = X.astype(np.float64)
    rc = np.atleast_2d(np.cov(X64, rowvar=False))
    assert np.max(np.abs(cov - rc)) <= 1e-13 * np.max(np.abs(rc))
    assert np.max(np.abs(mean - X64.mean(0))) <= 1e-13 * np.max(np.abs(X64.mean(0)))
    for k in range(G):
        if cnt[k]:
            ref = X64[g == k].mean(0)
            assert np.max(np.abs(gsum[k] / cnt[k] - ref)) <= 1e-13 * np.max(np.abs(ref))
        else:
            assert not gsum[k].any()
    assert int(cnt.sum()) == N
    assert np.array_equal(cov, cov.T)


def test_slicing_covers_every_row_once():
    for N in (1, 2, 255, 256, 257, 4097, 10 ** 6 + 3):
        for Z in (1, 9, 64, 65, 128, 512):
            S, R = slicing(N, Z)
            assert (S - 1) * R < N <= S * R and S <= 512


def _space(Z=4, seed=0, labels=("A", "B", "C"), counts=(3, 2, 0)):
    from zeggs_b200 import style_space
    rs = np.random.RandomState(seed)
    N = sum(counts)
    lab = np.concatenate([np.full(c, i, np.int64) for i, c in enumerate(counts)])
    emb = rs.randn(N, Z).astype(np.float32)
    e64 = emb.astype(np.float64)
    mean, cov = e64.mean(0), np.cov(e64, rowvar=False)
    var, comp = style_space.principal_axes(cov)
    cen = {n: e64[lab == i].mean(0) for i, n in enumerate(labels) if counts[i]}
    return style_space.StyleSpace(emb, lab, lab.copy(), np.arange(N, dtype=np.int64) * 64, mean, cov, comp, var, cen,
                                  dict(zip(labels, counts)), list(labels), 64, "nets")


def test_embedding_arithmetic():
    s = _space()
    got = s.embedding("A", {0: 1.5, 2: -1.0})
    want = s.centroids["A"] + 1.5 * np.sqrt(s.variances[0]) * s.components[:, 0] - np.sqrt(s.variances[2]) * s.components[:, 2]
    assert got.dtype == np.float32 and got.shape == (4,)
    assert np.array_equal(got, want.astype(np.float32))
    assert np.array_equal(s.embedding(), s.mean.astype(np.float32))
    v = np.arange(4.0)
    assert np.array_equal(s.embedding(v, {3: 2}), (v + 2 * np.sqrt(s.variances[3]) * s.components[:, 3]).astype(np.float32))
    assert np.array_equal(s.embedding("B"), s.centroids["B"].astype(np.float32))


def test_principal_axes_order_and_sign_rule():
    from zeggs_b200 import style_space
    rs = np.random.RandomState(4)
    A = rs.randn(40, 9)
    cov = np.cov(A, rowvar=False)
    var, comp = style_space.principal_axes(cov)
    assert np.all(np.diff(var) <= 0)
    lead = comp[np.argmax(np.abs(comp), axis=0), np.arange(9)]
    assert np.all(lead > 0)
    assert np.allclose(comp @ np.diag(var) @ comp.T, cov, atol=1e-12)
    assert np.allclose(comp.T @ comp, np.eye(9), atol=1e-12)
    # a diagonal covariance: the axes themselves, largest variance first, every entry positive
    var, comp = style_space.principal_axes(np.diag([1.0, 3.0, 2.0]))
    assert np.array_equal(var, [3.0, 2.0, 1.0])
    assert np.array_equal(comp, np.eye(3)[:, [1, 2, 0]])
    # rank-deficient: no negative variance
    var, _ = style_space.principal_axes(np.ones((3, 3)))
    assert np.all(var >= 0)


def test_window_tiling_matches_validation_windows():
    from zeggs_b200 import data, style_space
    ranges = np.array([[0, 300], [300, 420], [420, 900], [900, 960]], np.int64)
    labels = np.array([2, 0, 1, 1])
    starts, ri, lab = style_space.example_windows(ranges, labels, 64)
    vs, vr = data.validation_windows(ranges, 64)
    assert np.array_equal(starts, vs) and np.array_equal(ri, vr)
    assert np.array_equal(starts, [0, 64, 128, 192, 300, 420, 484, 548, 612, 676, 740, 804])
    assert np.array_equal(lab, labels[ri])
    for s, r in zip(starts, ri):
        assert ranges[r][0] <= s and s + 64 < ranges[r][1]        # inside its range, as the training windows are
    assert np.all(np.diff(starts) >= 64)                           # non-overlapping


def test_save_load_save_is_byte_identical(tmp_path):
    from zeggs_b200 import style_space
    s = _space(Z=9, counts=(5, 0, 4))
    s.save(tmp_path / "a.npz")
    t = style_space.load(tmp_path / "a.npz")
    t.save(tmp_path / "b.npz")
    assert (tmp_path / "a.npz").read_bytes() == (tmp_path / "b.npz").read_bytes()
    for k in ("embeddings", "labels", "range_index", "window_start", "mean", "cov", "components", "variances"):
        assert np.array_equal(getattr(s, k), getattr(t, k)), k
    assert t.label_names == s.label_names and t.counts == s.counts and t.example_length == 64 and t.network_path == "nets"
    assert set(t.centroids) == {"A", "C"} and all(np.array_equal(t.centroids[n], s.centroids[n]) for n in t.centroids)


def test_refusals():
    from zeggs_b200 import _lib
    s = _space()
    with pytest.raises(_lib.ZeggsError, match="unknown style label 'D'"):
        s.embedding("D")
    with pytest.raises(_lib.ZeggsError, match="'C' has no windows"):
        s.embedding("C")
    with pytest.raises(_lib.ZeggsError, match=r"component 4 does not exist: components are numbered 0\.\.3"):
        s.embedding("A", {4: 1.0})
    with pytest.raises(_lib.ZeggsError, match="component -1"):
        s.embedding("A", {-1: 1.0})
    with pytest.raises(_lib.ZeggsError, match="shape"):
        s.embedding(np.zeros(5))


def test_checkpoint_without_style_encoder_is_refused(tmp_path):
    from zeggs_b200 import _lib, style_space
    (tmp_path / "nets").mkdir()
    for n in ("speech_encoder", "decoder"):
        (tmp_path / "nets" / f"{n}.pt").write_bytes(b"")
    with pytest.raises(_lib.ZeggsError, match="no style_encoder.pt.*label-based model has none"):
        style_space.build(tmp_path / "nets", tmp_path / "data")


def test_example_length_and_paths_from_options(tmp_path):
    from zeggs_b200 import style_space
    out = tmp_path / "run"
    (out / "saved_models").mkdir(parents=True)
    assert style_space.checkpoint_example_length(out / "saved_models") == 256
    (out / "options.json").write_text(json.dumps({"net_opt": {"style_encoder": {"example_length": 128}}}))
    assert style_space.checkpoint_example_length(out / "saved_models") == 128
    opts = {"paths": {"base_path": "/d", "path_processed_data": "processed_v1", "output_dir": str(out), "models_dir": None}}
    assert style_space.paths_from_options(opts) == (out / "saved_models", style_space.Path("/d/processed_v1"))
    opts["paths"]["models_dir"] = "/m"
    assert style_space.paths_from_options(opts)[0] == style_space.Path("/m")
