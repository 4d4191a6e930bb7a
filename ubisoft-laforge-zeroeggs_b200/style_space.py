"""The style embedding space of an example-based model (beyond the reference code; the ZeroEGGS article's style-space edits).

`build()` encodes every non-overlapping example window of a processed dataset with a trained style encoder, on the device, and
reduces the embeddings to float64 statistics: the overall mean, the covariance, its principal directions and the centroid of each
style label.  `StyleSpace.embedding()` turns those into a style vector -- a label's centroid or the mean, moved along principal
directions in standard deviations -- that `generate.generate_gesture` takes as `styles=[(vector, name)]`.

    space = style_space.build("outputs/v1/saved_models", "data/processed_v1")
    vec = space.embedding("Happy", {0: 1.5})        # Happy, 1.5 standard deviations along the first principal direction
    generate_gesture(wav, [(vec, "happy_pc0")], ...)

Data flow: processed_data.npz -> HBM (data.DeviceWindowDataset) -> one zeggs_window_gather per batch of windows (the training
supplier's example rows, gaze slot zero) -> ops.normalize_rows with stats.npz -> style encoder (eval; mu with the VAE, z without it)
-> ops.embedding_moments (float64, fixed order) -> numpy.linalg.eigh of the Z x Z covariance on the host.

Command line: `python -m zeggs_b200.style_space -o options.json [--splits train valid] [--out style_space.npz]` builds and saves one
space from the `paths` of a training options file.
"""
import argparse
import json
from pathlib import Path

import numpy as np
import torch

from . import _lib, data, generate, ops
from .data_pipeline import savez_deterministic

DEFAULT_EXAMPLE_LENGTH = 256          # the v1 configuration's style_encoder.example_length


class StyleSpace:
    """Embeddings of a dataset's example windows and their statistics.

    embeddings [N, Z] float32; labels, range_index, window_start [N] int64 (label index, range of its split, first row)
    mean [Z], cov [Z, Z], variances [Z] (descending), components [Z, Z] (column k: unit direction of variances[k]) float64
    centroids {label name: [Z] float64} for every label with at least one window; counts {label name: windows}, every label
    label_names, example_length, network_path
    """

    def __init__(self, embeddings, labels, range_index, window_start, mean, cov, components, variances, centroids, counts, label_names,
                 example_length, network_path):
        self.embeddings, self.labels, self.range_index, self.window_start = embeddings, labels, range_index, window_start
        self.mean, self.cov, self.components, self.variances = mean, cov, components, variances
        self.centroids, self.counts = centroids, counts
        self.label_names, self.example_length, self.network_path = list(label_names), int(example_length), str(network_path)

    @property
    def Z(self):
        return int(self.mean.shape[0])

    def embedding(self, base="mean", pcs=None):
        """A style vector [Z] float32: `base` (a label name -> its centroid, "mean", or an explicit [Z] vector) plus, for every
        {k: a} of `pcs`, a * sqrt(variances[k]) * components[:, k] -- `a` standard deviations along principal direction k."""
        if isinstance(base, str):
            if base == "mean":
                v = self.mean.copy()
            elif base not in self.label_names:
                raise _lib.ZeggsError(f"unknown style label {base!r}: this space knows {self.label_names}")
            elif base not in self.centroids:
                raise _lib.ZeggsError(f"style label {base!r} has no windows in this space (no range of the encoded splits long enough for "
                                      f"a {self.example_length}-row example), so it has no centroid")
            else:
                v = self.centroids[base].copy()
        else:
            v = np.asarray(base, dtype=np.float64)
            if v.shape != (self.Z,):
                raise _lib.ZeggsError(f"base vector has shape {v.shape}, the space's embeddings have {self.Z} dimensions")
            v = v.copy()
        for k, a in (pcs or {}).items():
            if not (isinstance(k, (int, np.integer)) and 0 <= k < self.Z):
                raise _lib.ZeggsError(f"principal component {k!r} does not exist: components are numbered 0..{self.Z - 1}")
            v += float(a) * np.sqrt(self.variances[k]) * self.components[:, k]
        return v.astype(np.float32)

    def save(self, path):
        """One .npz; the same space always gives the same bytes."""
        G = len(self.label_names)
        cen = np.zeros((G, self.Z), np.float64)
        for i, n in enumerate(self.label_names):
            if n in self.centroids:
                cen[i] = self.centroids[n]
        savez_deterministic(path, dict(
            embeddings=self.embeddings, labels=self.labels, range_index=self.range_index, window_start=self.window_start,
            mean=self.mean, cov=self.cov, components=self.components, variances=self.variances, centroids=cen,
            counts=np.array([self.counts[n] for n in self.label_names], np.int64), label_names=np.array(self.label_names, dtype=str),
            example_length=np.int64(self.example_length), network_path=np.array(self.network_path, dtype=str)))


def load(path):
    """A StyleSpace saved by StyleSpace.save."""
    with np.load(path, allow_pickle=False) as d:
        names = [str(n) for n in d["label_names"]]
        counts = {n: int(c) for n, c in zip(names, d["counts"])}
        cen = d["centroids"]
        return StyleSpace(d["embeddings"], d["labels"], d["range_index"], d["window_start"], d["mean"], d["cov"], d["components"],
                          d["variances"], {n: cen[i] for i, n in enumerate(names) if counts[n] > 0}, counts, names,
                          int(d["example_length"]), str(d["network_path"]))


def principal_axes(cov):
    """numpy.linalg.eigh of a symmetric covariance in float64 -> (variances descending, components [Z, Z] by column).  Each column's
    largest-magnitude entry is made positive (the first such entry on a tie), so the same covariance always gives the same signs;
    eigenvalues that rounding leaves slightly negative (a rank-deficient covariance) are set to 0."""
    w, V = np.linalg.eigh(np.asarray(cov, dtype=np.float64))
    order = np.argsort(-w, kind="stable")
    w, V = np.maximum(w[order], 0.0), V[:, order]
    lead = V[np.argmax(np.abs(V), axis=0), np.arange(V.shape[1])]
    return w, V * np.where(lead < 0, -1.0, 1.0)[None, :]


def example_windows(ranges, labels, L):
    """Non-overlapping L-row windows of every range (data.validation_windows) -> (starts, range index, label) int64."""
    starts, ri = data.validation_windows(ranges, L)
    return starts, ri, np.asarray(labels, dtype=np.int64)[ri] if len(ri) else np.zeros(0, np.int64)


def checkpoint_example_length(network_path):
    """style_encoder.example_length of the options.json saved with a checkpoint (in the network directory or the training output
    directory above it), else DEFAULT_EXAMPLE_LENGTH."""
    network_path = Path(network_path)
    for p in (network_path / "options.json", network_path.parent / "options.json"):
        if p.exists():
            with open(p) as f:
                opts = json.load(f)
            L = opts.get("net_opt", {}).get("style_encoder", {}).get("example_length")
            if L is not None:
                return int(L)
    return DEFAULT_EXAMPLE_LENGTH


def _require_style_encoder(network_path):
    if not (Path(network_path) / "style_encoder.pt").exists():
        raise _lib.ZeggsError(f"{network_path} has no style_encoder.pt: a style space is built with the example-based model's style "
                              "encoder, and the label-based model has none")


@torch.no_grad()
def build(network_path, data_path, splits=("train",), example_length=None, batch=256, device="cuda"):
    """Encode every non-overlapping example window of the ranges of `splits` ("train", "valid") of data_path/processed_data.npz with
    network_path/style_encoder.pt and return their StyleSpace.  example_length defaults to the checkpoint's (options.json), else 256."""
    network_path, data_path = Path(network_path), Path(data_path)
    _require_style_encoder(network_path)
    for s in splits:
        if s not in ("train", "valid"):
            raise _lib.ZeggsError(f"unknown split {s!r} (train, valid)")
    L = int(example_length) if example_length is not None else checkpoint_example_length(network_path)
    if L < 1 or batch < 1:
        raise _lib.ZeggsError(f"example_length = {L} and batch = {batch} must be positive")
    dev = torch.device(device)
    enc = generate.load_networks(network_path, dev)["style_encoder"]
    ds = data.DeviceWindowDataset(str(data_path / "data_definition.json"), str(data_path / "processed_data.npz"), L, "example", L,
                                  device=dev)
    names = list(ds.details["label_names"])
    st = np.load(data_path / "stats.npz")
    in_mean = torch.as_tensor(st["anim_input_mean"], dtype=torch.float32, device=dev)
    in_std = torch.as_tensor(st["anim_input_std"], dtype=torch.float32, device=dev)
    if in_mean.numel() != ds.ex_width:
        raise _lib.ZeggsError(f"stats.npz normalises {in_mean.numel()} pose channels, the dataset's examples have {ds.ex_width}")
    parts = [example_windows(*((ds.ranges, ds.labels) if s == "train" else (ds.ranges_valid, ds.labels_valid)), L) for s in splits]
    starts, rng_idx, labels = (np.concatenate([p[i] for p in parts]) for i in range(3))
    N = len(starts)
    if N < 2:
        raise _lib.ZeggsError(f"{N} example window(s) of {L} rows in the splits {list(splits)}: a covariance needs at least 2")
    emb = torch.empty((N, enc.style_embedding_size), dtype=torch.float32, device=dev)
    ex_src = [ds.names.index(k) for k in ds._EX]
    for b0 in range(0, N, batch):
        B = min(batch, N - b0)
        ex = torch.empty((B, L, ds.ex_width), dtype=torch.float32, device=dev)
        # the gather's window part copies one row per array (T = 1, discarded); its example part is rows [start, start + L) of the
        # six pose arrays with a zero gaze slot, the training supplier's example of a window that fills it (data._example_vec)
        first = [torch.empty((B, ds.widths[k]), dtype=torch.float32, device=dev) for k in ex_src]
        st_dev = torch.from_numpy(starts[b0:b0 + B].astype(np.int32)).to(dev)
        n_dev = torch.full((B,), L, dtype=torch.int32, device=dev)
        a = _lib.GatherArgs(B=B, T=1, n_arrays=len(ex_src), start=st_dev.data_ptr(), ex_out=ex.data_ptr(), L=L, ex_width=ds.ex_width,
                            n_ex=len(ex_src), ex_start=st_dev.data_ptr(), ex_n=n_dev.data_ptr())
        for i, k in enumerate(ex_src):
            a.src[i], a.dst[i], a.width[i], a.ex_src[i] = ds.dev_arrays[k].data_ptr(), first[i].data_ptr(), ds.widths[k], i
        _lib.check(_lib.lib().zeggs_window_gather(a, _lib.stream_ptr()), "zeggs_window_gather")
        x = ops.normalize_rows(ex, in_mean, in_std)
        # the VAE's mu is the deterministic embedding: a zero eps keeps the encoder from drawing one
        eps = torch.zeros((B, enc.style_embedding_size), dtype=torch.float32, device=dev) if enc.use_vae else None
        z, mu, _ = enc(x, 1.0, eps=eps)
        emb[b0:b0 + B] = mu if enc.use_vae else z
    lab_dev = torch.from_numpy(labels.astype(np.int32)).to(dev)
    mean, cov, gsum, gcount = (t.cpu().numpy() for t in ops.embedding_moments(emb, lab_dev, len(names)))
    variances, components = principal_axes(cov)
    centroids = {n: gsum[i] / gcount[i] for i, n in enumerate(names) if gcount[i] > 0}
    counts = {n: int(gcount[i]) for i, n in enumerate(names)}
    return StyleSpace(emb.cpu().numpy(), labels, rng_idx.astype(np.int64), starts.astype(np.int64), mean, cov, components, variances,
                      centroids, counts, names, L, network_path)


def paths_from_options(options):
    """(network directory, processed-data directory) from a training options file's `paths`, as train() reads them: the data is
    base_path/path_processed_data, the networks models_dir or, when that is null, output_dir/saved_models."""
    p = options["paths"]
    base = Path(p["base_path"])
    models = p.get("models_dir")
    if models is None:
        if p.get("output_dir") is None:
            raise _lib.ZeggsError("options paths give neither models_dir nor output_dir: no network to build a style space with")
        models = Path(p["output_dir"]) / "saved_models"
    return Path(models), base / p["path_processed_data"]


def main(argv=None):
    ap = argparse.ArgumentParser(description="Build the style embedding space of a trained example-based ZeroEGGS model.")
    ap.add_argument("-o", "--options", required=True, help="training options file (its paths name the networks and the data)")
    ap.add_argument("--splits", nargs="+", default=["train"], choices=["train", "valid"])
    ap.add_argument("--out", default="style_space.npz")
    args = ap.parse_args(argv)
    with open(args.options) as f:
        options = json.load(f)
    network_path, data_path = paths_from_options(options)
    L = options.get("net_opt", {}).get("style_encoder", {}).get("example_length")
    space = build(network_path, data_path, splits=tuple(args.splits), example_length=L)
    space.save(args.out)
    w = max([len("label")] + [len(n) for n in space.label_names])
    print(f"{'label':<{w}}  windows")
    for n in space.label_names:
        print(f"{n:<{w}}  {space.counts[n]:7d}")
    print(f"{'total':<{w}}  {len(space.labels):7d}    -> {args.out}")


if __name__ == "__main__":
    main()
