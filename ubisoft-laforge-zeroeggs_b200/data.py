"""Window supplier with the reference's processed_data.npz schema (ZEGGS/data_pipeline.py:650-684,
ZEGGS/dataset.py:9-204): sliding training windows + the style-example window around each of them.
Whole arrays are kept pinned on the host and every batch is gathered with fancy indexing and copied with one
non-blocking H2D per tensor (the reference does 11 synchronous copies per step, train.py:215-225)."""
import json

import numpy as np
import torch

KEYS = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt", "gaze_pos"]


def validation_windows(ranges, window):
    """Fixed validation windows: in every range [s, e), non-overlapping windows of `window` rows at s, s+W, s+2W, ..., keeping only
    starts the reference's window enumeration also produces (dataset.py:89: start <= e - W - 1).  -> (starts, range index of each)."""
    starts, rng_idx = [], []
    for i, (s, e) in enumerate(ranges):
        st = np.arange(int(s), int(e) - window, window, dtype=np.int64)
        starts.append(st)
        rng_idx.append(np.full(len(st), i, dtype=np.int64))
    if not starts:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(starts), np.concatenate(rng_idx)


class WindowDataset:
    def __init__(self, path_data_definition, path_processed_data, window, style_encoding_type, example_window_length, seed=0):
        with open(path_data_definition, "r") as f:
            self.details = json.load(f)
        d = np.load(path_processed_data)
        self.window = window
        self.style_encoding_type = style_encoding_type
        self.example_window_length = example_window_length
        self.nlabels = len(self.details["label_names"])
        self.ranges = d["ranges_train"]
        self.labels = d["ranges_train_labels"]
        self.X = torch.as_tensor(d["X_audio_features"], dtype=torch.float32)
        self.Y = {k: torch.as_tensor(d["Y_" + k], dtype=torch.float32) for k in KEYS}
        self.stats = {k: d[k] for k in ("audio_input_mean", "audio_input_std", "anim_input_mean", "anim_input_std",
                                        "anim_output_mean", "anim_output_std")}
        starts, rng_idx = [], []
        for i, (s, e) in enumerate(self.ranges):                       # dataset.py:82-93
            n = max(0, int(e) - window - int(s))
            starts.append(np.arange(int(s), int(s) + n))
            rng_idx.append(np.full(n, i))
        self.starts = np.concatenate(starts) if starts else np.zeros(0, np.int64)
        self.rng_idx = np.concatenate(rng_idx) if rng_idx else np.zeros(0, np.int64)
        self.rs = np.random.RandomState(seed)
        # held-out split: fixed, non-overlapping windows (validation_windows); their style examples use the configured example length,
        # not the per-iteration random one.  No split when either key is missing or the ranges are empty.
        has_valid = "ranges_valid" in d.files and "ranges_valid_labels" in d.files and len(d["ranges_valid"]) > 0
        self.ranges_valid = d["ranges_valid"] if has_valid else np.zeros((0, 2), np.int64)
        self.labels_valid = d["ranges_valid_labels"] if has_valid else np.zeros(0, np.int64)
        self.valid_example_length = example_window_length
        self.valid_starts, self.valid_rng_idx = validation_windows(self.ranges_valid, window)
        if style_encoding_type == "example" and len(self.valid_starts):
            # the example rule can only double the rows a short range has (dataset.py:199-203): a tile whose example stays shorter
            # than L cannot be batched (the training draw raises on such windows), so validation leaves it out
            L, keep = example_window_length, []
            for s, r in zip(self.valid_starts.tolist(), self.valid_rng_idx.tolist()):
                a, b = self._example_rows(s, s + window - 1, int(self.ranges_valid[r][0]), int(self.ranges_valid[r][1]), L)
                keep.append(2 * (b - a) >= L)
            keep = np.array(keep, dtype=bool)
            self.valid_starts, self.valid_rng_idx = self.valid_starts[keep], self.valid_rng_idx[keep]

    def __len__(self):
        return len(self.starts)

    def get_shapes(self):
        return dict(num_audio_features=self.X.shape[1], pose_input_size=len(self.stats["anim_input_std"]),
                    pose_output_size=len(self.stats["anim_output_std"]))

    def _example_rows(self, first, last, s0, e0, L):
        """[a, b) rows of the style example around the rows first..last inside the range [s0, e0) (dataset.py:180-187)."""
        ext = (L - self.window) // 2
        ws, we = min(ext, first - s0), min(ext, e0 - last)
        s_ext, w_ext = ws + ext - we, we + ext - ws
        a = max(first - s_ext, s0)
        b = min(min(last + w_ext, e0) + 1, len(self.Y["root_vel"]))
        return a, b

    def _example_vec(self, a, b, L):
        """Rows [a, b) as [n, 1134] style-example features (gaze slot zero), tail-repeated up to L rows (dataset.py:188-204)."""
        n = b - a
        parts = [self.Y[k][a:b].reshape(n, -1) for k in ("root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt")]
        vec = torch.cat(parts + [torch.zeros(n, 3)], dim=1)
        if n < L:
            vec = torch.cat([vec, vec[-L + n:]], dim=0)
        return vec

    def _example(self, start, ri):
        """dataset.py:176-204."""
        L = self.example_window_length
        s0, e0 = int(self.ranges[ri][0]), int(self.ranges[ri][1])
        return self._example_vec(*self._example_rows(start, start + self.window - 1, s0, e0, L), L)

    def get_example(self, rows, sample_range, L):
        """dataset.py:176-204 with explicit arguments: rows = (first row, last row), as the reference's Rwindow[0] / Rwindow[-1]
        (train.py:544 passes the clip's [s, e] for both)."""
        return self._example_vec(*self._example_rows(int(rows[0]), int(rows[-1]), int(sample_range[0]), int(sample_range[1]), L), L)

    def get_sample(self, split, length=None, range_index=None, rs=None):
        """dataset.py:206-233: a whole range of `split` ("train" / "valid"), picked by `rs` (a RandomState) unless range_index is
        given, cut to at most `length` seconds (60 fps).  -> (dict of the 9 arrays + "audio" as [1, n, ...] tensors, label, [s, e],
        range_index)."""
        ranges, labels = (self.ranges, self.labels) if split == "train" else (self.ranges_valid, self.labels_valid)
        if range_index is None:
            range_index = int(rs.randint(len(ranges)))
        (s, e), label = (int(v) for v in ranges[range_index]), int(labels[range_index])
        if length is not None:
            e = min(s + length * 60, e)
        clip = {"audio": self.X[s:e][None]}
        for k in KEYS:
            clip[k] = self.Y[k][s:e][None]
        return clip, label, [s, e], range_index

    def valid_host_batch(self, idx):
        """Validation windows idx (indices into valid_starts) as a host batch with sample_host_batch's layout."""
        idx = np.asarray(idx)
        rows = torch.as_tensor(self.valid_starts[idx][:, None] + np.arange(self.window)[None, :])
        out = {"audio": self.X[rows]}
        for k in KEYS:
            out[k] = self.Y[k][rows]
        if self.style_encoding_type == "label":
            lab = torch.zeros(len(idx), self.nlabels)
            lab[torch.arange(len(idx)), torch.as_tensor(self.labels_valid[self.valid_rng_idx[idx]]).long()] = 1.0
            out["style"] = lab
        else:
            L = self.valid_example_length
            out["style"] = torch.stack([self.get_example((st, st + self.window - 1), self.ranges_valid[ri], L)
                                        for st, ri in zip(self.valid_starts[idx], self.valid_rng_idx[idx])])
        return out

    def valid_batch(self, idx, device):
        return {k: v.to(device) for k, v in self.valid_host_batch(idx).items()}

    def sample_batch(self, batchsize, device):
        return {k: v.to(device, non_blocking=True) for k, v in self.sample_host_batch(batchsize).items()}

    def sample_host_batch(self, batchsize):
        """Same draw as sample_batch, left in pinned host memory (for DevicePrefetcher.upload)."""
        idx = self.rs.randint(0, len(self.starts), size=batchsize)
        rows = torch.as_tensor(self.starts[idx][:, None] + np.arange(self.window)[None, :])
        out = {"audio": self.X[rows]}
        for k in KEYS:
            out[k] = self.Y[k][rows]
        if self.style_encoding_type == "label":
            lab = torch.zeros(batchsize, self.nlabels)
            lab[torch.arange(batchsize), torch.as_tensor(self.labels[self.rng_idx[idx]]).long()] = 1.0
            out["style"] = lab
        else:
            out["style"] = torch.stack([self._example(int(self.starts[i]), int(self.rng_idx[i])) for i in idx])
        pin = torch.cuda.is_available()
        return {k: (v.pin_memory() if pin else v.contiguous()) for k, v in out.items()}


class DeviceWindowDataset(WindowDataset):
    """The same windows, drawn by the same generator, with the processed arrays RESIDENT IN HBM and every batch produced by ONE
    gather launch (zeggs_window_gather) -- no per-sample host indexing, no host->device copies beyond three int32 vectors of length
    B (window starts, example starts, example lengths).  SURVEY.md 8f row 2; replaces dataset.py:110-153, 176-204 and
    train.py:215-225.  sample_batch() returns the dict TrainStep.step() takes; bit-identical to WindowDataset.sample_host_batch()
    for the same seed (pure row copies)."""
    _EX = ("root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt")

    def __init__(self, *args, device="cuda", **kw):
        super().__init__(*args, **kw)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            from . import _lib
            raise _lib.ZeggsError("DeviceWindowDataset keeps the data in HBM: needs a CUDA device")
        self.names = ["audio"] + KEYS
        flat = [self.X] + [self.Y[k] for k in KEYS]
        self.dev_arrays = [a.reshape(a.shape[0], -1).contiguous().to(self.device) for a in flat]
        self.shapes = [tuple(a.shape[1:]) for a in flat]
        self.widths = [a.shape[1] for a in self.dev_arrays]
        self.n_frames = flat[0].shape[0]
        self.ex_width = sum(self.widths[self.names.index(k)] for k in self._EX) + 3

    def _example_range(self, start, ri, ranges=None, L=None):
        """(first row, rows available) of the example window (dataset.py:176-198) -- the integer part of WindowDataset._example."""
        ranges = self.ranges if ranges is None else ranges
        a, b = self._example_rows(start, start + self.window - 1, int(ranges[ri][0]), int(ranges[ri][1]),
                                  self.example_window_length if L is None else L)
        return a, b - a

    def sample_batch(self, batchsize, device=None):
        idx = self.rs.randint(0, len(self.starts), size=batchsize)
        return self._gather(self.starts[idx], self.labels[self.rng_idx[idx]], self.rng_idx[idx], self.ranges, self.example_window_length)

    def valid_batch(self, idx, device=None):
        """Validation windows idx (indices into valid_starts) gathered on the device; bit-identical to valid_host_batch.  Draws
        nothing from self.rs."""
        idx = np.asarray(idx)
        ri = self.valid_rng_idx[idx]
        return self._gather(self.valid_starts[idx], self.labels_valid[ri], ri, self.ranges_valid, self.valid_example_length)

    def _gather(self, win_starts, labels, rng_idx, ranges, L):
        """One zeggs_window_gather launch: windows at win_starts, style = one-hot `labels` or the examples of length L around each
        window inside ranges[rng_idx]."""
        from . import _lib
        batchsize = len(win_starts)
        starts = np.asarray(win_starts).astype(np.int32)
        T = self.window
        dev = self.device
        out = {n: torch.empty((batchsize, T) + shp, dtype=torch.float32, device=dev) for n, shp in zip(self.names, self.shapes)}
        a = _lib.GatherArgs(B=batchsize, T=T, n_arrays=len(self.names))
        for k, n in enumerate(self.names):
            a.src[k], a.dst[k], a.width[k] = self.dev_arrays[k].data_ptr(), out[n].data_ptr(), self.widths[k]
        keep = [torch.from_numpy(starts).to(dev)]
        a.start = keep[0].data_ptr()
        if self.style_encoding_type == "label":
            lab = torch.zeros(batchsize, self.nlabels)
            lab[torch.arange(batchsize), torch.as_tensor(labels).long()] = 1.0
            out["style"] = lab.to(dev)
        else:
            rng = [self._example_range(int(s), int(r), ranges, L) for s, r in zip(win_starts, rng_idx)]
            for (_, n) in rng:
                if 2 * n < L:
                    raise _lib.ZeggsError("style example shorter than half the example window (dataset.py:201-203 cannot pad it)")
            ex = torch.empty((batchsize, L, self.ex_width), dtype=torch.float32, device=dev)
            keep += [torch.tensor([r[0] for r in rng], dtype=torch.int32).to(dev), torch.tensor([r[1] for r in rng], dtype=torch.int32).to(dev)]
            a.ex_out, a.L, a.ex_width, a.n_ex = ex.data_ptr(), L, self.ex_width, len(self._EX)
            for k, n in enumerate(self._EX):
                a.ex_src[k] = self.names.index(n)
            a.ex_start, a.ex_n = keep[1].data_ptr(), keep[2].data_ptr()
            out["style"] = ex
        _lib.check(_lib.lib().zeggs_window_gather(a, _lib.stream_ptr()), "zeggs_window_gather")
        return out


class DevicePrefetcher:
    """Double-buffered host->device input pipeline: `upload` enqueues the copies of the NEXT step's batch on a side stream
    so they overlap the current step's kernels; `acquire` makes the compute stream wait for them.  (The reference copies
    its 11 batch tensors synchronously at the top of every iteration, train.py:215-225.)  The device buffers are allocated
    once (grow-only, per tensor name) and re-used, so the steady state performs no allocation; a buffer is overwritten
    only after the step that read it has been enqueued two acquires ago (event-ordered, no host synchronisation)."""

    def __init__(self, device, nbuf=2):
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(self.device)
        self.flat = [dict() for _ in range(nbuf)]       # name -> 1-D device buffer (capacity)
        self.free_ev = [None] * nbuf                     # recorded on the compute stream when the buffer may be overwritten
        self.n = 0
        self.last = None

    def upload(self, host_batch):
        k = self.n % len(self.flat)
        self.n += 1
        views = {}
        for name, v in host_batch.items():
            buf = self.flat[k].get(name)
            if buf is None or buf.numel() < v.numel() or buf.dtype != v.dtype:
                buf = torch.empty(max(v.numel(), 1), dtype=v.dtype, device=self.device)
                self.flat[k][name] = buf
            views[name] = buf[:v.numel()].view(v.shape)
        with torch.cuda.stream(self.stream):
            if self.free_ev[k] is not None:
                self.stream.wait_event(self.free_ev[k])
            for name, v in host_batch.items():
                views[name].copy_(v, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        return k, views, ev

    def acquire(self, token):
        k, views, ev = token
        cur = torch.cuda.current_stream(self.device)
        if self.last is not None:                        # everything that read the previous buffer is enqueued by now
            fe = torch.cuda.Event()
            fe.record(cur)
            self.free_ev[self.last] = fe
        cur.wait_event(ev)
        self.last = k
        return views


class LaggedScalarReader:
    """Per-step device->host read of a scalar result (the loss) without draining the GPU: `push` enqueues a 4-byte copy into a
    pinned ring behind the step that produced the value and returns the values of the steps whose copies have certainly landed
    (those pushed `lag` calls ago); `drain` waits for the rest.  Every step's loss still reaches the host, one step late, so
    the next step's launches are enqueued while the current one runs (train.py:424-431 reads `loss.item()` synchronously)."""

    def __init__(self, device, lag=1, depth=8):
        self.device = torch.device(device)
        self.lag = lag
        self.ring = torch.empty(depth, dtype=torch.float32).pin_memory()
        self.pending = []                                 # (slot, event)
        self.n = 0

    def push(self, value):
        slot = self.n % self.ring.numel()
        self.n += 1
        self.ring[slot:slot + 1].copy_(value.detach().reshape(1), non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self.pending.append((slot, ev))
        out = []
        while len(self.pending) > self.lag:
            s, e = self.pending.pop(0)
            e.synchronize()
            out.append(float(self.ring[s]))
        return out

    def drain(self):
        out = []
        while self.pending:
            s, e = self.pending.pop(0)
            e.synchronize()
            out.append(float(self.ring[s]))
        return out

