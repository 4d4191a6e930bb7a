"""Training on the GPU path.  `train()` keeps the reference's call surface (ZEGGS/train.py:29-36, called from
main.py:64-71); `TrainStep` is the step body (train.py:196-432) with every stage running in libzeggs_b200.so:
speech encoder, style encoder (attn or gru, VAE on or off), persistent decoder window (fwd + BPTT), fused FK/L1 loss, fused RAdam,
and -- when torch.distributed is initialised -- ONE NCCL all-reduce of the flat gradient per step.
"""
import contextlib
import datetime
import json
import math
import os
import random
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

from . import _lib, dp, modules, ops
from .optimizers import RAdam

POSE_KEYS = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt"]
# the 19 entries of the loss vector (TrainStep.terms, TrainStep.evaluate): the total, the 17 L1 terms of train.py:340-395, the weighted KL
TERM_NAMES = ["total", "root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "lrot", "lvel", "lvrt", "cpos", "crot", "cvel", "cvrt",
              "ldvl", "ldvt", "cdvl", "cdvt", "gaze", "kl_div"]


def kl_weight(iteration, center=7500, rate=0.005, threshold=0.2):
    """modules.py:745-761, 784-788: logistic annealing clipped at 0.2."""
    return min(1.0 / (1.0 + math.exp(-rate * (iteration - center))), threshold)


def check_parents(parents, nj=75):
    """The skeleton's parent array (data_definition.json "parents") as int32, or ValueError unless it is a tree the loss kernel can
    walk: nj entries, parents[0] == -1 and 0 <= parents[i] < i for every other joint (so no cycles and no second root)."""
    a = np.asarray(parents)
    if a.shape != (nj,):
        raise ValueError(f"parents: expected {nj} joints, got shape {a.shape}")
    if not np.issubdtype(a.dtype, np.integer):
        raise ValueError(f"parents: expected integer joint indices, got {a.dtype}")
    if a[0] != -1:
        raise ValueError(f"parents[0] must be -1 (the root), got {a[0]}")
    i = np.arange(1, nj)
    bad = i[(a[1:] < 0) | (a[1:] >= i)]
    if bad.size:
        raise ValueError(f"parents[{bad[0]}] = {a[bad[0]]}: every joint's parent must come before it (0 <= parents[i] < i)")
    return a.astype(np.int32)


def pack_pose(root_vel, root_vrt, lpos, ltxy, lvel, lvrt):
    B, T = root_vel.shape[0], root_vel.shape[1]
    return torch.cat([root_vel.reshape(B, T, -1), root_vrt.reshape(B, T, -1), lpos.reshape(B, T, -1),
                      ltxy.reshape(B, T, -1), lvel.reshape(B, T, -1), lvrt.reshape(B, T, -1)], dim=2)


class TrainStep:
    """One optimisation step on one GPU (one rank).  Networks are zeggs_b200.modules.* instances.

    use_graph=True: the step body is captured ONCE per batch geometry into CUDA graphs (zero_grad + encoders + decoder window
    fwd/BPTT + loss + weight packs [+ RAdam]) and replayed; every step-dependent scalar lives in device memory (RAdam step count
    and hyper-parameters, KL weight, dropout seed), so replays need no host arithmetic: the host enqueues a handful of calls per
    step instead of ~265 launches through Python/ctypes/autograd.  Data parallel: graph A (backward done) -> ONE eager NCCL
    all-reduce of the flat gradient -> graph B (RAdam)."""

    def __init__(self, speech_encoder, decoder, style_encoder, stats, parents, dt, lr=1e-4, eps=1e-5,
                 world_size=1, process_group=None, use_graph=False, eval_seed=0):
        parents = check_parents(parents)          # before anything reaches the device
        self.se, self.dec, self.st = speech_encoder, decoder, style_encoder
        self.dev = next(decoder.parameters()).device
        f = lambda k: torch.as_tensor(stats[k], dtype=torch.float32, device=self.dev)
        self.audio_mean, self.audio_std = f("audio_input_mean"), f("audio_input_std")
        self.in_mean, self.in_std = f("anim_input_mean"), f("anim_input_std")
        self.out_mean, self.out_std = f("anim_output_mean"), f("anim_output_std")
        self.parents = torch.as_tensor(parents, device=self.dev)
        self.dt = float(dt)
        params = list(self.se.parameters()) + list(self.dec.parameters()) + \
            (list(self.st.parameters()) if self.st is not None else [])
        self.optimizer = RAdam(params, lr=lr, eps=eps)
        self.world_size = world_size
        self.pg = process_group
        self.optimizer.grad_scale = 1.0 / world_size
        self.iteration = 0
        self.terms = torch.zeros(19, dtype=torch.float32, device=self.dev)
        self.klw = torch.zeros(1, dtype=torch.float32, device=self.dev)      # annealed KL weight, device scalar
        self.use_graph = bool(use_graph)
        self.seed = ops.DeviceSeed(self.dev) if self.use_graph else None
        self.eval_seed = int(eval_seed)     # VAE noise of evaluate(): its own generator, re-seeded per call (see evaluate)
        self._graphs, self._seen, self._pool = {}, {}, None
        self.graph_min_seen = 1            # eager steps on a new batch geometry before it is captured
        self.graph_launches = 0            # library launches captured per replay (gpu_launches accounting)
        self.ar_events = None              # set to [] to record (start, end) CUDA events around every all-reduce
        # concurrent lanes: SpeechEncoder next to StyleEncoder in the forward; in the backward both encoders next to the decoder's
        # weight-gradient GEMMs (the many small, latency-bound encoder kernels fill the tail waves of the large GEMMs).  Each lane
        # has its own stream and its own GEMM scratch (ops.lane); fork/join by events, so the pattern captures into the graph as
        # parallel branches.  The side lanes carry the short latency-bound kernels: high priority, so their CTAs are placed ahead
        # of the queued GEMM tiles.
        self.lanes = self.dev.type == "cuda" and os.environ.get("ZEGGS_LANES", "1") == "1"
        self._lane_streams = [torch.cuda.Stream(self.dev, priority=-1) for _ in range(2)] if self.lanes else None

    def forward_backward(self, batch, eps=None, masks=None, train_mode=True):
        """batch: dict of DEVICE tensors: audio[B,T,81], the 8 pose tensors [B,T,...], gaze_pos[B,T,3], style (example
        [B,T_ex,1134] raw, or label [B,Z]).  Returns the loss tensor (device scalar); gradients land in optimizer.flat_grad."""
        capturing = torch.cuda.is_current_stream_capturing()
        if not capturing:
            self.klw.fill_(kl_weight(self.iteration))
        if self.seed is not None:
            self.seed.advance()
            with ops.device_seed(self.seed):
                return self._forward_backward(batch, eps, masks, train_mode)
        return self._forward_backward(batch, eps, masks, train_mode)

    @contextlib.contextmanager
    def _lane(self, i, name, after=None):
        """With lanes on: the block's calls go to side stream i, in lane `name` (its own GEMM scratch, ops.lane), behind the event
        `after` (_mark), else behind everything issued so far on the current stream.  With lanes off: the block runs in place."""
        if not self.lanes:
            yield
            return
        s = self._lane_streams[i]
        s.wait_event(after if after is not None else torch.cuda.current_stream(self.dev).record_event())
        with torch.cuda.stream(s), ops.lane(name):
            yield

    def _mark(self, i=None):
        """With lanes on: an event after the work issued so far on side stream i, or on the current stream (i=None).  None with
        lanes off."""
        if not self.lanes:
            return None
        return (torch.cuda.current_stream(self.dev) if i is None else self._lane_streams[i]).record_event()

    def _join(self, *marks):
        """The current stream waits for each mark (_mark); a None mark is nothing to wait for."""
        cur = torch.cuda.current_stream(self.dev)
        for ev in marks:
            if ev is not None:
                cur.wait_event(ev)

    def _forward(self, batch, eps, masks, save):
        """normalise -> SpeechEncoder (lane 0) | the StyleEncoder's draws, then the decoder's weight packs (lane 1) -> StyleEncoder ->
        decoder window, in the networks' current train / eval mode.  save: keep the activations and build the BPTT weight images for
        the backward.  -> (the loss's inputs: prediction Y, root_pos, root_rot and ground truth packed pose, root_pos, root_rot,
        gaze_pos; mu; logvar; the states of the backward), mu = logvar = None without the VAE."""
        se, dec, st = self.se, self.dec, self.st
        masks = masks or {}
        stats = (self.in_mean, self.in_std, self.out_mean, self.out_std)
        xa = ops.normalize_rows(batch["audio"], self.audio_mean, self.audio_std)
        with self._lane(0, "speech"):
            speech, se_state = ops.speech_encoder_fwd(se, xa, ops.speech_encoder_masks(se, xa, masks.get("speech")))
        # the StyleEncoder's dropout multipliers / VAE noise first (off the main stream's critical chain; seeded draws after the speech
        # encoder's), then the weight-only preparation of the decoder (bf16 weight images, folded layer-2 matrix, BPTT images)
        with self._lane(1, "style"):
            if st is not None:
                eps, smasks = ops.style_encoder_prepare(st, batch["style"], eps, masks.get("style"))
                drawn = self._mark(1)
            ops.decoder_prepack(dec, xa.shape[0], xa.shape[1], self.dev, stats, self.dt, backward=save)
        mu = logvar = st_state = None
        if st is not None:
            xs = ops.normalize_rows(batch["style"], self.in_mean, self.in_std)
            self._join(drawn)
            (z, mu, logvar), st_state = ops.style_encoder_fwd(st, xs, eps, smasks, 1.0)
        else:
            z = batch["style"]
        self._join(self._mark(0), self._mark(1))
        T = speech.shape[1]
        W = [batch[k] for k in POSE_KEYS]
        WY = pack_pose(*W[2:])                                   # ground-truth window, packed once
        Y, rp, rq, dstate = ops.decoder_window_forward(dec, W[0][:, 0], W[1][:, 0], WY[:, 0], batch["gaze_pos"], speech,
                                                       z.unsqueeze(1).expand(-1, T, -1), stats, self.dt, save=save)
        return (Y, rp, rq, WY, W[0], W[1], batch["gaze_pos"]), mu, logvar, (dstate, se_state, st_state)

    def _forward_backward(self, batch, eps, masks, train_mode):
        """Explicit forward + backward through the C ABI (no autograd engine on the step): every kernel writes its parameter
        gradients straight into the optimizer's flat gradient buffer (the views RAdam installed as p.grad)."""
        se, dec, st = self.se, self.dec, self.st
        for m in (se, dec, st):
            if m is not None:
                m.train(train_mode)
        loss_in, mu, logvar, (dstate, se_state, st_state) = self._forward(batch, eps, masks, save=True)
        loss, (dY, dRp, dRq, dmu, dlv) = ops.loss_fwd_bwd(*loss_in, self.parents, self.dt, mu, logvar,
                                                          kl_weight(self.iteration) if mu is not None else 0.0, self.terms,
                                                          self.klw if mu is not None else None)
        gv = lambda m: [p.grad for p in m._weights()]
        # phase 1 (recurrence + conditioning gradients), phase 2 (weight gradients); the encoders' backward passes need only phase 1:
        # with lanes on they run beside phase 2, with lanes off after it -> join
        _, dSpeech, dStyle, finish = ops.decoder_window_backward(dec, dstate, dY, dRp, dRq, grads_out=gv(dec), split=True)
        phase1 = self._mark()
        finish()
        with self._lane(0, "speech", after=phase1):
            ops.speech_encoder_bwd(se_state, dSpeech, grads_out=gv(se))
        if st is not None:
            with self._lane(1, "style", after=phase1):
                ops.style_encoder_bwd(st_state, dStyle.sum(dim=1), dmu, dlv, grads_out=gv(st))     # z was broadcast over the window
        self._join(self._mark(0), self._mark(1) if st is not None else None)
        return loss

    @torch.no_grad()
    def evaluate(self, batch, eps=None, index=0):
        """Forward only, in eval mode (no dropout): encoders -> decoder window -> the fused loss without its backward.  Returns the
        19 loss terms (TERM_NAMES) as a new device tensor, weighted with the same kl_weight(iteration) as training.
        The VAE noise is `eps` if given, else drawn from a generator seeded with (eval_seed, index) -- so the same weights and batch
        give bitwise-identical terms on every call.  Leaves the flat gradient, the optimizer state, `iteration`, `terms`, the
        dropout DeviceSeed, torch's / numpy's / Python's global generators and the captured training graphs alone."""
        if eps is None and self.st is not None and self.st.use_vae:
            g = torch.Generator(device=self.dev)
            g.manual_seed(self.eval_seed * 1000003 + int(index))
            eps = torch.randn((batch["style"].shape[0], self.dec.style_encoding_size), generator=g, device=self.dev)
        with eval_mode(self.se, self.dec, self.st):
            loss_in, mu, logvar, _ = self._forward(batch, eps, None, save=False)
            terms = torch.empty(19, dtype=torch.float32, device=self.dev)
            ops.loss_fwd_bwd(*loss_in, self.parents, self.dt, mu, logvar, kl_weight(self.iteration) if mu is not None else 0.0, terms,
                             grad=False)
        return terms

    def _allreduce(self):
        if self.ar_events is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        dp.allreduce_sum_(self.optimizer.flat_grad, group=self.pg)                  # the one collective of the step
        if self.ar_events is not None:
            e1.record()
            self.ar_events.append((e0, e1))

    def _eager_step(self, batch, eps=None, masks=None):
        self.optimizer.zero_grad()
        loss = self.forward_backward(batch, eps, masks)
        if self.world_size > 1:
            self._allreduce()
        self.optimizer.step()
        self.iteration += 1
        return loss

    def step(self, batch, eps=None, masks=None):
        if self.use_graph and eps is None and masks is None:
            return self._graph_step(batch)
        return self._eager_step(batch, eps, masks)

    # ---------------------------------------------------------------- CUDA-graph path
    def _graph_step(self, batch):
        key = tuple((k, tuple(v.shape), str(v.dtype)) for k, v in sorted(batch.items()))
        ent = self._graphs.get(key)
        if ent is None:
            seen = self._seen.get(key, 0)
            self._seen[key] = seen + 1
            if seen < self.graph_min_seen:        # first sight of a geometry: a real step, run eagerly (one-time initialisation, workspace growth)
                return self._eager_step(batch)
            ent = self._capture(key, batch)
            if ent is None:
                return self._eager_step(batch)
        static, g1, g2 = ent
        for k, v in batch.items():
            static[k].copy_(v, non_blocking=True)
        self.klw.fill_(kl_weight(self.iteration))
        self.optimizer.sync_hyper()
        g1.replay()
        if g2 is not None:
            self._allreduce()
            g2.replay()
        self.optimizer._step += 1
        ops.bump_weights_epoch()          # the replay rewrote the parameters: cached weight packs of eager callers are stale
        self.iteration += 1
        return self.terms[0]

    def _capture(self, key, batch):
        import sys
        static = {k: v.clone() for k, v in batch.items()}
        self.optimizer.sync_hyper()
        self.klw.fill_(kl_weight(self.iteration))
        torch.cuda.synchronize()
        n0 = _lib.lib().zeggs_launch_count()
        try:
            g1 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g1, **({} if self._pool is None else {"pool": self._pool})):
                self.optimizer.zero_grad()
                self.forward_backward(static)
                if self.world_size == 1:
                    self.optimizer.step()
            if self._pool is None:
                self._pool = g1.pool()
            g2 = None
            if self.world_size > 1:
                g2 = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g2, pool=self._pool):
                    self.optimizer.step()
        except Exception as e:       # capture refused (driver / library limitation): say so loudly and keep training eagerly
            print(f"[zeggs_b200] CUDA-graph capture of the train step FAILED ({type(e).__name__}: {e}); continuing with eager launches",
                  file=sys.stderr, flush=True)
            self.use_graph = False
            try:
                torch.cuda.synchronize()
            except Exception:
                pass
            ops.bump_weights_epoch()          # nothing captured has run: packs recorded during the capture never happened
            ops.WS.bufs.clear()
            return None
        self.graph_launches = int(_lib.lib().zeggs_launch_count() - n0)
        ops.bump_weights_epoch()
        self._graphs[key] = (static, g1, g2)
        return self._graphs[key]


class eval_mode:
    """Networks in eval mode for the block, restored afterwards together with their cached weight packs (`_zeggs_*`).  The packs a
    captured training graph writes were allocated in the graph's private memory pool; an eager call that re-packs would drop the
    module's last reference to them, and a later capture could then hand that memory to something else while the first graph still
    writes it.  Restoring keeps them referenced (their version keys are stale, so the next eager call packs afresh)."""

    def __init__(self, *nets):
        self.nets = [m for m in nets if m is not None]

    def __enter__(self):
        self.state = [(m, m.training, {k: v for k, v in m.__dict__.items() if k.startswith("_zeggs")}) for m in self.nets]
        for m in self.nets:
            m.eval()
        return self

    def __exit__(self, *exc):
        for m, training, caches in self.state:
            m.train(training)
            m.__dict__.update(caches)
        return False


def validate(stepper, ds, batchsize):
    """Held-out loss: every validation window of `ds` (data.validation_windows) through stepper.evaluate in batches of `batchsize`
    (the last one may be smaller).  -> (window-weighted mean of each of the 19 terms as float64 numpy [19], window count), or
    (None, 0) without a validation split.  Every term is a mean over its batch, so weighting by window count gives the exact mean
    over all windows."""
    n = len(ds.valid_starts)
    if n == 0:
        return None, 0
    acc = torch.zeros(19, dtype=torch.float64, device=stepper.dev)
    for k, i in enumerate(range(0, n, batchsize)):
        idx = np.arange(i, min(i + batchsize, n))
        terms = stepper.evaluate(ds.valid_batch(idx, stepper.dev), index=k)
        acc += terms.double() * len(idx)
    return (acc / n).cpu().numpy(), n


@torch.no_grad()
def write_samples(samples_dir, iteration, ds, se, de, st, stats, details, style_encoding_type, rs, device, splits=("train", "valid")):
    """train.py:511-729: for each split three clips of at most 30 s (dataset.py:206-233, ranges picked by `rs`), the networks in eval
    mode on the clip's audio from its first pose along its gaze track, and the ground truth and the prediction written as BVH files
    iteration_{it}_{split}_{ground|predict}_{i}_{label}.bvh.  The style is the clip's own example (get_example over the clip, the
    current example length; VAE noise from `rs`) or its one-hot label.  File-system errors are printed, not raised (:622-623)."""
    from . import bvhio
    f = lambda k: torch.as_tensor(stats[k], dtype=torch.float32, device=device)
    in_mean, in_std, out_mean, out_std = f("anim_input_mean"), f("anim_input_std"), f("anim_output_mean"), f("anim_output_std")
    parents, names, dt = details["parents"], details["bone_names"], float(details["dt"])
    with eval_mode(se, de, st):
        for split in splits:
            for i in range(3):
                clip, label, rng, _ = ds.get_sample(split, 30, rs=rs)
                c = {k: v.to(device) for k, v in clip.items()}
                speech = se((c["audio"] - f("audio_input_mean")) / f("audio_input_std"))
                if style_encoding_type == "example":
                    ex = (ds.get_example(rng, rng, ds.example_window_length).to(device) - in_mean) / in_std
                    eps = torch.from_numpy(rs.randn(1, de.style_encoding_size).astype(np.float32)).to(device) if st.use_vae else None
                    z, _, _ = st(ex[None], 1.0, eps=eps)
                else:
                    z = torch.zeros((1, len(details["label_names"])), dtype=torch.float32, device=device)
                    z[0, label] = 1.0
                T = speech.shape[1]
                V = de(*[c[k][:, 0] for k in POSE_KEYS], c["gaze_pos"], speech, z.unsqueeze(1).repeat(1, T, 1), None,
                       in_mean, in_std, out_mean, out_std, dt)
                V = dict(zip(POSE_KEYS, V))
                pos, eul = ops.pose_to_bvh_channels(*[torch.cat([c[k], V[k]], 0) for k in ("root_pos", "root_rot", "lpos", "ltxy")],
                                                    rebase=False)
                lab = details["label_names"][label]
                try:
                    for j, kind in enumerate(("ground", "predict")):
                        bvhio.save_bvh(str(Path(samples_dir) / f"iteration_{iteration}_{split}_{kind}_{i}_{lab}.bvh"), pos[j], eul[j],
                                       parents, names, "zyx", dt)
                except (PermissionError, OSError) as e:
                    print(e)


def pin_to_gpu_numa(local_rank):
    """Bind this process (the launch thread of one rank) to the CPUs of the NUMA node its GPU hangs off; returns the node or None.
    Un-pinned ranks of GPUs on the second socket otherwise enqueue from the remote socket."""
    try:
        p = torch.cuda.get_device_properties(local_rank)
        bus = f"{p.pci_domain_id:04x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0"
        with open(f"/sys/bus/pci/devices/{bus}/numa_node") as f:
            node = int(f.read().strip())
        if node < 0:
            return None
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            cpus = set()
            for part in f.read().strip().split(","):
                a, _, b = part.partition("-")
                cpus.update(range(int(a), int(b or a) + 1))
        allowed = os.sched_getaffinity(0) & cpus
        if allowed:
            os.sched_setaffinity(0, allowed)
        return node
    except Exception:
        return None


def build_networks(network_options, dimensions, style_encoding_type, nlabels, device):
    """train.py:96-139."""
    se_o, st_o, de_o = network_options["speech_encoder"], network_options["style_encoder"], network_options["decoder"]
    Z = nlabels if style_encoding_type == "label" else st_o["style_encoding_size"]
    se = modules.SpeechEncoder(dimensions["num_audio_features"], se_o["nhidden"], se_o["speech_encoding_size"]).to(device)
    de = modules.Decoder(pose_input_size=dimensions["pose_input_size"], pose_output_size=dimensions["pose_output_size"],
                         speech_encoding_size=se_o["speech_encoding_size"], style_encoding_size=Z,
                         hidden_size=de_o["nhidden"], num_rnn_layers=2, rnn_cond=de_o.get("rnn_cond", "normal")).to(device)
    st = None
    if style_encoding_type == "example":
        st = modules.StyleEncoder(dimensions["pose_input_size"], st_o["nhidden"], Z, type=st_o["type"],
                                  use_vae=st_o["use_vae"]).to(device)
    return se, de, st


def train(models_dir, logs_dir, path_processed_data, path_data_definition, train_options, network_options):
    """Drop-in for ZEGGS/train.py:29 (same arguments, same artefacts in models_dir).  Data-parallel when launched under
    torchrun (RANK/WORLD_SIZE set): each rank draws its own windows, one gradient all-reduce per step.  With `use_tensorboard`,
    rank 0 also writes logs_dir/tb (TensorBoardLog) from the loss terms every rank collects (LossLog)."""
    from .data import DevicePrefetcher, DeviceWindowDataset, WindowDataset
    use_tb = bool(train_options.get("use_tensorboard", False))
    if use_tb:
        summary_writer_class()               # a missing tensorboard package fails here, before any work, as the reference's import does
    np.random.seed(train_options["seed"])
    torch.manual_seed(train_options["seed"])
    if not (train_options["use_gpu"] and torch.cuda.is_available()):
        raise _lib.ZeggsError("zeggs_b200.train needs a CUDA device (no CPU fallback)")
    rank, world, local_rank = dp.env_rank_world()
    device = torch.device("cuda", local_rank)
    torch.cuda.set_device(device)
    pin_to_gpu_numa(local_rank)
    if world > 1 and not torch.distributed.is_initialized():
        torch.distributed.init_process_group("nccl")
    # additive option: recurrence engine ("auto": tensor-core bf16 operands / fp32 state where the hidden size is eligible -- the fast
    # path, pinned to the reference's loss/gradients by tests/golden/train_h384|h1024.npz and to the fp32 engine's loss curve by
    # test_short_training_curve_tc_tracks_fp32; "tc": the same but raises when ineligible; "fp32": SIMT parity-grade path)
    ops.set_decoder_engine(train_options.get("decoder_engine", "auto"))
    models_dir, logs_dir = Path(models_dir), Path(logs_dir)
    with open(path_data_definition, "r") as f:
        details = json.load(f)
    style_encoding_type = train_options["style_encoding_type"]
    # additive option "device_dataset" (default on): the processed arrays live in HBM and every batch is one gather launch; off: the
    # host supplier + double-buffered H2D prefetch
    on_device = bool(train_options.get("device_dataset", True))
    ds = (DeviceWindowDataset if on_device else WindowDataset)(
        path_data_definition, path_processed_data, train_options["window"], style_encoding_type,
        network_options["style_encoder"]["example_length"], seed=train_options["seed"] + rank, **({"device": device} if on_device else {}))
    se, de, st = build_networks(network_options, ds.get_shapes(), style_encoding_type, len(details["label_names"]), device)
    if train_options["resume"] and (models_dir / "checkpoints.pt").exists():
        for net, name in ((se, "speech_encoder"), (de, "decoder"), (st, "style_encoder")):
            if net is not None:
                net.load_state_dict(torch.load(models_dir / f"{name}.pt", weights_only=False).state_dict())
    stepper = TrainStep(se, de, st, ds.stats, details["parents"], details["dt"], lr=train_options["learning_rate"],
                        eps=train_options["eps"], world_size=world, use_graph=bool(train_options.get("cuda_graph", True)),
                        eval_seed=train_options["seed"])
    if train_options["resume"] and (models_dir / "checkpoints.pt").exists():
        ck = torch.load(models_dir / "checkpoints.pt", weights_only=False)
        stepper.iteration = ck["iteration"]
        stepper.optimizer.load_state_dict(ck["optimizer_state_dict"])
    decay = train_options["learning_rate_decay"]
    total = 1000 * train_options["niterations"]
    batchsize = train_options["batchsize"]
    ex_len = network_options["style_encoder"]["example_length"]
    start = datetime.datetime.now()
    samples_dir = logs_dir / "samples"
    sample_rs = np.random.RandomState(train_options["seed"])        # range picks and VAE noise of the sample animations
    if rank == 0:
        samples_dir.mkdir(parents=True, exist_ok=True)
    prefetch = None if on_device else DevicePrefetcher(device)
    token = None if on_device else prefetch.upload(ds.sample_host_batch(batchsize))
    # every rank collects (under data parallelism the blocks are averaged over ranks); rank 0 writes
    losslog = LossLog(device, group=stepper.pg) if use_tb else None
    tb = TensorBoardLog(logs_dir / "tb", network_options, train_options) if use_tb and rank == 0 else None
    log = (lambda steps, rows: tb.write("losses", steps, rows)) if tb is not None else (lambda steps, rows: None)
    while stepper.iteration < total:
        if on_device:
            batch = ds.sample_batch(batchsize)                                        # one gather launch out of the HBM-resident arrays
            ds.example_window_length = 2 * random.randint(ex_len // 2, ex_len)        # train.py:228-229 (applies to the next draw)
        else:
            batch = prefetch.acquire(token)
            ds.example_window_length = 2 * random.randint(ex_len // 2, ex_len)        # train.py:228-229
            token = prefetch.upload(ds.sample_host_batch(batchsize))                  # next step's windows copy under this step
        loss = stepper.step(batch)
        it = stepper.iteration
        if losslog is not None:
            log(*losslog.push(stepper))           # before the progress line's .item(): the writing overlaps the queued steps
        if it % 1000 == 0:
            for g in stepper.optimizer.param_groups:
                g["lr"] *= decay                                                     # ExponentialLR every 1000 its (:431-432)
        if rank == 0 and (it % 100 == 0 or it == 1):
            print(f"iteration {it}/{total} loss {loss.item():.5f} elapsed {datetime.datetime.now() - start}", flush=True)
        if losslog is not None and it % train_options["generate_samples_step"] == 0:
            log(*losslog.drain())                 # on every rank: a collective under data parallelism
        if rank == 0 and it % train_options["generate_samples_step"] == 0:
            train_loss = float(loss.item())
            save_checkpoint(models_dir, se, de, st, stepper, train_loss)
            save_checkpoint(models_dir / str(it), se, de, st, stepper, train_loss)             # train.py:493-509
            monitor(stepper, ds, batchsize, it, train_loss, logs_dir, samples_dir, se, de, st, details, style_encoding_type,
                    sample_rs, device, tb=tb)
    if losslog is not None:
        log(*losslog.drain())
    if rank == 0:
        save_checkpoint(models_dir, se, de, st, stepper, float(loss.item()))
    if tb is not None:
        tb.close()


def monitor(stepper, ds, batchsize, it, train_loss, logs_dir, samples_dir, se, de, st, details, style_encoding_type, rs, device, tb=None):
    """What train() does at every generate_samples_step besides saving: the sample animations (train.py:511-729) and the held-out
    loss (validate), printed and appended as one JSON line to logs_dir/valid_loss.jsonl, and written as `valid/*` at step `it` to
    the TensorBoardLog `tb` if given.  Touches nothing the training reads."""
    has_valid = len(ds.ranges_valid) > 0
    write_samples(samples_dir, it, ds, se, de, st, ds.stats, details, style_encoding_type, rs, device,
                  splits=("train", "valid") if has_valid else ("train",))
    terms, n = validate(stepper, ds, batchsize)
    if n == 0:
        return
    print(f"iteration {it} validation loss {terms[0]:.5f} over {n} windows (training loss {train_loss:.5f})", flush=True)
    rec = {"iteration": it, "train_loss": train_loss, "valid": {k: float(v) for k, v in zip(TERM_NAMES, terms)}, "windows": n}
    try:
        with open(Path(logs_dir) / "valid_loss.jsonl", "a") as fh:
            fh.write(json.dumps(rec) + "\n")
    except (PermissionError, OSError) as e:
        print(e)
    if tb is not None:
        tb.write("valid", [it], terms[None].astype(np.float32))


def flatten_options(d, prefix=""):
    """Nested option dicts -> one flat dict whose keys join the path with "_" ({"decoder": {"nhidden": 1024}} -> {"decoder_nhidden":
    1024}), the hyper-parameter names the reference's TensorBoard run carries (helpers.py:14-23)."""
    out = {}
    for k, v in d.items():
        key = f"{prefix}_{k}" if prefix else k
        if isinstance(v, dict):
            out.update(flatten_options(v, key))
        else:
            out[key] = v
    return out


def summary_writer_class():
    """torch.utils.tensorboard.SummaryWriter, or ZeggsError when the tensorboard package is missing."""
    try:
        from torch.utils.tensorboard import SummaryWriter
    except ImportError as e:
        raise _lib.ZeggsError(f"use_tensorboard is set but torch.utils.tensorboard cannot be imported ({e}): install the tensorboard "
                              "package or set use_tensorboard to false") from e
    return SummaryWriter


class TensorBoardLog:
    """The reference's TensorBoard run (train.py:179-187, 437-463) in directory `tb_dir`: the flattened network and training options as
    hyper-parameters once, then per step `<prefix>/total_loss` and `<prefix>/losses` with the 18 named terms (`loss_root_pos` ...
    `loss_gaze`, `loss_kl_div` = the weighted KL), one sub-run per term (tb/<prefix>_losses_loss_*/) as add_scalars lays them out.
    train() writes prefix "losses" for every optimizer step and "valid" for the held-out loss."""

    def __init__(self, tb_dir, network_options, train_options):
        self.writer = summary_writer_class()(str(tb_dir), flush_secs=10)
        h = flatten_options(network_options)
        h.update(flatten_options(train_options))
        self.writer.add_hparams(h, {"No Metric": 0.0})

    def write(self, prefix, steps, rows):
        """rows[i] (the 19 TERM_NAMES values) at step steps[i]."""
        for s, r in zip(steps, rows):
            s = int(s)
            self.writer.add_scalar(f"{prefix}/total_loss", r[0], s)
            self.writer.add_scalars(f"{prefix}/losses", {"loss_" + n: r[j] for j, n in enumerate(TERM_NAMES[1:], 1)}, s)

    def close(self):
        self.writer.close()


class LossLog:
    """Every step's 19 loss terms (TrainStep.terms) brought to the host without a per-step device sync.  `push(stepper)` after each
    step enqueues one device-to-device copy of the terms into the next row of a [block, 19] device history, on the current stream:
    behind the step that wrote them, ahead of the next one that overwrites them.  When a block fills, its rows are averaged over the
    ranks of `group` (one all-reduce per block; exact, since every term is a batch mean and the per-rank batches are equal) and
    copied to pinned host memory behind an event; the PREVIOUS block's rows, long landed, are returned then.  So a push that does
    not fill a block returns nothing and waits for nothing, and the host gets the rows at most two blocks late.  `drain()` closes the
    open block, waits and returns everything pending; under data parallelism every rank must push and drain at the same steps.
    Both return (steps int64 [n], rows float32 [n, 19]); a row's step is stepper.iteration - 1, the 0-based optimizer step."""

    def __init__(self, device, block=100, group=None):
        self.dev = torch.device(device)
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        self.hist = torch.zeros(block, 19, dtype=torch.float32, device=self.dev)
        self.host = torch.zeros(block, 19, dtype=torch.float32).pin_memory()
        self.steps = []                # steps of the rows in the open block
        self.pending = None            # (steps, event) of the closed block whose copy to `host` is in flight

    def push(self, stepper):
        self.hist[len(self.steps)].copy_(stepper.terms, non_blocking=True)
        self.steps.append(stepper.iteration - 1)
        if len(self.steps) < self.hist.shape[0]:
            return np.zeros(0, np.int64), np.zeros((0, 19), np.float32)
        return self._close()

    def drain(self):
        s0, r0 = self._close()
        s1, r1 = self._collect()
        return np.concatenate([s0, s1]), np.concatenate([r0, r1])

    def _collect(self):
        if self.pending is None:
            return np.zeros(0, np.int64), np.zeros((0, 19), np.float32)
        steps, ev = self.pending
        self.pending = None
        ev.synchronize()
        return np.asarray(steps, np.int64), self.host[:len(steps)].numpy().copy()

    def _close(self):
        out = self._collect()                  # before the next copy into `host`
        n = len(self.steps)
        if n:
            rows = self.hist[:n]
            if self.world > 1:
                dist.all_reduce(rows, op=dist.ReduceOp.SUM, group=self.group)
                rows.mul_(1.0 / self.world)
            self.host[:n].copy_(rows, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.dev))
            self.pending, self.steps = (self.steps, ev), []
        return out


def save_checkpoint(models_dir, se, de, st, stepper, loss):
    """train.py:477-509: whole-module pickles + optimizer state."""
    models_dir = Path(models_dir)
    models_dir.mkdir(parents=True, exist_ok=True)

    def clean(m):
        """A standalone CPU copy of the module: parameters cloned out of the optimizer's shared flat buffer (each pickle would otherwise
        drag the whole 100 MB storage along), cached weight packs (`_zeggs_*`) dropped."""
        import copy
        c = copy.copy(m)
        c.__dict__ = {k: v for k, v in m.__dict__.items() if not k.startswith("_zeggs")}
        c = copy.deepcopy(c)
        for p in c.parameters():
            p.data = p.data.detach().clone().cpu()
            p.grad = None
        return c.cpu()

    torch.save(clean(se), models_dir / "speech_encoder.pt")
    torch.save(clean(de), models_dir / "decoder.pt")
    if st is not None:
        torch.save(clean(st), models_dir / "style_encoder.pt")
    torch.save({"iteration": stepper.iteration, "epoch": 0, "loss": loss,
                "optimizer_state_dict": stepper.optimizer.state_dict()}, models_dir / "checkpoints.pt")
