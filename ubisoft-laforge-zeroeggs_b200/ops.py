"""Launchers: torch tensors -> C-ABI calls (libzeggs_b200.so).  Plumbing only (buffers, streams,
autograd wiring); all arithmetic is in csrc/*.cu."""
import ctypes as C

import torch

from . import _lib

NJ, P_IN, P_OUT = 75, 1134, 1131


def _f32c(t, device=None):
    t = t.detach() if t.requires_grad else t
    if device is not None and t.device != device:
        t = t.to(device)
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


class _Workspace:
    """Grow-only per-device scratch buffers owned by the caller side (the library allocates nothing)."""

    def __init__(self):
        self.bufs = {}

    def get(self, key, nbytes, device):
        b = self.bufs.get((key, str(device)))
        if b is None or b.numel() < nbytes:
            b = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
            self.bufs[(key, str(device))] = b
        return b


WS = _Workspace()

_scratch = {}
_ctx = {}
GEMM_MODE = 1          # 0: fp32 SIMT everywhere, 1: tensor-core split-bf16 (~fp32 accuracy)


def set_gemm_mode(mode):
    """GEMM engine of the batched (non-recurrent) products for subsequent calls from this process."""
    global GEMM_MODE
    if mode not in (0, 1):
        raise _lib.ZeggsError("gemm mode must be 0 (fp32 SIMT) or 1 (tensor-core bf16x3)")
    GEMM_MODE = mode
    for c in _ctx.values():
        c.gemm_mode = mode


# Lanes: calls that run CONCURRENTLY on different CUDA streams (the two encoders next to each other, the encoders' backward next to the
# decoder's weight-gradient GEMMs) must not share the GEMM front end's scratch buffer.  `with ops.lane("speech"):` makes every call issued
# inside the block travel with that lane's own zeggs_ctx (own scratch); the default lane is "main".
_lane_local = __import__("threading").local()


def current_lane():
    return getattr(_lane_local, "name", "main")


class lane:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        self.prev = current_lane()
        _lane_local.name = self.name
        return self

    def __exit__(self, *exc):
        _lane_local.name = self.prev
        return False


def ensure_scratch(dev):
    """Caller-owned scratch for the tensor-core GEMM front end (bf16 operand copies); ZEGGS_SCRATCH_MB (main lane) / ZEGGS_LANE_SCRATCH_MB
    (side lanes) override the size.  The buffer, the GEMM mode and the weight-gradient mode travel to the library in a per-(device, lane)
    zeggs_ctx passed with every call (ctx_ptr): the library keeps no mutable global state for them."""
    import os
    ln = current_lane()
    key = (str(dev), ln)
    if key not in _scratch:
        mb = int(os.environ.get("ZEGGS_SCRATCH_MB", "1536")) if ln == "main" else int(os.environ.get("ZEGGS_LANE_SCRATCH_MB", "768"))
        buf = torch.empty(mb << 20, dtype=torch.uint8, device=dev)
        _scratch[key] = buf
        _ctx[key] = _lib.Ctx(scratch=buf.data_ptr(), scratch_bytes=buf.numel(), gemm_mode=GEMM_MODE,
                             fast_wgrad=0 if DECODER_ENGINE == "fp32" else 1)
    return _scratch[key]


def ctx_ptr(dev):
    """Address of the current lane's zeggs_ctx on this device (for the `ctx` field of the args structs)."""
    ensure_scratch(dev)
    return C.addressof(_ctx[(str(dev), current_lane())])


_weights_epoch = 0

# decoder recurrence engine: "fp32" (SIMT, parity grade), "tc" (wgmma, bf16 operands / fp32 state) or "auto" (tc where the
# geometry is eligible, fp32 otherwise).  An explicit "tc" request on an ineligible geometry RAISES (it never silently
# runs the other engine).
DECODER_ENGINE = __import__("os").environ.get("ZEGGS_DECODER_ENGINE", "fp32")


def tc_eligible(H, S, Z):
    """The tensor-core recurrence (forward AND BPTT kernels) covers H % 128 == 0, 384 <= H <= 1024: the library's
    zeggs_decoder_packed_tc_bytes / _bwd_tc_bytes report 0 for anything else."""
    l = _lib.lib()
    return l.zeggs_decoder_packed_tc_bytes(H, S, Z) > 0 and l.zeggs_decoder_packed_bwd_tc_bytes(H, S, Z) > 0


def set_decoder_engine(name):
    global DECODER_ENGINE
    if name not in ("fp32", "tc", "auto"):
        raise _lib.ZeggsError("decoder engine must be 'fp32', 'tc' or 'auto'")
    DECODER_ENGINE = name
    # the tensor-core engine's weight gradients are single-pass bf16: the encoders' weight-gradient GEMMs follow it
    for c in _ctx.values():
        c.fast_wgrad = 0 if name == "fp32" else 1


def resolve_engine(H, S, Z, film=False):
    """-> True when the tensor-core engine runs this geometry under the current setting.  A FiLM decoder always runs on the fp32
    engine ("auto" picks it); an explicit "tc" raises."""
    if DECODER_ENGINE == "fp32":
        return False
    if film:
        if DECODER_ENGINE == "tc":
            raise _lib.ZeggsError("decoder engine 'tc' requested for a FiLM decoder (rnn_cond='film'): its layer2 is followed by an ELU "
                                  "and the FiLM modulation, so the tensor-core engine's fold of layer2 into the next step does not "
                                  "apply; use 'fp32' or 'auto'")
        return False
    ok = tc_eligible(H, S, Z)
    if DECODER_ENGINE == "tc" and not ok:
        raise _lib.ZeggsError(f"decoder engine 'tc' requested but hidden size {H} is not eligible (needs H % 128 == 0 and "
                              f"384 <= H <= 1024); use 'fp32' or 'auto'")
    return ok


def bump_weights_epoch():
    """Called by anything that rewrites parameters without going through torch (the fused optimizer)."""
    global _weights_epoch
    _weights_epoch += 1


def weights_key(params):
    return (_weights_epoch,) + tuple(p._version for p in params) + tuple(p.data_ptr() for p in params)


def normalize_rows(x, mean, std):
    """(x - mean) / std over the last dimension in one pass (zeggs_normalize_rows); same arithmetic as the two torch ops."""
    if x.device.type != "cuda":
        raise _lib.ZeggsError("zeggs_b200.ops.normalize_rows runs on CUDA tensors only")
    x = _f32c(x)
    Cn = x.shape[-1]
    try:                                    # statistics broadcast over the channel dimension (the audio std is a scalar)
        mean = _f32c(mean, x.device).reshape(-1).expand(Cn).contiguous() if mean.numel() in (1, Cn) else None
        std = _f32c(std, x.device).reshape(-1).expand(Cn).contiguous() if std.numel() in (1, Cn) else None
    except RuntimeError:
        mean = std = None
    if mean is None or std is None:
        raise _lib.ZeggsError("normalize_rows: mean / std must be scalars or have the size of the last dimension")
    out = torch.empty_like(x)
    _lib.check(_lib.lib().zeggs_normalize_rows(x.data_ptr(), mean.data_ptr(), std.data_ptr(), out.data_ptr(), x.numel() // Cn, Cn,
                                               _lib.stream_ptr()), "zeggs_normalize_rows")
    return out


def split_pose(Y, root_pos, root_rot):
    """[B,T,1131] pose vectors -> the reference's 8-tuple (modules.py:153-162, 731-736)."""
    B, T = Y.shape[0], Y.shape[1]
    o = 6
    return (root_pos, root_rot, Y[..., 0:3], Y[..., 3:6],
            Y[..., o:o + NJ * 3].reshape(B, T, NJ, 3),
            Y[..., o + NJ * 3:o + NJ * 9].reshape(B, T, NJ, 2, 3),
            Y[..., o + NJ * 9:o + NJ * 12].reshape(B, T, NJ, 3),
            Y[..., o + NJ * 12:o + NJ * 15].reshape(B, T, NJ, 3))


def _weight_pack(dec, kind, a, dev):
    """Device buffer of the decoder's weight pack `kind` -- "" (fp32 forward), "_tc", "_bwd", "_bwd_tc", "_film" or "_bwd_film": the output of
    zeggs_decoder_pack_weights<kind> -- cached on the module as `_zeggs_packed<kind>` and re-packed whenever any parameter's version
    counter moved or the device changed."""
    l = _lib.lib()
    ver = weights_key(dec._weights())
    cache = dec.__dict__.get("_zeggs_packed" + kind)
    if cache is None or cache[0] != ver or cache[1].device != dev:
        d = a.dec if isinstance(a, _lib.DecoderFilmFwdArgs) else a
        nbytes = getattr(l, f"zeggs_decoder_packed{kind}_bytes")(d.H, d.S, d.Z)
        if nbytes == 0:
            raise _lib.ZeggsError(f"decoder hidden size {d.H} unsupported")
        packed = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        name = f"zeggs_decoder_pack_weights{kind}"
        _lib.check(getattr(l, name)(a, packed.data_ptr(), _lib.stream_ptr()), name)
        cache = dec.__dict__["_zeggs_packed" + kind] = (ver, packed)
    return cache[1]


_FILM_NAMES = ["Wm", "bm", "Wg", "bg", "Wb", "bb"]


def _decoder_args(dec, B, T, dev, tensors, stats, dt, save, pack_only=False):
    """Fill a DecoderFwdArgs (a DecoderFilmFwdArgs for a FiLM decoder); returns (args, keepalive list, workspace).  pack_only: stop
    after the weight packs (decoder_prepack)."""
    H, S, Z = dec.hidden_size, dec.speech_encoding_size, dec.style_encoding_size
    film = dec.film
    kind = "_film" if film else ""
    l = _lib.lib()
    w = [_f32c(p, dev) for p in dec._weights()]
    names = ["W0", "b0", "W_ih0", "b_ih0", "W_hh0", "b_hh0", "W_ih1", "b_ih1", "W_hh1", "b_hh1", "W2", "b2",
             "Wc0", "bc0", "Wc1", "bc1", "Wc2", "bc2"]
    a = _lib.DecoderFwdArgs(B=B, T=T, H=H, S=S, Z=Z, dt=dt, ctx=ctx_ptr(dev))
    for n, t in zip(names, w):
        setattr(a, n, _lib.ptr(t))
    keep = list(w)
    st = [_f32c(s, dev).reshape(-1) for s in stats]
    for n, t in zip(["in_mean", "in_std", "out_mean", "out_std"], st):
        setattr(a, n, _lib.ptr(t))
    keep += st
    for n, t in tensors.items():
        setattr(a, n, _lib.ptr(t))
        keep.append(t)
    use_tc = resolve_engine(H, S, Z, film)          # a FiLM decoder: fp32, or raises on an explicit "tc"
    args = a
    if film:
        args = _lib.DecoderFilmFwdArgs(dec=a)
        for n, t in zip(_FILM_NAMES, w[18:]):
            setattr(args, n, _lib.ptr(t))
        a = args.dec                                 # a view of the copy inside args
    # each engine packs only its own slices
    if use_tc and B > 32:
        raise _lib.ZeggsError("tensor-core decoder engine: one call covers one 32-sample batch tile (decoder_window splits larger batches)")
    if use_tc:
        ptc = _weight_pack(dec, "_tc", a, dev)
        wtc = WS.get("dec_tc", l.zeggs_decoder_tc_workspace_bytes(H, S, Z), dev)
        a.engine, a.packed_tc, a.workspace_tc = 1, ptc.data_ptr(), wtc.data_ptr()
        keep += [ptc, wtc]
    else:
        packed = _weight_pack(dec, kind, args, dev)
        a.packed = packed.data_ptr()
        keep.append(packed)
    if pack_only:
        return args, keep, None
    wsb = getattr(l, f"zeggs_decoder{kind}_workspace_bytes")(B, T, H, S, Z, int(save))
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev) if save else WS.get("dec_fwd", wsb, dev)
    a.workspace = ws.data_ptr()
    a.workspace_bytes = wsb
    a.save_for_backward = int(save)
    keep.append(ws)
    return args, keep, ws


def decoder_prepack(dec, B, T, dev, stats, dt, backward=True):
    """Everything the decoder derives from its WEIGHTS alone -- the engine's packed / bf16 weight images, the folded layer-2 matrix and
    (backward=True) the transposed images of the BPTT kernel -- issued on the current stream and lane.  The window calls find the caches
    fresh and skip the work, so a training step can run this next to the encoders' forward instead of in front of the recurrence."""
    a, keep, _ = _decoder_args(dec, B, T, dev, {}, stats, dt, False, pack_only=True)
    if backward and dec.film:
        _weight_pack(dec, "_bwd_film", a, dev)
    elif backward and a.engine == 1:
        _weight_pack(dec, "_bwd_tc", a, dev)
    return keep


def decoder_window_forward(dec, root_pos0, root_rot0, pose0, gaze_pos, speech, style, stats, dt, save=False):
    dev = speech.device
    if dev.type != "cuda":
        raise _lib.ZeggsError("zeggs_b200.Decoder runs on CUDA tensors only (no CPU fallback)")
    ensure_scratch(dev)
    B, T = speech.shape[0], speech.shape[1]
    tensors = dict(root_pos0=_f32c(root_pos0, dev).reshape(B, 3), root_rot0=_f32c(root_rot0, dev).reshape(B, 4),
                   pose0=_f32c(pose0, dev).reshape(B, P_OUT), gaze_pos=_f32c(gaze_pos, dev).reshape(B, T, 3),
                   speech=_f32c(speech, dev), style=_f32c(style, dev))
    if tensors["style"].shape[:2] != (B, T):
        raise _lib.ZeggsError("style_encoding must be [B,T,Z] (modules.py:119)")
    Y = torch.empty((B, T, P_OUT), dtype=torch.float32, device=dev)
    rp = torch.empty((B, T, 3), dtype=torch.float32, device=dev)
    rq = torch.empty((B, T, 4), dtype=torch.float32, device=dev)
    tensors.update(Y=Y, root_pos=rp, root_rot=rq)
    a, keep, ws = _decoder_args(dec, B, T, dev, tensors, stats, dt, save)
    fn = "zeggs_decoder_film_window_fwd" if dec.film else "zeggs_decoder_window_fwd"
    _lib.check(getattr(_lib.lib(), fn)(a, _lib.stream_ptr()), fn)
    return Y, rp, rq, (a, keep, ws)


_DEC_GRAD_NAMES = ["dW0", "db0", "dW_ih0", "db_ih0", "dW_hh0", "db_hh0", "dW_ih1", "db_ih1", "dW_hh1", "db_hh1",
                   "dW2", "db2", "dWc0", "dbc0", "dWc1", "dbc1", "dWc2", "dbc2"]


def _grad_targets(weights, grads_out):
    """Gradient buffers for `weights`: fresh tensors, or the caller's (e.g. the views of the optimizer's flat gradient buffer:
    the kernels then write every parameter gradient straight to its final place -- no autograd accumulation pass)."""
    if grads_out is None:
        return [torch.empty_like(w, dtype=torch.float32, memory_format=torch.contiguous_format) for w in weights]
    for w, g in zip(weights, grads_out):
        if g.shape != w.shape or not g.is_contiguous() or g.dtype != torch.float32:
            raise _lib.ZeggsError("gradient target must be a contiguous fp32 tensor of the parameter's shape")
    return list(grads_out)


def decoder_window_backward(dec, state, dY, dRp, dRq, grads_out=None, split=False):
    """BPTT of one decoder window (zeggs_decoder_window_bwd).  state = the 4th result of decoder_window_forward(save=True).
    Returns (weight gradients in dec._weights() order, dSpeech [B,T,S], dStyle [B,T,Z]).
    split=True: run phase 1 only (recurrence, CellStateEncoder gradients, dSpeech / dStyle) and return a 4th value `finish`;
    calling it issues phase 2 (all remaining parameter gradients) on the then-current stream of the same lane -- the caller may run the
    encoders' backward passes on other streams / lanes in between."""
    l = _lib.lib()
    fa, keep, ws = state
    film = dec.film
    kind = "_film" if film else ""
    fb = _lib.DecoderFilmBwdArgs() if film else _lib.DecoderBwdArgs()
    a, b = (fa.dec, fb.dec) if film else (fa, fb)
    dev = ws.device
    B, T, H, S, Z = a.B, a.T, a.H, a.S, a.Z
    hold = []
    for name, g in (("dY", dY), ("dRootPos", dRp), ("dRootRot", dRq)):
        if g is not None:
            g = g.contiguous().float()
            hold.append(g)
            setattr(b, name, g.data_ptr())
    # transposed weight slices for the backward recurrence
    if a.engine == 1:
        ptc = _weight_pack(dec, "_bwd_tc", a, dev)
        wtc = WS.get("dec_bwd_tc", l.zeggs_decoder_bwd_tc_workspace_bytes(H, S, Z), dev)
        b.packed_bwd_tc, b.workspace_tc = ptc.data_ptr(), wtc.data_ptr()
        hold += [ptc, wtc]
    else:
        packed = _weight_pack(dec, "_bwd" + kind, fa, dev)
        b.packed_bwd = packed.data_ptr()
        hold.append(packed)
    grads = _grad_targets(dec._weights(), grads_out)
    for n, g in zip(_DEC_GRAD_NAMES, grads):
        setattr(b, n, g.data_ptr())
    for n, g in zip(_FILM_NAMES, grads[18:]):
        setattr(fb, "d" + n, g.data_ptr())
    dSpeech = torch.empty((B, T, S), dtype=torch.float32, device=dev)
    dStyle = torch.empty((B, T, Z), dtype=torch.float32, device=dev)
    b.dSpeech, b.dStyle = dSpeech.data_ptr(), dStyle.data_ptr()
    wsb = getattr(l, f"zeggs_decoder{kind}_bwd_workspace_bytes")(B, T, H, S, Z)
    bws = WS.get("dec_bwd", wsb, dev)
    b.workspace, b.workspace_bytes = bws.data_ptr(), wsb
    name = f"zeggs_decoder{kind}_window_bwd"
    run = lambda: getattr(l, name)(fa, fb, _lib.stream_ptr())
    if not split:
        _lib.check(run(), name)
        return grads, dSpeech, dStyle
    b.phase = 1
    _lib.check(run(), name + " (phase 1)")

    def finish():
        b.phase = 2
        _lib.check(run(), name + " (phase 2)")
        return hold, bws, grads, state, fb    # everything phase 2 reads stays referenced until it has been issued
    return grads, dSpeech, dStyle, finish


def loss_fwd_bwd(Y, rp, rq, WY, Wrp, Wrq, gaze, parents_i32, dt, mu, logvar, kl_weight, terms_out=None, kl_weight_dev=None, grad=True):
    """train.py:277-421 forward and gradient in one call (zeggs_loss_fwd_bwd) -> (loss = terms[0], (dY, dRp, dRq, dmu, dlogvar)).
    grad=False: the 19 terms only (dY == NULL: no backward kernels) -> (loss, None)."""
    l = _lib.lib()
    dev = Y.device
    B, T = Y.shape[0], Y.shape[1]
    f = _f32c
    Y, rp, rq, WY, Wrp, Wrq, gaze = f(Y), f(rp), f(rq), f(WY), f(Wrp), f(Wrq), f(gaze)
    losses = terms_out if terms_out is not None else torch.empty(19, dtype=torch.float32, device=dev)
    a = _lib.LossArgs(B=B, T=T, Z=(mu.shape[1] if mu is not None else 0), dt=dt, kl_weight=kl_weight)
    if kl_weight_dev is not None:          # device scalar (graph-replayable): overrides the by-value weight
        a.kl_weight_dev = kl_weight_dev.data_ptr()
    a.Y, a.root_pos, a.root_rot = Y.data_ptr(), rp.data_ptr(), rq.data_ptr()
    a.WY, a.W_root_pos, a.W_root_rot = WY.data_ptr(), Wrp.data_ptr(), Wrq.data_ptr()
    a.gaze_pos, a.parents, a.losses = gaze.data_ptr(), parents_i32.data_ptr(), losses.data_ptr()
    if grad:
        dY, dRp, dRq = torch.empty_like(Y), torch.empty_like(rp), torch.empty_like(rq)
        a.dY, a.dRootPos, a.dRootRot = dY.data_ptr(), dRp.data_ptr(), dRq.data_ptr()
    dmu = dlv = None
    if mu is not None:
        mu, logvar = f(mu), f(logvar)
        a.mu, a.logvar = mu.data_ptr(), logvar.data_ptr()
        if grad:
            dmu, dlv = torch.empty_like(mu), torch.empty_like(logvar)
            a.dmu, a.dlogvar = dmu.data_ptr(), dlv.data_ptr()
    wsb = l.zeggs_loss_workspace_bytes(B, T)
    ws = WS.get("loss", wsb, dev)
    a.workspace, a.workspace_bytes = ws.data_ptr(), wsb
    _lib.check(l.zeggs_loss_fwd_bwd(a, _lib.stream_ptr()), "zeggs_loss_fwd_bwd")
    return losses[0], ((dY, dRp, dRq, dmu, dlv) if grad else None)


def decoder_window(dec, root_pos0, root_rot0, pose0, gaze_pos, speech, style,
                   in_mean, in_std, out_mean, out_std, dt):
    if speech.device.type != "cuda":
        raise _lib.ZeggsError("zeggs_b200.Decoder runs on CUDA tensors only (no CPU fallback)")
    B = speech.shape[0]
    if B > 32 and resolve_engine(dec.hidden_size, dec.speech_encoding_size, dec.style_encoding_size, dec.film):
        # the tensor-core recurrence works on one 32-sample batch tile: independent windows -> run the tiles back to back
        outs = [decoder_window(dec, root_pos0[i:i + 32], root_rot0[i:i + 32], pose0[i:i + 32], gaze_pos[i:i + 32],
                               speech[i:i + 32], style[i:i + 32], in_mean, in_std, out_mean, out_std, dt)
                for i in range(0, B, 32)]
        return tuple(torch.cat(o, 0) for o in zip(*outs))
    needs_grad = torch.is_grad_enabled() and (
        any(p.requires_grad for p in dec.parameters()) or speech.requires_grad or style.requires_grad)
    if needs_grad:
        from .autograd import DecoderWindowFn
        return DecoderWindowFn.apply(dec, root_pos0, root_rot0, pose0, gaze_pos, speech, style,
                                     in_mean, in_std, out_mean, out_std, dt, *dec._weights())
    Y, rp, rq, _ = decoder_window_forward(dec, root_pos0, root_rot0, pose0, gaze_pos, speech, style,
                                          (in_mean, in_std, out_mean, out_std), dt, save=False)
    return Y, rp, rq


def sgemm(A, B, bias=None, act=0, trans_a=False, out=None, accumulate=False):
    """trans_a False: act(A[M,K] @ B[N,K]^T + bias);  True: A[K,M]^T @ B[K,N]."""
    if trans_a:
        K, M = A.shape
        N = B.shape[1]
    else:
        M, K = A.shape
        N = B.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=A.device)
    _lib.check(_lib.lib().zeggs_sgemm(int(trans_a), M, N, K, _lib.ptr(A), A.stride(0), _lib.ptr(B), B.stride(0),
                                     _lib.ptr(bias) if bias is not None else None, _lib.ptr(out), out.stride(0),
                                     act, int(accumulate), _lib.stream_ptr()), "zeggs_sgemm")
    return out


def split_bf16(x, want_lo=True, pad_to=8):
    """fp32 [rows, cols] -> (hi, lo) bf16 [rows, ld] with ld = cols rounded up to `pad_to` (zero padded)."""
    rows, cols = x.shape
    ld = (cols + pad_to - 1) // pad_to * pad_to
    hi = torch.empty((rows, ld), dtype=torch.bfloat16, device=x.device)
    lo = torch.empty((rows, ld), dtype=torch.bfloat16, device=x.device) if want_lo else None
    _lib.check(_lib.lib().zeggs_split_bf16(_lib.ptr(x), rows, cols, x.stride(0), hi.data_ptr(),
                                          lo.data_ptr() if want_lo else None, ld, _lib.stream_ptr()), "zeggs_split_bf16")
    return hi, lo


def tc_gemm(A_hi, B_hi, A_lo=None, B_lo=None, K=None, bias=None, act=0, out=None, accumulate=False):
    """tensor-core GEMM: act(A[M,K] @ B[N,K]^T + bias); bf16 operands (optionally split hi/lo), fp32 result."""
    M, N = A_hi.shape[0], B_hi.shape[0]
    K = K or A_hi.shape[1]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=A_hi.device)
    _lib.check(_lib.lib().zeggs_tc_gemm_bf16(
        M, N, K, A_hi.data_ptr(), A_lo.data_ptr() if A_lo is not None else None, A_hi.stride(0),
        B_hi.data_ptr(), B_lo.data_ptr() if B_lo is not None else None, B_hi.stride(0),
        _lib.ptr(bias) if bias is not None else None, _lib.ptr(out), out.stride(0), act, int(accumulate),
        _lib.stream_ptr()), "zeggs_tc_gemm_bf16")
    return out


# ---------------------------------------------------------------------------------------------- encoders
class DeviceSeed:
    """Dropout seed in DEVICE memory (zeggs_dropout_mask_dev): a captured CUDA graph of the train step draws fresh masks on every
    replay because `advance()` -- one in-graph increment -- is part of the step.  `salt` separates the masks within a step."""

    def __init__(self, device):
        self.t = torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).to(device)      # torch.manual_seed() -> reproducible runs
        self.salt = 0

    def advance(self):
        self.t.add_(1)
        self.salt = 0


_dev_seed = None


class device_seed:
    """Context: dropout masks drawn inside it use `seed` (a DeviceSeed) instead of the host generator."""

    def __init__(self, seed):
        self.seed = seed

    def __enter__(self):
        global _dev_seed
        self.prev, _dev_seed = _dev_seed, self.seed

    def __exit__(self, *exc):
        global _dev_seed
        _dev_seed = self.prev


def _drop_mask(shape, p, device):
    """Dropout mask (u >= p) / (1 - p) in one kernel; the seed comes from torch's CPU generator, so torch.manual_seed()
    makes training runs reproducible (and no device synchronisation is involved) -- or from a DeviceSeed inside a
    `device_seed` context (graph-replayable)."""
    out = torch.empty(shape, dtype=torch.float32, device=device)
    if _dev_seed is not None:
        _dev_seed.salt += 1
        _lib.check(_lib.lib().zeggs_dropout_mask_dev(out.data_ptr(), out.numel(), float(p), _dev_seed.t.data_ptr(), _dev_seed.salt,
                                                    _lib.stream_ptr()), "zeggs_dropout_mask_dev")
        return out
    seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    _lib.check(_lib.lib().zeggs_dropout_mask(out.data_ptr(), out.numel(), float(p), seed, _lib.stream_ptr()), "zeggs_dropout_mask")
    return out


def speech_enc_args(enc, x, masks, y, ws):
    w = [_f32c(p, x.device) for p in enc._weights()]
    H, Cin = w[0].shape[0], w[0].shape[1]
    O = w[2].shape[0]
    B, T = x.shape[0], x.shape[1]
    a = _lib.SpeechEncArgs(B=B, T=T, C_in=Cin, H=H, O=O, ctx=ctx_ptr(x.device))
    for n, t in zip(("W0", "b0", "W1", "b1", "W2", "b2"), w):
        setattr(a, n, t.data_ptr())
    a.x, a.y = x.data_ptr(), y.data_ptr()
    if masks is not None:
        a.mask0, a.mask1 = masks[0].data_ptr(), masks[1].data_ptr()
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    return a, w


def speech_encoder_masks(enc, x, masks=None):
    """Dropout multipliers of modules.py:263-270 (sampled in train mode unless injected)."""
    B, T = x.shape[0], x.shape[1]
    H, O = enc.layer0.weight.shape[0], enc.layer1.weight.shape[0]
    if masks is None and enc.training:
        masks = (_drop_mask((B, T, H), 0.2, x.device), _drop_mask((B, T, O), 0.2, x.device))
    if masks is not None:
        masks = tuple(_f32c(m, x.device) for m in masks)
    return masks


def speech_encoder_fwd(enc, x, masks):
    """zeggs_speech_enc_fwd -> (y [B,T,O], state for speech_encoder_bwd)."""
    if x.device.type != "cuda":
        raise _lib.ZeggsError("zeggs_b200.SpeechEncoder runs on CUDA tensors only (no CPU fallback)")
    l = _lib.lib()
    ensure_scratch(x.device)
    x = _f32c(x)
    weights = enc._weights()
    B, T = x.shape[0], x.shape[1]
    Cin, H, O = weights[0].shape[1], weights[0].shape[0], weights[2].shape[0]
    y = torch.empty((B, T, O), dtype=torch.float32, device=x.device)
    ws = torch.empty(l.zeggs_speech_enc_workspace_bytes(B, T, Cin, H, O), dtype=torch.uint8, device=x.device)
    a, keep = speech_enc_args(enc, x, masks, y, ws)
    _lib.check(l.zeggs_speech_enc_fwd(a, _lib.stream_ptr()), "zeggs_speech_enc_fwd")
    return y, (a, keep, x, masks, y, ws, weights)


def speech_encoder_bwd(state, dy, grads_out=None):
    a, keep, x, masks, y, ws, weights = state
    a.ctx = ctx_ptr(x.device)              # the lane this call is issued from (may differ from the forward's)
    dy = dy.contiguous().float()
    grads = _grad_targets(weights, grads_out)
    g = _lib.SpeechEncGrads(dy=dy.data_ptr())
    for n, t in zip(("dW0", "db0", "dW1", "db1", "dW2", "db2"), grads):
        setattr(g, n, t.data_ptr())
    _lib.check(_lib.lib().zeggs_speech_enc_bwd(a, g, _lib.stream_ptr()), "zeggs_speech_enc_bwd")
    return grads


def speech_encoder(enc, x, masks=None):
    if x.device.type != "cuda":
        raise _lib.ZeggsError("zeggs_b200.SpeechEncoder runs on CUDA tensors only (no CPU fallback)")
    from .autograd import SpeechEncoderFn
    return SpeechEncoderFn.apply(enc, x, speech_encoder_masks(enc, x, masks), *enc._weights())


_pe_cache = {}


def style_enc_args(enc, x, eps, masks, temperature, outs, ws):
    dev = x.device
    w = [_f32c(p, dev) for p in enc._weights()]
    B, T, Cin = x.shape
    Hs, E = w[0].shape[0], w[4].shape[0]
    nh = enc.encoder.blocks[0].attention.multi_head_attention.num_heads
    a = _lib.StyleEncArgs(B=B, T=T, C_in=Cin, H=Hs, E=E, nheads=nh, temperature=temperature, ctx=ctx_ptr(dev))
    for n, t in zip(_lib.STYLE_W, w):
        setattr(a, n, t.data_ptr())
    key = (T, E, str(dev))
    if key not in _pe_cache:
        _pe_cache[key] = enc.encoder.pos_enc.table(T).to(dev).contiguous()
    pe = _pe_cache[key]
    a.x, a.pe = x.data_ptr(), pe.data_ptr()
    if eps is not None:
        a.eps = eps.data_ptr()
    if masks is not None:
        for n in ("c1", "c2", "attn", "ao", "ff"):
            setattr(a, "mask_" + n, masks[n].data_ptr())
    if outs[1] is not None:
        a.mu, a.logvar = outs[1].data_ptr(), outs[2].data_ptr()
    a.z = outs[0].data_ptr()
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    return a, w + [pe]


def style_gru_args(enc, x, eps, temperature, outs, ws):
    dev = x.device
    w = [_f32c(p, dev) for p in enc._weights()]
    B, T, Cin = x.shape
    H, E = w[0].shape[0], w[12].shape[0]
    a = _lib.StyleEncGruArgs(B=B, T=T, C_in=Cin, H=H, E=E, temperature=temperature, ctx=ctx_ptr(dev))
    for n, t in zip(_lib.STYLE_GRU_W, w):
        setattr(a, n, t.data_ptr())
    a.x = x.data_ptr()
    if eps is not None:
        a.eps = eps.data_ptr()
    if outs[1] is not None:
        a.mu, a.logvar = outs[1].data_ptr(), outs[2].data_ptr()
    a.z = outs[0].data_ptr()
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    return a, w


def _style_outputs(enc, B, E, dev):
    """[z, mu, logvar] each [B, E/2] with the VAE; [z [B, E], None, None] without it (modules.py:303-304)."""
    if enc.use_vae:
        return [torch.empty((B, E // 2), dtype=torch.float32, device=dev) for _ in range(3)]
    return [torch.empty((B, E), dtype=torch.float32, device=dev), None, None]


def style_encoder_fwd(enc, x, eps, masks, temperature):
    """zeggs_style_enc_fwd (attn) / zeggs_style_enc_gru_fwd (gru) -> ([z, mu, logvar], state for style_encoder_bwd);
    mu = logvar = None without the VAE."""
    l = _lib.lib()
    x = _f32c(x)
    weights = enc._weights()
    B, T, Cin = x.shape
    if enc.encoder_type == "gru":
        H, E = weights[0].shape[0], weights[12].shape[0]
        outs = _style_outputs(enc, B, E, x.device)
        # 0 bytes when the library refuses the shape (hidden size, odd encoding with the VAE, batch): the call below says why
        nb = l.zeggs_style_enc_gru_workspace_bytes(B, T, Cin, H, E, int(bool(enc.use_vae)))
        ws = torch.empty(nb, dtype=torch.uint8, device=x.device)
        a, keep = style_gru_args(enc, x, eps, temperature, outs, ws)
        _lib.check(l.zeggs_style_enc_gru_fwd(a, _lib.stream_ptr()), "zeggs_style_enc_gru_fwd")
        return outs, ("gru", a, keep, x, eps, masks, outs, ws, weights)
    Hs, E = weights[0].shape[0], weights[4].shape[0]
    nh = enc.encoder.blocks[0].attention.multi_head_attention.num_heads
    outs = _style_outputs(enc, B, E, x.device)
    ws = torch.empty(l.zeggs_style_enc_workspace_bytes(B, T, Cin, Hs, E, nh), dtype=torch.uint8, device=x.device)
    a, keep = style_enc_args(enc, x, eps, masks, temperature, outs, ws)
    _lib.check(l.zeggs_style_enc_fwd(a, _lib.stream_ptr()), "zeggs_style_enc_fwd")
    return outs, ("attn", a, keep, x, eps, masks, outs, ws, weights)


def style_encoder_bwd(state, dz, dmu, dlv, grads_out=None):
    kind, a, keep, x, eps, masks, outs, ws, weights = state
    a.ctx = ctx_ptr(x.device)              # the lane this call is issued from (may differ from the forward's)
    g = _lib.StyleEncGruGrads() if kind == "gru" else _lib.StyleEncGrads()
    hold = []
    for n, t in (("dz", dz), ("dmu", dmu), ("dlogvar", dlv)):
        if t is not None:
            t = t.contiguous().float()
            hold.append(t)
            setattr(g, n, t.data_ptr())
    if outs[1] is None and dz is None:     # without the VAE z is the only output: the library needs its gradient
        dz = torch.zeros_like(outs[0])
        hold.append(dz)
        g.dz = dz.data_ptr()
    grads = _grad_targets(weights, grads_out)
    for n, t in zip(_lib.STYLE_GRU_W if kind == "gru" else _lib.STYLE_W, grads):
        setattr(g, "d" + n, t.data_ptr())
    if kind == "gru":
        _lib.check(_lib.lib().zeggs_style_enc_gru_bwd(a, g, _lib.stream_ptr()), "zeggs_style_enc_gru_bwd")
    else:
        _lib.check(_lib.lib().zeggs_style_enc_bwd(a, g, _lib.stream_ptr()), "zeggs_style_enc_bwd")
    return grads


def _draw_eps(shape, dev):
    if _dev_seed is not None:                               # device-seeded draw (replayable graph), else torch's generator
        eps = torch.empty(shape, dtype=torch.float32, device=dev)
        _dev_seed.salt += 1
        _lib.check(_lib.lib().zeggs_randn_dev(eps.data_ptr(), eps.numel(), _dev_seed.t.data_ptr(), _dev_seed.salt, _lib.stream_ptr()),
                   "zeggs_randn_dev")
        return eps
    return torch.randn(shape, device=dev)                   # modules.py:299


def style_encoder_prepare(enc, x, eps=None, masks=None):
    """VAE noise (modules.py:299; drawn only with use_vae) and dropout multipliers (attn encoder only: StyleEncoderGRU has no
    dropout; sampled in train mode unless injected) -> (eps or None, masks or None)."""
    dev = x.device
    ensure_scratch(dev)
    B, T = x.shape[0], x.shape[1]
    gru = enc.encoder_type == "gru"
    E = (enc.encoder.projection_layer.linear_layer.weight if gru else enc.encoder.convs[4].conv.weight).shape[0]
    if not enc.use_vae:
        eps = None
    elif eps is None:
        eps = _draw_eps((B, E // 2), dev)
    if gru:
        masks = None
    else:
        Hs = enc.encoder.convs[0].conv.weight.shape[0]
        nh = enc.encoder.blocks[0].attention.multi_head_attention.num_heads
        if masks is None and enc.training:
            masks = dict(c1=_drop_mask((B, T, Hs), 0.2, dev), c2=_drop_mask((B, T, E), 0.2, dev),
                         attn=_drop_mask((B, nh, T, T), 0.1, dev), ao=_drop_mask((B, T, E), 0.1, dev),
                         ff=_drop_mask((B, T, E), 0.1, dev))
        if masks is not None:
            masks = {k: _f32c(v, dev) for k, v in masks.items()}
    return (None if eps is None else _f32c(eps, dev)), masks


def style_encoder(enc, x, temperature=1.0, eps=None, masks=None):
    """-> (z, mu, logvar); (z, None, None) without the VAE, as modules.py:303-304 returns."""
    if x.device.type != "cuda":
        raise _lib.ZeggsError("zeggs_b200.StyleEncoder runs on CUDA tensors only (no CPU fallback)")
    from .autograd import StyleEncoderFn
    eps, masks = style_encoder_prepare(enc, x, eps, masks)
    out = StyleEncoderFn.apply(enc, x, eps, masks, temperature, *enc._weights())
    return tuple(out) if enc.use_vae else (out, None, None)


# ---------------------------------------------------------------------------------------------- pose -> BVH channel values
def pose_to_bvh_channels(root_pos, root_rot, lpos, ltxy, start_position=(0.0, 0.0, 0.0), start_rotation=(1.0, 0.0, 0.0, 0.0),
                         rebase=True, want_lrot=False):
    """Device post-step of generate.py:389-406 / utils.py:47-87: [N,T,...] pose tensors -> (positions [N,T,J,3], euler degrees
    [N,T,J,3] in 'zyx' channel order[, local rotations [N,T,J,4]]).  rebase: move the root's first frame to start_position /
    start_rotation, as write_bvh does when both are given."""
    if root_pos.device.type != "cuda":
        raise _lib.ZeggsError("pose_to_bvh_channels runs on CUDA tensors only (no CPU fallback)")
    rp, rq, lp, xy = _f32c(root_pos), _f32c(root_rot), _f32c(lpos), _f32c(ltxy)
    if rp.dim() == 2:
        rp, rq, lp, xy = rp[None], rq[None], lp[None], xy[None]
    N, T, J = lp.shape[0], lp.shape[1], lp.shape[2]
    pos = torch.empty((N, T, J, 3), dtype=torch.float32, device=lp.device)
    eul = torch.empty((N, T, J, 3), dtype=torch.float32, device=lp.device)
    lrot = torch.empty((N, T, J, 4), dtype=torch.float32, device=lp.device) if want_lrot else None
    a = _lib.PosePostArgs(N=N, T=T, J=J, rebase=int(bool(rebase)), root_pos=rp.data_ptr(), root_rot=rq.data_ptr(), lpos=lp.data_ptr(),
                          ltxy=xy.data_ptr(), positions=pos.data_ptr(), euler_deg=eul.data_ptr(),
                          lrot=lrot.data_ptr() if want_lrot else None)
    for i in range(3):
        a.start_pos[i] = float(start_position[i])
    for i in range(4):
        a.start_rot[i] = float(start_rotation[i])
    _lib.check(_lib.lib().zeggs_pose_to_bvh_channels(a, _lib.stream_ptr()), "zeggs_pose_to_bvh_channels")
    return (pos, eul, lrot) if want_lrot else (pos, eul)


# ---------------------------------------------------------------------------------------------- training-set construction
_EULER_AXIS = {"x": 0, "y": 1, "z": 2}
_TO_EULER = {"zyx": 0, "xzy": 1}


def _f64c(t, device):
    return torch.as_tensor(t).to(device=device, dtype=torch.float64).contiguous()


def anim_features(rotations, positions, parents, order, dt, spine2, hips, head, device="cuda"):
    """data_pipeline.py:90-228 on the device for one take: rotations [T,J,3] (degrees, BVH channel order `order`), positions [T,J,3],
    parents [J] -> dict of float32 CUDA tensors root_pos, root_rot, root_vel, root_vrt, lpos, ltxy, lvel, lvrt, gaze_pos, gaze_dir
    with the reference's shapes.  The arithmetic is float64."""
    dev = torch.device(device)
    rot, pos = _f64c(rotations, dev), _f64c(positions, dev)
    T, J = int(rot.shape[0]), int(rot.shape[1])
    par = torch.as_tensor(parents, dtype=torch.int32).to(dev).contiguous()
    shapes = dict(root_pos=(T, 3), root_rot=(T, 4), root_vel=(T, 3), root_vrt=(T, 3), lpos=(T, J, 3), ltxy=(T, J, 2, 3), lvel=(T, J, 3),
                  lvrt=(T, J, 3), gaze_pos=(T, 3), gaze_dir=(T, 3))
    out = {k: torch.empty(s, dtype=torch.float32, device=dev) for k, s in shapes.items()}
    _anim_call(rot, pos, par, order, dt, (spine2, hips, head), out, None)
    return out


def unrolled_quaternions(rotations, parents, order, device="cuda"):
    """quat.unroll(quat.from_euler(radians(rotations), order)) on the device: [T,J,3] degrees -> [T,J,4] float64 CUDA tensor."""
    dev = torch.device(device)
    rot = _f64c(rotations, dev)
    par = torch.as_tensor(parents, dtype=torch.int32).to(dev).contiguous()
    q = torch.empty((rot.shape[0], rot.shape[1], 4), dtype=torch.float64, device=dev)
    _anim_call(rot, None, par, order, 1.0, (0, 0, 0), None, q)
    return q


def _anim_call(rot, pos, par, order, dt, joints, out, quat_out):
    l = _lib.lib()
    T, J = int(rot.shape[0]), int(rot.shape[1])
    if rot.shape[2:] != (3,) or (pos is not None and tuple(pos.shape) != (T, J, 3)) or par.numel() != J:
        raise _lib.ZeggsError(f"anim_features: rotations {tuple(rot.shape)}, positions {None if pos is None else tuple(pos.shape)}, "
                              f"{par.numel()} parents")
    if len(order) != 3 or any(c not in _EULER_AXIS for c in order):
        raise _lib.ZeggsError(f"anim_features: Euler order {order!r}")
    wsb = l.zeggs_anim_features_workspace_bytes(T, J)
    ws = WS.get("anim_features", max(wsb, 1), rot.device)
    a = _lib.AnimFeaturesArgs(T=T, J=J, spine2=int(joints[0]), hips=int(joints[1]), head=int(joints[2]), dt=float(dt),
                              rotations=rot.data_ptr(), positions=pos.data_ptr() if pos is not None else None, parents=par.data_ptr(),
                              quat_out=quat_out.data_ptr() if quat_out is not None else None, workspace=ws.data_ptr(), workspace_bytes=wsb)
    for i, c in enumerate(order):
        a.order[i] = _EULER_AXIS[c]
    if out is not None:
        for k, t in out.items():
            setattr(a, k, t.data_ptr())
    _lib.check(l.zeggs_anim_features(a, _lib.stream_ptr()), "zeggs_anim_features")


def quat_to_euler_deg(q, order):
    """quat.normalize -> quat.to_euler(order) -> np.degrees on the device: [..., 4] float64 CUDA -> [..., 3] float64."""
    if order not in _TO_EULER:
        raise _lib.ZeggsError(f"to_euler converts to 'zyx' or 'xzy' only, not {order!r} (the reference raises NotImplementedError)")
    q = q.to(torch.float64).contiguous()
    e = torch.empty(q.shape[:-1] + (3,), dtype=torch.float64, device=q.device)
    _lib.check(_lib.lib().zeggs_quat_to_euler_deg(_lib.ptr(q), _lib.ptr(e), q.numel() // 4, _TO_EULER[order], _lib.stream_ptr()),
               "zeggs_quat_to_euler_deg")
    return e


def spline_resample(x, m):
    """griddata(arange(n), x, linspace(0, n-1, m), method="cubic") along dim 0 (data_pipeline.py:415-432): x [n] or [n, ...] float32 /
    float64 CUDA tensor -> [m] or [m, ...] float64."""
    if not x.is_cuda:
        raise _lib.ZeggsError("spline_resample runs on CUDA tensors only (no CPU fallback)")
    if x.dtype not in (torch.float32, torch.float64):
        x = x.to(torch.float64)
    x = x.contiguous()
    n = int(x.shape[0])
    C = int(x[0].numel()) if n else 1
    l = _lib.lib()
    y = torch.empty((int(m),) + tuple(x.shape[1:]), dtype=torch.float64, device=x.device)
    wsb = l.zeggs_spline_resample_workspace_bytes(n, C)
    ws = WS.get("spline", max(wsb, 1), x.device)
    a = _lib.SplineArgs(n=n, m=int(m), C=C, in_f64=int(x.dtype == torch.float64), x=x.data_ptr(), y=y.data_ptr(), workspace=ws.data_ptr(),
                        workspace_bytes=wsb)
    _lib.check(l.zeggs_spline_resample(a, _lib.stream_ptr()), "zeggs_spline_resample")
    return y


def masked_moments(groups, rows):
    """Per-channel mean and population std, and the pooled population std of each group, over the rows `rows` (data_pipeline.py:562-648).
    groups: list of float32 CUDA tensors [n_rows, ...] (flattened per row); rows: int index tensor.  -> (mean [sum widths] f64,
    std [sum widths] f64, group_std [len(groups)] f64), CUDA tensors."""
    if not 1 <= len(groups) <= _lib.MOMENTS_MAX_GROUPS:
        raise _lib.ZeggsError(f"masked_moments: {len(groups)} groups (1..{_lib.MOMENTS_MAX_GROUPS})")
    dev = groups[0].device
    srcs = [g.reshape(g.shape[0], -1).to(torch.float32).contiguous() for g in groups]
    rows = torch.as_tensor(rows, dtype=torch.int32).to(dev).contiguous()
    W = sum(int(s.shape[1]) for s in srcs)
    mean = torch.empty(W, dtype=torch.float64, device=dev)
    std = torch.empty(W, dtype=torch.float64, device=dev)
    gstd = torch.empty(len(srcs), dtype=torch.float64, device=dev)
    l = _lib.lib()
    wsb = l.zeggs_masked_moments_workspace_bytes(int(rows.numel()), W)
    ws = WS.get("moments", max(wsb, 1), dev)
    a = _lib.MomentsArgs(n_groups=len(srcs), rows=_lib.ptr(rows), n_sel=int(rows.numel()), mean=mean.data_ptr(), std=std.data_ptr(),
                         group_std=gstd.data_ptr(), workspace=ws.data_ptr(), workspace_bytes=wsb)
    for i, s in enumerate(srcs):
        a.src[i] = _lib.ptr(s)
        a.width[i] = int(s.shape[1])
    _lib.check(l.zeggs_masked_moments(a, _lib.stream_ptr()), "zeggs_masked_moments")
    return mean, std, gstd


def embedding_moments(X, group, n_groups):
    """float64 statistics of embedding rows (zeggs_embedding_moments): X [N, Z] float32 CUDA tensor, group [N] ints in 0..n_groups-1
    -> (mean [Z], cov [Z, Z] = Xc^T Xc / (N - 1), group_sum [n_groups, Z] f64, group_count [n_groups] int64), CUDA tensors.  Two
    passes and a fixed reduction order: the same input gives the same bits on every call."""
    if not X.is_cuda:
        raise _lib.ZeggsError("embedding_moments runs on CUDA tensors only (no CPU fallback)")
    if X.dim() != 2:
        raise _lib.ZeggsError(f"embedding_moments: X must be [N, Z], got shape {tuple(X.shape)}")
    N, Z, G = int(X.shape[0]), int(X.shape[1]), int(n_groups)
    dev = X.device
    X = X.to(torch.float32).contiguous()
    group = torch.as_tensor(group, device=dev).to(torch.int32).contiguous()
    if group.shape != (N,):
        raise _lib.ZeggsError(f"embedding_moments: group has shape {tuple(group.shape)}, X has {N} rows")
    if N and not (0 <= int(group.min()) and int(group.max()) < G):
        raise _lib.ZeggsError(f"embedding_moments: group ids must lie in 0..{G - 1}")
    l = _lib.lib()
    wsb = l.zeggs_embedding_moments_workspace_size(N, Z, G)   # 0 for a shape the call below refuses, naming the limit
    ws = WS.get("embedding_moments", max(wsb, 1), dev)
    f64 = dict(dtype=torch.float64, device=dev)
    mean, cov, gsum = torch.empty(Z, **f64), torch.empty((Z, Z), **f64), torch.empty((G, Z), **f64)
    gcount = torch.empty(G, dtype=torch.int64, device=dev)
    a = _lib.EmbeddingMomentsArgs(N=N, Z=Z, G=G, X=_lib.ptr(X), group=_lib.ptr(group), mean=mean.data_ptr(), cov=cov.data_ptr(),
                                  group_sum=gsum.data_ptr(), group_count=gcount.data_ptr(), workspace=ws.data_ptr(), workspace_bytes=wsb)
    _lib.check(l.zeggs_embedding_moments(a, _lib.stream_ptr()), "zeggs_embedding_moments")
    return mean, cov, gsum, gcount
