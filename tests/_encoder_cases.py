"""Inputs, float64 oracles and modelled faults of the speech encoder and the attention style encoder, shared by
tests/test_encoders_f64_cpu.py (no GPU: the bounds mean something) and tests/test_encoders_f64_gpu.py (the kernels meet them).

* Inputs: `synth` audio features / style examples normalised with the shipped stats, explicit dropout multipliers (0 or 1/(1-p)) so
  train mode is deterministic, an injected VAE eps and random cotangents.
* `run_oracle`: `oracle/model_oracle` with parameters, inputs, masks and eps cast to float64 (or float32), plus autograd.  The
  positional-encoding table stays the float32 table the module and the reference compute: at T = 3600 a float64 table differs from
  it by ~2e-4, which is not a kernel error.
* `run_restated`: the same networks restated from primitives, with two options `model_oracle` does not have:
  - `matched`: the weight gradients of the products the kernels run as ONE bf16 tensor-core pass under `fast_wgrad = 1`
    (dW = bf16(dpre)^T bf16(input), accumulated in float64; bias and input gradients keep full precision, as in the kernels);
  - `fault`: one modelled kernel error (FAULTS), to show that every bound is tight enough to see it.
  Without either it equals `model_oracle` to 1e-12 (tests/test_encoders_f64_cpu.py).
* `margined_style_params`: style parameters whose three ReLU sites (conv1, conv2, first feed-forward conv) keep every pre-activation
  well away from zero, so a gate cannot flip between fp32 and float64 and gradients can be compared tightly.
"""
import math
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn.functional as F

from tests._util import stats_tensors

SPEECH_SEED, STYLE_SEED = 21, 22
NHEADS = 4

# The tensor-core dispatch rule of gemm_f32_auto / conv_gemm_wgrad (csrc/tc_gemm.cu): a product runs on the tensor cores when the
# GEMM mode is not 0 and M*N*K >= 4e6 (and the scratch holds its operands); smaller products run on the fp32 SIMT kernel.
TC_MIN_MNK = 4.0e6

# Bounds (docstring of tests/test_encoders_f64_gpu.py; DESIGN.md §2).
FWD_TOL = 2e-5          # outputs: max-abs / max(1, max|ref|)
GRAD_TOL = 1e-4         # every gradient, fp32-grade settings: relative L2 per tensor

# (name the restatement gives the product, parameter key of its weight): the weight gradients that fast_wgrad = 1 runs in one bf16 pass
SPEECH_WGRADS = ["speech_encoder.layer0.weight", "speech_encoder.layer1.weight", "speech_encoder.layer2.weight"]
_SE = "style_encoder.encoder."
STYLE_WGRADS = [_SE + "convs.0.conv.weight", _SE + "convs.4.conv.weight", _SE + "blocks.0.feed_forward.convs.0.conv.weight",
                _SE + "blocks.0.feed_forward.convs.2.conv.weight", _SE + "blocks.0.attention.multi_head_attention.in_proj_weight",
                _SE + "blocks.0.attention.multi_head_attention.out_proj.weight"]
# Single-pass bf16 weight gradients vs the bf16-matched oracle, relative L2 per tensor.  Where the kernel's dpre and the float64 one
# round to different sides of a bf16 boundary the operand moves by a whole bf16 step, so the error grows with the error of dpre: the
# style conv1 gradient sits at the end of the whole backward (and behind two LayerNorm backwards), and the speech weights see the
# fewest rows.  The unmatched float64 oracle is >= 1.3e-4 (style), >= 2.3e-3 (style conv1, speech) away.
MATCHED_TOL = {**{k: 3.5e-4 for k in SPEECH_WGRADS}, **{k: 6e-5 for k in STYLE_WGRADS}, STYLE_WGRADS[0]: 2.5e-4}

FAULTS = {
    "speech": ["zero_pad", "taps_reversed", "cross_clip"],
    "style": ["cross_clip", "attn_scale_E", "heads_order", "attn_mask_T", "softmax_bwd_Pd", "pe_shift", "ln_unbiased", "pool_T-1",
              "mask_missing_bwd", "bias_rows8"],
}


# ---------------------------------------------------------------------------------------------- inputs
def speech_params():
    from zeggs_b200 import synth
    return {k: v for k, v in synth.make_params(H=64, seed=SPEECH_SEED).items() if k.startswith("speech_encoder.")}


def style_params(vae=True):
    """Style encoder of the shipped configs (hidden 512, E = 128 with the VAE, 64 without it)."""
    from zeggs_b200 import synth
    P = synth.make_params(H=64, seed=STYLE_SEED, style_embed=128 if vae else 64)
    return {k: v for k, v in P.items() if k.startswith("style_encoder.")}


def _mask(rs, shape, p):
    return torch.from_numpy(((rs.rand(*shape) >= p) / (1 - p)).astype(np.float32))


def speech_case(B, T, train=True, grads=True, seed=0):
    """x [B,T,81] normalised, masks (m0, m1) [B,T,64] or None, cotangent [B,T,64] or None."""
    from zeggs_b200 import synth
    st = synth.load_stats()
    x = (synth.make_audio_features(B, T, seed=seed) - st["audio_input_mean"]) / st["audio_input_std"]
    rs = np.random.RandomState(1000 + seed)
    masks = [_mask(rs, (B, T, 64), 0.2) for _ in range(2)] if train else None
    cots = [torch.from_numpy(rs.randn(B, T, 64).astype(np.float32))] if grads else None
    return SimpleNamespace(kind="speech", B=B, T=T, x=torch.from_numpy(x.astype(np.float32)), masks=masks, cots=cots, train=train)


def style_case(B, T, train=True, grads=True, vae=True, eps=True, temperature=1.3, seed=0):
    """x [B,T,1134] normalised, masks dict or None, eps [B,Z] or None (z = mu), cotangents of (z, mu, logvar) or of z alone."""
    from zeggs_b200 import synth
    st = stats_tensors()
    E = 128 if vae else 64
    x = (torch.from_numpy(synth.make_style_example(B, T, seed=seed)) - st["anim_input_mean"]) / st["anim_input_std"]
    rs = np.random.RandomState(2000 + seed)
    masks = None
    if train:
        masks = dict(c1=_mask(rs, (B, T, 512), 0.2), c2=_mask(rs, (B, T, E), 0.2), attn=_mask(rs, (B, NHEADS, T, T), 0.1),
                     ao=_mask(rs, (B, T, E), 0.1), ff=_mask(rs, (B, T, E), 0.1))
    Z = E // 2 if vae else E
    e = torch.from_numpy(rs.randn(B, Z).astype(np.float32)) if (vae and eps) else None
    cots = [torch.from_numpy(rs.randn(B, Z).astype(np.float32)) for _ in range(3 if vae else 1)] if grads else None
    return SimpleNamespace(kind="style", B=B, T=T, x=x.float(), masks=masks, eps=e, cots=cots, train=train, vae=vae,
                           temperature=temperature)


# The cases of tests/test_encoders_f64_gpu.py: id -> constructor arguments.
SPEECH_CASES = {
    "B32_T256": dict(B=32, T=256),                                  # the training shape
    **{f"B{B}_T{T}": dict(B=B, T=T) for B, T in [(1, 1), (1, 2), (2, 15), (2, 16), (3, 31)]},   # replicate padding of k = 31
    "B1_T9000_eval": dict(B=1, T=9000, train=False, grads=False),   # a 150 s clip
}
STYLE_CASES = {
    "B32_T384_vae": dict(B=32, T=384),                              # the training shape
    "B32_T384_novae": dict(B=32, T=384, vae=False),
    **{f"B{B}_T{T}": dict(B=B, T=T) for B, T in [(1, 1), (2, 127), (2, 128), (2, 129),    # narrow-N attention GEMMs at M >= 128
                                                   (4, 400), (8, 256), (5, 413)]},          # column reduction: 25, 32, 33 rows per block
    **{f"B1_T{T}_gen": dict(B=1, T=T, train=False, grads=False, eps=False) for T in (1000, 3600)},   # generate_gesture's whole clip
}


def make_case(kind, cid):
    kw = dict(SPEECH_CASES[cid] if kind == "speech" else STYLE_CASES[cid])
    kw.setdefault("seed", 10000 * kw["B"] + kw["T"])
    return speech_case(**kw) if kind == "speech" else style_case(**kw)


# ---------------------------------------------------------------------------------------------- model_oracle runner
def _leaves(P, dtype, grads):
    return {k: torch.from_numpy(np.asarray(v)).to(dtype).requires_grad_(grads) for k, v in P.items()}


def _finish(outs, Pt, cots):
    """-> (outputs, {key: gradient of sum(out * cot)} or None)."""
    if cots is None:
        return [o.detach() for o in outs], None
    keys = sorted(Pt)
    loss = sum((o * c.to(o.dtype)).sum() for o, c in zip(outs, cots))
    gs = torch.autograd.grad(loss, [Pt[k] for k in keys])
    return [o.detach() for o in outs], dict(zip(keys, gs))


def run_oracle(P, case, dtype=torch.float64):
    """model_oracle in `dtype` -> (outputs, gradients or None).  Speech: [y]; style: [z, mu, logvar] or [z] without the VAE."""
    from oracle import model_oracle as mo
    grads = case.cots is not None
    Pt = _leaves(P, dtype, grads)
    with torch.set_grad_enabled(grads):
        if case.kind == "speech":
            masks = None if case.masks is None else [m.to(dtype).transpose(1, 2) for m in case.masks]
            outs = [mo.speech_encoder(Pt, case.x.to(dtype), masks)]
        else:
            masks = None if case.masks is None else {k: v.to(dtype) for k, v in case.masks.items()}
            eps = None if case.eps is None else case.eps.to(dtype)
            outs = mo.style_encoder(Pt, case.x.to(dtype), eps=eps, temperature=case.temperature, masks=masks, use_vae=case.vae)
            outs = list(outs) if case.vae else [outs[0]]
    return _finish(outs, Pt, case.cots)


# ---------------------------------------------------------------------------------------------- restatement: primitives
def _bf16(t):
    return t.to(torch.bfloat16).double()


class _Linear(torch.autograd.Function):
    """y = x W^T + b over rows of x.  matched: dW = bf16(dy)^T bf16(x) accumulated in float64 (the single-pass weight-gradient
    product).  drop_rows: the bias gradient leaves out the last rows (a modelled reduction-tail fault)."""

    @staticmethod
    def forward(ctx, x, W, b, matched, drop_rows):
        ctx.save_for_backward(x, W)
        ctx.matched, ctx.drop_rows = matched, drop_rows
        return x @ W.T + b

    @staticmethod
    def backward(ctx, dy):
        x, W = ctx.saved_tensors
        d2, x2 = dy.reshape(-1, dy.shape[-1]), x.reshape(-1, x.shape[-1])
        dW = (_bf16(d2).T @ _bf16(x2)).to(dy.dtype) if ctx.matched else d2.T @ x2
        db = d2[:d2.shape[0] - ctx.drop_rows].sum(0)
        return dy @ W, dW, db, None, None


class _MaskMul(torch.autograd.Function):
    """h * mask; fault: the backward forgets the mask."""

    @staticmethod
    def forward(ctx, h, m, drop_in_bwd):
        ctx.save_for_backward(m)
        ctx.drop_in_bwd = drop_in_bwd
        return h * m

    @staticmethod
    def backward(ctx, g):
        (m,) = ctx.saved_tensors
        return (g if ctx.drop_in_bwd else g * m), None, None


class _SoftmaxDropout(torch.autograd.Function):
    """Pd = softmax(S) * mask; backward dS = P (dP - sum(dP P)), dP = dPd * mask.  fault: Pd where P belongs."""

    @staticmethod
    def forward(ctx, S, m, use_pd):
        P = torch.softmax(S, dim=-1)
        Pd = P * m
        ctx.save_for_backward(P, Pd, m)
        ctx.use_pd = use_pd
        return Pd

    @staticmethod
    def backward(ctx, g):
        P, Pd, m = ctx.saved_tensors
        Q = Pd if ctx.use_pd else P
        dP = g * m
        return Q * (dP - (dP * Q).sum(-1, keepdim=True)), None, None


class Opts:
    """matched: round the weight-gradient operands of products that meet the tensor-core rule; fault: one FAULTS entry.
    After a run, `rounded` lists (weight key, M, N, K) of every product whose weight gradient was rounded."""

    def __init__(self, matched=False, fault=None):
        self.matched, self.fault = matched, fault
        self.rounded = []


def _lin(x, W, b, o, key):
    K, N = W.shape[1], W.shape[0]
    M = x.numel() // K
    rnd = o.matched and M * N * K >= TC_MIN_MNK           # the weight-gradient product is [N, K] over M rows
    if rnd:
        o.rounded.append((key, M, N, K))
    drop = 8 if (o.fault == "bias_rows8" and key.endswith("feed_forward.convs.2.conv.weight")) else 0
    return _Linear.apply(x, W, b, rnd, drop)


def _conv(x, W, b, o, key, replicate):
    """'same' 1-D convolution of x [B,T,C] (channels last) as unfold + GEMM: col[(b,t)][c*k + kk] = x[b][t + kk - k//2][c]."""
    B, T, C = x.shape
    N, _, k = W.shape
    pad = k // 2
    if o.fault == "taps_reversed":
        W = W.flip(-1)
    mode = "replicate" if (replicate and o.fault != "zero_pad") else "constant"
    if o.fault == "cross_clip":          # the batch read as one long sequence: padding only at its two ends
        xp = F.pad(x.reshape(1, B * T, C).transpose(1, 2), (pad, pad), mode=mode).transpose(1, 2)
        col = xp.unfold(1, k, 1).reshape(B, T, C * k)
    else:
        xp = F.pad(x.transpose(1, 2), (pad, pad), mode=mode).transpose(1, 2)
        col = xp.unfold(1, k, 1).reshape(B, T, C * k)
    return _lin(col, W.reshape(N, C * k), b, o, key)


def _drop(h, masks, name, o):
    if masks is None:
        return h
    m = masks[name].to(h.dtype)
    return _MaskMul.apply(h, m, o.fault == "mask_missing_bwd" and name == "ao")


def _ln(x, g, b, o):
    if o.fault == "ln_unbiased":
        mu = x.mean(-1, keepdim=True)
        return (x - mu) / torch.sqrt(x.var(-1, unbiased=True, keepdim=True) + 1e-5) * g + b
    return F.layer_norm(x, (x.shape[-1],), g, b)


# ---------------------------------------------------------------------------------------------- restatement: the two encoders
def speech_forward(P, x, masks, o):
    """modules.py:265-272 with x [B,T,81] and masks [B,T,64] (channels last, as the module takes them)."""
    g = lambda k: P["speech_encoder." + k]
    W0 = g("layer0.weight")
    h = F.elu(_lin(x, W0.reshape(W0.shape[0], -1), g("layer0.bias"), o, "speech_encoder.layer0.weight"))
    h = _drop(h, None if masks is None else dict(m0=masks[0]), "m0", o)
    h = F.elu(_conv(h, g("layer1.weight"), g("layer1.bias"), o, "speech_encoder.layer1.weight", replicate=True))
    h = _drop(h, None if masks is None else dict(m1=masks[1]), "m1", o)
    return F.elu(_lin(h, g("layer2.weight"), g("layer2.bias"), o, "speech_encoder.layer2.weight"))


def style_forward(P, x, eps, temperature, masks, vae, o, internals=None):
    """modules.py:289-304, 391-420 -> [z, mu, logvar] or [z].  internals: dict that receives the three ReLU pre-activations."""
    from oracle import model_oracle as mo
    g = lambda k: P[_SE + k]
    B, T, _ = x.shape
    pre = internals if internals is not None else {}
    pre["c1"] = _conv(x, g("convs.0.conv.weight"), g("convs.0.conv.bias"), o, _SE + "convs.0.conv.weight", replicate=False)
    h = _drop(_ln(F.relu(pre["c1"]), g("convs.2.weight"), g("convs.2.bias"), o), masks, "c1", o)
    pre["c2"] = _conv(h, g("convs.4.conv.weight"), g("convs.4.conv.bias"), o, _SE + "convs.4.conv.weight", replicate=False)
    h = _drop(_ln(F.relu(pre["c2"]), g("convs.6.weight"), g("convs.6.bias"), o), masks, "c2", o)
    E = h.shape[-1]
    shift = 1 if o.fault == "pe_shift" else 0
    x0 = h + mo.positional_encoding(T + shift, E)[shift:].to(h.dtype)[None]
    a = "blocks.0.attention."
    qkv = _lin(x0, g(a + "multi_head_attention.in_proj_weight"), g(a + "multi_head_attention.in_proj_bias"), o,
               _SE + a + "multi_head_attention.in_proj_weight")
    d = E // NHEADS
    if o.fault == "heads_order":         # heads interleaved: head j gets channels j, j + 4, ...
        split = lambda t: t.reshape(B, T, d, NHEADS).permute(0, 3, 1, 2)
        merge = lambda t: t.permute(0, 2, 3, 1).reshape(B, T, E)
    else:
        split = lambda t: t.reshape(B, T, NHEADS, d).transpose(1, 2)
        merge = lambda t: t.transpose(1, 2).reshape(B, T, E)
    q, k, v = (split(t) for t in qkv.split(E, dim=-1))
    scale = 1.0 / math.sqrt(E if o.fault == "attn_scale_E" else d)
    s = torch.matmul(q * scale, k.transpose(-1, -2))
    if masks is None:
        p = torch.softmax(s, dim=-1)
    else:
        m = masks["attn"].to(s.dtype)
        if o.fault == "attn_mask_T":
            m = m.transpose(-1, -2)
        p = _SoftmaxDropout.apply(s, m, o.fault == "softmax_bwd_Pd")
    att = _lin(merge(torch.matmul(p, v)), g(a + "multi_head_attention.out_proj.weight"), g(a + "multi_head_attention.out_proj.bias"),
               o, _SE + a + "multi_head_attention.out_proj.weight")
    x1 = _ln(_drop(att, masks, "ao", o) + x0, g(a + "layer_norm.weight"), g(a + "layer_norm.bias"), o)
    f = "blocks.0.feed_forward."
    pre["f1"] = _conv(x1, g(f + "convs.0.conv.weight"), g(f + "convs.0.conv.bias"), o, _SE + f + "convs.0.conv.weight", replicate=False)
    y = _conv(F.relu(pre["f1"]), g(f + "convs.2.conv.weight"), g(f + "convs.2.conv.bias"), o, _SE + f + "convs.2.conv.weight",
              replicate=False)
    x2 = _ln(_drop(y, masks, "ff", o) + x1, g(f + "layer_norm.weight"), g(f + "layer_norm.bias"), o)
    pooled = x2.sum(1) / float(T - 1 if o.fault == "pool_T-1" else T)
    if not vae:
        return [pooled]
    Z = pooled.shape[1] // 2
    mu, logvar = pooled[:, :Z], pooled[:, Z:]
    z = mu if eps is None else mu + eps * torch.exp(0.5 * logvar) / temperature
    return [z, mu, logvar]


def run_restated(P, case, dtype=torch.float64, matched=False, fault=None):
    """The restatement in `dtype` -> (outputs, gradients or None, Opts of the run)."""
    o = Opts(matched, fault)
    grads = case.cots is not None
    Pt = _leaves(P, dtype, grads)
    with torch.set_grad_enabled(grads):
        x = case.x.to(dtype)
        if case.kind == "speech":
            outs = [speech_forward(Pt, x, None if case.masks is None else [m.to(dtype) for m in case.masks], o)]
        else:
            eps = None if case.eps is None else case.eps.to(dtype)
            outs = style_forward(Pt, x, eps, case.temperature, case.masks, case.vae, o)
    outs, gs = _finish(outs, Pt, case.cots)
    return outs, gs, o


# ---------------------------------------------------------------------------------------------- ReLU gate margins
RELU_SITES = [("c1", "convs.0.conv.bias"), ("c2", "convs.4.conv.bias"), ("f1", "blocks.0.feed_forward.convs.0.conv.bias")]
GATE_SHIFT = 4.0          # bias = -mean +- GATE_SHIFT * std of the bias-free pre-activation, sign alternating by channel
GATE_RATIO = 16.0         # required: min |pre-activation| >= GATE_RATIO x the fp32 pre-activation error of its layer


def _style_internals(P, case, dtype):
    pre = {}
    Pt = _leaves(P, dtype, False)
    with torch.no_grad():
        eps = None if case.eps is None else case.eps.to(dtype)
        style_forward(Pt, case.x.to(dtype), eps, case.temperature, case.masks, case.vae, Opts(), internals=pre)
    return pre


def margined_style_params(P, case):
    """Style parameters with every ReLU pre-activation of `case` (its input and masks) far from zero: layer by layer in float64, each
    ReLU conv's bias is set per channel to -mean +- 4 std of its bias-free pre-activation (std over all rows; over the whole layer
    when there is one row), + on even channels and - on odd ones: about half the channels almost always pass, half almost never."""
    P = dict(P)
    for site, bkey in RELU_SITES:
        P[_SE + bkey] = np.zeros_like(P[_SE + bkey])
        z = _style_internals(P, case, torch.float64)[site]
        z = z.reshape(-1, z.shape[-1])
        mean = z.mean(0)
        std = z.std(0) if z.shape[0] > 1 else z.std().expand_as(mean)
        sign = torch.ones_like(mean)
        sign[1::2] = -1.0
        P[_SE + bkey] = (-mean + sign * GATE_SHIFT * std).float().numpy()
    return P


def gate_margins(P, case):
    """-> {site: (min |pre-activation| in float64, max |fp32 - float64| of the pre-activation)} at the three ReLU sites."""
    p64, p32 = _style_internals(P, case, torch.float64), _style_internals(P, case, torch.float32)
    return {s: (float(p64[s].abs().min()), float((p32[s].double() - p64[s]).abs().max())) for s, _ in RELU_SITES}


# ---------------------------------------------------------------------------------------------- comparisons
def fwd_err(got, ref):
    """max-abs error / max(1, max|ref|)."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    assert got.shape == ref.shape and bool(torch.isfinite(got).all())
    return float((got - ref).abs().max()) / max(1.0, float(ref.abs().max()))


def rel_l2(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    assert got.shape == ref.shape and bool(torch.isfinite(got).all())
    return float((got - ref).norm()) / max(float(ref.norm()), 1e-30)


def errors(outs, grads, ref_outs, ref_grads, rounded=()):
    """-> [(name, error, bound)] for every output (FWD_TOL) and gradient (GRAD_TOL; MATCHED_TOL for the keys in `rounded`)."""
    res = [(f"out{i}", fwd_err(o, r), FWD_TOL) for i, (o, r) in enumerate(zip(outs, ref_outs))]
    if grads is not None:
        for k in sorted(ref_grads):
            res.append((k, rel_l2(grads[k], ref_grads[k]), MATCHED_TOL[k] if k in rounded else GRAD_TOL))
    return res
