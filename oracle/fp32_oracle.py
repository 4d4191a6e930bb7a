"""CPU restatement of what the fp32 decoder engine (engine 0: csrc/decoder_fwd.cu, csrc/decoder_bwd.cu) computes, normal and FiLM.

TEST INFRASTRUCTURE ONLY.  run() evaluates the decoder window and the gradients of sum(out * cot) the way the engine splits the work:

  * the recurrence (every per-step product, gate, ELU, FiLM modulation and the root integration) is plain arithmetic in `dtype`;
  * the weight and bias gradients of the recurrent decoder are formed afterwards from the per-step histories, as phase 2 of the
    backward does: dW = sum over slots t = 1..T-1 of g(t)^T x(t), db = the row sums of g(t);
  * gemm=True models GEMM mode 1: the products that go through the tensor-core front end (CellStateEncoder forward and input
    gradient, FiLM predictors, and -- for the normal decoder -- the weight gradients of wgrad_gemms) are split-bf16: both operands are
    split into a bf16 hi and a bf16 lo part, lo * lo is dropped and the rest is evaluated in float32.  gemm=False is GEMM mode 0
    (every product plain, the SIMT kernels).

With dtype = float64 and no perturbation, run() equals autograd through model_oracle.decoder_forward / film_oracle.decoder_forward_film
(tests/test_decoder_fp32_oracle_cpu.py).  `perturb` injects one small, plausible kernel fault (PERTURBATIONS), to show that the
tolerances below catch what a subtly wrong kernel would do.
"""
import torch
import torch.nn.functional as F

from oracle import model_oracle as mo

P_IN, P_OUT = 1134, 1131
NAMES = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt"]

# Tolerances of the fp32 engine against the float64 oracle (model_oracle / film_oracle), for both decoders.
# Forward: per pose-channel group, max-abs error <= FP32_FWD_TOL * max(1, max|ref|) in de-normalised units.
# Gradients: per parameter / dSpeech / dStyle tensor, max-abs error <= tol * max|ref|, with FP32_GRAD_TOL in GEMM mode 0 (SIMT weight
# gradients) and FP32_GEMM_GRAD_TOL in GEMM mode 1 (split-bf16 products).  tests/test_decoder_fp32_oracle_cpu.py shows that a
# float32 evaluation meets them with at least 4x headroom and that each modelled fault exceeds them.
FP32_FWD_TOL = 3e-5
FP32_GRAD_TOL = 2e-5
FP32_GEMM_GRAD_TOL = 5e-5
# the bounds the older tests used, for comparison: forward / max-abs gradient of the normal decoder, forward / rel-L2 gradient of FiLM
OLD_FWD_TOL, OLD_GRAD_TOL, OLD_FILM_TOL = 2e-4, 3e-4, 2e-3

PERTURBATIONS = ("kchunk", "zcols", "bhn_outside", "stale_h1", "tile_rootv",                         # forward
                 "drop_carry", "wgrad_shift", "wgrad_lastslot", "bias_slot0", "dstyle_cse",  # backward
                 "film_gamma", "film_beta_prev")                                             # FiLM


def units_per_cta(H):
    """U of csrc/decoder_common.cuh pick_U: CTA c owns hidden units c*U .. c*U+U-1 of every gate block."""
    return 4 if H % 4 == 0 and H // 4 <= 132 else 8


def bad_units(H):
    """The hidden units of the CTA the perturbations hit (the middle one)."""
    U = units_per_cta(H)
    c = (H // U) // 2
    return torch.arange(c * U, c * U + U)


def _bf16(x):
    return x.to(torch.bfloat16).to(torch.float32)


def split_mm(a, b):
    """a @ b as the split-bf16 tensor-core GEMMs form it: hi and lo parts of both operands, lo * lo dropped, float32 accumulation."""
    a, b = a.float(), b.float()
    ah, bh = _bf16(a), _bf16(b)
    al, bl = _bf16(a - ah), _bf16(b - bh)
    return ah @ bh + (ah @ bl + al @ bh)


def _front_end(split, M, N, K):
    """True when the GEMM front end runs an [M, K] x [K, N] product on the tensor cores (plan_tc_operands: >= 4e6 multiply-adds)."""
    return split and float(M) * N * K >= 4.0e6


def _mm(a, b, split):
    return split_mm(a, b).to(a.dtype) if split else a @ b


class _Front(torch.autograd.Function):
    """y = x W^T + b through the GEMM front end: forward and input gradient split-bf16 when large enough in GEMM mode 1, weight gradient
    split or SIMT as `wsplit` says."""

    @staticmethod
    def forward(ctx, x, W, b, split, wsplit):
        ctx.save_for_backward(x, W)
        ctx.split, ctx.wsplit = split, wsplit
        y = _mm(x, W.T, _front_end(split, x.shape[0], W.shape[0], x.shape[1]))
        return y + b if b is not None else y

    @staticmethod
    def backward(ctx, g):
        x, W = ctx.saved_tensors
        dx = _mm(g, W, _front_end(ctx.split, g.shape[0], W.shape[1], g.shape[1]))
        dW = _mm(g.T, x, _front_end(ctx.wsplit, g.shape[1], x.shape[1], g.shape[0]))
        return dx, dW, g.sum(0), None, None


class _Rec(torch.autograd.Function):
    """One product of the recurrence, y = x W^T + b, plain.  Its backward passes dx = g W on and records (g, x) of this step for the
    weight / bias gradients formed after the recurrence; W and b get no gradient here."""

    @staticmethod
    def forward(ctx, x, W, b, tape, key, t):
        ctx.save_for_backward(x, W)
        ctx.tape, ctx.key, ctx.t = tape, key, t
        return x @ W.T + b

    @staticmethod
    def backward(ctx, g):
        x, W = ctx.saved_tensors
        ctx.tape.setdefault(ctx.key, {})[ctx.t] = (g, x)
        return g @ W, None, None, None, None, None


def _gru(gi, gh, h, b_hn=None, units=None, carry=True):
    """nn.GRU cell on precomputed products (gate order r, z, n).  units: b_hn (part of gh) is added outside r * (.) for these units.
    carry=False: the dh * z carry to h(t-1) is dropped from the backward."""
    H = h.shape[-1]
    r = torch.sigmoid(gi[:, :H] + gh[:, :H])
    z = torch.sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
    pre = gi[:, 2 * H:] + r * gh[:, 2 * H:]
    if units is not None:
        pre = pre.clone()
        pre[:, units] = pre[:, units] + (1.0 - r[:, units]) * b_hn[units]
    n = torch.tanh(pre)
    return (1.0 - z) * n + z * (h if carry else h.detach())


def _window(Pt, first, gaze, sp, sy, st, film, perturb, gemm, tape):
    """Forward of one window; returns the 8-tuple of model_oracle.decoder_forward."""
    im, is_, om, os_, dt = st
    pr, pc = "decoder.recurrent_decoder.", "decoder.cell_state_encoder."
    g = lambda k: Pt[pr + k]
    H = g("layer0.weight").shape[0]
    B, T = sp.shape[0], sp.shape[1]
    nj = first[4].shape[1]
    units = bad_units(H)
    O = [[t] for t in first]
    x0 = mo.vectorize_input(*first, gaze[:, 0], im, is_)
    # CellStateEncoder (decoder_fwd_prologue: three front-end GEMMs; backward: SIMT weight gradients, front-end input gradients)
    s0 = sy[:, 0].detach() if perturb == "dstyle_cse" else sy[:, 0]
    c = lambda k: Pt[pc + k]
    h = F.elu(_Front.apply(torch.cat([x0, s0], -1), c("layer0.weight"), c("layer0.bias"), gemm, False))
    h = F.elu(_Front.apply(h, c("layer1.weight"), c("layer1.bias"), gemm, False))
    o = _Front.apply(h, c("layer2.weight"), c("layer2.bias"), gemm, False)
    h0, h1 = o[:, :H], o[:, H:]
    h1_prev = h1
    if film:                                          # the predictors of every frame: two front-end GEMMs over B*T rows
        Z = sy.shape[-1]
        flat = sy.reshape(B * T, Z)
        gam = _Front.apply(flat, g("gammas_predictor.linear_layer.weight"), g("gammas_predictor.linear_layer.bias"), gemm, gemm)
        bet = _Front.apply(flat, g("betas_predictor.linear_layer.weight"), g("betas_predictor.linear_layer.bias"), gemm, gemm)
        gam, bet = gam.reshape(B, T, 2 * H), bet.reshape(B, T, 2 * H)
    W_hh1 = g("layer1.weight_hh_l1")
    if perturb == "kchunk":                           # the CTA's gate rows of W_hh1 miss one 16-row k-chunk
        k0 = 16 * min(1, H // 16 - 1)
        keep = torch.ones_like(W_hh1)
        keep[torch.cat([units + q * H for q in range(3)]), k0:k0 + 16] = 0.0
        W_hh1 = W_hh1 * keep
    if perturb == "zcols":                            # the CTA's z-gate rows of W_hh1 miss the last 4 k-columns
        keep = torch.ones_like(W_hh1)
        keep[units + H, H - 4:] = 0.0
        W_hh1 = W_hh1 * keep
    for t in range(1, T):
        pose = mo.vectorize_input(*[o_[-1] for o_ in O], gaze[:, t], im, is_)
        u = torch.cat([pose, sp[:, t]] + ([] if film else [sy[:, t]]), -1)
        a = F.elu(_Rec.apply(u, g("layer0.weight"), g("layer0.bias"), tape, "layer0", t))
        if film:
            tb = t - 1 if perturb == "film_beta_prev" else t
            a = a * (1.0 + gam[:, t, :H]) + bet[:, tb, :H]
        v = torch.cat([a, u], -1)
        gi0 = _Rec.apply(v, g("layer1.weight_ih_l0"), g("layer1.bias_ih_l0"), tape, "l0_ih", t)
        gh0 = _Rec.apply(h0, g("layer1.weight_hh_l0"), g("layer1.bias_hh_l0"), tape, "l0_hh", t)
        h0n = _gru(gi0, gh0, h0)
        gi1 = _Rec.apply(h0n, g("layer1.weight_ih_l1"), g("layer1.bias_ih_l1"), tape, "l1_ih", t)
        gh1 = _Rec.apply(h1, W_hh1, g("layer1.bias_hh_l1"), tape, "l1_hh", t)
        if perturb == "stale_h1" and t >= 2:          # the CTA's rows read h1 from two steps back
            rows = torch.cat([units + q * H for q in range(3)])
            gh1 = gh1.clone()
            gh1[:, rows] = h1_prev @ W_hh1[rows].T + g("layer1.bias_hh_l1")[rows]
        h1n = _gru(gi1, gh1, h1, g("layer1.bias_hh_l1")[2 * H:], units if perturb == "bhn_outside" else None,
                   carry=not (perturb == "drop_carry" and t == T // 2))
        if film:
            gm = 1.0 + gam[:, t, H:]
            if perturb == "film_gamma":               # the CTA's layer-2 units scale by gamma instead of 1 + gamma
                gm = gm.clone()
                gm[:, units] = gm[:, units] - 1.0
            cm = F.elu(_Rec.apply(h1n, g("layer2.weight"), g("layer2.bias"), tape, "layer2", t)) * gm + bet[:, tb, H:]
            y = _Rec.apply(cm, g("layer3.weight"), g("layer3.bias"), tape, "layer3", t)
        else:
            y = _Rec.apply(h1n, g("layer2.weight"), g("layer2.bias"), tape, "layer2", t)
        new = mo.devectorize_output(y, O[0][-1], O[1][-1], dt, om, os_, nj)
        if perturb == "tile_rootv" and B > 32:        # the second batch tile integrates the root with the first tile's velocities
            yr = torch.cat([y[:32], y[:B - 32]], 0)
            new = mo.devectorize_output(yr, O[0][-1], O[1][-1], dt, om, os_, nj)[:2] + new[2:]
        for k in range(8):
            O[k].append(new[k])
        h1_prev = h1
        h0, h1 = h0n, h1n
    return tuple(torch.stack(o_, dim=1) for o_ in O)


# recurrence product -> (weight, bias) state-dict suffix
_REC = {"layer0": ("layer0.weight", "layer0.bias"), "l0_ih": ("layer1.weight_ih_l0", "layer1.bias_ih_l0"),
        "l0_hh": ("layer1.weight_hh_l0", "layer1.bias_hh_l0"), "l1_ih": ("layer1.weight_ih_l1", "layer1.bias_ih_l1"),
        "l1_hh": ("layer1.weight_hh_l1", "layer1.bias_hh_l1"), "layer2": ("layer2.weight", "layer2.bias"),
        "layer3": ("layer3.weight", "layer3.bias")}


def run(P, win, speech, style, cot, stats, dtype=torch.float64, film=False, perturb=None, gemm=False, grads=True):
    """The window of the fp32 engine and the gradients of sum(out * cot).
    P: the decoder's state dict (reference names, numpy or tensors); win: {name: [B,T,...]} windows (frame 0 and gaze_pos used);
    speech [B,T,S], style [B,T,Z]; cot: 8 cotangents; stats: (in_mean, in_std, out_mean, out_std, dt).
    -> (8 outputs, {state-dict name / "speech" / "style": gradient}) in `dtype`; grads=False -> (outputs, None)."""
    assert perturb is None or perturb in PERTURBATIONS, perturb
    cast = lambda x: torch.as_tensor(x).to(dtype)
    Pt = {k: cast(v).requires_grad_(grads) for k, v in P.items() if k.startswith("decoder.")}
    sp, sy = cast(speech).requires_grad_(grads), cast(style).requires_grad_(grads)
    first = [cast(win[n][:, 0]) for n in NAMES]
    st = tuple(cast(s) for s in stats[:4]) + (float(stats[4]),)
    tape = {}
    with torch.set_grad_enabled(grads):
        out = _window(Pt, first, cast(win["gaze_pos"]), sp, sy, st, film, perturb, gemm, tape)
    if not grads:
        return [o.detach() for o in out], None
    loss = sum((o * cast(c)).sum() for o, c in zip(out, cot))
    keys = sorted(Pt)
    res = {}
    if loss.requires_grad:
        gs = torch.autograd.grad(loss, [Pt[k] for k in keys] + [sp, sy], allow_unused=True)
        res = {k: gv for k, gv in zip(keys + ["speech", "style"], gs) if gv is not None}
    # phase 2: weight / bias gradients of the recurrence from the per-step histories (slots t = 1 .. T-1)
    T = sp.shape[1]
    wsplit = gemm and not film                        # wgrad_gemms (normal decoder, GEMM mode 1); FiLM: always SIMT
    for key, (wn, bn) in _REC.items():
        steps = tape.get(key, {})
        ts = [t for t in range(1, T) if t in steps]
        if not ts:
            continue
        gs_ = [steps[t][0] for t in ts]
        xs = [steps[t][1] for t in ts]
        if perturb == "wgrad_shift" and key == "l1_ih":        # x operand one slot early: h0(t-1) with the gate gradients of t
            xs = [tape["l0_hh"][t][1] for t in ts]
        if perturb == "wgrad_lastslot" and key == "l1_hh":     # the contraction misses the last slot
            gs_, xs = gs_[:-1], xs[:-1]
        G, X = torch.cat(gs_, 0), torch.cat(xs, 0)
        dW = split_mm(G.T, X).to(dtype) if wsplit else G.T @ X
        db = G.sum(0)
        if perturb == "bias_slot0" and key == "l0_ih":         # the row sum starts at slot 0, which holds a stale copy of slot 1
            db = db + steps[1][0].sum(0)
        res["decoder.recurrent_decoder." + wn] = dW
        res["decoder.recurrent_decoder." + bn] = db
    for k in keys + ["speech", "style"]:
        if k not in res:
            res[k] = torch.zeros_like(Pt[k] if k in Pt else (sp if k == "speech" else sy))
    return [o.detach() for o in out], {k: v.detach() for k, v in res.items()}


def forward_errors(out, ref):
    """Per output group: max-abs error / max(1, max|ref|)."""
    res = {}
    for n, o, q in zip(NAMES, out, ref):
        o, q = o.detach().double().cpu(), q.detach().double().cpu()
        res[n] = float((o - q).abs().max()) / max(1.0, float(q.abs().max()))
    return res


def grad_errors(grads, ref):
    """Per gradient: max-abs error / max|ref| (0 when both are exactly zero)."""
    res = {}
    for k, r in ref.items():
        a, r = grads[k].detach().double().cpu(), r.detach().double().cpu()
        err, sc = float((a - r).abs().max()), float(r.abs().max())
        res[k] = err / sc if sc > 0 else (0.0 if err == 0 else float("inf"))
    return res


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm()) / max(float(b.norm()), 1e-30)
