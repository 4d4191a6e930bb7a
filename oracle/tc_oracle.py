"""CPU restatement (float64 PyTorch) of what the tensor-core decoder engine (engine 1) computes.

TEST INFRASTRUCTURE ONLY.  decoder_forward_tc() has the signature of model_oracle.decoder_forward and restates the FOLDED recurrence
of csrc/decoder_fwd_tc.cu (header; the algebra is checked by tests/test_fold_algebra_cpu.py), built from model_oracle's blocks:

  [pre_a ; gi0](1)   = Wx x(1) + cond(1) + [b0 ; b_ih0]                          x(1) = the given pose (fp32 XP row)
  [pre_a ; gi0](t+1) = Mfold h1(t) + cfold + Wx[:, 1131:1134] gaze(t+1) + cond(t+1) + [b0 ; b_ih0]
  root(t)            integrated from the six fold-chain rows y(t)[0:6] = W2[0:6] h1(t) + b2[0:6]
  Y(t)               = one layer-2 product over the h1 history

bf16=False: plain float64 arithmetic -- outputs and autograd gradients equal model_oracle.decoder_forward's (tests/test_tc_oracle_cpu.py).
bf16=True: every MMA operand is rounded to bf16 (round to nearest even) exactly where the kernels round; everything else stays float64.

Forward rounding points (decoder_fwd_tc.cu):
  * packed weight slices, __float2bfloat16_rn at :159 / :163 of pack_decoder_tc_kernel: W_ih0[:, :H], W_hh0, W_ih1, W_hh1 (:148-151),
    Mfold (:146) and the root rows W2[0:6] (:147) of the fold chain;
  * Mfold is rounded after its fp32-grade product (three-pass split-bf16 GEMM under a fast_wgrad = 0 copy of the context, :655-657, :679);
  * w2b = bf16(W2) for the batched layer 2 (zeggs_split_bf16, :670; product at :753);
  * activation images a(t) (:483), h0(t) (:526), h1(t) (:566) and the bf16 h1 history of the layer-2 product (:574), plus the images of
    h0(0) / h1(0) that the CellStateEncoder state seeds (image_from_kmajor_kernel :178, launched at :744-745).
  Not rounded (fp32-grade): the hoisted S01 cond product (:736-737), cfold / bfold (fold_const_kernel :100-112), the first step's pose
  term (fold_first_step_kernel :114-123), the gaze columns (c_wgz :251-254, :476), the CellStateEncoder, and the gate, ELU and
  root-integration epilogues.

Backward rounding points (decoder_bwd_tc.cu, decoder_bwd.cu); _Prod / _PoseTerm / _W2Grad give autograd the same products:
  * the G1 / G0 gate-gradient images dpr, dpz, dpn, dpn*r (decoder_bwd_tc.cu:374-375, :430-431) against the transposed bf16 weight
    images of pack_decoder_bwd_tc_kernel (:97) -- dh0 = W_ih1^T dgi1, dh1 += W_hh1^T dgh1, da = W_ih0a^T dgi0, dh0 += W_hh0^T dgh0;
  * the d pre_a image (:463) and the G0 image against Mfold^T and the gaze rows (fold part of dh1, gaze adjoint);
  * dYs = bf16(out_std * dY) against bf16(W2) (dy_scale_bf16_kernel :495, product in decoder_window_bwd_tc);
  * phase 2, single pass bf16 (fast_wgrad = 1): every weight gradient (wgrad_gemms, decoder_bwd.cu) over bf16 histories, d cond
    and the x_pose gradient DXP (decoder_window_bwd_tc) that joins dY and dch in DY before dW2 is formed.
  fp32-grade in the kernels, hence unrounded here: the root / gaze adjoint and its W2[0:6] rows (decoder_bwd_tc.cu:163, :369), the gate
  and ELU adjoints, every bias gradient (row sums of the fp32 histories), and the CellStateEncoder's gradients and input adjoints.
"""
import torch
import torch.nn.functional as F

from oracle import model_oracle as mo

P_IN, P_OUT = 1134, 1131
NAMES = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "ltxy", "lvel", "lvrt"]

# Tolerances of the tensor-core kernels against decoder_forward_tc(bf16=True), asserted by tests/test_tc_engine_gpu.py and shown to
# discriminate small kernel faults by tests/test_tc_oracle_cpu.py.  Forward: per pose-channel group, max-abs error over
# max(1, max|ref|) in de-normalised units.  Gradients: relative L2 error per parameter / dSpeech / dStyle tensor.
# Set from the H100 (DESIGN.md 2): worst measured 1.8e-3 forward (lvel), 3.1e-3 gradient (layer0.weight).  The kernels differ from
# this float64 restatement by less than from the fp32 oracle, but only by about 2x, not 10x: a value that fp32 and float64 round to
# different sides of a bf16 boundary moves by a whole bf16 step (identical samples match to 3e-7, distinct ones do not).
TC_FWD_TOL = 2.5e-3
TC_GRAD_TOL = 4e-3
# the tolerances the tensor-core tests against the fp32 oracle (model_oracle) use, for comparison
FP32_ORACLE_FWD_TOL = 2e-2
FP32_ORACLE_GRAD_TOL = 3e-2


def bf16_rn(x):
    return x.to(torch.bfloat16).to(x.dtype)


def bf16_trunc(x):
    """bf16 by truncation (the low 16 bits of the fp32 pattern dropped): a packing fault the tolerance must catch."""
    return (x.float().view(torch.int32) & -65536).view(torch.float32).to(x.dtype)


def _ident(x):
    return x


class _Prod(torch.autograd.Function):
    """value = rx(x) @ rw(W)^T (or the given fp32-grade value);  dx = rg(g) @ rw(W),  dW = rg(g)^T @ rx(x)."""

    @staticmethod
    def forward(ctx, x, W, value, rx, rw):
        ctx.save_for_backward(x, W)
        ctx.rx, ctx.rw = rx, rw
        return value.clone() if value is not None else rx(x) @ rw(W).T

    @staticmethod
    def backward(ctx, g):
        x, W = ctx.saved_tensors
        gr = ctx.rx(g)
        return gr @ ctx.rw(W), gr.T @ ctx.rx(x), None, None, None


class _PoseTerm(torch.autograd.Function):
    """The pose-input term Wx x(t) of [pre_a ; gi0](t), with the value the forward kernel forms (folded for t >= 2) and the gradients
    the BPTT kernel forms: dh1 = r(g) r(Mfold) (B3 / B4 chains), dx = r(g) r(Wx) (DXP product and gaze adjoint rows),
    dWx = r(g)^T r(x) (phase-2 weight gradient over the x_pose history).  h1 / Mf are None for the first step."""

    @staticmethod
    def forward(ctx, h1, x, Wx, value, Mf, r, rw):
        ctx.save_for_backward(h1, x, Wx)
        ctx.Mf, ctx.r, ctx.rw = Mf, r, rw
        return value.clone()

    @staticmethod
    def backward(ctx, g):
        h1, x, Wx = ctx.saved_tensors
        gr = ctx.r(g)
        dh1 = gr @ ctx.rw(ctx.Mf) if h1 is not None else None
        return dh1, gr @ ctx.rw(Wx), gr.T @ ctx.r(x), None, None, None, None


class _W2Grad(torch.autograd.Function):
    """Value 0; gathers every consumer's gradient of y(t) (pose output, next x_pose, root rows) so that dW2 = r(DY)^T r(h1) rounds the
    SUM once, as the kernels' single DY history does."""

    @staticmethod
    def forward(ctx, W2, h1, r):
        ctx.save_for_backward(h1)
        ctx.r = r
        return h1.new_zeros(h1.shape[0], W2.shape[0])

    @staticmethod
    def backward(ctx, g):
        (h1,) = ctx.saved_tensors
        return ctx.r(g).T @ ctx.r(h1), None, None


def _gru(gi, gh, h):
    H = h.shape[-1]
    r = torch.sigmoid(gi[:, :H] + gh[:, :H])
    z = torch.sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
    n = torch.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
    return (1.0 - z) * n + z * h


def units_per_cta(H):
    """U of csrc/library.cuh units_per_cta: CTA c owns hidden units c*U .. c*U+U-1 of every gate block."""
    return 4 if H % 4 == 0 and H // 4 <= 132 else 8


PERTURBATIONS = ("drop_kblock", "stale_h1", "zero_gaze", "truncate")


def decoder_forward_tc(P, root_pos, root_rot, root_vel, root_vrt, lpos, ltxy, lvel, lvrt, gaze_pos, speech, style,
                       in_mean, in_std, out_mean, out_std, dt, bf16=True, perturb=None):
    """Arguments as model_oracle.decoder_forward (P: reference state-dict names, "decoder." prefix).  Computes in float64.
    perturb (for the sensitivity test): one of PERTURBATIONS, a model of a small kernel fault --
      drop_kblock  the middle CTA's W_hh1 chain misses its second 64-wide k-block;
      stale_h1     the middle CTA's units reach the next step's chains with the h1 image of the step before;
      zero_gaze    the gaze columns Wx[:, 1131:1134] of the folded steps are zero;
      truncate     every weight operand is packed by truncation instead of round-to-nearest-even."""
    assert perturb is None or perturb in PERTURBATIONS, perturb
    f = lambda t: t.double()
    pd = "decoder.recurrent_decoder."
    w = lambda k: f(P[pd + k])
    W0, b0, W2, b2 = w("layer0.weight"), w("layer0.bias"), w("layer2.weight"), w("layer2.bias")
    Wih0, bih0, Whh0, bhh0 = w("layer1.weight_ih_l0"), w("layer1.bias_ih_l0"), w("layer1.weight_hh_l0"), w("layer1.bias_hh_l0")
    Wih1, bih1, Whh1, bhh1 = w("layer1.weight_ih_l1"), w("layer1.bias_ih_l1"), w("layer1.weight_hh_l1"), w("layer1.bias_hh_l1")
    H = W0.shape[0]
    im, is_, om, os_ = f(in_mean), f(in_std), f(out_mean), f(out_std)
    r = bf16_rn if bf16 else _ident
    rw = bf16_trunc if perturb == "truncate" else r
    first = [f(t) for t in (root_pos, root_rot, root_vel, root_vrt, lpos, ltxy, lvel, lvrt)]
    gaze_pos, speech, style = f(gaze_pos), f(speech), f(style)
    B, T = speech.shape[0], speech.shape[1]
    nj = lpos.shape[1]
    O = [[t] for t in first]
    x0 = mo.vectorize_input(*first, gaze_pos[:, 0], im, is_)
    pc = "decoder.cell_state_encoder."
    state = mo.cell_state_encoder({k: f(v) for k, v in P.items() if k.startswith(pc)}, x0, style[:, 0])
    h0, h1 = state[0], state[1]
    if T == 1:
        return tuple(torch.stack(o, dim=1) for o in O)

    Wx = torch.cat([W0[:, :P_IN], Wih0[:, H:H + P_IN]], 0)            # pose columns of layer0 / GRU0   [4H, 1134]
    Wc = torch.cat([W0[:, P_IN:], Wih0[:, H + P_IN:]], 0)             # speech / style columns          [4H, S+Z]
    bx = torch.cat([b0, bih0])
    Wa = Wih0[:, :H]
    with torch.no_grad():
        Mf = (Wx[:, :P_OUT] * (os_ / is_[:P_OUT])) @ W2                # fold matrix            [4H, H]
        cfold = Wx[:, :P_OUT] @ ((b2 * os_ + om - im[:P_OUT]) / is_[:P_OUT])
    U = units_per_cta(H)
    c_bad = (H // U) // 2                                              # the CTA the perturbations hit
    units = torch.arange(c_bad * U, c_bad * U + U)
    Whh1_used = Whh1
    if perturb == "drop_kblock":
        keep = torch.ones_like(Whh1)
        keep[torch.cat([units + q * H for q in range(3)]), 64:128] = 0.0
        Whh1_used = Whh1 * keep
    Wx_fold = Wx
    if perturb == "zero_gaze":
        keep = torch.ones_like(Wx)
        keep[:, P_OUT:] = 0.0
        Wx_fold = Wx * keep

    x = mo.vectorize_input(*first, gaze_pos[:, 1], im, is_).detach()   # x(1): the given pose, no gradient
    h1_img = h1
    for t in range(1, T):
        cond = torch.cat([speech[:, t], style[:, t]], -1)
        S = _Prod.apply(cond, Wc, (cond @ Wc.T).detach(), r, rw) + bx
        if t == 1:
            S = S + _PoseTerm.apply(None, x, Wx, (x @ Wx.T).detach(), None, r, rw)
        else:
            with torch.no_grad():
                val = r(h1_img) @ rw(Mf).T + cfold + x[:, P_OUT:] @ Wx_fold[:, P_OUT:].T
            S = S + _PoseTerm.apply(h1_img, x, Wx_fold, val, Mf, r, rw)
        a = F.elu(S[:, :H])
        gi0 = S[:, H:] + _Prod.apply(a, Wa, None, r, rw)
        gh0 = _Prod.apply(h0, Whh0, None, r, rw) + bhh0
        h0n = _gru(gi0, gh0, h0)
        gi1 = _Prod.apply(h0n, Wih1, None, r, rw) + bih1
        gh1 = _Prod.apply(h1_img, Whh1_used, None, r, rw) + bhh1
        h1n = _gru(gi1, gh1, h1)
        # layer 2: yo carries dh1 = r(out_std dY) r(W2) only; yw (value b2) carries dW2 / db2 from every consumer of y(t)
        yo = _Prod.apply(h1n, W2.detach(), None, r, rw)
        yw = _W2Grad.apply(W2, h1n.detach(), r) + b2
        y6g = h1n @ W2[:6].detach().T                                  # root rows: fp32-grade adjoint
        y6 = y6g + (yo[:, :6] - y6g).detach() + yw[:, :6]
        p6 = y6 * os_[:6] + om[:6]
        rp, rq = O[0][-1], O[1][-1]
        new_pos = mo.quat_mul_vec(rq, p6[:, 0:3] * dt) + rp           # modules.py:739-740 (as model_oracle.devectorize_output)
        new_rot = mo.quat_mul(mo.quat_from_helical(mo.quat_mul_vec(rq, p6[:, 3:6] * dt)), rq)
        rest = mo.devectorize_output(yo + yw, rp, rq, dt, om, os_, nj)[2:]
        for k, v in enumerate((new_pos, new_rot) + tuple(rest)):
            O[k].append(v)
        if t + 1 < T:
            xpose = ((yo.detach() + yw) * os_ + om - im[:P_OUT]) / is_[:P_OUT]
            gz = (mo.quat_inv_mul_vec(new_rot, gaze_pos[:, t + 1] - new_pos) - im[P_OUT:]) / is_[P_OUT:]
            x = torch.cat([xpose, gz], -1)
        h1_img = h1n
        if perturb == "stale_h1" and t >= 2:
            h1_img = h1n.clone()
            h1_img[:, units] = h1[:, units]
        h0, h1 = h0n, h1n
    return tuple(torch.stack(o, dim=1) for o in O)


def forward_errors(out, ref):
    """Per output group: max-abs error / max(1, max|ref|)."""
    res = {}
    for n, o, q in zip(NAMES, out, ref):
        o, q = o.detach().double().cpu(), q.detach().double().cpu()
        res[n] = float((o - q).abs().max()) / max(1.0, float(q.abs().max()))
    return res


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm()) / max(float(b.norm()), 1e-30)
