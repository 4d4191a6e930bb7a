"""Inputs, float64 oracle and modelled faults of the GRU style encoder (`style_type: "gru"`: csrc/style_gru.cu and
zeggs_style_enc_gru_fwd / _bwd in csrc/encoders.cu), shared by tests/test_style_gru_f64_cpu.py (no GPU: the bounds mean something) and
tests/test_style_gru_f64_gpu.py (the kernels meet them).

* Inputs: `synth` style examples normalised with the shipped stats, an injected VAE eps and random cotangents.  The GRU encoder has
  no dropout.
* `run_oracle`: oracle/style_oracle.style_encoder(type="gru") with everything cast to float64 (or float32), plus autograd.  It scans
  the reverse direction in full; its output at T-1 is the one cell the kernel runs.
* `run_restated`: the encoder restated in the kernels' decomposition -- conv, conv, GI = x W_ih^T + b_ih for all steps, the T-step
  forward scan (GH = h(t-1) W_hh^T + b_hh, then the gate cell, whose backward is the BPTT kernel's phase A), the reverse cell at
  T-1 from h = 0, the projection of [h(T-1), h_r] and the VAE split -- with two options the oracle does not have:
  - `matched`: the weight gradients of the products that run as ONE bf16 tensor-core pass under `fast_wgrad = 1` (the rule of
    tests/_encoder_cases.py: M*N*K >= 4e6) are formed from bf16-rounded operands, accumulated in float64;
  - `fault`: one modelled kernel error (FAULTS).
  Without either it equals `run_oracle` to 1e-12 (tests/test_style_gru_f64_cpu.py).
* `margined_params`: parameters whose two ReLU convolutions keep every pre-activation well away from zero, so fp32 cannot flip a gate
  that float64 does not, and gradients can be compared tightly.
"""
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn.functional as F

from tests import _encoder_cases as ec
from tests._util import stats_tensors

SEED = 23
GRU_KC = 512              # rows of h(t-1) the forward kernel stages per K chunk (csrc/style_gru.cu)

_SE = "style_encoder.encoder."
CONV1, CONV2 = _SE + "convs.0.conv.weight", _SE + "convs.2.conv.weight"
W_IH, W_HH = _SE + "rnn_layer.weight_ih_l0", _SE + "rnn_layer.weight_hh_l0"
W_IH_R, W_HH_R = _SE + "rnn_layer.weight_ih_l0_reverse", _SE + "rnn_layer.weight_hh_l0_reverse"
W_P = _SE + "projection_layer.linear_layer.weight"
WGRADS = [CONV1, CONV2, W_IH, W_HH, W_IH_R, W_P]      # the weight gradients fast_wgrad = 1 may run in one bf16 pass

FWD_TOL = ec.FWD_TOL      # outputs: max-abs / max(1, max|ref|)
GRAD_TOL = ec.GRAD_TOL    # every gradient in fp32-grade settings: relative L2 per tensor
# Single-pass bf16 weight gradients vs the bf16-matched float64 oracle, relative L2 per tensor.  Where the kernel's operand and the
# float64 one round to different sides of a bf16 boundary, the operand moves by a whole bf16 step, so the distance grows with the
# error of the operands: <= 5.3e-5 with fp32 arithmetic, but with the forward and input-gradient products of GEMM mode 1 emulated
# as split-bf16 (hi*hi + hi*lo + lo*hi, ~1e-5 relative) up to 2.4e-4 at the training shape and at H = 1056.  The unmatched float64
# oracle is >= 1.48e-3 away: a kernel that ran the fp32-grade product instead fails by 3x or more.
MATCHED_TOL = {k: 5e-4 for k in WGRADS}

# fault -> what it models
FAULTS = {
    "tile_offset": "samples b >= 32 stage tile 0's h(t-1) (the b0 offset of the batch tile lost)",
    "k_chunk_dropped": "the last GRU_KC chunk of h(t-1) never reaches the product (H > 512 only)",
    "rev_row_T-2": "the reverse cell reads row T-2 of c2 instead of T-1 (the T*H stride of the strided operand)",
    "rev_row_0": "the reverse cell reads row 0 of c2 instead of T-1",
    "bptt_no_z_carry": "BPTT drops the dh(t) * z carry into dh(t-1)",
    "n_gate_no_r": "the n gate's hidden-side gradient omits the factor r",
    "hcat_T-2": "the projection reads h(T-2) instead of h(T-1)",
}


def hidden_sizes():
    """Every H style_gru_units accepts: H % 4 == 0, H <= 528 (4 units per CTA) and H % 8 == 0, H <= 1056 (8 units per CTA)."""
    return [H for H in range(4, 1057, 4) if H <= 528 or H % 8 == 0]


# ---------------------------------------------------------------------------------------------- inputs
def gru_params(H, E):
    from zeggs_b200 import synth
    P = synth.make_params(H=64, seed=SEED, style_hidden=H, style_embed=E, style_type="gru")
    return {k: v for k, v in P.items() if k.startswith("style_encoder.")}


def gru_case(B, T, H, vae=True, E=None, grads=True, eps=True, temperature=1.3, seed=0):
    """x [B,T,1134] normalised, eps [B,E/2] or None (z = mu), cotangents of (z, mu, logvar) or of z alone."""
    from zeggs_b200 import synth
    st = stats_tensors()
    E = E if E is not None else (128 if vae else 64)
    x = (torch.from_numpy(synth.make_style_example(B, T, seed=seed)) - st["anim_input_mean"]) / st["anim_input_std"]
    rs = np.random.RandomState(3000 + seed)
    Z = E // 2 if vae else E
    e = torch.from_numpy(rs.randn(B, Z).astype(np.float32)) if (vae and eps) else None
    cots = [torch.from_numpy(rs.randn(B, Z).astype(np.float32)) for _ in range(3 if vae else 1)] if grads else None
    return SimpleNamespace(B=B, T=T, H=H, E=E, vae=vae, x=x.float(), eps=e, cots=cots, temperature=temperature)


H_EDGES = [4, 512, 516, 528, 536, 1056]     # one CTA; 4 units: one K chunk, full / 4-row / 16-row tail chunk; 8 units: 2 / 3 chunks
B_EDGES = [1, 31, 32, 33, 64, 65]           # 1, 2 and 3 batch tiles, full and one-sample tiles

# The cases with gradients of tests/test_style_gru_f64_gpu.py: id -> gru_case arguments.
CASES = {
    "H512_B32_T384_vae": dict(B=32, T=384, H=512),                   # the training shape
    "H512_B32_T384_novae": dict(B=32, T=384, H=512, vae=False),
    **{f"H{H}_B{B}_T17_vae": dict(B=B, T=17, H=H) for H in H_EDGES for B in B_EDGES},
    **{f"H{H}_B{B}_T{T}_novae": dict(B=B, T=T, H=H, vae=False) for H in H_EDGES for B in (1, 33) for T in (1, 2)},
    **{f"H{H}_B33_T17_E63": dict(B=33, T=17, H=H, vae=False, E=63) for H in H_EDGES},    # odd-width encoding without the VAE
}
# Forward only: generate_gesture's whole style clip (no eps: z = mu).
GEN_CASES = {f"H512_B1_T{T}_gen": dict(B=1, T=T, H=512, grads=False, eps=False) for T in (1000, 3600)}
TRAIN, LARGEST = "H512_B32_T384_vae", "H1056_B65_T17_vae"
# Where each fault can appear.
FAULT_CASE = {"tile_offset": "H512_B65_T17_vae", "k_chunk_dropped": LARGEST, **{f: TRAIN for f in FAULTS if f not in
                                                                                    ("tile_offset", "k_chunk_dropped")}}


def make_case(cid):
    kw = dict(CASES[cid] if cid in CASES else GEN_CASES[cid])
    kw.setdefault("seed", 10000 * kw["B"] + 10 * kw["T"] + kw["H"])
    return gru_case(**kw)


def sweep_case(H):
    """The hidden-size sweep: B = 3, T = 5, forward only."""
    return gru_case(B=3, T=5, H=H, grads=False, seed=H)


# ---------------------------------------------------------------------------------------------- the oracle
def run_oracle(P, case, dtype=torch.float64):
    """style_oracle in `dtype` -> (outputs, gradients or None): [z, mu, logvar], or [z] without the VAE."""
    from oracle import style_oracle as so
    grads = case.cots is not None
    Pt = ec._leaves(P, dtype, grads)
    with torch.set_grad_enabled(grads):
        eps = None if case.eps is None else case.eps.to(dtype)
        outs = so.style_encoder(Pt, case.x.to(dtype), eps=eps, temperature=case.temperature, use_vae=case.vae, type="gru")
        outs = list(outs) if case.vae else [outs[0]]
    return ec._finish(outs, Pt, case.cots)


# ---------------------------------------------------------------------------------------------- restatement
class _Cell(torch.autograd.Function):
    """h = (1 - z) n + z hp, r = sigmoid(gi_r + gh_r), z = sigmoid(gi_z + gh_z), n = tanh(gi_n + r gh_n) (nn.GRU's gate order
    r, z, n).  The backward is phase A of gru_bwd_kernel (rev_cell_bwd_kernel with hp = 0).  Faults: drop_carry (no dh z into
    dh(t-1)), n_no_r (the n gate's hidden-side gradient without r)."""

    @staticmethod
    def forward(ctx, gi, gh, hp, drop_carry, n_no_r):
        H = hp.shape[-1]
        r = torch.sigmoid(gi[:, :H] + gh[:, :H])
        z = torch.sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
        n = torch.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
        ctx.save_for_backward(r, z, n, gh[:, 2 * H:], hp)
        ctx.drop_carry, ctx.n_no_r = drop_carry, n_no_r
        return (1.0 - z) * n + z * hp

    @staticmethod
    def backward(ctx, dh):
        r, z, n, ghn, hp = ctx.saved_tensors
        dpn = dh * (1.0 - z) * (1.0 - n * n)
        dpr = dpn * ghn * r * (1.0 - r)
        dpz = dh * (hp - n) * z * (1.0 - z)
        dgi = torch.cat([dpr, dpz, dpn], dim=1)
        dgh = torch.cat([dpr, dpz, dpn if ctx.n_no_r else dpn * r], dim=1)
        return dgi, dgh, torch.zeros_like(dh) if ctx.drop_carry else dh * z, None, None


def _rounded(o, key, M, N, K):
    """Whether the weight gradient [N, K] over M rows runs as one bf16 pass (and is matched as such)."""
    rnd = o.matched and M * N * K >= ec.TC_MIN_MNK
    if rnd:
        o.rounded.append((key, M, N, K))
    return rnd


def gru_forward(P, x, eps, temperature, vae, o, internals=None):
    """modules.py:289-304, 307-343 -> [z, mu, logvar] or [z].  internals: dict that receives the two ReLU pre-activations."""
    g = lambda k: P[_SE + k]
    B, T, _ = x.shape
    f = o.fault
    pre = internals if internals is not None else {}
    pre["c1"] = ec._conv(x, P[CONV1], g("convs.0.conv.bias"), o, CONV1, replicate=False)
    pre["c2"] = ec._conv(F.relu(pre["c1"]), P[CONV2], g("convs.2.conv.bias"), o, CONV2, replicate=False)
    c2 = F.relu(pre["c2"])
    Whh, bhh = P[W_HH], g("rnn_layer.bias_hh_l0")
    H = Whh.shape[1]
    GI = ec._lin(c2, P[W_IH], g("rnn_layer.bias_ih_l0"), o, W_IH)                     # [B,T,3H], all steps in one product
    rnd = _rounded(o, W_HH, B * T, 3 * H, H)                                          # dW_hh = sum_t dG_hh(t)^T h(t-1)
    kd = (H - 1) // GRU_KC * GRU_KC if (f == "k_chunk_dropped" and H > GRU_KC) else H
    tile = torch.arange(B) % 32
    h, hs = x.new_zeros(B, H), []
    for t in range(T):
        hin = h[tile] if (f == "tile_offset" and B > 32) else h
        gh = ec._Linear.apply(hin[:, :kd], Whh[:, :kd], bhh, rnd, 0)
        h = _Cell.apply(GI[:, t], gh, h, f == "bptt_no_z_carry", f == "n_gate_no_r")
        hs.append(h)
    hf = hs[-2] if (f == "hcat_T-2" and T > 1) else hs[-1]
    row = {"rev_row_T-2": max(T - 2, 0), "rev_row_0": 0}.get(f, T - 1)
    GIr = ec._lin(c2[:, row], P[W_IH_R], g("rnn_layer.bias_ih_l0_reverse"), o, W_IH_R)
    h0 = x.new_zeros(B, H)
    ghr = ec._Linear.apply(h0, P[W_HH_R], g("rnn_layer.bias_hh_l0_reverse"), False, 0)   # W_hh_r h(=0) + b_hh_r: dW_hh_r is 0
    hr = _Cell.apply(GIr, ghr, h0, False, False)
    out = ec._lin(torch.cat([hf, hr], dim=1), P[W_P], g("projection_layer.linear_layer.bias"), o, W_P)
    if not vae:
        return [out]
    Z = out.shape[1] // 2
    mu, logvar = out[:, :Z], out[:, Z:]
    z = mu if eps is None else mu + eps * torch.exp(0.5 * logvar) / temperature
    return [z, mu, logvar]


def run_restated(P, case, dtype=torch.float64, matched=False, fault=None):
    """The restatement in `dtype` -> (outputs, gradients or None, ec.Opts of the run)."""
    assert fault is None or fault in FAULTS, fault
    o = ec.Opts(matched, fault)
    grads = case.cots is not None
    Pt = ec._leaves(P, dtype, grads)
    with torch.set_grad_enabled(grads):
        eps = None if case.eps is None else case.eps.to(dtype)
        outs = gru_forward(Pt, case.x.to(dtype), eps, case.temperature, case.vae, o)
    outs, gs = ec._finish(outs, Pt, case.cots)
    return outs, gs, o


# ---------------------------------------------------------------------------------------------- ReLU gate margins
RELU_SITES = [("c1", "convs.0.conv.bias"), ("c2", "convs.2.conv.bias")]


def _internals(P, case, dtype):
    pre = {}
    Pt = ec._leaves(P, dtype, False)
    with torch.no_grad():
        eps = None if case.eps is None else case.eps.to(dtype)
        gru_forward(Pt, case.x.to(dtype), eps, case.temperature, case.vae, ec.Opts(), internals=pre)
    return pre


GATE_GAP = 0.5           # bias margin, in std of the channel's bias-free pre-activation


def margined_params(P, case):
    """Parameters with every ReLU pre-activation of `case` at least GATE_GAP std from zero: layer by layer in float64, each ReLU
    conv's bias is set per channel so that even channels pass on every row (bias = -min + GATE_GAP std of the bias-free
    pre-activation) and odd channels on none (bias = -max - GATE_GAP std); std over all rows, over the whole layer when there is
    one row.  Unlike ec.margined_style_params' -mean +- 4 std, no row can land near zero by chance, at any batch."""
    P = dict(P)
    for site, bkey in RELU_SITES:
        P[_SE + bkey] = np.zeros_like(P[_SE + bkey])
        z = _internals(P, case, torch.float64)[site]
        z = z.reshape(-1, z.shape[-1])
        std = z.std(0) if z.shape[0] > 1 else z.std().expand(z.shape[1])
        b = -z.max(0).values - GATE_GAP * std
        b[0::2] = (-z.min(0).values + GATE_GAP * std)[0::2]
        P[_SE + bkey] = b.float().numpy()
    return P


def gate_margins(P, case):
    """-> {site: (min |pre-activation| in float64, max |fp32 - float64| of the pre-activation)} at the two ReLU sites."""
    p64, p32 = _internals(P, case, torch.float64), _internals(P, case, torch.float32)
    return {s: (float(p64[s].abs().min()), float((p32[s].double() - p64[s]).abs().max())) for s, _ in RELU_SITES}


# ---------------------------------------------------------------------------------------------- comparisons
def errors(outs, grads, ref_outs, ref_grads, rounded=()):
    """-> [(name, error, bound)] for every output (FWD_TOL) and gradient (GRAD_TOL; MATCHED_TOL for the keys in `rounded`)."""
    res = [(f"out{i}", ec.fwd_err(o, r), FWD_TOL) for i, (o, r) in enumerate(zip(outs, ref_outs))]
    if grads is not None:
        for k in sorted(ref_grads):
            res.append((k, ec.rel_l2(grads[k], ref_grads[k]), MATCHED_TOL[k] if k in rounded else GRAD_TOL))
    return res
