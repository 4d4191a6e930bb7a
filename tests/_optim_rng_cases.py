"""Cases, bounds and restatements for the RAdam step and the device-seeded draws of csrc/radam.cu.

RAdam (zeggs_radam_step_dev through optimizers.RAdam)
* The reference is oracle/model_oracle.radam_step in float64, with lr, the betas and eps as Python doubles and the gradient
  multiplied by grad_scale in float64, fed the same fp32 state (p, g, m, v) as the kernel.
* Bounds, with e = 2^-24 (half an fp32 ulp, relative) and the fp32 results m', v', p' against the float64 m*, v*, p*:
    |m' - m*| <= M_TOL e (|b1 m| + |(1 - b1) g|)                  the sum of the magnitudes of m's two terms (they may cancel)
    |v' - v*| <= V_TOL e v*                                       both terms of v are >= 0
    |p' - p*| <= e (P_TOL |p*| + U_TOL U)                          U = lr s (|b1 m| + |(1 - b1) g|) / (sqrt(v*) + eps), adaptive
                                                                  U = lr s (|b1 m| + |(1 - b1) g|), SGD branch (s = step size)
  each plus FLOOR, a few denormal ulps (tiny gradients square to fp32 denormals).  With p = 0 the update is p' in one rounding,
  so U_TOL measures the update itself: the parent kernel formed 1.0f - (float)beta2, which scales every v term and the step
  size by about 1 - 1.3e-5 at beta2 = 0.999, about 200 e, far past U_TOL.
* Trajectories: from a zero state, the update of every step (p reset to 0 before each step, which changes nothing else since
  weight_decay = 0) against a float64 trajectory on the same gradients, as a rel-L2 per step bounded by traj_bound(t): fp32
  state drifts from the float64 state, mostly through v's 1000-step memory, so the bound grows with t.
* `emulate_step` restates the kernel's fp32 arithmetic in torch float32 (one rounding per operation); with `fault` it models a
  mistake the bounds must reject (FAULTS).  tests/test_optim_rng_f64_cpu.py shows the reference's own fp32 arithmetic meets
  every bound with >= 4x headroom and that every fault breaks one.

The draws: oracle/rng_oracle.py.
"""
import math

import numpy as np
import torch

from oracle import model_oracle as mo

E = 2.0 ** -24
M_TOL, V_TOL, P_TOL, U_TOL = 16.0, 24.0, 8.0, 32.0
FLOOR = 2.0 ** -146                              # 8 fp32 denormal ulps

N_MODEL = 25_543_147                             # the shipped v1 networks (attn style encoder): one flat buffer
SIZES = [1, 255, 256, 257, 1023, 1024, 1025, 1212415, 1212416, 1212417, N_MODEL]   # grid cap 1184 blocks of 1024 from 1212416
STEPS = [1, 2, 3, 4, 5, 6, 7, 8, 50, 999, 1000, 1001, 10 ** 4, 10 ** 5]
GRAD_SCALES = [1.0, 0.5, 1.0 / 3.0, 0.125]
BETAS = [(0.9, 0.999), (0.8, 0.99)]
EPSS = [1e-5, 1e-8]
LRS = [1e-3, 1e-4]
GRID_N = 4099                                    # the hyper-parameter grid: 5 blocks, the last one ragged

TRAJ_N, TRAJ_STEPS, TRAJ_LR_STEP, TRAJ_DECAY = 4096, 1200, 1000, 0.995

FAULTS = {
    "parent": "rectification from the fp32 betas and 1 - beta formed from the fp32 betas (the kernel before this fix)",
    "scale_m_only": "grad_scale applied to m's gradient but not to v's",
    "step_before_increment": "the rectification evaluated at the step count before its increment",
    "adaptive_previous": "the adaptive flag of the previous step",
    "eps_in_sqrt": "eps inside the square root: sqrt(v + eps)",
}


# ---------------------------------------------------------------------------------------------- state
def make_state(n, seed, p_zero=False):
    """fp32 (p, g, m, v) [n] on the CPU.  Element classes cycle through the index so every size has each: p = 0 exactly (p' is the
    update in one rounding), g = 0, g tiny (g^2 below FLT_MIN: denormal v terms), g large (up to 1e17), v = 0 (the (1 - b2) g^2
    term is all of v'), g^2 >> v, m = 0, and a general mixture with magnitudes over ten decades.  p_zero: p = 0 everywhere."""
    rs = np.random.RandomState(seed)
    mag = lambda lo, hi: 10.0 ** rs.uniform(lo, hi, n)
    g = rs.randn(n) * mag(-4, 2)
    m = rs.randn(n) * mag(-5, 1)
    v = np.abs(rs.randn(n)) * mag(-10, 2)
    p = rs.randn(n) * mag(-3, 1)
    cls = np.arange(n) % 8
    g[cls == 1] = 0.0
    g[cls == 2] = rs.randn(int(np.sum(cls == 2))) * 1e-21
    g[cls == 3] = rs.randn(int(np.sum(cls == 3))) * 1e17
    v[cls == 4] = 0.0
    sel = cls == 5
    v[sel] = (g[sel] * 1e-4) ** 2
    m[cls == 6] = 0.0
    p[(cls % 2 == 0) | (np.arange(n) % 3 == 0)] = 0.0
    if p_zero:
        p[:] = 0.0
    f = lambda a: torch.from_numpy(a.astype(np.float32))
    return f(p), f(g), f(m), f(v)


# ---------------------------------------------------------------------------------------------- oracle and bounds
def rectification(step, b1, b2):
    """(step size, adaptive) of optimizers.py:64-78 in Python doubles."""
    b2t = b2 ** step
    n_max = 2 / (1 - b2) - 1
    n_sma = n_max - 2 * step * b2t / (1 - b2t)
    if n_sma >= 5:
        return math.sqrt((1 - b2t) * (n_sma - 4) / (n_max - 4) * (n_sma - 2) / n_sma * n_max / (n_max - 2)) / (1 - b1 ** step), True
    return 1.0 / (1 - b1 ** step), False


def oracle_step(p, g, m, v, step, lr, b1, b2, eps, gs):
    """model_oracle.radam_step in float64 from the fp32 state (any device) -> (p*, m*, v*) float64."""
    P, M, V = p.double(), m.double(), v.double()
    mo.radam_step(P, g.double() * gs, M, V, step, lr, beta1=b1, beta2=b2, eps=eps)
    return P, M, V


def step_ratios(out, ref, state, step, lr, b1, b2, eps, gs):
    """Worst ratio to its bound of each of p', m', v' (fp32 results `out`, float64 `ref`, the fp32 input `state`)
    -> {"p": (ratio, index), "m": ..., "v": ...}.  A non-finite result is an infinite ratio."""
    p, g, m, v = (x.double() for x in state)
    ge = g * gs
    mterm = (b1 * m).abs() + ((1 - b1) * ge).abs()
    ss, adaptive = rectification(step, b1, b2)
    U = lr * ss * mterm / ((ref[2].sqrt() + eps) if adaptive else 1.0)
    bounds = dict(p=E * (P_TOL * ref[0].abs() + U_TOL * U) + FLOOR, m=M_TOL * E * mterm + FLOOR, v=V_TOL * E * ref[2] + FLOOR)
    res = {}
    for k, o, r in zip("pmv", out, ref):
        d = (o.double() - r).abs()
        q = torch.where(torch.isfinite(d), d / bounds[k], torch.full_like(d, math.inf))
        i = int(torch.argmax(q))
        res[k] = (float(q[i]), i)
    return res


def worst(res):
    return max(r for r, _ in res.values())


# ---------------------------------------------------------------------------------------------- fp32 restatements
def reference_fp32_step(state, step, lr, b1, b2, eps, gs):
    """The reference's own arithmetic: model_oracle.radam_step on fp32 tensors (torch rounds each Python scalar to fp32 once),
    with the gradient scaled in fp32 -> (p', m', v')."""
    p, g, m, v = (x.clone() for x in state)
    mo.radam_step(p, g * np.float32(gs), m, v, step, lr, beta1=b1, beta2=b2, eps=eps)
    return p, m, v


def emulate_step(state, step, lr, b1, b2, eps, gs, fault=None):
    """The kernel's fp32 arithmetic (radam_prep_kernel + radam_dev_kernel), one rounding per operation -> (p', m', v')."""
    p, g, m, v = (x.clone() for x in state)
    f = np.float32
    if fault == "parent":
        b1h, b2h = float(f(b1)), float(f(b2))                # the prep kernel read fp32 betas
        omb1, omb2 = f(1.0) - f(b1), f(1.0) - f(b2)
    else:
        b1h, b2h = b1, b2
        omb1, omb2 = f(1.0 - b1), f(1.0 - b2)
    if fault == "step_before_increment":
        ss, adaptive = rectification(step - 1, b1h, b2h) if step > 1 else (math.inf, False)     # 1 / (1 - b1^0)
    else:
        ss, adaptive = rectification(step, b1h, b2h)
    if fault == "adaptive_previous":
        adaptive = rectification(step - 1, b1h, b2h)[1] if step > 1 else False
    step_lr = f(ss * lr)
    gi = g * f(gs)
    gv = g if fault == "scale_m_only" else gi
    v = v * f(b2) + (gv * omb2) * gv
    m = m * f(b1) + gi * omb1
    if adaptive:
        den = (v + f(eps)).sqrt() if fault == "eps_in_sqrt" else v.sqrt() + f(eps)
        p = p - (m * step_lr) / den
    else:
        p = p - m * step_lr
    return p, m, v


# ---------------------------------------------------------------------------------------------- trajectories
def traj_grads(n=TRAJ_N, steps=TRAJ_STEPS, seed=3):
    """fp32 gradients [steps, n]: per-element scale over six decades and a per-element mean (so m does not average out), a
    sixteenth of the elements always zero and another sixteenth zero on every other step."""
    rs = np.random.RandomState(seed)
    scale = 10.0 ** rs.uniform(-5, 1, n)
    mean = rs.randn(n) * 0.5
    g = (mean[None, :] + rs.randn(steps, n)) * scale[None, :]
    idx = np.arange(n)
    g[:, idx % 16 == 0] = 0.0
    g[0::2, idx % 16 == 1] = 0.0
    return torch.from_numpy(g.astype(np.float32))


def traj_lr(t, lr=1e-4):
    """lr of step t (1-based): decayed once after TRAJ_LR_STEP steps, as train.py's ExponentialLR does every 1000 iterations."""
    return lr * TRAJ_DECAY if t > TRAJ_LR_STEP else lr


def traj_oracle(grads, b1=0.9, b2=0.999, eps=1e-5):
    """float64 updates [steps, n] (p_t - p_{t-1}) from a zero state."""
    n = grads.shape[1]
    m, v = torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    out = torch.empty(grads.shape, dtype=torch.float64)
    for t in range(1, grads.shape[0] + 1):
        p = torch.zeros(n, dtype=torch.float64)
        mo.radam_step(p, grads[t - 1].double(), m, v, t, traj_lr(t), beta1=b1, beta2=b2, eps=eps)
        out[t - 1] = p
    return out


def traj_fp32(grads, step_fn, b1=0.9, b2=0.999, eps=1e-5):
    """fp32 updates [steps, n] of step_fn(state, step, lr, b1, b2, eps, gs) (reference_fp32_step or emulate_step) from a zero
    state, p reset to 0 before every step."""
    n = grads.shape[1]
    m, v = torch.zeros(n), torch.zeros(n)
    out = torch.empty(grads.shape)
    for t in range(1, grads.shape[0] + 1):
        p, m, v = step_fn((torch.zeros(n), grads[t - 1], m, v), t, traj_lr(t), b1, b2, eps, 1.0)
        out[t - 1] = p
    return out


def traj_bound(t):
    """rel-L2 bound on the update of step t: 15 e at step 1, growing like sqrt(t) with the rounding v accumulates (the
    reference's own fp32 arithmetic reaches about 1.5 sqrt(t) e)."""
    return E * (8.0 + 7.0 * math.sqrt(t))


def traj_ratios(upd, ref):
    """-> per-step ratio of ||upd_t - ref_t|| / ||ref_t|| to traj_bound(t), float64 [steps]."""
    d = (upd.double() - ref).norm(dim=1) / ref.norm(dim=1)
    b = torch.tensor([traj_bound(t) for t in range(1, upd.shape[0] + 1)], dtype=torch.float64)
    r = d / b
    return torch.where(torch.isfinite(r), r, torch.full_like(r, math.inf))
