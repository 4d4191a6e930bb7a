"""The training-loss kernel (zeggs_loss_fwd_bwd, csrc/loss.cu) against model_oracle.train_losses in float64.

Inputs are synth.make_pose_windows windows (O = decoder-output stand-in, W = ground truth).  Per case: the total and the 17 terms
within TERM_TOL relative (floor 1e-3 on |ref|), the KL term, dmu and dlogvar within KL_TOL, and the pose gradients (dY unpacked per
pose tensor, dRootPos, dRootRot), each relative to its own max, within GRAD_TOL on the frames tests/_util.loss_ambiguous_frames
leaves in.  A residual within fp32 rounding of zero may take either sign, and every gradient element is a weighted sum of signs,
so the frames such residuals reach are excluded (values there must still be finite).  Each case prints its worst errors and the
fraction of frames excluded; more than EXCLUDED_MAX excluded fails, so the test cannot quietly stop testing.
tests/test_loss_oracle_cpu.py shows that small modelled faults fail these tolerances and that an exact fp32 implementation
passes them."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import model_oracle as mo
from tests._util import (NAMES, ensure_built, loss_ambiguous_frames, loss_case, masked_grad_errors, oracle_loss_grads,
                         unpack_pose_grad, LOSS_KL_ITER)

pytestmark = pytest.mark.gpu

# About 4x the worst errors measured on an H100 80GB HBM3 (shipped tree: terms 4.0e-7, clean-frame gradients 4.9e-7, KL / dmu /
# dlogvar 2.3e-7; star and random trees below those; 75-deep chain: terms 1.9e-6, gradients 1.6e-6).
TERM_TOL = 2e-6
KL_TOL = 1e-6
GRAD_TOL = 2.5e-6
EXCLUDED_MAX = 0.10
# 75 chained rotations: the deep joints' fp32 rounding is several times the shipped tree's, so their errors and the share of
# residuals within rounding of zero are larger
TERM_TOL_CHAIN = 8e-6
GRAD_TOL_CHAIN = 6.5e-6
EXCLUDED_MAX_CHAIN = 0.20


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


def _stats():
    from zeggs_b200 import synth
    st = synth.load_stats()
    return np.asarray(st["parents"]), float(st["dt"])


def _tree(name):
    if name == "star":                                   # 74 children of joint 0: one level five passes wide
        return np.array([-1] + [0] * 74)
    if name == "chain":                                  # 75 levels deep
        return np.arange(-1, 74)
    rs = np.random.RandomState(7)                        # a random tree with parents[i] < i
    return np.array([-1] + [rs.randint(0, i) for i in range(1, 75)])


def _kernel(dev, O, W, gaze, parents, dt, mu, lv, autograd=False, kl_weight_dev=None):
    """One zeggs_loss_fwd_bwd call -> (terms[19] on the CPU, {pose name / mu / logvar: gradient})."""
    from zeggs_b200 import ops
    from zeggs_b200.autograd import TrainLossFn
    from zeggs_b200.train import kl_weight, pack_pose
    Og, Wg = [o.to(dev) for o in O], [w.to(dev) for w in W]
    mu_g, lv_g = (None, None) if mu is None else (mu.to(dev), lv.to(dev))
    WY, gz = pack_pose(*Wg[2:]), gaze.to(dev)
    par = torch.as_tensor(parents, dtype=torch.int32, device=dev)
    kw = kl_weight(LOSS_KL_ITER) if mu is not None else 0.0
    terms = torch.zeros(19, device=dev)
    if autograd:
        Og = [o.requires_grad_(True) for o in Og]
        leaves = Og + ([mu_g.requires_grad_(True), lv_g.requires_grad_(True)] if mu is not None else [])
        loss = TrainLossFn.apply(pack_pose(*Og[2:]), Og[0], Og[1], WY, Wg[0], Wg[1], gz, par, dt, mu_g, lv_g, kw, terms)
        gs = torch.autograd.grad(loss, leaves)
        g = dict(zip(NAMES + ["mu", "logvar"], gs))
    else:
        _, (dY, dRp, dRq, dmu, dlv) = ops.loss_fwd_bwd(pack_pose(*Og[2:]), Og[0], Og[1], WY, Wg[0], Wg[1], gz, par, dt, mu_g, lv_g, kw,
                                                       terms, kl_weight_dev)
        g = unpack_pose_grad(dY, dRp, dRq)
        g["mu"], g["logvar"] = dmu, dlv
    torch.cuda.synchronize()
    return terms.cpu(), {k: (None if v is None else v.detach().cpu()) for k, v in g.items()}


def _kernel_forward_only(dev, O, W, gaze, parents, dt, mu, lv):
    """zeggs_loss_fwd_bwd with dY == NULL (the header's forward-only call) -> terms[19] on the CPU."""
    from zeggs_b200 import _lib
    from zeggs_b200.train import kl_weight, pack_pose
    l = _lib.lib()
    Og, Wg = [o.to(dev).contiguous() for o in O], [w.to(dev).contiguous() for w in W]
    B, T = O[0].shape[:2]
    Y, WY, gz = pack_pose(*Og[2:]).contiguous(), pack_pose(*Wg[2:]).contiguous(), gaze.to(dev).contiguous()
    mu_g, lv_g = mu.to(dev).contiguous(), lv.to(dev).contiguous()
    par = torch.as_tensor(parents, dtype=torch.int32, device=dev)
    terms = torch.zeros(19, device=dev)
    wsb = l.zeggs_loss_workspace_bytes(B, T)
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    a = _lib.LossArgs(B=B, T=T, Z=mu.shape[1], dt=dt, kl_weight=kl_weight(LOSS_KL_ITER))
    a.Y, a.root_pos, a.root_rot = Y.data_ptr(), Og[0].data_ptr(), Og[1].data_ptr()
    a.WY, a.W_root_pos, a.W_root_rot = WY.data_ptr(), Wg[0].data_ptr(), Wg[1].data_ptr()
    a.gaze_pos, a.parents, a.losses = gz.data_ptr(), par.data_ptr(), terms.data_ptr()
    a.mu, a.logvar = mu_g.data_ptr(), lv_g.data_ptr()
    a.workspace, a.workspace_bytes = ws.data_ptr(), wsb
    assert not a.dY and not a.dmu
    _lib.check(l.zeggs_loss_fwd_bwd(C.byref(a), _lib.stream_ptr()), "zeggs_loss_fwd_bwd (forward only)")
    torch.cuda.synchronize()
    return terms.cpu()


def _term_errors(terms, total64, L64):
    """Relative errors (floor 1e-3 on |ref|) of the total and the 17 terms, and the KL term's relative error."""
    e = {"total": abs(float(terms[0]) - total64) / max(1e-3, abs(total64))}
    for i, k in enumerate(mo.LOSS_NAMES):
        e[k] = abs(float(terms[1 + i]) - L64[k]) / max(1e-3, abs(L64[k]))
    kl = L64.get("kl_div", 0.0)
    e_kl = abs(float(terms[18]) - kl) / max(abs(kl), 1e-30) if kl else abs(float(terms[18]))
    return e, e_kl


def _check_case(dev, B, T, parents, dt, seed, copy_frame0, label, autograd=False, term_tol=TERM_TOL, grad_tol=GRAD_TOL,
                excluded_max=EXCLUDED_MAX):
    O, W, gaze, mu, lv = loss_case(B, T, seed=seed, copy_frame0=copy_frame0)
    total64, L64, g64 = oracle_loss_grads(O, W, gaze, parents, dt, mu, lv)
    amb_y, amb_rot = loss_ambiguous_frames(O, W, gaze, parents, dt)
    terms, g = _kernel(dev, O, W, gaze, parents, dt, mu, lv, autograd=autograd)
    te, e_kl = _term_errors(terms, total64, L64)
    ge = masked_grad_errors(g, g64, amb_y, amb_rot)
    e_mu = float((g["mu"].double() - g64["mu"]).abs().max() / g64["mu"].abs().max())
    e_lv = float((g["logvar"].double() - g64["logvar"]).abs().max() / g64["logvar"].abs().max())
    fy, fr = float(amb_y.float().mean()), float(amb_rot.float().mean())
    wt, wg = max(te, key=te.get), max(ge, key=ge.get)
    print(f"  [{label} B={B} T={T}] worst term {te[wt]:.2e} ({wt}); KL {e_kl:.2e}, dmu {e_mu:.2e}, dlogvar {e_lv:.2e}; "
          f"worst clean-frame gradient {ge[wg]:.2e} ({wg}); excluded {fy:.3f} of frames (dRootRot {fr:.3f})")
    assert max(fy, fr) <= excluded_max, (fy, fr)
    assert te[wt] <= term_tol, te
    assert max(e_kl, e_mu, e_lv) <= KL_TOL, (e_kl, e_mu, e_lv)
    assert ge[wg] <= grad_tol, ge


# T=2: every frame ends its window.  B*T = 165 and 287 leave a dead half-warp in the backward kernel (two frames per warp);
# 8192 frames leave a partial last CTA of the backward (6 frames per CTA).  The long windows copy frame 0 from the ground truth,
# as the decoder returns it, so every direct residual of frame 0 is exactly 0.
SHAPES = [(1, 2, False), (2, 2, False), (5, 33, False), (7, 41, False), (16, 120, True), (32, 256, True)]


@pytest.mark.parametrize("B,T,copy_frame0", SHAPES)
def test_loss_kernel_vs_float64_oracle(dev, B, T, copy_frame0):
    parents, dt = _stats()
    _check_case(dev, B, T, parents, dt, seed=41 + B + T, copy_frame0=copy_frame0, label="shipped")


def test_loss_autograd_wrapper_vs_float64_oracle(dev):
    """The same check through autograd.TrainLossFn (loss.backward() with the implicit unit gradient)."""
    parents, dt = _stats()
    _check_case(dev, 5, 33, parents, dt, seed=79, copy_frame0=True, label="TrainLossFn", autograd=True)


@pytest.mark.parametrize("tree", ["star", "chain", "random"])
@pytest.mark.parametrize("B,T", [(4, 17), (16, 120)])
def test_loss_kernel_other_skeletons(dev, tree, B, T):
    """Trees other than the shipped one (13 levels, at most 12 joints wide): a star makes the level loops and joint 0's child
    gather run 74 wide, a chain makes the level walk 75 deep."""
    _, dt = _stats()
    tol = dict(term_tol=TERM_TOL_CHAIN, grad_tol=GRAD_TOL_CHAIN, excluded_max=EXCLUDED_MAX_CHAIN) if tree == "chain" else {}
    _check_case(dev, B, T, _tree(tree), dt, seed=141 + B + T, copy_frame0=T > 100, label=tree, **tol)


@pytest.mark.parametrize("vae", [True, False])
def test_equal_windows_give_exact_zeros(dev, vae):
    """O == W: every residual is exactly 0, so are the 17 terms and the pose gradients; the total is the KL term / 18."""
    parents, dt = _stats()
    _, W, gaze, mu, lv = loss_case(7, 41, seed=5)
    if not vae:
        mu = lv = None
    terms, g = _kernel(dev, [w.clone() for w in W], W, gaze, parents, dt, mu, lv)
    assert torch.all(terms[1:18] == 0), terms
    for n in NAMES:
        assert torch.all(g[n] == 0), n
    if vae:
        kl = float(terms[18])
        assert kl > 0
        assert abs(float(terms[0]) - kl / 18.0) <= float(np.spacing(np.float32(kl / 18.0))), (float(terms[0]), kl)
    else:
        assert torch.all(terms == 0), terms


def test_repeated_calls_are_bitwise_identical(dev):
    parents, dt = _stats()
    case = loss_case(16, 120, seed=9, copy_frame0=True)
    t1, g1 = _kernel(dev, *case[:3], parents, dt, *case[3:])
    t2, g2 = _kernel(dev, *case[:3], parents, dt, *case[3:])
    assert torch.equal(t1, t2)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k


def test_device_kl_weight_matches_the_value(dev):
    """kl_weight_dev (read by the kernel, for CUDA-graph replays) gives the same bits as the same weight passed by value."""
    from zeggs_b200.train import kl_weight
    parents, dt = _stats()
    case = loss_case(5, 33, seed=13)
    t1, g1 = _kernel(dev, *case[:3], parents, dt, *case[3:])
    kw = torch.tensor([kl_weight(LOSS_KL_ITER)], dtype=torch.float32, device=dev)
    t2, g2 = _kernel(dev, *case[:3], parents, dt, *case[3:], kl_weight_dev=kw)
    assert torch.equal(t1, t2)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k
    # and the device scalar really is read: another weight there changes the KL term and dmu
    kw.fill_(0.5 * kl_weight(LOSS_KL_ITER))
    t3, g3 = _kernel(dev, *case[:3], parents, dt, *case[3:], kl_weight_dev=kw)
    assert torch.equal(t3[1:18], t1[1:18]) and float(t3[18]) != float(t1[18])
    assert not torch.equal(g3["mu"], g1["mu"])


def test_loss_without_vae(dev):
    """mu = logvar = NULL (use_vae: false, and the label-style path): terms 1..17 are the with-VAE call's bits, the KL term is 0,
    the total matches float64, and the pose gradients are the with-VAE call's."""
    parents, dt = _stats()
    O, W, gaze, mu, lv = loss_case(16, 120, seed=17, copy_frame0=True)
    t_vae, g_vae = _kernel(dev, O, W, gaze, parents, dt, mu, lv)
    t, g = _kernel(dev, O, W, gaze, parents, dt, None, None)
    assert torch.equal(t[1:18], t_vae[1:18])
    assert float(t[18]) == 0.0
    assert g["mu"] is None and g["logvar"] is None
    for n in NAMES:
        assert torch.equal(g[n], g_vae[n]), n
    total64, L64, _ = oracle_loss_grads(O, W, gaze, parents, dt)
    te, _ = _term_errors(t, total64, L64)
    print(f"  [no VAE] total rel err {te['total']:.2e}")
    assert te["total"] <= TERM_TOL


@pytest.mark.parametrize("B,T", [(2, 2), (7, 41), (32, 256)])
def test_forward_only_call(dev, B, T):
    """dY == NULL runs the frame-difference sums in their own kernel.  Terms 1-12 and gaze are bitwise the fwd+bwd call's; the four
    difference terms are summed in another order (1e-6 relative); all 17 match float64."""
    parents, dt = _stats()
    O, W, gaze, mu, lv = loss_case(B, T, seed=23 + T, copy_frame0=T > 100)
    t_fb, _ = _kernel(dev, O, W, gaze, parents, dt, mu, lv)
    t = _kernel_forward_only(dev, O, W, gaze, parents, dt, mu, lv)
    same = list(range(1, 13)) + [17, 18]
    assert torch.equal(t[same], t_fb[same])
    d = (t[13:17].double() - t_fb[13:17].double()).abs() / t_fb[13:17].double().abs()
    total64, L64, _ = oracle_loss_grads(O, W, gaze, parents, dt, mu, lv)
    te, _ = _term_errors(t, total64, L64)
    wt = max(te, key=te.get)
    print(f"  [forward only B={B} T={T}] difference terms vs fwd+bwd {float(d.max()):.2e}; worst term vs float64 {te[wt]:.2e} ({wt})")
    assert float(d.max()) <= 1e-6
    assert te[wt] <= TERM_TOL
