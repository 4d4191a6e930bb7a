"""GPU: the fused RAdam step (zeggs_radam_step_dev through optimizers.RAdam) against oracle/model_oracle.radam_step in float64,
and the counter-based draws (zeggs_dropout_mask, zeggs_dropout_mask_dev, zeggs_randn_dev) against their restatement in
oracle/rng_oracle.py, at every size, step and seed the cases name (tests/_optim_rng_cases.py).

* RAdam, one step from a given fp32 state: p', m' and v' within the bounds of _optim_rng_cases, at every size across the grid
  cap (1184 blocks of 1024 elements from n = 1212416) up to the shipped model's 25,543,147 parameters, and over the grid of
  steps (set through step_dev), grad_scale, betas, eps and lr.  States with p = 0 make p' the update in one rounding.
* RAdam trajectories: 1200 eager steps from a zero state, lr decayed through param_groups after step 1000; each step's update
  within traj_bound(t) in rel-L2 of the float64 trajectory.
* RAdam in a CUDA graph (captured as train.py does): every replay equals the one-step oracle from the state before it and the
  bits of an eager twin; step_dev follows the host's step count.  Resume from a zeggs or a reference state_dict at step 5
  equals an uninterrupted run bit for bit.
* Dropout masks: bit-exact against the restatement for both kernels, at sizes across the grid cap (2368 blocks of 1024 from
  n = 2424832) up to the training attention mask, for p from 0 to the largest float below 1, four seeds and salts 1-4.
  p = 1, -0.1 and NaN are refused before any launch.
* VAE noise: zeggs_randn_dev within RANDN_ULPS fp32 ulps of the restatement (u1 and the angle formed in fp32 as the kernel does,
  log / sqrt / sin / cos in float64): CUDA documents logf within 1 ulp and sinf / cosf within 2 ulp, and sqrtf and the products
  round correctly, about 3.5 * 2^-23 relative in all, at most 7 ulps.
* A captured graph of DeviceSeed.advance() and the draws of one step draws the restatement's values at seed t0 + k on replay k.
tests/test_optim_rng_f64_cpu.py shows the reference's fp32 arithmetic meets the RAdam bounds with >= 4x headroom, every
modelled kernel fault breaks one, and the restatement of the draws is right.
"""
import copy

import numpy as np
import pytest
import torch

from oracle import rng_oracle as ro
from tests import _optim_rng_cases as oc
from tests._util import ensure_built

pytestmark = pytest.mark.gpu

RANDN_ULPS = 8.0
RANDN_FLOOR = 2.0 ** -140


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


# ---------------------------------------------------------------------------------------------- RAdam
def _opt(n, dev, lr=1e-4, betas=(0.9, 0.999), eps=1e-5):
    from zeggs_b200.optimizers import RAdam
    return RAdam([torch.nn.Parameter(torch.zeros(n, device=dev))], lr=lr, betas=betas, eps=eps)


def _one_step(opt, st, step, lr, b1, b2, eps, gs):
    """Load the fp32 state, set the hyper-parameters through param_groups / grad_scale and the step count through step_dev, take
    one step -> (p', m', v') on the device."""
    g = opt.param_groups[0]
    g["lr"], g["betas"], g["eps"] = lr, (b1, b2), eps
    opt.grad_scale = gs
    for dst, src in zip((opt.flat_param, opt.flat_grad, opt.exp_avg, opt.exp_avg_sq), st):
        dst.copy_(src)
    opt.step_dev.fill_(step - 1)
    opt._step = step - 1
    opt.step()
    assert int(opt.step_dev.item()) == step == opt._step
    return opt.flat_param, opt.exp_avg, opt.exp_avg_sq


def _check_step(out, st, hp):
    res = oc.step_ratios(out, oc.oracle_step(*st, *hp), st, *hp)
    return oc.worst(res), res


@pytest.mark.parametrize("n", oc.SIZES)
def test_radam_one_step_sizes(dev, n):
    """Every element of a buffer of n parameters, at steps 6 and 1000 (the rectification at its most biased in the kernel before
    the fix), grad_scale 1/3, on a mixed state and on one with p = 0.  The float64 oracle runs on the device."""
    opt = _opt(n, dev)
    worst = (0.0, None)
    for seed, p_zero in ((n % 997, False), (n % 997 + 1, True)):
        st = [x.to(dev) for x in oc.make_state(n, seed, p_zero)]
        for step in (6, 1000):
            hp = (step, 1e-4, 0.9, 0.999, 1e-5, 1.0 / 3.0)
            r, res = _check_step(_one_step(opt, st, *hp), st, hp)
            print(f"  [n {n} step {step} p=0 {p_zero}] p {res['p'][0]:.3g} m {res['m'][0]:.3g} v {res['v'][0]:.3g} of the bound")
            worst = max(worst, (r, (p_zero, step)), key=lambda w: w[0])
        del st
    print(f"  [n {n}] worst {worst[0]:.3g} of the bound at (p=0, step) = {worst[1]}")
    assert worst[0] <= 1.0, worst


@pytest.mark.parametrize("eps", oc.EPSS)
@pytest.mark.parametrize("betas", oc.BETAS, ids=str)
def test_radam_one_step_grid(dev, betas, eps):
    """n = 4099 (a ragged last block): every step, grad_scale and lr at these betas and eps, mixed state and p = 0."""
    b1, b2 = betas
    opt = _opt(oc.GRID_N, dev)
    states = [[x.to(dev) for x in oc.make_state(oc.GRID_N, seed, p_zero)] for seed, p_zero in ((1, False), (2, True))]
    bad, per_step = [], {}
    for step in oc.STEPS:
        for gs in oc.GRAD_SCALES:
            for lr in oc.LRS:
                for k, st in enumerate(states):
                    hp = (step, lr, b1, b2, eps, gs)
                    r, _ = _check_step([x.clone() for x in _one_step(opt, st, *hp)], st, hp)
                    per_step[step] = max(per_step.get(step, 0.0), r)
                    if not r <= 1.0:
                        bad.append((step, gs, lr, k, r))
    print(f"  [betas {betas} eps {eps}] worst ratio per step: " + ", ".join(f"{s}: {r:.3g}" for s, r in per_step.items()))
    assert not bad, bad[:20]


def test_radam_trajectory(dev):
    """1200 eager steps from a zero state on fp32 gradients; lr decayed by 0.995 through param_groups after step 1000.  p is
    reset to 0 before every step, so each step's p' is its update in one rounding (m and v are untouched by it)."""
    G = oc.traj_grads()
    ref = oc.traj_oracle(G)
    opt = _opt(oc.TRAJ_N, dev)
    Gd = G.to(dev)
    upd = torch.empty_like(Gd)
    for t in range(1, oc.TRAJ_STEPS + 1):
        opt.param_groups[0]["lr"] = oc.traj_lr(t)
        opt.flat_param.zero_()
        opt.flat_grad.copy_(Gd[t - 1])
        opt.step()
        upd[t - 1].copy_(opt.flat_param)
    assert int(opt.step_dev.item()) == oc.TRAJ_STEPS == opt._step
    r = oc.traj_ratios(upd.cpu(), ref)
    t = int(torch.argmax(r)) + 1
    print(f"  [trajectory] worst {float(r.max()):.3g} of the bound at step {t}; at steps 1 / 6 / 100 / 1000 / 1001 / 1200: "
          + " / ".join(f"{float(r[s - 1]):.3g}" for s in (1, 6, 100, 1000, 1001, 1200)))
    assert float(r.max()) <= 1.0, t


def test_radam_graph_replay(dev):
    """optimizer.step() captured in a CUDA graph as train.py's _capture does, replayed 6 times from step 3 (across the switch to
    the adaptive branch at step 6) with new gradients before each replay, sync_hyper() between replays and lr changed once.
    Every replay: within the one-step bounds of the oracle from the state before it, bit-identical to an eager twin, and
    step_dev equal to the host's count."""
    n = 5000
    opt, twin = _opt(n, dev), _opt(n, dev)
    st = [x.to(dev) for x in oc.make_state(n, 4)]
    for o in (opt, twin):
        for dst, src in zip((o.flat_param, o.flat_grad, o.exp_avg, o.exp_avg_sq), st):
            dst.copy_(src)
        o.step_dev.fill_(2)
        o._step = 2
    opt.sync_hyper()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()
    assert int(opt.step_dev.item()) == 2                   # captured, not run
    grads = [torch.from_numpy((np.random.RandomState(k).randn(n) * 10.0 ** np.random.RandomState(k + 50).uniform(-4, 1, n))
                              .astype(np.float32)).to(dev) for k in range(6)]
    worst = 0.0
    for k in range(6):
        lr = 1e-4 if k < 3 else 3e-4
        for o in (opt, twin):
            o.param_groups[0]["lr"] = lr
            o.flat_grad.copy_(grads[k])
        before = [x.clone() for x in (opt.flat_param, opt.flat_grad, opt.exp_avg, opt.exp_avg_sq)]
        opt.sync_hyper()
        graph.replay()
        opt._step += 1
        twin.step()
        step = k + 3
        assert int(opt.step_dev.item()) == opt._step == step
        for a, b in zip((opt.flat_param, opt.exp_avg, opt.exp_avg_sq), (twin.flat_param, twin.exp_avg, twin.exp_avg_sq)):
            assert torch.equal(a, b), step
        hp = (step, lr, 0.9, 0.999, 1e-5, 1.0)
        r, _ = _check_step((opt.flat_param, opt.exp_avg, opt.exp_avg_sq), before, hp)
        print(f"  [graph replay {k + 1}, step {step}, lr {lr}] worst {r:.3g} of the bound")
        worst = max(worst, r)
    assert worst <= 1.0


def _params(dev, seed=6):
    rs = np.random.RandomState(seed)
    return [torch.nn.Parameter(torch.from_numpy(rs.randn(*s).astype(np.float32)).to(dev)) for s in ((33, 7), (129,), (4, 5, 6))]


@pytest.mark.parametrize("fmt", ["zeggs", "reference"])
def test_radam_resume(dev, fmt):
    """state_dict at step 5, loaded into a fresh optimizer over parameters holding the step-5 values, then steps 6-8 (the switch
    to the adaptive branch): the bits of an uninterrupted run.  `reference` is the reference optimizer's per-parameter layout."""
    from zeggs_b200.optimizers import RAdam
    rs = np.random.RandomState(8)
    n = sum(p.numel() for p in _params(dev))
    grads = [torch.from_numpy((rs.randn(n) * 10.0 ** rs.uniform(-3, 1, n)).astype(np.float32)).to(dev) for _ in range(8)]

    def run(opt, steps):
        for k in steps:
            opt.flat_grad.copy_(grads[k])
            opt.step()

    full = RAdam(_params(dev), lr=2e-4, eps=1e-5)
    run(full, range(8))
    head = RAdam(_params(dev), lr=2e-4, eps=1e-5)
    run(head, range(5))
    if fmt == "zeggs":
        sd = copy.deepcopy(head.state_dict())
    else:
        sd = dict(param_groups=[dict(lr=2e-4, betas=(0.9, 0.999), eps=1e-5, weight_decay=0, params=[0, 1, 2])], state={})
        off = 0
        for i, p in enumerate(head.param_groups[0]["params"]):
            k = p.numel()
            sd["state"][i] = dict(step=5, exp_avg=head.exp_avg[off:off + k].view(p.shape).clone(),
                                  exp_avg_sq=head.exp_avg_sq[off:off + k].view(p.shape).clone())
            off += k
    ps = _params(dev)
    for p, q in zip(ps, head.param_groups[0]["params"]):
        p.data.copy_(q.data)
    resumed = RAdam(ps, lr=1e-3, eps=1e-8)                 # the checkpoint's lr and eps replace these
    resumed.load_state_dict(sd)
    assert resumed._step == 5 and int(resumed.step_dev.item()) == 5
    run(resumed, range(5, 8))
    assert resumed._step == 8 == full._step and int(resumed.step_dev.item()) == 8
    for a, b in zip((resumed.flat_param, resumed.exp_avg, resumed.exp_avg_sq), (full.flat_param, full.exp_avg, full.exp_avg_sq)):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------- dropout masks
MASK_SIZES = [1, 2, 255, 256, 257, 1024, 1025, 2424831, 2424832, 2424833, 32 * 4 * 384 * 384]
MASK_PS = [0.0, 0.1, 0.2, 0.5, 0.99999994]


def _mask(dev, n, p, seed=None, t=None, salt=None):
    from zeggs_b200 import _lib
    out = torch.empty(n, dtype=torch.float32, device=dev)
    if t is None:
        _lib.check(_lib.lib().zeggs_dropout_mask(out.data_ptr(), n, float(p), seed, _lib.stream_ptr()), "zeggs_dropout_mask")
    else:
        td = torch.tensor([t], dtype=torch.int64, device=dev)
        _lib.check(_lib.lib().zeggs_dropout_mask_dev(out.data_ptr(), n, float(p), td.data_ptr(), salt, _lib.stream_ptr()),
                   "zeggs_dropout_mask_dev")
    return out


@pytest.mark.parametrize("n", MASK_SIZES)
def test_dropout_masks_bit_exact(dev, n):
    """Both kernels against the restatement, bit for bit, at every p; seeds 0, 1, 2^62 - 1 and a random one, salts 1-4 (at the
    attention-mask size two seeds and two (seed, salt) pairs)."""
    seeds = [0, 1, 2 ** 62 - 1, int(np.random.RandomState(n % 1000).randint(0, 2 ** 62, dtype=np.int64))]
    big = n > 2424833
    host = seeds[1:3] if big else seeds
    devs = [(seeds[2], 1), (seeds[3], 4)] if big else [(t, s) for t in seeds for s in (1, 2, 3, 4)]
    cases = [("host", s, None, ro.words(n, s)) for s in host] + [("dev", t, s, ro.words(n, ro.device_seed(t, s))) for t, s in devs]
    checked = 0
    for kind, s, salt, u in cases:
        for p in MASK_PS:
            want = torch.from_numpy(ro.mask_from_words(u, p)).to(dev)
            got = _mask(dev, n, p, seed=s) if kind == "host" else _mask(dev, n, p, t=s, salt=salt)
            if not torch.equal(got.view(torch.int32), want.view(torch.int32)):
                bad = int((got != want).nonzero()[0])
                raise AssertionError(f"{kind} seed {s} salt {salt} p {p}: first mismatch at {bad} of {n}")
            checked += 1
    print(f"  [n {n}] {checked} masks bit-exact")


@pytest.mark.parametrize("p", [1.0, -0.1, float("nan")])
def test_dropout_refuses_bad_p_before_launch(dev, p):
    from zeggs_b200 import _lib
    out = torch.full((1000,), 7.0, device=dev)
    td = torch.zeros(1, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    before = _lib.lib().zeggs_launch_count()
    assert _lib.lib().zeggs_dropout_mask(out.data_ptr(), 1000, p, 5, _lib.stream_ptr()) != 0
    assert _lib.lib().zeggs_dropout_mask_dev(out.data_ptr(), 1000, p, td.data_ptr(), 1, _lib.stream_ptr()) != 0
    assert _lib.lib().zeggs_launch_count() == before
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())


def test_dropout_host_seed_follows_torch_manual_seed(dev):
    """ops._drop_mask outside a device_seed context draws its seed from torch's CPU generator: the same mask after the same
    torch.manual_seed, a new one on the next call, and the restatement's mask at that seed."""
    from zeggs_b200 import ops
    shape = (64, 257, 33)
    n = int(np.prod(shape))
    for p in (0.1, 0.2):
        torch.manual_seed(5)
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        torch.manual_seed(5)
        a = ops._drop_mask(shape, p, dev)
        b = ops._drop_mask(shape, p, dev)
        torch.manual_seed(5)
        a2 = ops._drop_mask(shape, p, dev)
        assert torch.equal(a, a2) and not torch.equal(a, b)
        assert torch.equal(a.flatten().cpu(), torch.from_numpy(ro.dropout_mask(n, p, seed)))


# ---------------------------------------------------------------------------------------------- VAE noise
def _randn(dev, n, t, salt):
    from zeggs_b200 import _lib
    out = torch.empty(n, dtype=torch.float32, device=dev)
    td = torch.tensor([t], dtype=torch.int64, device=dev)
    _lib.check(_lib.lib().zeggs_randn_dev(out.data_ptr(), n, td.data_ptr(), salt, _lib.stream_ptr()), "zeggs_randn_dev")
    return out


def _randn_ulps(got, want):
    """-> (worst |got - want| in fp32 ulps of want, worst ratio to the bound, index)."""
    want32 = np.abs(want).astype(np.float32)
    ulp = np.spacing(want32).astype(np.float64)
    d = np.abs(got.astype(np.float64) - want)
    ratio = d / (RANDN_ULPS * ulp + RANDN_FLOOR)
    i = int(np.argmax(ratio))
    return float(np.max(d / ulp)), float(ratio[i]), i


@pytest.mark.parametrize("n", [1, 2, 3, 606207, 606208, 606209, 2000001])
def test_randn_dev_against_restatement(dev, n):
    """Every element within RANDN_ULPS fp32 ulps (plus a 2^-140 floor) of the restatement, for two (seed word, salt) pairs; the
    grid of 1184 x 256 pair-threads is exactly full at n = 606208."""
    for t, salt in ((0, 1), (2 ** 62 - 1 - n, 3)):
        got = _randn(dev, n, t, salt).cpu().numpy()
        want = ro.randn_dev(n, t, salt)
        assert np.all(np.isfinite(got))
        ulps, r, i = _randn_ulps(got, want)
        print(f"  [n {n} seed {t} salt {salt}] worst {ulps:.2f} ulp, {r:.3g} of the bound (element {i}: {got[i]!r} vs {want[i]!r})")
        assert r <= 1.0, i


# ---------------------------------------------------------------------------------------------- graph replay
def test_graph_replay_draws_fresh_values(dev):
    """DeviceSeed.advance() and one step's draws (two dropout masks, the VAE noise) captured in a CUDA graph inside
    ops.device_seed: replay k draws the restatement's masks and noise at seed word t0 + k, salts 1, 2 and 3."""
    from zeggs_b200 import ops
    seed = ops.DeviceSeed(dev)
    t0 = int(seed.t.item())
    with ops.device_seed(ops.DeviceSeed(dev)):            # load the kernels before the capture
        ops._drop_mask((3, 5), 0.2, dev)
        ops._draw_eps((3, 4), dev)
    torch.cuda.synchronize()
    shapes = ((32, 34, 256), (32, 4, 34, 34), (32, 64))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        seed.advance()
        with ops.device_seed(seed):
            a = ops._drop_mask(shapes[0], 0.2, dev)
            b = ops._drop_mask(shapes[1], 0.1, dev)
            e = ops._draw_eps(shapes[2], dev)
    assert int(seed.t.item()) == t0
    for k in range(1, 4):
        g.replay()
        assert int(seed.t.item()) == t0 + k
        assert torch.equal(a.flatten().cpu(), torch.from_numpy(ro.dropout_mask_dev(a.numel(), 0.2, t0 + k, 1)))
        assert torch.equal(b.flatten().cpu(), torch.from_numpy(ro.dropout_mask_dev(b.numel(), 0.1, t0 + k, 2)))
        ulps, r, _ = _randn_ulps(e.flatten().cpu().numpy(), ro.randn_dev(e.numel(), t0 + k, 3))
        print(f"  [replay {k}] masks bit-exact, noise worst {ulps:.2f} ulp")
        assert r <= 1.0
