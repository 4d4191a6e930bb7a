"""GPU: the GRU style encoder (`style_type: "gru"`; csrc/style_gru.cu, zeggs_style_enc_gru_fwd / _bwd) against the float64 oracle at
every hidden size it accepts, at the batch-tile, K-chunk and sequence edges of its recurrences, at the training shape and at the
generation shape.  Cases and oracles: tests/_gru_cases.py.

* Every accepted hidden size (198: H % 4 == 0 up to 528, H % 8 == 0 up to 1056), forward at B = 3, T = 5, GEMM modes 0 and 1.
* Forward and backward at H in {4, 512, 516, 528, 536, 1056} x B in {1, 31, 32, 33, 64, 65} (T = 17, VAE), T in {1, 2} at B in
  {1, 33} without the VAE, an odd-width encoding (E = 63) without the VAE, and the training shape (B = 32, T = 384, H = 512) with
  and without the VAE -- each in three settings: GEMM mode 0 (fp32 SIMT), mode 1 (tensor-core split-bf16) with fast_wgrad = 0, and
  mode 1 with fast_wgrad = 1 (what the tensor-core decoder engine selects: weight gradients in one bf16 pass).
* Generation: B = 1, T = 1000 and 3600, forward only, no eps (z = mu).
* Refusals: H = 6, 532, 1064 and an odd encoding with the VAE raise ZeggsError before any launch.
Bounds:
  outputs (z / mu / logvar), natural and margined parameters    max-abs <= 2e-5 * max(1, max|ref|) vs the float64 oracle
  every gradient (margined parameters), first two settings       relative L2 per tensor <= 1e-4 vs the float64 oracle
  fast_wgrad = 1: the weight gradients whose product meets the   relative L2 per tensor <= 5e-4 vs the bf16-matched float64
    tensor-core rule (M*N*K >= 4e6); every other gradient 1e-4     restatement
  the reverse direction's W_hh gradient                           exactly zero
tests/test_style_gru_f64_cpu.py shows the float32 oracle meets them with >= 4x headroom and each modelled kernel fault exceeds them.
"""
import pytest
import torch

from tests import _gru_cases as gc
from tests._util import ensure_built

pytestmark = pytest.mark.gpu

SETTINGS = ["mode0", "mode1", "mode1_fast_wgrad"]
_PREFIX = "style_encoder."


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


@pytest.fixture
def setting(dev):
    """Select GEMM mode and weight-gradient mode (through the decoder engine, as a user does) for one test; restore afterwards."""
    from zeggs_b200 import ops
    prev = ops.DECODER_ENGINE

    def apply(name):
        ops.set_gemm_mode(0 if name == "mode0" else 1)
        ops.set_decoder_engine("tc" if name == "mode1_fast_wgrad" else "fp32")
    yield apply
    ops.set_gemm_mode(1)
    ops.set_decoder_engine(prev)


def _module(P, case, dev):
    from zeggs_b200 import modules
    mod = modules.StyleEncoder(1134, case.H, case.E // 2 if case.vae else case.E, type="gru", use_vae=case.vae)
    mod.load_state_dict({k[len(_PREFIX):]: torch.from_numpy(v) for k, v in P.items()})
    return mod.to(dev)


def _run_gpu(P, case, dev, grads):
    """-> (outputs, {key: gradient} or None) of the CUDA module."""
    from zeggs_b200 import ops
    mod = _module(P, case, dev)
    x = case.x.to(dev)
    with torch.set_grad_enabled(grads):
        if case.vae and case.eps is None:      # generation: no eps at all, z = mu (the kernel's eps == NULL branch)
            outs = [o for o in ops.style_encoder_fwd(mod, x, None, None, case.temperature)[0] if o is not None]
        else:
            eps = None if case.eps is None else case.eps.to(dev)
            outs = [o for o in mod(x, case.temperature, eps=eps) if o is not None]
    if not grads:
        torch.cuda.synchronize()
        return outs, None
    named = dict(mod.named_parameters())
    keys = sorted(P)
    gs = torch.autograd.grad(sum((o * c.to(dev)).sum() for o, c in zip(outs, case.cots)), [named[k[len(_PREFIX):]] for k in keys])
    torch.cuda.synchronize()
    return outs, dict(zip(keys, gs))


def _report(tag, errs):
    for n, e, b in errs:
        print(f"  [{tag}] {n}: {e:.2e} (bound {b:.1e})")
    n, e, b = max(errs, key=lambda x: x[1] / x[2])
    print(f"  [{tag}] WORST {n}: {e:.2e} = {e / b:.3f} of its bound")
    bad = [x for x in errs if not x[1] <= x[2]]
    assert not bad, bad


_oracles = {}


def _oracle(cid):
    """Cached per case: (case, natural parameters, margined parameters, natural outputs, margined outputs, gradients, matched
    gradients, keys the matched oracle rounded).  The settings of one case run one after another: only that case is kept."""
    if cid not in _oracles:
        _oracles.clear()
        case = gc.make_case(cid)
        P = gc.gru_params(case.H, case.E)
        Pm = gc.margined_params(P, case)
        nat_o = gc.run_oracle(P, case)[0]
        o, g = gc.run_oracle(Pm, case)
        _, mg, opts = gc.run_restated(Pm, case, matched=True)
        _oracles[cid] = (case, P, Pm, nat_o, o, g, mg, {r[0] for r in opts.rounded})
    return _oracles[cid]


@pytest.mark.parametrize("H", gc.hidden_sizes())
def test_forward_at_every_hidden_size(dev, setting, H):
    case = gc.sweep_case(H)
    P = gc.gru_params(H, case.E)
    ref = gc.run_oracle(P, case)[0]
    for name in ("mode0", "mode1"):
        setting(name)
        _report(f"H{H} B3 T5 {name}", gc.errors(_run_gpu(P, case, dev, False)[0], None, ref, None))


@pytest.mark.parametrize("name", SETTINGS)
@pytest.mark.parametrize("cid", list(gc.CASES))
def test_gru_style_encoder_vs_float64(dev, setting, cid, name):
    setting(name)
    case, P, Pm, nat_o, o, g, mg, rounded = _oracle(cid)
    fast = name == "mode1_fast_wgrad"
    errs = [(f"natural {n}", e, b) for n, e, b in gc.errors(_run_gpu(P, case, dev, False)[0], None, nat_o, None)]
    go, gg = _run_gpu(Pm, case, dev, True)
    errs += gc.errors(go, gg, o, mg if fast else g, rounded if fast else ())
    # the reverse direction's W_hh multiplied h = 0: exactly zero gradient, as the reference's autograd gives
    assert float(gg[gc.W_HH_R].abs().max()) == 0.0
    _report(f"{cid} {name}", errs)


@pytest.mark.parametrize("name", ["mode0", "mode1"])
@pytest.mark.parametrize("cid", list(gc.GEN_CASES))
def test_generation_forward_vs_float64(dev, setting, cid, name):
    setting(name)
    if cid not in _oracles:
        _oracles.clear()
        case = gc.make_case(cid)
        P = gc.gru_params(case.H, case.E)
        _oracles[cid] = (case, P, gc.run_oracle(P, case)[0])
    case, P, ref = _oracles[cid]
    _report(f"{cid} {name}", gc.errors(_run_gpu(P, case, dev, False)[0], None, ref, None))


@pytest.mark.parametrize("H,E", [(6, 128), (532, 128), (1064, 128), (512, 63)])
def test_unsupported_shapes_are_refused_before_any_launch(dev, H, E):
    """Hidden sizes style_gru_units rejects, and an odd encoding with the VAE (mu and logvar split it in halves)."""
    from zeggs_b200 import _lib, modules
    mod = modules.StyleEncoder(1134, H, 64, type="gru", use_vae=True)
    if E % 2:
        mod.encoder.projection_layer = modules.LinearNorm(2 * H, E, w_init_gain="linear")
    mod = mod.to(dev)
    x = torch.zeros(2, 5, 1134, device=dev)
    torch.cuda.synchronize()
    launches = _lib.lib().zeggs_launch_count()
    with pytest.raises(_lib.ZeggsError) as ei:
        mod(x, 1.0, eps=torch.zeros(2, E // 2, device=dev))
    print(f"  [H{H} E{E}] {ei.value}")
    assert _lib.lib().zeggs_launch_count() == launches
