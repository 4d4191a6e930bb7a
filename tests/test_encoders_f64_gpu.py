"""GPU: the speech encoder and the attention style encoder (csrc/encoders.cu) against float64 oracles at the shapes they run at --
training (32 x 256 speech, 32 x 384 style), the padding / narrow-N / column-reduction edges and generation (150 s of speech, style
clips of 1000 and 3600 frames).  Cases and oracles: tests/_encoder_cases.py.

Every case runs in three settings: GEMM mode 0 (fp32 SIMT), mode 1 (tensor-core split-bf16) with fast_wgrad = 0, and mode 1 with
fast_wgrad = 1 (what the tensor-core decoder engine selects; the encoders' weight gradients run as ONE bf16 pass).  Bounds:
  outputs (z / mu / logvar, speech features), natural parameters     max-abs <= 2e-5 * max(1, max|ref|) vs float64 model_oracle
  every gradient (gate-margined style parameters), first two settings  relative L2 per tensor <= 1e-4 vs float64 model_oracle autograd
  fast_wgrad = 1: the weight gradients whose product meets the         relative L2 per tensor vs the bf16-matched float64 oracle:
    tensor-core rule (M*N*K >= 4e6); every other gradient 1e-4           speech 3.5e-4, style conv1 2.5e-4, the other style weights 6e-5
tests/test_encoders_f64_cpu.py shows the float32 oracle meets them with >= 4x headroom and each modelled kernel fault exceeds them.
The single-pass weight-gradient product at the encoders' shapes is checked on its own in tests/test_gemm_f64_gpu.py.
"""
import pytest
import torch

from tests import _encoder_cases as ec
from tests._util import ensure_built

pytestmark = pytest.mark.gpu

SETTINGS = ["mode0", "mode1", "mode1_fast_wgrad"]


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


_oracles = {}


def _oracle(kind, cid):
    """Cached per case: (case, natural parameters, margined parameters, natural outputs, margined outputs, gradients, matched
    gradients, keys the matched oracle rounded)."""
    if (kind, cid) not in _oracles:
        case = ec.make_case(kind, cid)
        P = ec.speech_params() if kind == "speech" else ec.style_params(case.vae)
        Pm = P if (kind == "speech" or case.cots is None) else ec.margined_style_params(P, case)
        nat_o = ec.run_oracle(P, case)[0] if Pm is not P else None
        o, g = ec.run_oracle(Pm, case)
        mg, rounded = None, ()
        if g is not None:
            _, mg, opts = ec.run_restated(Pm, case, matched=True)
            rounded = {r[0] for r in opts.rounded}
        _oracles[(kind, cid)] = (case, P, Pm, nat_o if nat_o is not None else o, o, g, mg, rounded)
    return _oracles[(kind, cid)]


def _module(kind, P, vae, dev):
    from zeggs_b200 import modules
    prefix = kind + "_encoder."
    mod = modules.SpeechEncoder(81, 64, 64) if kind == "speech" else \
        modules.StyleEncoder(1134, 512, 64, type="attn", use_vae=vae)
    mod.load_state_dict({k[len(prefix):]: torch.from_numpy(v) for k, v in P.items()})
    return mod.to(dev)


def _run_gpu(kind, P, case, dev, grads):
    """-> (outputs, {key: gradient} or None) of the CUDA module."""
    from zeggs_b200 import ops
    vae = getattr(case, "vae", True)
    mod = _module(kind, P, vae, dev).train(case.train)
    x = case.x.to(dev)
    with torch.set_grad_enabled(grads):
        if kind == "speech":
            outs = [mod(x, None if case.masks is None else [m.to(dev) for m in case.masks])]
        elif vae and case.eps is None:     # generation: no eps at all, z = mu (the kernel's eps == NULL branch)
            outs = [o for o in ops.style_encoder_fwd(mod, x, None, None, case.temperature)[0] if o is not None]
        else:
            masks = None if case.masks is None else {k: v.to(dev) for k, v in case.masks.items()}
            eps = None if case.eps is None else case.eps.to(dev)
            outs = [o for o in mod(x, case.temperature, eps=eps, masks=masks) if o is not None]
    if not grads:
        torch.cuda.synchronize()
        return outs, None
    named = dict(mod.named_parameters())
    keys = sorted(P)
    prefix = kind + "_encoder."
    gs = torch.autograd.grad(sum((o * c.to(dev)).sum() for o, c in zip(outs, case.cots)), [named[k[len(prefix):]] for k in keys])
    torch.cuda.synchronize()
    return outs, dict(zip(keys, gs))


def _check(kind, cid, name, dev):
    case, P, Pm, nat_o, o, g, mg, rounded = _oracle(kind, cid)
    fast = name == "mode1_fast_wgrad"
    errs = [(f"natural {n}", e, b) for n, e, b in ec.errors(_run_gpu(kind, P, case, dev, False)[0], None, nat_o, None)]
    if g is not None:
        go, gg = _run_gpu(kind, Pm, case, dev, True)
        errs += ec.errors(go, gg, o, mg if fast else g, rounded if fast else ())
    for n, e, b in errs:
        print(f"  [{kind} {cid} {name}] {n}: {e:.2e} (bound {b:.1e})")
    n, e, b = max(errs, key=lambda x: x[1] / x[2])
    print(f"  [{kind} {cid} {name}] WORST {n}: {e:.2e} = {e / b:.3f} of its bound")
    bad = [x for x in errs if not x[1] <= x[2]]
    assert not bad, bad


@pytest.mark.parametrize("name", SETTINGS)
@pytest.mark.parametrize("cid", list(ec.SPEECH_CASES))
def test_speech_encoder_vs_float64(dev, setting, cid, name):
    setting(name)
    _check("speech", cid, name, dev)


@pytest.mark.parametrize("name", SETTINGS)
@pytest.mark.parametrize("cid", list(ec.STYLE_CASES))
def test_style_encoder_vs_float64(dev, setting, cid, name):
    setting(name)
    _check("style", cid, name, dev)
