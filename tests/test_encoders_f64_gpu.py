"""GPU: the speech encoder and the attention style encoder (csrc/encoders.cu) against float64 oracles at the shapes they run at --
training (32 x 256 speech, 32 x 384 style), the padding / narrow-N / column-reduction edges and generation (150 s of speech, style
clips of 1000 and 3600 frames).  Cases and oracles: tests/_encoder_cases.py.

Every case runs in three settings: GEMM mode 0 (fp32 SIMT), mode 1 (tensor-core split-bf16) with fast_wgrad = 0, and mode 1 with
fast_wgrad = 1 (what the tensor-core decoder engine selects; the encoders' weight gradients run as ONE bf16 pass).  Bounds:
  outputs (z / mu / logvar, speech features), natural parameters     max-abs <= 2e-5 * max(1, max|ref|) vs float64 model_oracle
  every gradient (gate-margined style parameters), first two settings  relative L2 per tensor <= 1e-4 vs float64 model_oracle autograd
  fast_wgrad = 1: the weight gradients whose product meets the         relative L2 per tensor vs the bf16-matched float64 oracle:
    tensor-core rule (M*N*K >= 4e6); every other gradient 1e-4           speech 3.5e-4, style conv1 2.5e-4, the other style weights 6e-5
  zeggs_gemm_f32_ctx mode 1, fast_wgrad = 1, encoder wgrad shapes     max-abs <= 2e-5 * max|C| vs float64 of the bf16-rounded operands
tests/test_encoders_f64_cpu.py shows the float32 oracle meets them with >= 4x headroom and each modelled kernel fault exceeds them.
"""
import ctypes as C

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


@pytest.mark.parametrize("M,N,K", [(512, 3402, 12288), (64, 1984, 8192), (384, 128, 12288)])   # style conv1, speech conv (split-K), in_proj
def test_single_pass_bf16_weight_gradient_gemm(dev, M, N, K):
    """zeggs_gemm_f32_ctx, mode 1 (C = A[K,M]^T B[K,N]) with a fast_wgrad = 1 context: the float64 product of the bf16-rounded
    operands to 2e-5 of max|C| (worst 7.0e-6, at K = 12288), and 100x further from the fp32-grade product of the unrounded ones (2.0e-3)."""
    from zeggs_b200 import _lib
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    ctx = _lib.Ctx(scratch=scratch.data_ptr(), scratch_bytes=scratch.numel(), gemm_mode=1, fast_wgrad=1)
    assert M * N * K >= ec.TC_MIN_MNK
    g = torch.Generator().manual_seed(M + N + K)
    A, B = torch.randn(K, M, generator=g), torch.randn(K, N, generator=g)
    ref = A.to(torch.bfloat16).double().T @ B.to(torch.bfloat16).double()
    Ad, Bd = A.to(dev), B.to(dev)
    out = torch.empty(M, N, device=dev)
    _lib.check(_lib.lib().zeggs_gemm_f32_ctx(C.addressof(ctx), 1, M, N, K, Ad.data_ptr(), M, Bd.data_ptr(), N, None, out.data_ptr(), N,
                                             0, 0, _lib.stream_ptr()), "zeggs_gemm_f32_ctx")
    torch.cuda.synchronize()
    got = out.cpu().double()
    sc = float(ref.abs().max())
    err = float((got - ref).abs().max())
    err_exact = float((got - A.double().T @ B.double()).abs().max())
    print(f"  [gemm fast_wgrad {M}x{N} over {K}] vs bf16 operands {err / sc:.2e}, vs unrounded {err_exact / sc:.2e} of max|C|")
    assert err <= 2e-5 * sc
    assert err_exact > 50 * 2e-5 * sc
