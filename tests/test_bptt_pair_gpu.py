"""The tensor-core BPTT kernel at the hidden sizes whose cluster-pair grid differs from the others: H = 512 (U = 4, 128 CTAs = 64
pairs, the narrowest chains: B2 24 columns, B3 40 / 56) and H = 768 (U = 8, 96 CTAs = 48 pairs).  Same contract as
test_tc_engine_gpu.test_tc_backward_vs_matched_oracle: every decoder parameter gradient, dSpeech and dStyle against autograd through the
bf16-operand-matched oracle, relative L2 error <= TC_GRAD_TOL."""
import pytest

from oracle import tc_oracle as tco
from tests._util import run_with_grads
from tests.test_tc_engine_gpu import _case, _run_gpu, dev, engine  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("H,B,T", [(H, B, T) for H in (512, 768) for B, T in ((1, 5), (16, 12), (32, 17))])
def test_bptt_pair_backward_vs_matched_oracle(dev, engine, H, B, T):  # noqa: F811
    engine("tc")
    case = _case(H, B, T, 64, seed=1700 + H + B + T)
    _, g_got = _run_gpu(dev, *case, H, 64, grads=True)
    _, g_tc = run_with_grads(tco.decoder_forward_tc, *case, bf16=True)
    bad = []
    for k in g_tc:
        e = tco.rel_l2(g_got[k], g_tc[k])
        print(f"  [tc bwd H{H} B{B} T{T}] {k:48s} relL2 vs matched {e:.3e}")
        if not e <= tco.TC_GRAD_TOL:
            bad.append((k, e))
    assert not bad, bad
