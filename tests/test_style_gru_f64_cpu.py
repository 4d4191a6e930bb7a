"""No GPU: the bounds of tests/test_style_gru_f64_gpu.py mean something.

* The fault-injectable restatement of the GRU style encoder (tests/_gru_cases.py), without a fault, equals the float64 oracle
  (oracle/style_oracle.py, full bidirectional scans) to 1e-12.
* The float32 oracle meets every bound with at least 4x headroom at the training shape and at the largest case (H = 1056, B = 65).
* The ReLU gate-margin precondition holds for every case the GPU file runs with gradients.
* The bf16-matched oracle evaluated in float32 passes the matched bound, and the unmatched float64 oracle fails it: a kernel that
  silently ran the fp32-grade weight-gradient product would fail.
* Every modelled kernel fault exceeds its bound at a case where it can appear.
"""
import pytest
import torch

from tests import _encoder_cases as ec
from tests import _gru_cases as gc

_cases = {}


def _main(cid):
    """(margined parameters, case, float64 oracle outputs, gradients), cached per case."""
    if cid not in _cases:
        case = gc.make_case(cid)
        P = gc.margined_params(gc.gru_params(case.H, case.E), case)
        _cases[cid] = (P, case) + tuple(gc.run_oracle(P, case))
    return _cases[cid]


def _show(tag, errs):
    for n, e, b in errs:
        print(f"  [{tag}] {n}: {e:.2e} (bound {b:.1e}, {b / max(e, 1e-30):.1f}x headroom)")


def test_hidden_sizes_are_every_size_the_kernel_accepts():
    hs = gc.hidden_sizes()
    assert len(hs) == 198 and hs[0] == 4 and hs[131] == 528 and hs[132] == 536 and hs[-1] == 1056
    assert set(gc.H_EDGES) <= set(hs)


@pytest.mark.parametrize("cid", [gc.TRAIN, "H512_B32_T384_novae", gc.LARGEST, "H4_B1_T1_novae", "H536_B33_T2_novae",
                                 "H516_B33_T17_E63"])
def test_restatement_equals_float64_oracle(cid):
    case = gc.make_case(cid)
    P = gc.gru_params(case.H, case.E) if cid not in (gc.TRAIN, gc.LARGEST) else _main(cid)[0]
    ref_o, ref_g = gc.run_oracle(P, case)
    o, g, _ = gc.run_restated(P, case)
    for a, b in zip(o, ref_o):
        assert float((a - b).abs().max()) <= 1e-12 * max(1.0, float(b.abs().max()))
    for k in ref_g:
        assert float((g[k] - ref_g[k]).abs().max()) <= 1e-12 * max(1e-30, float(ref_g[k].abs().max())), k
    assert float(ref_g[gc.W_HH_R].abs().max()) == 0.0 and float(g[gc.W_HH_R].abs().max()) == 0.0


@pytest.mark.parametrize("cid", [gc.TRAIN, gc.LARGEST])
def test_float32_oracle_meets_every_bound_with_4x_headroom(cid):
    P, case, ref_o, ref_g = _main(cid)
    errs = gc.errors(*gc.run_oracle(P, case, torch.float32), ref_o, ref_g)
    _show(f"{cid} fp32", errs)
    assert not [x for x in errs if not 4 * x[1] <= x[2]]
    # the natural parameters' outputs too (the GPU file checks forwards with them)
    Pn = gc.gru_params(case.H, case.E)
    errs = gc.errors(gc.run_oracle(Pn, case, torch.float32)[0], None, gc.run_oracle(Pn, case)[0], None)
    _show(f"{cid} fp32 natural", errs)
    assert not [x for x in errs if not 4 * x[1] <= x[2]]


def test_float32_oracle_meets_the_forward_bound_at_the_generation_shape():
    case = gc.make_case("H512_B1_T3600_gen")
    P = gc.gru_params(case.H, case.E)
    errs = gc.errors(gc.run_oracle(P, case, torch.float32)[0], None, gc.run_oracle(P, case)[0], None)
    _show("T3600 fp32", errs)
    assert not [x for x in errs if not 4 * x[1] <= x[2]]


@pytest.mark.parametrize("cid", list(gc.CASES))
def test_gate_margins_hold_for_every_gpu_case(cid):
    """Every ReLU pre-activation of the margined parameters lies at least GATE_RATIO x the float32 error of its layer from zero."""
    if cid in _cases:
        P, case = _cases[cid][:2]
    else:
        case = gc.make_case(cid)
        P = gc.margined_params(gc.gru_params(case.H, case.E), case)
    for site, (margin, err) in gc.gate_margins(P, case).items():
        print(f"  [{cid} {site}] nearest |pre| {margin:.2e}, fp32 error {err:.2e}: {margin / max(err, 1e-30):.0f}x")
        assert margin >= ec.GATE_RATIO * err, site


@pytest.mark.parametrize("cid", [gc.TRAIN, gc.LARGEST])
def test_matched_bound_separates_single_pass_bf16_from_fp32_grade(cid):
    P, case, ref_o, ref_g = _main(cid)
    mo, mg, opts = gc.run_restated(P, case, matched=True)
    # at these shapes every weight gradient fast_wgrad = 1 can run in one bf16 pass meets the tensor-core rule
    rounded = {key: M * N * K for key, M, N, K in opts.rounded}
    assert sorted(rounded) == sorted(gc.WGRADS)
    assert all(mnk >= ec.TC_MIN_MNK for mnk in rounded.values())
    for k in ref_g:
        if k not in rounded:
            assert float((mg[k] - ref_g[k]).abs().max()) <= 1e-12 * max(1e-30, float(ref_g[k].abs().max())), k
    m32o, m32g, _ = gc.run_restated(P, case, torch.float32, matched=True)
    errs = gc.errors(m32o, m32g, mo, mg, rounded)
    _show(f"{cid} matched fp32", errs)
    assert not [x for x in errs if not 4 * x[1] <= x[2]]
    for k in rounded:
        e = ec.rel_l2(ref_g[k], mg[k])
        print(f"  [{cid} unmatched float64] {k}: {e:.2e} = {e / gc.MATCHED_TOL[k]:.1f}x the bound {gc.MATCHED_TOL[k]:.1e}")
        assert e > gc.MATCHED_TOL[k], k


def test_small_products_are_not_matched():
    """Below the tensor-core rule the single-pass setting leaves a weight gradient fp32-grade: at H = 4 only conv1 (4 x 3402 over
    1105 rows) is rounded, and without the VAE the B = 32 projection (64 x 1024 over 32 rows) is not."""
    _, _, o = gc.run_restated(gc.gru_params(4, 128), gc.make_case("H4_B65_T17_vae"), matched=True)
    assert [r[0] for r in o.rounded] == [gc.CONV1]
    case = gc.make_case("H512_B32_T384_novae")
    _, _, o = gc.run_restated(gc.gru_params(512, 64), case, matched=True)
    assert sorted(r[0] for r in o.rounded) == sorted(k for k in gc.WGRADS if k != gc.W_P)


@pytest.mark.parametrize("fault", list(gc.FAULTS))
def test_modelled_fault_exceeds_its_bound(fault):
    cid = gc.FAULT_CASE[fault]
    P, case, ref_o, ref_g = _main(cid)
    o, g, _ = gc.run_restated(P, case, fault=fault)
    # the looser matched bounds on the single-pass weight gradients too: the fault shows in every setting
    errs = gc.errors(o, g, ref_o, ref_g, gc.WGRADS)
    n, e, b = max(errs, key=lambda x: x[1] / x[2])
    print(f"  [{fault} at {cid}] worst {n}: {e:.2e} = {e / b:.0f}x its bound")
    assert e > b
