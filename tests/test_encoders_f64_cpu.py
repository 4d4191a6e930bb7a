"""No GPU: the bounds of tests/test_encoders_f64_gpu.py mean something.

* The fault-injectable restatement (tests/_encoder_cases.py), without a fault, equals model_oracle to 1e-12.
* The float32 oracle meets every bound with at least 4x headroom at the training shapes: the bounds leave room for fp32 arithmetic.
* The ReLU gate-margin precondition holds for every style case the GPU file runs with gradients.
* The bf16-matched oracle evaluated in float32 passes the matched bound, and the unmatched float64 oracle fails it: a kernel that
  silently ran the fp32-grade weight-gradient product would fail.
* Every modelled kernel fault exceeds its bound at the training shape.
"""
import pytest
import torch

from tests import _encoder_cases as ec

MAIN = dict(speech="B32_T256", style="B32_T384_vae")


@pytest.fixture(scope="module")
def main_cases():
    """kind -> (parameters as the GPU file uses them for gradients, case, float64 model_oracle outputs, gradients)."""
    out = {}
    for kind, cid in MAIN.items():
        case = ec.make_case(kind, cid)
        P = ec.speech_params() if kind == "speech" else ec.margined_style_params(ec.style_params(), case)
        out[kind] = (P, case) + tuple(ec.run_oracle(P, case))
    return out


def _show(tag, errs):
    for n, e, b in errs:
        print(f"  [{tag}] {n}: {e:.2e} (bound {b:.1e})")


@pytest.mark.parametrize("kind,cid", [("speech", "B32_T256"), ("speech", "B2_T15"), ("style", "B32_T384_vae"), ("style", "B1_T1"),
                                      ("style", "B2_T129"), ("style", "B32_T384_novae")])
def test_restatement_equals_model_oracle(main_cases, kind, cid):
    if cid == MAIN[kind]:
        P, case, ref_o, ref_g = main_cases[kind]
    else:
        case = ec.make_case(kind, cid)
        P = ec.speech_params() if kind == "speech" else ec.style_params(case.vae)
        ref_o, ref_g = ec.run_oracle(P, case)
    o, g, _ = ec.run_restated(P, case)
    for a, b in zip(o, ref_o):
        assert float((a - b).abs().max()) <= 1e-12 * max(1.0, float(b.abs().max()))
    for k in ref_g:
        assert float((g[k] - ref_g[k]).abs().max()) <= 1e-12 * max(1e-30, float(ref_g[k].abs().max())), k


@pytest.mark.parametrize("kind", ["speech", "style"])
def test_float32_oracle_meets_every_bound_with_4x_headroom(main_cases, kind):
    P, case, ref_o, ref_g = main_cases[kind]
    errs = ec.errors(*ec.run_oracle(P, case, torch.float32), ref_o, ref_g)
    _show(f"{kind} fp32", errs)
    assert not [x for x in errs if not 4 * x[1] <= x[2]]
    if kind == "style":                    # the natural parameters' outputs too (the GPU file checks forwards with them)
        errs = ec.errors(ec.run_oracle(ec.style_params(), case, torch.float32)[0], None,
                         ec.run_oracle(ec.style_params(), case)[0], None)
        assert not [x for x in errs if not 4 * x[1] <= x[2]]


@pytest.mark.parametrize("cid", [c for c, kw in ec.STYLE_CASES.items() if kw.get("grads", True)])
def test_gate_margins_hold_for_every_gpu_style_case(main_cases, cid):
    """Every ReLU pre-activation of the margined parameters lies at least GATE_RATIO x the float32 error of its layer from zero."""
    if cid == MAIN["style"]:
        P, case = main_cases["style"][:2]
    else:
        case = ec.make_case("style", cid)
        P = ec.margined_style_params(ec.style_params(case.vae), case)
    for site, (margin, err) in ec.gate_margins(P, case).items():
        print(f"  [{cid} {site}] nearest |pre| {margin:.2e}, fp32 error {err:.2e}: {margin / max(err, 1e-30):.0f}x")
        assert margin >= ec.GATE_RATIO * err, site


@pytest.mark.parametrize("kind", ["speech", "style"])
def test_matched_bound_separates_single_pass_bf16_from_fp32_grade(main_cases, kind):
    P, case, ref_o, ref_g = main_cases[kind]
    mo, mg, opts = ec.run_restated(P, case, matched=True)
    # every weight gradient fast_wgrad = 1 runs in one bf16 pass meets the tensor-core rule at this shape, so the oracle rounds them all
    rounded = {key: M * N * K for key, M, N, K in opts.rounded}
    assert sorted(rounded) == sorted(ec.SPEECH_WGRADS if kind == "speech" else ec.STYLE_WGRADS)
    assert all(mnk >= ec.TC_MIN_MNK for mnk in rounded.values())
    # non-rounded gradients are the plain oracle's
    for k in ref_g:
        if k not in rounded:
            assert float((mg[k] - ref_g[k]).abs().max()) <= 1e-12 * max(1e-30, float(ref_g[k].abs().max())), k
    m32o, m32g, _ = ec.run_restated(P, case, torch.float32, matched=True)
    errs = ec.errors(m32o, m32g, mo, mg, rounded)
    _show(f"{kind} matched fp32", errs)
    assert not [x for x in errs if not 4 * x[1] <= x[2]]
    for k in rounded:
        e = ec.rel_l2(ref_g[k], mg[k])
        print(f"  [{kind} unmatched float64] {k}: {e:.2e} (bound {ec.MATCHED_TOL[k]:.1e})")
        assert e > ec.MATCHED_TOL[k], k


@pytest.mark.parametrize("kind,fault", [(k, f) for k, fs in ec.FAULTS.items() for f in fs])
def test_modelled_fault_exceeds_its_bound(main_cases, kind, fault):
    P, case, ref_o, ref_g = main_cases[kind]
    o, g, _ = ec.run_restated(P, case, fault=fault)
    # the looser matched bounds on the single-pass weight gradients too: the fault shows in every setting
    errs = ec.errors(o, g, ref_o, ref_g, ec.SPEECH_WGRADS if kind == "speech" else ec.STYLE_WGRADS)
    n, e, b = max(errs, key=lambda x: x[1] / x[2])
    print(f"  [{kind} {fault}] worst {n}: {e:.2e} = {e / b:.0f}x its bound")
    assert e > b
