"""No GPU: GRU style encoders wider than 1056 hidden units (16 units per CTA, H % 16 == 0, 1056 < H <= 2112; csrc/style_gru.cu).

* The library's workspace query accepts exactly the size rule: H % 4 == 0 up to 528, H % 8 == 0 up to 1056, H % 16 == 0 up to 2112.
* At H = 2112 one call takes at most 1792 samples (the BPTT's carry, W_hh streamed); one more is refused before any launch.
* The float32 oracle meets the bounds of tests/test_style_gru_wide_f64_gpu.py with at least 4x headroom at H = 2112, B = 33 (VAE on).
* Modelled faults of the wide path exceed them: the second 8-unit half of each CTA multiplying the first half's W_hh rows, the last
  (64-row) K chunk of h(t-1) dropped at H = 2112, and a column-sum slab that drops or shifts the bias-gradient columns >= 4096.
"""
import ctypes

import pytest
import torch

from tests import _encoder_cases as ec
from tests import _gru_cases as gc
from tests._util import ensure_built

WIDE_H = list(range(1072, 2112 + 1, 16))
COLRED_MAXD = 4096          # columns per column-sum slab (csrc/encoders.cu)
B_HH, B_IH = gc._SE + "rnn_layer.bias_hh_l0", gc._SE + "rnn_layer.bias_ih_l0"


@pytest.fixture(scope="module")
def lib():
    ensure_built()
    from zeggs_b200 import _lib
    return _lib


def accepted(H):
    return (H % 4 == 0 and H <= 528) or (H % 8 == 0 and H <= 1056) or (H % 16 == 0 and 1056 < H <= 2112)


def test_workspace_query_accepts_exactly_the_size_rule(lib):
    l = lib.lib()
    got = [H for H in range(1, 2300) if l.zeggs_style_enc_gru_workspace_bytes(1, 5, 1134, H, 128, 1) > 0]
    assert got == [H for H in range(1, 2300) if accepted(H)]
    assert [H for H in got if H > 1056] == WIDE_H and len(WIDE_H) == 66
    for H in (6, 532, 1064, 2120, 2128):
        assert l.zeggs_style_enc_gru_workspace_bytes(1, 5, 1134, H, 128, 1) == 0, H


def test_largest_batch_at_2112_and_one_more_is_refused(lib):
    """U = 16 keeps no weights resident, so the BPTT's shared memory holds the 16-unit carry of 56 batch tiles (116736 + 56 * 2048
    bytes <= 227 KB) at every wide H.  The workspace query reports 0 above that, and both entry points refuse, naming the limit."""
    l = lib.lib()
    for H in (1072, 2112):
        assert l.zeggs_style_enc_gru_workspace_bytes(1792, 17, 1134, H, 128, 1) > 0
        assert l.zeggs_style_enc_gru_workspace_bytes(1793, 17, 1134, H, 128, 1) == 0
    dummy = ctypes.create_string_buffer(64)
    p = ctypes.addressof(dummy)
    a = lib.StyleEncGruArgs(B=1793, T=17, C_in=1134, H=2112, E=128, temperature=1.0, x=p, z=p, mu=p, logvar=p, workspace=p,
                            workspace_bytes=1 << 40)
    g = lib.StyleEncGruGrads(dz=p, dmu=p, dlogvar=p)
    launches = l.zeggs_launch_count()
    assert l.zeggs_style_enc_gru_fwd(ctypes.byref(a), None) != 0
    assert "at most 1792 samples" in l.zeggs_last_error().decode()
    assert l.zeggs_style_enc_gru_bwd(ctypes.byref(a), ctypes.byref(g), None) != 0
    assert "at most 1792 samples" in l.zeggs_last_error().decode()
    assert l.zeggs_launch_count() == launches


# ---------------------------------------------------------------------------------------------- bounds at H = 2112
_main = {}


def _case2112():
    """(margined parameters, case, float64 oracle outputs, gradients) at H = 2112, B = 33, T = 17 with the VAE, cached."""
    if not _main:
        case = gc.gru_case(B=33, T=17, H=2112, seed=2112)
        P = gc.margined_params(gc.gru_params(case.H, case.E), case)
        _main["v"] = (P, case) + tuple(gc.run_oracle(P, case))
    return _main["v"]


def _show(tag, errs):
    for n, e, b in errs:
        print(f"  [{tag}] {n}: {e:.2e} (bound {b:.1e}, {b / max(e, 1e-30):.1f}x headroom)")


def test_float32_oracle_meets_every_bound_with_4x_headroom_at_2112():
    P, case, ref_o, ref_g = _case2112()
    errs = gc.errors(*gc.run_oracle(P, case, torch.float32), ref_o, ref_g)
    _show("H2112 B33 T17 fp32", errs)
    assert not [x for x in errs if not 4 * x[1] <= x[2]]
    for site, (margin, err) in gc.gate_margins(P, case).items():
        assert margin >= ec.GATE_RATIO * err, site


def _half_rows(Whh):
    """W_hh as a CTA reads it when units 8..15 of each 16-unit CTA multiply the W_hh rows of units 0..7."""
    H = Whh.shape[1]
    W = Whh.copy()
    for g in range(3):
        for c0 in range(0, H, 16):
            W[g * H + c0 + 8:g * H + c0 + 16] = Whh[g * H + c0:g * H + c0 + 8]
    return W


def _worst(errs):
    return max(errs, key=lambda x: x[1] / x[2])


def test_second_half_of_a_cta_on_the_first_halfs_rows_exceeds_the_bound():
    P, case, ref_o, _ = _case2112()
    outs = gc.run_oracle(dict(P, **{gc.W_HH: _half_rows(P[gc.W_HH])}), case)[0]
    n, e, b = _worst(gc.errors(outs, None, ref_o, None))
    print(f"  [half rows at H2112] worst {n}: {e:.2e} = {e / b:.0f}x its bound")
    assert e > b


def test_last_64_row_k_chunk_dropped_at_2112_exceeds_the_bound():
    P, case, ref_o, ref_g = _case2112()
    assert (case.H - 1) // gc.GRU_KC * gc.GRU_KC == 2048          # the fault drops rows 2048 .. 2111
    o, g, _ = gc.run_restated(P, case, fault="k_chunk_dropped")
    n, e, b = _worst(gc.errors(o, g, ref_o, ref_g, gc.WGRADS))
    print(f"  [k_chunk_dropped at H2112] worst {n}: {e:.2e} = {e / b:.0f}x its bound")
    assert e > b


@pytest.mark.parametrize("fault", ["dropped", "shifted"])
@pytest.mark.parametrize("key", [B_HH, B_IH])
def test_column_sum_slab_fault_exceeds_the_bound(fault, key):
    """3H = 6336 bias columns are summed as slabs [0, 4096) and [4096, 6336): a second slab that is never written, or that reads the
    first slab's columns (its column offset lost), moves the bias gradient by more than the bound."""
    _, _, _, ref_g = _case2112()
    ref = ref_g[key]
    assert ref.shape[0] == 6336
    bad = ref.clone()
    bad[COLRED_MAXD:] = 0.0 if fault == "dropped" else ref[:ref.shape[0] - COLRED_MAXD]
    e = ec.rel_l2(bad, ref)
    print(f"  [slab {fault} in {key}] {e:.2e} = {e / gc.GRAD_TOL:.0f}x the bound")
    assert e > gc.GRAD_TOL
