"""CPU checks for decoders wider than 1056 hidden units (the fp32 engine at 16 units per CTA, H % 16 == 0, 1056 < H <= 2112):
(1) the library's fp32 pack, workspace and FiLM size queries accept exactly H % 16 == 0, H <= 2112, and the tensor-core rule stays
    H <= 1024;
(2) the units-per-CTA mapping the tests use (U = 16 above 1056) is the one the library packs with;
(3) a float32 evaluation of oracle/fp32_oracle.py meets the fp32 bounds with 4x headroom at H = 2112, B = 33 (two batch tiles), and the
    modelled kernel faults, aimed at one 16-unit CTA, break them.
No GPU involved."""
import numpy as np
import pytest
import torch

from oracle import fp32_oracle as f3
from tests._util import NAMES, ensure_built, stats_tensors, tt
from zeggs_b200 import synth

WIDE_H = list(range(1072, 2112 + 1, 16))


def units_per_cta(H):
    """U of csrc/decoder_common.cuh pick_U at every accepted H: 4 up to 528, 8 up to 1056, 16 up to 2112."""
    return f3.units_per_cta(H) if H <= 1056 else 16


@pytest.fixture(scope="module")
def lib():
    ensure_built()
    from zeggs_b200 import _lib
    return _lib.lib()


def _sizes(l, H, S=64, Z=64, B=33, T=17):
    return {"packed": l.zeggs_decoder_packed_bytes(H, S, Z), "packed_bwd": l.zeggs_decoder_packed_bwd_bytes(H, S, Z),
            "ws": l.zeggs_decoder_workspace_bytes(B, T, H, S, Z, 1), "ws_nosave": l.zeggs_decoder_workspace_bytes(B, T, H, S, Z, 0),
            "bwd_ws": l.zeggs_decoder_bwd_workspace_bytes(B, T, H, S, Z), "film_packed": l.zeggs_decoder_packed_film_bytes(H, S, Z),
            "film_packed_bwd": l.zeggs_decoder_packed_bwd_film_bytes(H, S, Z),
            "film_ws": l.zeggs_decoder_film_workspace_bytes(B, T, H, S, Z, 1),
            "film_bwd_ws": l.zeggs_decoder_film_bwd_workspace_bytes(B, T, H, S, Z)}


def test_fp32_sizes_accept_exactly_h16_up_to_2112(lib):
    for H in range(16, 2112 + 1, 16):
        s = _sizes(lib, H)
        assert all(v > 0 for v in s.values()), (H, s)
    for H in (1000, 2120, 2128, 2144, 4096):
        s = _sizes(lib, H)
        assert all(v == 0 for v in s.values()), (H, s)


def test_tensor_core_rule_stays_at_1024():
    from zeggs_b200 import ops
    for H in range(1040, 2112 + 1, 16):
        assert not ops.tc_eligible(H, 64, 64), H


@pytest.mark.parametrize("H", [16, 528, 544, 1056] + WIDE_H)
def test_units_per_cta_is_the_library_packing(lib, H):
    """The pack is H*1136*4 floats (P1) + 2 * 6*H*H (P2, P3) + G * n4t * H * 16 (P4: ceil(1131 / G) layer-2 rows per CTA in 16-row
    tiles), so its size fixes the grid G = H / U."""
    U = units_per_cta(H)
    G = H // U
    n4t = -(-(-(-1131 // G)) // 16)
    assert lib.zeggs_decoder_packed_bytes(H, 64, 64) == 4 * (H * 1136 * 4 + 12 * H * H + G * n4t * H * 16)
    assert G <= 132 and (U == 16) == (H > 1056)


@pytest.fixture(scope="module")
def stats():
    st = stats_tensors()
    return tuple(st[k] for k in ("anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")) + (st["dt"],)


def _case(H, B, T, seed, film=False):
    P = synth.make_params(H=H, S=64, Z=64, seed=seed, with_style=False, rnn_cond="film" if film else "normal")
    win = tt(synth.make_pose_windows(B, T, seed=seed))
    rs = np.random.RandomState(seed)
    speech = torch.from_numpy((rs.randn(B, T, 64) * 0.5).astype(np.float32))
    style = torch.from_numpy(rs.randn(B, T, 64).astype(np.float32))
    cot = [torch.from_numpy(rs.randn(*win[n].shape).astype(np.float32)) for n in NAMES]
    return P, win, speech, style, cot


def _worst(d):
    return max(d.items(), key=lambda kv: kv[1])


@pytest.mark.parametrize("film", [False, True])
def test_float32_has_4x_headroom_at_2112(stats, film):
    case = _case(2112, 33, 9, seed=17, film=film)
    out64, g64 = f3.run(*case, stats, film=film)
    for gemm in (False, True):
        out32, g32 = f3.run(*case, stats, dtype=torch.float32, film=film, gemm=gemm)
        fn, fe = _worst(f3.forward_errors(out32, out64))
        tol = f3.FP32_GEMM_GRAD_TOL if gemm else f3.FP32_GRAD_TOL
        gn, ge = _worst(f3.grad_errors(g32, g64))
        print(f"  [{'film ' if film else ''}H2112 B33 T9 gemm mode {int(gemm)}] float32 forward worst {fn} {fe:.2e} "
              f"({f3.FP32_FWD_TOL / max(fe, 1e-30):.1f}x headroom)  gradient worst {gn} {ge:.2e} ({tol / max(ge, 1e-30):.1f}x headroom)")
        assert 4 * fe <= f3.FP32_FWD_TOL, (gemm, fn, fe)
        assert 4 * ge <= tol, (gemm, gn, ge)


@pytest.fixture(scope="module")
def wide_fault_base(stats):
    res = {}
    for film in (False, True):
        case = _case(1536, 33, 9, seed=2025, film=film)
        res[film] = case, f3.run(*case, stats, film=film)
    return res


@pytest.mark.parametrize("fault", f3.PERTURBATIONS)
def test_bounds_catch_faults_in_one_16_unit_cta(stats, wide_fault_base, fault, monkeypatch):
    """H = 1536 (U = 16, 96 CTAs), B = 33, T = 9: each modelled fault, aimed at the 16 units of the middle CTA, moves some output group
    or gradient by more than its bound."""
    monkeypatch.setattr(f3, "units_per_cta", units_per_cta)
    assert len(f3.bad_units(1536)) == 16
    film = fault.startswith("film")
    case, (out0, g0) = wide_fault_base[film]
    out, g = f3.run(*case, stats, film=film, perturb=fault)
    fn, fe = _worst(f3.forward_errors(out, out0))
    gn, ge = _worst(f3.grad_errors(g, g0))
    print(f"  [{fault}] forward worst {fn} {fe:.2e} (bound {f3.FP32_FWD_TOL:.0e})  gradient worst {gn} {ge:.2e} "
          f"(bound {f3.FP32_GEMM_GRAD_TOL:.0e})")
    assert fe > f3.FP32_FWD_TOL or ge > f3.FP32_GEMM_GRAD_TOL, (fault, fn, fe, gn, ge)
