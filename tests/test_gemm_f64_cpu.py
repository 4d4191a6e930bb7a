"""CPU-only: the GEMM front end's bounds mean something.  Cases, planner rule, oracles and restatements: tests/_gemm_cases.py.

* The restatements without a fault equal plain float64 where they should (the three-pass scheme without rounding, the matched oracle
  on bf16-exact operands), to 1e-12.
* The fp32 / bf16 restatement of each path meets tau with >= 4x headroom: SIMT, three-pass tensor cores with and without split-K,
  one-pass against the bf16-matched oracle, each epilogue, randn and dynamic-range operands, K from 1 to 12288.
* Each modelled fault of FAULTS breaks its bound (or the guard band around the output window); the factor is printed.
* On the dynamic-range case an unwritten M tail passes the earlier 4e-5 max|C| check and fails the elementwise bound.
* expected_path at each planner boundary, on devices of several SM counts.
tests/test_gemm_front_end_cpu.py checks that a zeggs_ctx whose gemm_mode is neither 0 nor 1 is refused before anything is launched.
"""
import math

import pytest
import torch

from tests import _gemm_cases as gc

# (path, mode, M, N, K, splits): every path, the tails of a 128-row tile, K below one k-block, Kp padding and the weight gradients' K
HEADROOM_CASES = [
    ("simt", 0, 65, 33, 1, 1), ("simt", 1, 129, 31, 1000, 1), ("simt", 2, 63, 129, 65, 1), ("simt", 0, 16, 17, 12288, 1),
    ("tc3", 0, 65, 33, 1, 1), ("tc3", 1, 129, 257, 9, 1), ("tc3", 2, 128, 127, 513, 1), ("tc3", 0, 64, 64, 4096, 4),
    ("tc3", 1, 32, 33, 12288, 2), ("tc1", 1, 65, 33, 7, 1), ("tc1", 1, 129, 256, 513, 1), ("tc1", 1, 32, 32, 12288, 6),
]
HEADROOM = 4.0


def _restate(path, mode, A, B, bias, act, C0, splits, fault=None, **kw):
    if path == "simt":
        return gc.restate_simt(mode, A, B, bias, act, C0, fault, **kw)
    return gc.restate_tc(mode, A, B, bias, act, C0, path == "tc3", splits, fault)


def _ref(path, mode, A, B, bias, act, C0):
    return (gc.matched if path == "tc1" else gc.oracle)(mode, A, B, bias, act, C0)


def _worst(path, mode, A, B, bias, act, C0, got):
    K = gc.op_a(mode, A).shape[1]
    return float(gc.ratio(got, _ref(path, mode, A, B, bias, act, C0), gc.scale(mode, A, B, bias), gc.tau(path, K)).max())


def test_restatements_equal_float64_where_they_should():
    A, B, _, _ = gc.make_operands(0, 33, 17, 40, seed=3)
    ah, al = gc.split_hi_lo(A)
    bh, bl = gc.split_hi_lo(B.T)
    exact = ah @ bh + al @ bh + ah @ bl
    assert float((gc.split3(0, A, B) - exact).abs().max()) <= 1e-12 * float(exact.abs().max())
    # bf16-exact operands: the matched oracle, the three-pass emulation and plain float64 agree
    Ab, Bb = gc.bf16(A).float(), gc.bf16(B).float()
    ref = gc.oracle(0, Ab, Bb)
    for f in (gc.matched, gc.split3):
        assert float((f(0, Ab, Bb) - ref).abs().max()) <= 1e-12 * float(ref.abs().max())
    # the epilogue: act(P + bias) + C0 in every layout
    for mode in (0, 1, 2):
        A, B, bias, C0 = gc.make_operands(mode, 9, 5, 7, seed=mode)
        a = A.double().T if mode == 1 else A.double()
        b = B.double().T if mode == 0 else B.double()
        want = torch.nn.functional.elu(a @ b + bias.double()) + C0.double()
        assert float((gc.oracle(mode, A, B, bias, 1, C0) - want).abs().max()) <= 1e-12 * float(want.abs().max())


@pytest.mark.parametrize("dyn", [False, True], ids=["randn", "dynrange"])
@pytest.mark.parametrize("path,mode,M,N,K,splits", HEADROOM_CASES)
def test_restated_path_meets_tau_with_headroom(path, mode, M, N, K, splits, dyn):
    A, B, bias, C0 = gc.make_operands(mode, M, N, K, seed=M + N + K, dyn=dyn)
    worst = 0.0
    for act, b, c in [(0, None, None), (1, bias, C0), (2, bias, None), (0, None, C0)]:
        got = _restate(path, mode, A, B, b, act, c, splits)
        worst = max(worst, _worst(path, mode, A, B, b, act, c, got))
    print(f"  [{path} mode{mode} {M}x{N}x{K} splits {splits} {'dynrange' if dyn else 'randn'}] worst {worst:.3f} of tau "
          f"({gc.tau(path, K):.2e}): headroom {1 / worst:.1f}x")
    assert worst * HEADROOM <= 1.0


# fault -> (path, mode, M, N, K, splits, act, bias, accumulate)
FAULT_CASES = {
    "lo_hi_dropped": ("tc3", 0, 129, 129, 513, 1, 0, False, False),
    "k_tail_dropped": ("tc3", 2, 65, 65, 513, 1, 0, False, False),
    "m_tail_unwritten": ("tc3", 0, 200, 64, 256, 1, 0, False, False),
    "bias_twice": ("tc3", 0, 32, 64, 4096, 4, 0, True, False),
    "accumulate_ignored": ("tc3", 1, 64, 64, 512, 1, 0, False, True),
    "act_before_bias": ("simt", 0, 64, 64, 64, 1, 2, True, False),
    "splitk_partial_missing": ("tc3", 0, 32, 64, 4096, 4, 0, False, False),
    "mode1_lda_is_M": ("simt", 1, 40, 24, 64, 1, 0, False, False),
    "n_tail_past_N": ("tc3", 0, 64, 33, 64, 1, 0, False, False),
    "n32_last_chunk_dropped": ("simt", 2, 129, 31, 1000, 1, 0, False, False),
    "fast_wgrad_in_mode0": ("tc3", 0, 128, 128, 512, 1, 0, False, False),
}


@pytest.mark.parametrize("fault", list(gc.FAULTS))
def test_each_modelled_fault_breaks_its_bound(fault):
    path, mode, M, N, K, splits, act, with_bias, acc = FAULT_CASES[fault]
    A, B, bias, C0 = gc.make_operands(mode, M, N, K, seed=11)
    bias = bias if with_bias else None
    C0 = C0 if acc else None
    kw = {}
    if fault == "mode1_lda_is_M":
        store = torch.randn(K, M + 8, generator=torch.Generator().manual_seed(2))
        A, kw = store[:, :M], {"A_store": store}
    good = _restate(path, mode, A, B, bias, act, C0, splits, **kw)
    assert _worst(path, mode, A, B, bias, act, C0, good) < 1.0
    if fault == "n_tail_past_N":
        # the output window [M, N] of a [M, N + 1] buffer pre-filled with a NaN sentinel: the store of column N leaves the window
        buf = torch.full((M, N + 1), float("nan"), dtype=torch.float64)
        buf[:, :N] = good
        buf[:, N] = good[:, N - 1]
        changed = int((~torch.isnan(buf[:, N])).sum())
        print(f"  [{fault}] guard band: {changed} elements beside the window overwritten")
        assert changed > 0
        return
    bad = good if fault == "m_tail_unwritten" else _restate(path, mode, A, B, bias, act, C0, splits, fault, **kw)
    if fault == "m_tail_unwritten":
        bad = gc.m_tail_unwritten(good, M)
    w = _worst(path, mode, A, B, bias, act, C0, bad)
    print(f"  [{fault}] {gc.FAULTS[fault]}: {w:.3g}x its bound")
    assert w > 1.0


def test_unwritten_m_tail_passes_the_max_c_check_on_the_dynamic_range_case():
    """M = 65: row 64 is the second consumer warpgroup's only row.  With seed 4 its row of op(A) is scaled by 10^-1.4 and every element
    of it is below 4e-5 of max|C|, so a kernel that never stores it passes the max|C| check -- and fails the elementwise bound."""
    M, N, K = 65, 33, 64
    A, B, _, _ = gc.make_operands(0, M, N, K, seed=4, dyn=True)
    ref = gc.oracle(0, A, B)
    good = gc.restate_tc(0, A, B)
    bad = gc.m_tail_unwritten(good, M)
    w = float(gc.ratio(bad, ref, gc.scale(0, A, B), gc.tau("tc3", K)).max())
    print(f"  unwritten M tail: old check passes, {w:.3g}x the elementwise bound")
    assert gc.old_check(good, ref) and gc.old_check(bad, ref)
    assert w > 1.0


# ---------------------------------------------------------------------------------------------- planner boundaries
BIG = gc.Ctx(1, 1 << 40, 0)
FAST = gc.Ctx(1, 1 << 40, 1)


@pytest.mark.parametrize("sms", [132, 114, 78, 16])
def test_expected_path_at_each_planner_boundary(sms):
    ep = lambda mode, M, N, K, ctx=BIG: gc.expected_path(mode, M, N, K, ctx, sms)
    for mode in (0, 1, 2):
        # the MAC threshold: 160 x 125 x 200 = 4e6 runs on the tensor cores, one k less stays on SIMT
        assert ep(mode, 160, 125, 200).kind == "tc3" and ep(mode, 160, 125, 199).kind == "simt"
        # no scratch, GEMM mode 0
        assert ep(mode, 256, 384, 512, gc.Ctx(1, None, 0)).kind.startswith("simt")
        assert ep(mode, 256, 384, 512, gc.Ctx(0, 1 << 40, 0)).kind.startswith("simt")
        # the carve: exactly enough -> tensor cores, no room for split-K partials; one byte short -> SIMT
        carve = gc.carve_bytes(256, 384, 512, True)
        assert carve == 2 * (256 * 512 * 2 + 384 * 512 * 2)
        assert ep(mode, 256, 384, 512, gc.Ctx(1, carve, 0)) == gc.Path("tc3", 1, 128)
        assert ep(mode, 256, 384, 512, gc.Ctx(1, carve - 1, 0)).kind == "simt"
        # fast_wgrad reaches mode-1 products only
        assert ep(mode, 256, 384, 512, gc.Ctx(1, 1 << 40, 1)).kind == ("tc1" if mode == 1 else "tc3")
    # Kp padding and the 256-byte rounding of each piece
    assert gc.carve_bytes(3, 5, 9, False) == 256 + 256 and gc.carve_bytes(300, 5, 9, True) == 2 * (9728 + 256)
    # the n32 kernel: modes 1 and 2, N <= 32, M >= 128
    assert ep(1, 128, 32, 5).kind == "simt_n32" and ep(2, 128, 1, 5).kind == "simt_n32"
    assert ep(1, 127, 32, 5).kind == "simt" and ep(1, 128, 33, 5).kind == "simt" and ep(0, 128, 32, 5).kind == "simt"
    # BN = 256 for one pass with N >= 256 only
    assert [ep(1, 512, n, 384, FAST).BN for n in (255, 256, 257)] == [128, 256, 256]
    assert ep(0, 512, 256, 384).BN == 128
    # split-K: tiles <= sms / 2 and at least 8 k-blocks; the count from the SMs, half the k-blocks, the workspace, then re-rounded
    half = sms // 2
    K8, K7 = 8 * 64, 7 * 64
    assert gc.tc_splits(128, 128 * half, K8 * 8, 128, sms, 1 << 40) > 1
    assert gc.tc_splits(128, 128 * (half + 1), K8 * 8, 128, sms, 1 << 40) == 1
    assert gc.tc_splits(128, 128, K8, 128, sms, 1 << 40) == min(sms, 4) and gc.tc_splits(128, 128, K7, 128, sms, 1 << 40) == 1
    assert gc.tc_splits(128, 128, 9 * 64, 128, sms, 1 << 40) == (3 if sms >= 4 else 2)    # kbs = ceil(9 / 4) = 3 -> 3 splits
    per = 128 * 128 * 4
    assert gc.tc_splits(128, 128, 64 * 64, 128, sms, 2 * per) == 2
    assert gc.tc_splits(128, 128, 64 * 64, 128, sms, 2 * per - 1) == 1
    assert gc.tc_splits(128, 128, 64 * 64, 128, sms, None) == 1
    m = gc.expected_path(0, 32, 300, 4096, BIG, sms)
    kbs = math.ceil(64 / min(sms // 3, 32))
    assert m.kind == "tc3" and m.splits == math.ceil(64 / kbs)
    # launches: SIMT once per 65535 row tiles, tensor cores 2 + slices (+ the reduction)
    assert gc.Path("simt", 1, 0).launches(65535 * 64) == 1 and gc.Path("simt", 1, 0).launches(65535 * 64 + 1) == 2
    assert gc.Path("simt_n32", 1, 0).launches(65535 * 128 + 1) == 2
    assert gc.Path("tc3", 1, 128).launches(65535 * 128) == 3 and gc.Path("tc3", 1, 128).launches(65535 * 128 + 1) == 4
    assert gc.Path("tc1", 4, 128).launches(64) == 4
