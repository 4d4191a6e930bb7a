"""CPU (no GPU): the restatement of the loudness kernel's scheme (tests/_loudness_cases.py) meets every bound
tests/test_loudness_f64_gpu.py holds the kernel to, against oracle/loudness_oracle.py, with >= 4x headroom; each modelled
kernel fault breaks a bound; and the host's gating geometry (LoudnessMeter._geometry) equals the oracle's block bounds with the
last block clamped, at every rate and length the GPU sweep runs."""
import numpy as np
import pytest

from oracle import loudness_oracle as lo
from tests import _loudness_cases as lc

HEADROOM = 4.0


def _worst(cases):
    """cases: [(tag, x, rate)] -> the worst (ratio, tag) of the restatement against the oracle, printing the three worst."""
    out = []
    for tag, x, rate in cases:
        L, g = lc.oracle(x, rate)
        out.append((lc.ratio(*lc.meter(x, rate), L, g), tag))
    out.sort(reverse=True)
    for r, tag in out[:3]:
        print(f"  [restatement {tag}] {r:.3g} of the bound (headroom {1.0 / max(r, 1e-30):.3g}x)")
    return out[0]


# ---------------------------------------------------------------------------------------------- the restatement meets the bounds
def test_restatement_meets_the_bounds_at_16k_lengths():
    cases = [(f"n{n} {k}", lc.content(k, n, 16000, 7), 16000) for n in lc.LEN_16K for k in lc.CONTENTS]
    r, tag = _worst(cases)
    assert r * HEADROOM <= 1.0, tag


def test_restatement_meets_the_bounds_at_long_clips():
    """The block counts around the former shared-memory limit and cap, and 20 minutes."""
    cases = [(f"{nb} blocks", lc.content("speech", lc.samples_for_blocks(nb), 16000, nb), 16000) for nb in lc.BLOCK_COUNTS]
    cases.append(("20 min", lc.content("gate_sections", lc.MIN_20, 16000, 3), 16000))
    r, tag = _worst(cases)
    assert r * HEADROOM <= 1.0, tag


@pytest.mark.parametrize("rate", lc.OTHER_RATES)
def test_restatement_meets_the_bounds_at_other_rates(rate):
    cases = [(f"{rate} Hz n{n} {k}", lc.content(k, n, rate, 11), rate) for n in lc.rate_lengths(rate) for k in lc.CONTENTS]
    r, tag = _worst(cases)
    assert r * HEADROOM <= 1.0, tag


def test_restatement_meets_the_bounds_on_int16_pcm():
    x = lc.to_pcm16(lc.batch(10, lc.clamped_length(16000), 16000, 5))
    r, tag = _worst([(f"int16 {k}", x[i], 16000) for i, k in enumerate(lc.CONTENTS)])
    assert r * HEADROOM <= 1.0, tag


def test_cases_reach_every_gate_outcome():
    """Zero and sub-gate clips give -inf in the oracle; the gate-sections clip has a relative threshold below -70 LUFS with
    blocks between it and -70 (so the absolute term of the second pass decides); the burst's relative gate drops most blocks."""
    n = 160000
    for k in ("zeros", "below_gate", "const1e-5"):
        assert lc.oracle(lc.content(k, n, 16000), 16000)[0] == -np.inf, k
    z = _block_loudness(lc.content("gate_sections", n, 16000), 16000)
    gamma_r = -0.691 + 10.0 * np.log10(np.mean(10.0 ** ((z[z >= -70.0] + 0.691) / 10.0))) - 10.0
    print(f"  [gate sections] relative threshold {gamma_r:.2f} LUFS, {np.sum((z > gamma_r) & (z <= -70.0))} blocks between it and -70")
    assert gamma_r < -70.0 and np.sum((z > gamma_r) & (z <= -70.0)) >= 10
    z = _block_loudness(lc.content("burst", n, 16000), 16000)
    gamma_r = -0.691 + 10.0 * np.log10(np.mean(10.0 ** ((z[z >= -70.0] + 0.691) / 10.0))) - 10.0
    print(f"  [burst] {np.sum(z > gamma_r)} of {len(z)} blocks pass the relative gate; {np.sum(z >= -70)} the absolute one")
    assert np.sum(z > gamma_r) < len(z) // 4 and np.sum(z >= -70.0) == len(z)


def _block_loudness(x, rate):
    y = x.copy()
    for b, a in lo.k_weighting(rate):
        y[:] = lo.signal.lfilter(b, a, y)
    lo_, hi_ = lo.block_bounds(len(x), rate)
    z = np.array([np.sum(np.square(y[l:u], dtype=np.float64)) / (lo.T_G * rate) for l, u in zip(lo_, hi_)])
    return -0.691 + 10.0 * np.log10(z)


# ---------------------------------------------------------------------------------------------- faults break a bound
def _fault_case(fault):
    """-> (x, rate, next clip) of the case that shows `fault`."""
    n_clamp = lc.clamped_length(16000)
    if fault == "warm0":
        return lc.content("tone38_dc", 160000, 16000), 16000, None
    if fault == "seg_off_by_one":
        return lc.content("burst", 160000, 16000, 2), 16000, None
    if fault == "no_clamp":
        return lc.content("speech", n_clamp, 16000, 2) * np.float32(0.1), 16000, lc.content("square", n_clamp, 16000)
    if fault == "clamped_len":
        return lc.content("speech", n_clamp, 16000, 2), 16000, None
    if fault == "no_abs_in_rel":
        return lc.content("gate_sections", 160000, 16000), 16000, None
    if fault == "i16_32767":
        return lc.to_pcm16(lc.content("speech", n_clamp, 16000, 4)), 16000, None
    raise KeyError(fault)


@pytest.mark.parametrize("fault", list(lc.FAULTS))
def test_fault_breaks_a_bound(fault):
    x, rate, nxt = _fault_case(fault)
    L, g = lc.oracle(x, rate)
    lufs, gain = lc.meter(x, rate, fault, nxt)
    dl, dg = abs(float(lufs) - L) / lc.LUFS_TOL, abs(float(gain) - g) / (lc.GAIN_RTOL * g)
    print(f"  [fault {fault}: {lc.FAULTS[fault]}] LUFS {dl:.3g}, gain {dg:.3g} of their bounds")
    assert max(dl, dg) > 1.0


# ---------------------------------------------------------------------------------------------- host geometry
GEOMETRY_CASES = ([(16000, n) for n in lc.LEN_16K + [lc.samples_for_blocks(nb) for nb in lc.BLOCK_COUNTS] + [lc.MIN_20]]
                  + [(r, n) for r in lc.OTHER_RATES for n in lc.rate_lengths(r)])


def test_host_geometry_matches_the_oracle_block_bounds():
    """LoudnessMeter._geometry (host tables, built on a CPU device here) against loudness_oracle.block_bounds: each block's
    segments tile exactly [lo_j, min(hi_j, n)), and at least one length per rate clamps its last block."""
    from zeggs_b200 import audio
    clamped = set()
    for rate, n in GEOMETRY_CASES:
        g = audio.LoudnessMeter("cpu", rate)._geometry(n)
        bounds, blo, bhi = g["bounds"].numpy(), g["lo"].numpy(), g["hi"].numpy()
        lo_, hi_ = lo.block_bounds(n, rate)
        assert g["n_blocks"] == len(lo_) == len(blo) and g["n_seg"] == len(bounds) - 1, (rate, n)
        assert np.array_equal(bounds[blo], lo_) and np.array_equal(bounds[bhi], np.minimum(hi_, n)), (rate, n)
        assert bounds[0] == 0 and bounds[-1] <= n and np.all(np.diff(bounds) > 0), (rate, n)
        rb, rlo, rhi = lc.geometry(n, rate)
        assert np.array_equal(bounds, rb) and np.array_equal(blo, rlo) and np.array_equal(bhi, rhi), (rate, n)
        if hi_[-1] > n:
            clamped.add(rate)
    assert clamped == {16000} | set(lc.OTHER_RATES)


def test_too_short_is_refused_by_the_host():
    from zeggs_b200 import _lib, audio
    with pytest.raises(_lib.ZeggsError):
        audio.LoudnessMeter("cpu", 16000)._geometry(lc.TOO_SHORT)


def test_block_counts_and_uneven_segments():
    assert [lc.n_blocks(lc.samples_for_blocks(nb), 16000) for nb in lc.BLOCK_COUNTS] == lc.BLOCK_COUNTS
    assert lc.n_blocks(lc.MIN_20, 16000) > 6001
    b, _, _ = lc.geometry(10 * 11025, 11025)
    assert set(np.diff(b).tolist()) == {1102, 1103}
